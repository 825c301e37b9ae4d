// flat.cu -- exhaustive (flat) search on the Hopper tensor cores (SURVEY.md §8 f2).
//
// Replaces, for ground truth and re-ranking: svs::Flat / FlatIndex::search
// (include/svs/index/flat/flat.h:159,421-465) -- the one place on this path where a query block x base block
// forms a dense GEMM.  Three steps, the result being EXACT (the same ids and the same bit-exact distances as the
// scan with the search path's distance code, ties by id):
//
//   1. flat_gemm_topk_kernel: S = Q . X^T in fp16 with fp32 accumulation.  One CTA per (128-query tile, range of
//      256-row base tiles); operands are pre-tiled in HBM in the canonical K-major layout of the warpgroup MMA
//      (8x8 core matrices, no swizzle) so that every k-block of a tile is one contiguous blob moved by ONE
//      `cp.async.bulk` into a 6-stage shared-memory ring signalled through mbarriers by a producer warp.  Two
//      consumer warpgroups each issue `wgmma.mma_async.m64n256k16.f32.f16.f16` on 64 of the tile's 128 query rows,
//      keep the 64 x 256 fp32 accumulator in registers, turn scores into keys (|x|^2 - 2 q.x for L2, -q.x for
//      inner product) and keep, per query, the KC smallest keys seen in this CTA's base range: KC = 33 in one list per
//      column half (k <= 25), or KC = 129 in one list per query row (k <= 121, the flat index's deep lists).  Either
//      way a list covers one (row, base range) pair and the ranges of a query are disjoint.
//   2. flat_rescore_kernel: every candidate of a query (all ranges) is re-scored with the search path's own
//      bit-exact distance code (eval_pass) and the k best by (key, id) are written out.
//   3. verification: fp16 rounding moves a key by at most E(q) (derived below); a base row that is NOT a
//      candidate has an approximate key >= T, the smallest per-range list maximum.  If T > kth-smallest approximate
//      key + 2 E(q), no excluded row can belong to the exact top k, so the rescored result IS the exact result.
//      Queries that fail the test (rare) are searched again with the exact scan kernel -- the result is exact
//      in every case.
//
// Error bound, over the whole float32 range: q~, x~ are the fp16-rounded operands (float16 and integer inputs are not
// rounded at all).  Per element, |fl16(v) - v| <= 2^-11 |v| + 2^-25: relative in fp16's normal range, absolute (half
// the subnormal spacing 2^-24) below 2^-14.  So a rounded operand moves by
//   dq = ||q~ - q|| <= 2^-11 ||q|| + 2^-25 sqrt(dim),   dx = ||x~ - x|| <= 2^-11 Xmax + 2^-25 sqrt(dim)
// (0 for an operand that is not rounded), and ||q~|| <= ||q|| + dq, ||x~|| <= Xmax + dx.  Then
//   |q~.x~ - q.x| <= ||q~ - q|| ||x~|| + ||q|| ||x~ - x|| <= dq (Xmax + dx) + ||q|| dx;
// the products are exact in fp32 (fp16 x fp16, down to 2^-48) and the tensor-core accumulation of `dim` of them adds
// at most dim 2^-22 ||q~|| ||x~||; for L2 the bias |x~|^2 differs from |x|^2 by at most ||x~ - x|| ||x~ + x|| <=
// dx (2 Xmax + dx).  So
//   E_ip(q) = dq (Xmax + dx) + ||q|| dx + dim 2^-22 (||q|| + dq)(Xmax + dx),
//   E_l2(q) = 2 E_ip(q) + dx (2 Xmax + dx)   (+ the integer term below),
// both times 1.0001 for the float32 norms.  The rescoring kernel rounds every operation of E and of kth + 2E upward, so
// neither underflows nor falls below the true bound.  In fp16's normal range this is the relative bound
// (r 2^-11 + dim 2^-22) ||q|| Xmax, r the number of rounded operands; for unit vectors at dim 96 the absolute term
// 2^-25 sqrt(96) ~ 3e-7 is about 6e-4 of the 2^-11 one.  An element of magnitude >= 65520 rounds to +-inf: its
// row's key becomes +-inf or NaN (NaN and +inf keys are never offered to a list), which no finite bound covers.  The
// tile kernel gives such a row -- query or base -- the norm +inf (so Xmax = +inf), and a query whose ||q||, Xmax or E
// is not finite is never verified: it runs on the exact scan.  tests/test_flat_bound_model.py checks the formula on a
// numpy model of the lists and the certificate.
// int8 / uint8 data with float32 queries takes this path too: integers up to 255 are exact in fp16, so only the query
// is rounded (dx = 0).  The bias is the exact integer |x|^2 converted once (at most 2^-24 Xmax^2 off), and the fp32 key
// bias - 2 s~ is itself rounded once (2^-24 of |x|^2 + 2 |q| |x|), so integer data adds an explicit [integer data]
// 2^-23 Xmax^2 to E_l2.  The 2^-23 |q| |x| part is NOT inside dq Xmax, which the query's rounding uses up: it is
// covered by the accumulation term, whose dim 2^-22 (doubled in E_l2) is twice the dim 2^-23 that a truncating fp32
// accumulator can lose (four times round-to-nearest's); the spare dim 2^-22 >= 2^-23 holds it.  Tightening the dim
// term below 2x would have to add 2^-23 |q| Xmax explicitly.  (The same margin holds the key rounding of float data.)
//
// Integer path: (int8, int8) and (uint8, uint8) with dim <= 32768 run `wgmma.mma_async.m64n256k32.s32.{s8.s8,u8.u8}`
// instead, over tiles of the raw codes (64-element k-blocks: one blob has the bytes of an fp16 blob, so the ring, the
// producer and the work split are the same).  Every sum is exact in int32 (32768 * 255^2 < 2^31), and so is the key
// K = |x|^2 - 2 s (L2) or -s (inner product).  The lists hold the KC smallest (K, id) PAIRS of their range, so each
// is exact, ties included.  The reported distance is a monotone function F of K: float(|q|^2 + K) for L2, float(K) for
// the key of inner product (-float(s)); call v(K) the integer inside the float.  Every row outside the candidates has
// a pair above T, the smallest list-maximum pair, and the k-th result has the pair (K_k, id_k).  The result is exact iff
// every excluded row ranks after the k-th result by (F, id), which holds when either
//   (a) F(T.K) > F(K_k): then F(K) >= F(T.K) > F(K_k) for every excluded row, or
//   (b) |v(T.K)| < 2^24 and T > (K_k, id_k): v(T.K) - 1, v(T.K) and v(T.K) + 1 are exact floats, so
//       F(T.K - 1) < F(T.K) < F(T.K + 1).  An excluded row has K >= T.K >= K_k.  If K_k < T.K, then
//       F(K_k) <= F(T.K - 1) < F(T.K) <= F(K).  If K_k = T.K, a row with K > T.K has F(K) >= F(T.K + 1) > F(K_k), and
//       one with K = T.K has an id above T.id > id_k.  (At |v| = 2^24 the bound fails: 2^24 + 1 rounds to 2^24.)
// Below 2^24 (b) always holds, so no query falls back.  The GEMM key is also checked against the rescored distance,
// F(K) == the exact distance for every candidate: a wrong integer GEMM shows as a fallback, not a wrong answer.
//
// Filtered search (DESIGN.md §9d): the GEMM reads a per-call copy of the bias in which every disallowed column has the
// empty bias, so such a column is never offered to a list (fp16: its key is +inf or NaN; integer kinds: the MASKED
// epilogue gives it the empty key).  The certificate keeps its form and needs no new proof: every allowed row that is
// not a candidate still has an approximate key >= T, and the excluded rows are now a subset of those it already
// covered.  Xmax stays the index's (or the Valid slots'): sound, if looser than the allowed rows' maximum.
#include "host.cuh"
#include "search_kernel.cuh"

#include <cuda_fp16.h>

#include <climits>
#include <type_traits>

namespace svsb200 {

constexpr uint32_t FLAT_BM = 128, FLAT_BN = 256, FLAT_BK = 32;      // tile sizes (rows, rows, k elements per blob)
constexpr uint32_t FLAT_A_BYTES = FLAT_BM * FLAT_BK * 2, FLAT_B_BYTES = FLAT_BN * FLAT_BK * 2;
constexpr uint32_t FLAT_STAGE_BYTES = FLAT_A_BYTES + FLAT_B_BYTES;
constexpr uint32_t FLAT_STAGES = 6;
constexpr uint32_t FLAT_KC = 33;                                     // list entries per (query, base range)
constexpr uint32_t FLAT_KC_DEEP = 129;                               // ... of the deep lists (Flat handle, k <= 121)
constexpr uint32_t FLAT_LEAD = 4;                                   // tiles a CTA may run ahead of its segment's slowest CTA
constexpr uint32_t FLAT_CMAX = 1024;                                 // candidates per query the rescoring kernel holds
constexpr uint32_t FLAT_BK8 = 64;                                    // k elements per blob of 8-bit operands (same bytes)
constexpr uint32_t FLAT_INT_MAX_DIM = 32768;                         // integer GEMM: every int32 sum and key is exact
// Operand kind of the GEMM: fp16 (float data, or integer data with float32 queries) or the raw int8 / uint8 codes.
enum FlatKind : int { FLAT_F16 = 0, FLAT_S8 = 1, FLAT_U8 = 2 };

// ---- PTX helpers -------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return static_cast<uint32_t>(__cvta_generic_to_shared(p)); }
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint64_t* bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
    asm volatile(
        "{\n\t"
        ".reg .pred p;\n\t"
        "WAIT_LOOP:\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n\t"
        "@p bra DONE;\n\t"
        "bra WAIT_LOOP;\n\t"
        "DONE:\n\t"
        "}\n" ::"r"(smem_u32(bar)),
        "r"(parity)
        : "memory");
}
__device__ __forceinline__ void bulk_copy_g2s(void* smem_dst, const void* gmem_src, uint32_t bytes, uint64_t* bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(smem_u32(smem_dst)),
                 "l"(gmem_src), "r"(bytes), "r"(smem_u32(bar))
                 : "memory");
}
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N> __device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }
// Warpgroup-MMA shared-memory matrix descriptor, K-major, no swizzle (layout type 0): 8x8-element core matrices of
// 128 contiguous bytes; LBO = byte distance between the two 8-element k-chunks of one K=16 MMA, SBO = byte distance
// between 8-row groups.
__device__ __forceinline__ uint64_t wgmma_desc(uint32_t smem_addr, uint32_t lbo_bytes, uint32_t sbo_bytes) {
    return uint64_t((smem_addr >> 4) & 0x3FFFu) | (uint64_t((lbo_bytes >> 4) & 0x3FFFu) << 16) |
           (uint64_t((sbo_bytes >> 4) & 0x3FFFu) << 32);
}
// D (64 x 256, in registers) [+]= A (64 x K) . B (256 x K)^T, both K-major in shared memory: fp16 with fp32
// accumulation (m64n256k16), or int8 (KIND FLAT_S8) / uint8 (FLAT_U8) with int32 accumulation (m64n256k32) under the
// same descriptors, a core matrix being 8 rows x 16 one-byte elements.  `C` is the accumulator's register constraint;
// the fp16 form adds its scale and transpose operands.
#define FLAT_D8(C, i) C(d[i]), C(d[i + 1]), C(d[i + 2]), C(d[i + 3]), C(d[i + 4]), C(d[i + 5]), C(d[i + 6]), C(d[i + 7])
#define FLAT_WGMMA(SHAPE, C, TAIL)                                                                                    \
    asm volatile(                                                                                                     \
        "{\n\t"                                                                                                       \
        ".reg .pred p;\n\t"                                                                                           \
        "setp.ne.b32 p, %130, 0;\n\t"                                                                                 \
        "wgmma.mma_async.sync.aligned." SHAPE " "                                                                     \
        "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "                                     \
        "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, "                            \
        "%32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, "                            \
        "%48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63, "                            \
        "%64, %65, %66, %67, %68, %69, %70, %71, %72, %73, %74, %75, %76, %77, %78, %79, "                            \
        "%80, %81, %82, %83, %84, %85, %86, %87, %88, %89, %90, %91, %92, %93, %94, %95, "                            \
        "%96, %97, %98, %99, %100, %101, %102, %103, %104, %105, %106, %107, %108, %109, %110, %111, "                 \
        "%112, %113, %114, %115, %116, %117, %118, %119, %120, %121, %122, %123, %124, %125, %126, %127}, "           \
        "%128, %129, p" TAIL ";\n\t"                                                                                  \
        "}\n"                                                                                                         \
        : FLAT_D8(C, 0), FLAT_D8(C, 8), FLAT_D8(C, 16), FLAT_D8(C, 24), FLAT_D8(C, 32), FLAT_D8(C, 40),               \
          FLAT_D8(C, 48), FLAT_D8(C, 56), FLAT_D8(C, 64), FLAT_D8(C, 72), FLAT_D8(C, 80), FLAT_D8(C, 88),             \
          FLAT_D8(C, 96), FLAT_D8(C, 104), FLAT_D8(C, 112), FLAT_D8(C, 120)                                           \
        : "l"(adesc), "l"(bdesc), "r"(accumulate))
template <int KIND, typename T>
__device__ __forceinline__ void wgmma_m64n256(T (&d)[128], uint64_t adesc, uint64_t bdesc, uint32_t accumulate) {
    if constexpr (KIND == FLAT_F16) FLAT_WGMMA("m64n256k16.f32.f16.f16", "+f", ", 1, 1, 0, 0");
    else if constexpr (KIND == FLAT_S8) FLAT_WGMMA("m64n256k32.s32.s8.s8", "+r", "");
    else FLAT_WGMMA("m64n256k32.s32.u8.u8", "+r", "");
}
#undef FLAT_WGMMA
#undef FLAT_D8
// keeps the compiler from moving reads of an accumulator register across the wait that completes it
__device__ __forceinline__ void reg_fence(float& r) { asm volatile("" : "+f"(r)::"memory"); }
__device__ __forceinline__ void reg_fence(int& r) { asm volatile("" : "+r"(r)::"memory"); }
// Per-query list of the KC smallest keys: shared memory, [query row][KC] with KC odd, so that a warp reading one row
// side by side is bank-conflict free.  Keys are stored as order-preserving unsigned integers (REDUX.MAX works on them);
// a list starts full of +inf / no-id entries, so there is no fill count -- an update always replaces the current
// maximum, and the row's threshold is the new maximum.  A lane holds ceil(KC / 32) entries of the row: two for
// KC = FLAT_KC, five for FLAT_KC_DEEP.
static_assert(FLAT_KC % 2 == 1 && FLAT_KC > 32 && FLAT_KC <= 64, "list layout");
static_assert(FLAT_KC_DEEP % 2 == 1 && FLAT_KC_DEEP > 64, "list layout");
__device__ __forceinline__ uint32_t flat_ord(float f) {
    const uint32_t u = __float_as_uint(f);
    return u ^ (uint32_t(int32_t(u) >> 31) | 0x80000000u);
}
__device__ __forceinline__ float flat_unord(uint32_t o) {
    return __uint_as_float(o ^ ((o >> 31) ? 0x80000000u : 0xFFFFFFFFu));
}
// Integer lists are ordered by the pair (key, id); their keys are uint32(K) ^ 0x80000000 and an empty entry is
// (0xFFFFFFFF, 0xFFFFFFFF), above every real pair.  flat_pair_max: the largest pair over the warp.
__device__ __forceinline__ uint64_t flat_pair_max(uint64_t v) {
    const uint32_t hi = __reduce_max_sync(0xFFFFFFFFu, uint32_t(v >> 32));
    const uint32_t lo = __reduce_max_sync(0xFFFFFFFFu, uint32_t(v >> 32) == hi ? uint32_t(v) : 0u);
    return (uint64_t(hi) << 32) | lo;
}
// The whole warp offers the ordered key `okey` with `id` to the list of row `list_row`; returns the ordered key of the
// row's new largest entry -- its threshold, warp-uniform.  By key (fp16 lists, BY_PAIR = false): the caller offers only
// keys below the threshold, and the key replaces the first entry holding the largest key.  By (key, id) pair (integer
// lists): a pair not below the largest pair is rejected (an equal key with a larger id), otherwise it replaces the first
// entry holding the largest pair; a pair can only be below the largest pair if its key does not exceed that key, so the
// largest key is still the threshold.  Only the keys stay in registers: the ids are read where a key equals the largest.
template <uint32_t KC, bool BY_PAIR>
__device__ __forceinline__ uint32_t flat_list_offer(uint32_t* lkey, uint32_t* lid, uint32_t list_row, uint32_t lane,
                                                    uint32_t okey, uint32_t id) {
    constexpr uint32_t NW = (KC + 31) / 32;
    uint32_t* rk = lkey + list_row * KC;
    uint32_t* ri = lid + list_row * KC;
    uint32_t v[NW], m = 0;
#pragma unroll
    for (uint32_t w = 0; w < NW; ++w) {
        v[w] = lane + 32 * w < KC ? rk[lane + 32 * w] : 0u;
        m = max(m, v[w]);
    }
    const uint32_t hi = __reduce_max_sync(0xFFFFFFFFu, m);
    uint32_t lo = 0;   // (by pair) the largest id among the entries holding the largest key
    bool take = true;  // (warp-uniform; a rejected pair leaves the list as it is -- no early return, which would make the
                       // compiler guard every collective below against a divergent warp)
    if constexpr (BY_PAIR) {
#pragma unroll
        for (uint32_t w = 0; w < NW; ++w)
            if (lane + 32 * w < KC && v[w] == hi) lo = max(lo, ri[lane + 32 * w]);
        lo = __reduce_max_sync(0xFFFFFFFFu, lo);
        take = ((uint64_t(okey) << 32) | id) < ((uint64_t(hi) << 32) | lo);
    }
    uint32_t slot = 0;   // the first entry holding the largest key (pair)
#pragma unroll
    for (int w = int(NW) - 1; w >= 0; --w) {
        const uint32_t in =
            __ballot_sync(0xFFFFFFFFu, lane + 32 * w < KC && v[w] == hi && (!BY_PAIR || ri[lane + 32 * w] == lo));
        if (in) slot = 32 * w + uint32_t(__ffs(int(in)) - 1);
    }
    const bool mine = take && lane == (slot & 31u);
    if (mine) {
        rk[slot] = okey;
        ri[slot] = id;
    }
    m = 0;
#pragma unroll
    for (uint32_t w = 0; w < NW; ++w) m = max(m, mine && w == slot / 32 ? okey : v[w]);
    return __reduce_max_sync(0xFFFFFFFFu, m);
}

struct FlatParams {
    const __half* a_tiles;    // [mtiles][KB] blobs of FLAT_A_BYTES
    const __half* b_tiles;    // [ntiles][KB] blobs of FLAT_B_BYTES
    const float* b_bias;      // [ntiles * FLAT_BN]: |x~|^2 (L2) / 0 (inner product), +inf for padding rows
                              // (integer kinds: int32 |x|^2 / 0, INT32_MAX for padding rows)
    uint32_t KB, ntiles, mtiles, nlists;
    uint32_t share;           // R: CTAs that walk the same base tiles at the same time, on R consecutive query tiles
    uint32_t* progress;       // [gridDim.x] tiles started by each CTA (zeroed before the launch)
    float key_scale;          // key = bias + key_scale * s (-2 or -1)
    float* cand_key;          // [mtiles * FLAT_BM][nlists][KC], pre-filled with (+inf, no id)
                              // (integer kinds: ordered int32 keys, pre-filled with 0xFFFFFFFF)
    uint32_t* cand_id;
};

// Work split: query tiles are taken R at a time ("row groups"); the (row group, base tile) pairs form one row-major
// sequence, cut into G = gridDim.x / R contiguous, equal segments -- every SM gets the same number of tiles whatever
// the batch size.  Segment g is walked by R CTAs (blockIdx g, g + G, ...: all resident at once, started together, doing
// identical work), one per query tile of the row group: they ask for the same base tile within microseconds of each
// other, so all but the first request are served by L2 -- without this, one CTA per SM streams as many different
// places of a base that is many times the L2, and every operand byte comes from DRAM.  A segment may run over a
// row-group boundary (the lists are flushed there), and a query tile is covered by a few consecutive segments
// ("pieces"); each piece keeps two lists per query, one per half of the 256 tile columns -- or, with the deep lists
// (KC = FLAT_KC_DEEP), one list per query that both halves share.
__host__ __device__ inline uint64_t flat_seg_begin(uint64_t total, uint32_t ctas, uint32_t b) { return total * b / ctas; }
__host__ __device__ inline uint32_t flat_cta_of_tile(uint64_t t, uint64_t total, uint32_t ctas) {
    uint32_t b = uint32_t(t * ctas / total);
    while (b + 1 < ctas && flat_seg_begin(total, ctas, b + 1) <= t) ++b;
    while (b > 0 && flat_seg_begin(total, ctas, b) > t) --b;
    return b;
}

// Threads: warps 0-7 are the two consumer warpgroups (a warpgroup is four consecutive warps starting at a multiple of
// four), warp 8 the producer.  Shared memory: stages | list keys [H][128][KC] | list ids [H][128][KC] | barriers, with
// H lists per query row: two (one per column half) with FLAT_KC entries and a 6-stage ring, one with FLAT_KC_DEEP
// entries and a 4-stage ring (4 x 24 576 + 128 x 129 x 8 + 128 = 230 528 bytes).
constexpr uint32_t FLAT_CONSUMER_WARPS = 8, FLAT_THREADS = 32 * FLAT_CONSUMER_WARPS + 32;
template <uint32_t KC> struct FlatShape {
    static constexpr uint32_t HALVES = KC == FLAT_KC ? 2 : 1;   // lists per query row and piece
    static constexpr uint32_t STAGES = KC == FLAT_KC ? FLAT_STAGES : 4;
    static constexpr size_t SMEM = size_t(STAGES) * FLAT_STAGE_BYTES + 2 * HALVES * size_t(KC) * FLAT_BM * 4 + 128;
    static_assert(SMEM <= kSmemOptInMax, "flat GEMM shared memory exceeds the 227 KB a block may use");
    // index of the list of query row `row` for column half `half` (the deep lists: of `row`, both halves sharing it)
    static __device__ __forceinline__ uint32_t list_row(uint32_t row, uint32_t half) {
        return HALVES == 2 ? half * FLAT_BM + row : row;
    }
};
template struct FlatShape<FLAT_KC>;
template struct FlatShape<FLAT_KC_DEEP>;

// A key of the epilogue: float (fp16 GEMM) or the ordered key itself (integer GEMM), and its conversions to and from
// the ordered keys the lists store.
template <int KIND> using flat_key_t = std::conditional_t<KIND == FLAT_F16, float, uint32_t>;
template <int KIND> __device__ __forceinline__ uint32_t flat_to_ord(flat_key_t<KIND> key) {
    if constexpr (KIND == FLAT_F16) return flat_ord(key);
    else return key;
}
template <int KIND> __device__ __forceinline__ flat_key_t<KIND> flat_from_ord(uint32_t o) {
    if constexpr (KIND == FLAT_F16) return flat_unord(o);
    else return o;
}
// Ordered key of an empty list entry (its flat_from_ord is the threshold of an empty list).
template <int KIND> __device__ __forceinline__ uint32_t flat_empty_key() {
    if constexpr (KIND == FLAT_F16) return flat_ord(INFINITY);
    else return 0xFFFFFFFFu;
}
// Whether a key is offered to a list of threshold `thr`.  fp16: strictly below it, compared as float (the ordered
// integers would order -0 / +0 and negative NaNs differently).  Integer: at or below it, the list comparing the ids --
// but never the empty key, which padding rows (bias INT32_MAX, above every real key) have.
template <int KIND> __device__ __forceinline__ bool flat_beats(flat_key_t<KIND> key, flat_key_t<KIND> thr) {
    if constexpr (KIND == FLAT_F16) return key < thr;
    else return key != 0xFFFFFFFFu && key <= thr;
}

// (The shape is named through the type alias `Shape` only: a kernel-local constant would make the compiler order the
// main loop's stage counters differently and change the FLAT_KC instantiations' code.)
// MASKED (integer kinds, the filtered search): a column whose bias is the empty bias INT32_MAX gets the empty key
// whatever its blob holds.  The wrapping key bias - 2 s of such a column over a non-zero blob looks like an ordinary key
// (and would send the query to the scan through the rescoring's mismatch check); no real |x|^2 reaches INT32_MAX.
template <int KIND, uint32_t KC, bool MASKED = false>
__global__ void __launch_bounds__(FLAT_THREADS, 1) flat_gemm_topk_kernel(const __grid_constant__ FlatParams fp) {
    using acc_t = std::conditional_t<KIND == FLAT_F16, float, int>;
    using Shape = FlatShape<KC>;
    extern __shared__ __align__(1024) uint8_t smem[];
    uint8_t* stages = smem;
    uint32_t* lkey = reinterpret_cast<uint32_t*>(smem + size_t(Shape::STAGES) * FLAT_STAGE_BYTES);   // [H][128][KC] ordered keys
    uint32_t* lid = lkey + Shape::HALVES * size_t(KC) * FLAT_BM;
    uint64_t* bars = reinterpret_cast<uint64_t*>(lid + Shape::HALVES * size_t(KC) * FLAT_BM);
    uint64_t* full = bars;                       // [STAGES] bytes of a stage have landed
    uint64_t* empty = bars + Shape::STAGES;      // [STAGES] the MMAs of every consumer warp reading a stage have completed

    const uint32_t warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const uint32_t nseg = gridDim.x / fp.share, seg = blockIdx.x % nseg, member = blockIdx.x / nseg;
    const uint32_t ngroups = (fp.mtiles + fp.share - 1) / fp.share;
    const uint64_t total = uint64_t(ngroups) * fp.ntiles;
    const uint64_t t_lo = flat_seg_begin(total, nseg, seg), t_hi = flat_seg_begin(total, nseg, seg + 1);
    // (a CTA's query tile advances by `share` at a row-group boundary; tiles of a query tile past the last one are skipped
    // by every role alike)
    const uint32_t mtile0 = uint32_t(t_lo / fp.ntiles) * fp.share + member, nt0 = uint32_t(t_lo % fp.ntiles);

    if (threadIdx.x == 0) {
        for (uint32_t i = 0; i < Shape::STAGES; ++i) {
            mbar_init(full + i, 1);
            mbar_init(empty + i, FLAT_CONSUMER_WARPS);
        }
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();

    if (warp == FLAT_CONSUMER_WARPS) {
        // ===== producer: one bulk copy per operand blob =====
        if (lane == 0) {
            uint32_t s = 0, ph = 0, mtile = mtile0, nt = nt0;
            // Pacing: the R CTAs of a segment do identical work but drift apart by their data-dependent list updates, and a
            // base tile only stays in L2 for some tens of microseconds while the other segments stream through it.  Every
            // other tile the producer publishes its progress and, if it is more than FLAT_LEAD tiles ahead of the
            // segment's slowest CTA, waits (bounded: all CTAs of the grid are resident -- one per SM -- but nothing is
            // assumed; after a timeout this CTA stops looking).  Only for wide rows: with few k-blocks per tile the
            // operands are not DRAM-bound and the L2 round trips of the exchange would cost more than they save.
            bool in_step = fp.share > 1 && fp.KB >= 8;
            for (uint64_t t = t_lo; t < t_hi; ++t) {
                if (in_step && ((t - t_lo) & 1u) == 0) {
                    const uint32_t mine = uint32_t(t - t_lo) + 1u;
                    volatile uint32_t* prog = fp.progress;
                    prog[blockIdx.x] = mine;
                    for (uint32_t spin = 0;; ++spin) {
                        uint32_t slowest = mine;
                        for (uint32_t m = 0; m < fp.share; ++m) slowest = min(slowest, prog[seg + m * nseg]);
                        if (slowest + FLAT_LEAD >= mine) break;
                        if (spin > (1u << 16)) {
                            in_step = false;
                            break;
                        }
                        __nanosleep(200);
                    }
                }
                for (uint32_t kb = 0; kb < fp.KB && mtile < fp.mtiles; ++kb) {
                    mbar_wait(empty + s, ph ^ 1u);
                    mbar_arrive_expect_tx(full + s, FLAT_STAGE_BYTES);
                    uint8_t* st = stages + size_t(s) * FLAT_STAGE_BYTES;
                    bulk_copy_g2s(st, reinterpret_cast<const uint8_t*>(fp.a_tiles) + (size_t(mtile) * fp.KB + kb) * FLAT_A_BYTES,
                                  FLAT_A_BYTES, full + s);
                    bulk_copy_g2s(st + FLAT_A_BYTES,
                                  reinterpret_cast<const uint8_t*>(fp.b_tiles) + (size_t(nt) * fp.KB + kb) * FLAT_B_BYTES,
                                  FLAT_B_BYTES, full + s);
                    if (++s == Shape::STAGES) {
                        s = 0;
                        ph ^= 1u;
                    }
                }
                if (++nt == fp.ntiles) {
                    nt = 0;
                    mtile += fp.share;
                }
            }
            if (fp.share > 1) fp.progress[blockIdx.x] = 0xFFFFFFFFu;   // finished: never the slowest again
        }
        return;
    }

    // ===== consumers: warpgroup wg computes query rows 64 wg .. 64 wg + 63 of the tile against all 256 base rows.
    // Accumulator element d[4c + 2i + e] of a thread is (row 16 (warp % 4) + lane / 4 + 8 i, column 8c + 2 (lane % 4) + e)
    // of its warpgroup's 64 x 256 block, so the four lanes of a quad share two rows; a row keeps one list per column
    // half (deep lists: one list), updated by the whole warp (all lanes of a quad see the new threshold) =====
    const uint32_t wg = warp >> 2;
    const uint32_t row0 = wg * 64 + (warp & 3u) * 16 + (lane >> 2);   // the thread's rows: row0, row0 + 8
    const uint32_t frow = wg * 64 + (warp & 3u) * 16 + (lane >> 1), fhalf = lane & 1u;   // the (row, half) list this lane clears / writes out
    acc_t d[128];
#pragma unroll
    for (uint32_t i = 0; i < 128; ++i) d[i] = acc_t(0);
    // [row i][list]: the largest key of that list (integer kinds: the ordered key of its largest (key, id) pair)
    flat_key_t<KIND> thr[2][Shape::HALVES];
    // Writes the lane's list out to (ok, oi) unless ok is NULL, and empties every list of the warp and its thresholds.
    // (deep lists: the two lanes of a row clear / write out alternate entries of its one list)
    auto reset_lists = [&](flat_key_t<KIND>* ok, uint32_t* oi) {
        uint32_t* rk = lkey + Shape::list_row(frow, fhalf) * KC;
        uint32_t* ri = lid + Shape::list_row(frow, fhalf) * KC;
        for (uint32_t e = Shape::HALVES == 2 ? 0u : fhalf; e < KC; e += 3 - Shape::HALVES) {
            if (ok) {
                ok[e] = flat_from_ord<KIND>(rk[e]);
                oi[e] = ri[e];
            }
            rk[e] = flat_empty_key<KIND>();
            ri[e] = 0xFFFFFFFFu;
        }
        __syncwarp();
#pragma unroll
        for (uint32_t i = 0; i < 2 * Shape::HALVES; ++i)
            thr[i / Shape::HALVES][i % Shape::HALVES] = flat_from_ord<KIND>(flat_empty_key<KIND>());
    };
    reset_lists(nullptr, nullptr);
    uint32_t s = 0, ph = 0, mtile = mtile0, nt = nt0;
    for (uint64_t t = t_lo; t < t_hi; ++t) {
        if (mtile >= fp.mtiles) {
            if (++nt == fp.ntiles) {
                nt = 0;
                mtile += fp.share;
            }
            continue;
        }
        // ---- mainloop: one k-block per stage, two MMAs each (K = 16 fp16 / K = 32 8-bit elements); a stage is released
        // once the MMAs of the next one have been issued and its own have completed ----
        uint32_t prev = 0;
        for (uint32_t kb = 0; kb < fp.KB; ++kb) {
            mbar_wait(full + s, ph);
            const uint32_t a_addr = smem_u32(stages + size_t(s) * FLAT_STAGE_BYTES) + wg * 1024u;   // 8 row groups of 128 B
            const uint32_t b_addr = smem_u32(stages + size_t(s) * FLAT_STAGE_BYTES + FLAT_A_BYTES);
            wgmma_fence();
#pragma unroll
            for (uint32_t j = 0; j < FLAT_BK / 16; ++j) {
                // k-chunks 2j and 2j+1 of the blob: [kc][rows/8][8][16 bytes]
                const uint64_t adesc = wgmma_desc(a_addr + 2 * j * (FLAT_BM * 16), FLAT_BM * 16, 128);
                const uint64_t bdesc = wgmma_desc(b_addr + 2 * j * (FLAT_BN * 16), FLAT_BN * 16, 128);
                wgmma_m64n256<KIND>(d, adesc, bdesc, (kb | j) != 0 ? 1u : 0u);
            }
            wgmma_commit();
            wgmma_wait<1>();
            if (kb > 0 && lane == 0) mbar_arrive(empty + prev);
            prev = s;
            if (++s == Shape::STAGES) {
                s = 0;
                ph ^= 1u;
            }
        }
        wgmma_wait<0>();
#pragma unroll
        for (uint32_t i = 0; i < 128; ++i) reg_fence(d[i]);
        if (lane == 0) mbar_arrive(empty + prev);

        // ---- epilogue: keys of the thread's 128 elements; only columns whose keys beat a row's threshold (rare once
        // the lists have settled) are looked at key by key, the lanes with such a key served in turn by the whole warp.
        // Integer kinds: exact int32 keys (wrapping arithmetic: the true key always fits), ordered as uint32 ----
        const uint32_t* bias = reinterpret_cast<const uint32_t*>(fp.b_bias) + size_t(nt) * FLAT_BN + 2 * (lane & 3u);
#pragma unroll
        for (uint32_t c = 0; c < FLAT_BN / 8; ++c) {
            const uint32_t h = Shape::HALVES == 2 ? c / (FLAT_BN / 16) : 0u;   // the list of this column
            const uint2 b2 = __ldg(reinterpret_cast<const uint2*>(bias + 8 * c));
            flat_key_t<KIND> key[4];
#pragma unroll
            for (uint32_t v = 0; v < 4; ++v) {
                const uint32_t b = v & 1u ? b2.y : b2.x;
                if constexpr (KIND == FLAT_F16) key[v] = fmaf(fp.key_scale, d[4 * c + v], __uint_as_float(b));
                else key[v] = (b + uint32_t(int(fp.key_scale)) * uint32_t(d[4 * c + v])) ^ 0x80000000u;
                if constexpr (MASKED && KIND != FLAT_F16)
                    if (b == 0x7FFFFFFFu) key[v] = 0xFFFFFFFFu;
            }
            const bool any = flat_beats<KIND>(min(key[0], key[1]), thr[0][h]) || flat_beats<KIND>(min(key[2], key[3]), thr[1][h]);
            if (!__any_sync(0xFFFFFFFFu, any)) continue;
#pragma unroll
            for (uint32_t v = 0; v < 4; ++v) {
                const uint32_t i = v >> 1;
                bool pending = flat_beats<KIND>(key[v], thr[i][h]);
                uint32_t hits = __ballot_sync(0xFFFFFFFFu, pending);
                while (hits) {
                    const uint32_t src = uint32_t(__ffs(int(hits)) - 1);
                    const uint32_t o_src = flat_to_ord<KIND>(__shfl_sync(0xFFFFFFFFu, key[v], src));
                    const uint32_t id = nt * FLAT_BN + 8 * c + 2 * (src & 3u) + (v & 1u);
                    const uint32_t tnew = flat_list_offer<KC, KIND != FLAT_F16>(
                        lkey, lid, Shape::list_row(row0 - (lane >> 2) + (src >> 2) + 8 * i, h), lane, o_src, id);
                    if ((lane >> 2) == (src >> 2)) thr[i][h] = flat_from_ord<KIND>(tnew);
                    // another lane of the quad may hold a key of the same row that no longer beats the new threshold
                    pending = pending && lane != src && flat_beats<KIND>(key[v], thr[i][h]);
                    hits = __ballot_sync(0xFFFFFFFFu, pending);
                }
            }
        }
        if (++nt == fp.ntiles || t + 1 == t_hi) {
            // the query tile (or this CTA's part of it) is finished: lists out, lists reset
            const uint32_t piece = seg - flat_cta_of_tile(uint64_t(mtile / fp.share) * fp.ntiles, total, nseg);
            const size_t q = size_t(mtile) * FLAT_BM + frow;
            const size_t list = q * fp.nlists + piece * Shape::HALVES + (Shape::HALVES == 2 ? fhalf : 0u);
            // (the sync before a write-out is not in reset_lists: one ahead of the first reset makes the compiler stop
            // proving the consumer warps converged, and the main loop loses the uniform datapath)
            __syncwarp();
            reset_lists(reinterpret_cast<flat_key_t<KIND>*>(fp.cand_key) + list * KC, fp.cand_id + list * KC);
            nt = 0;
            mtile += fp.share;
        }
    }
}

// ---- operand tiling: rows -> blobs in the canonical K-major layout of the warpgroup MMA ---------------------------
// K-blocks of a row: a blob holds FLAT_BK fp16 or FLAT_BK8 8-bit elements, FLAT_BK * 2 bytes of a row either way.
__host__ __device__ inline uint32_t flat_kblocks(int kind, uint32_t dim) {
    return kind == FLAT_F16 ? (dim + FLAT_BK - 1) / FLAT_BK : (dim + FLAT_BK8 - 1) / FLAT_BK8;
}
// Element (row r, k e) -- row rr = r % TR of tile t = r / TR of TR rows -- with E elements per 16 bytes (8 fp16, 16
// 8-bit) and so 4E per blob: blob t*KB + e/(4E), 16-byte k-chunk (e%(4E))/E of it, 8-row group rr/8, row rr%8, element e%E.
template <uint32_t E> __host__ __device__ inline size_t flat_blob_offset(uint32_t t, uint32_t rr, uint32_t e, uint32_t TR, uint32_t KB) {
    return ((size_t(t) * KB + e / (4 * E)) * 4 + (e % (4 * E)) / E) * (size_t(TR) * E) + (rr / 8) * (8 * E) + (rr % 8) * E + e % E;
}

// rows -> fp16 blobs, with the bias, the row norms and their maximum (the error bound's ||q|| and Xmax)
template <int SRCT>
__global__ void flat_tile_kernel(const char* __restrict__ src, uint32_t row_stride, uint32_t n, uint32_t dim, uint32_t TR,
                                 uint32_t KB, float scale, int l2, __half* __restrict__ dst, float* __restrict__ bias,
                                 float* __restrict__ norms, unsigned int* __restrict__ max_norm_bits) {
    const uint32_t r = blockIdx.x * (blockDim.x / 32) + threadIdx.x / 32;
    const uint32_t lane = threadIdx.x & 31;
    const uint32_t rows_padded = (n + TR - 1) / TR * TR;
    if (r >= rows_padded) return;
    if (r >= n) {
        if (bias && lane == 0) bias[r] = INFINITY;   // padding rows never become candidates
        return;
    }
    const char* row = src + size_t(r) * row_stride;
    const uint32_t t = r / TR, rr = r % TR;
    float sq_rounded = 0.f, sq_exact = 0.f;
    int sq_int = 0;           // integer rows: |x|^2, exact
    bool overflow = false;    // an element rounded to +-inf in fp16 (float rows only)
    for (uint32_t e = lane; e < dim; e += 32) {
        float x;
        if constexpr (SRCT == SVSB200_F32) {
            x = reinterpret_cast<const float*>(row)[e];
        } else if constexpr (SRCT == SVSB200_F16) {
            x = __half2float(reinterpret_cast<const __half*>(row)[e]);
        } else {
            const int v = SRCT == SVSB200_I8 ? int(reinterpret_cast<const int8_t*>(row)[e]) : int(reinterpret_cast<const uint8_t*>(row)[e]);
            sq_int += v * v;
            x = float(v);   // exact in fp16
        }
        const __half h = __float2half_rn(x * scale);
        if constexpr (SRCT == SVSB200_F32) overflow |= bool(__hisinf(h));
        const float xr = __half2float(h) / scale;
        sq_rounded = fmaf(xr, xr, sq_rounded);
        sq_exact = fmaf(x, x, sq_exact);
        dst[flat_blob_offset<8>(t, rr, e, TR, KB)] = h;
    }
    if constexpr (SRCT == SVSB200_I8 || SRCT == SVSB200_U8) {
        for (int o = 16; o; o >>= 1) sq_int += __shfl_xor_sync(0xFFFFFFFFu, sq_int, o);
        sq_rounded = sq_exact = float(sq_int);   // one rounding, 2^-24 |x|^2 at most (E_l2 in the header)
    } else {
        for (int o = 16; o; o >>= 1) {
            sq_rounded += __shfl_xor_sync(0xFFFFFFFFu, sq_rounded, o);
            sq_exact += __shfl_xor_sync(0xFFFFFFFFu, sq_exact, o);
        }
    }
    if constexpr (SRCT == SVSB200_F32) overflow = __any_sync(0xFFFFFFFFu, overflow);
    if (lane == 0) {
        if (bias) bias[r] = l2 ? sq_rounded : 0.f;
        // a row with an infinite fp16 element gets the norm +inf (and so Xmax = +inf): its queries never verify
        const float nrm = overflow ? INFINITY : sqrtf(sq_exact) * 1.000001f;
        if (norms) norms[r] = nrm;
        if (max_norm_bits) atomicMax(max_norm_bits, __float_as_uint(nrm));
    }
}

// int8 / uint8 rows -> blobs of their raw codes; zero padding adds nothing to any integer sum.  bias: |x|^2 (L2) / 0,
// INT32_MAX for padding rows (above every real key, so they never enter a list).
template <int SRCT>
__global__ void flat_tile8_kernel(const char* __restrict__ src, uint32_t row_stride, uint32_t n, uint32_t dim, uint32_t TR,
                                  uint32_t KB, int l2, uint8_t* __restrict__ dst, int* __restrict__ bias) {
    const uint32_t r = blockIdx.x * (blockDim.x / 32) + threadIdx.x / 32;
    const uint32_t lane = threadIdx.x & 31;
    const uint32_t rows_padded = (n + TR - 1) / TR * TR;
    if (r >= rows_padded) return;
    if (r >= n) {
        if (bias && lane == 0) bias[r] = INT_MAX;
        return;
    }
    const uint8_t* row = reinterpret_cast<const uint8_t*>(src + size_t(r) * row_stride);
    const uint32_t t = r / TR, rr = r % TR;
    int sq = 0;
    for (uint32_t e = lane; e < dim; e += 32) {
        const uint8_t c = row[e];
        const int v = SRCT == SVSB200_I8 ? int(int8_t(c)) : int(c);
        sq += v * v;
        dst[flat_blob_offset<16>(t, rr, e, TR, KB)] = c;
    }
    for (int o = 16; o; o >>= 1) sq += __shfl_xor_sync(0xFFFFFFFFu, sq, o);
    if (bias && lane == 0) bias[r] = l2 ? sq : 0;
}

// ---- exact re-scoring + verification: one warp per query ----------------------------------------------------------
struct RescoreParams {
    const float* cand_key;    // [nq_padded][nsplit][KC], nsplit * KC <= FLAT_CMAX
    const uint32_t* cand_id;
    uint32_t nsplit, nq, k, n;
    const float* qnorm;       // [nq] ||q||
    const unsigned int* xmax_bits;
    uint64_t* out_ids;        // [nq][k]
    float* out_dists;
    uint32_t* unverified;     // list of query indices that need the exact scan
    uint32_t* n_unverified;
    float ksign;
    int data_rounded;         // the base vectors were float32 (rounded to fp16 for the GEMM)
    int data_int;             // the base vectors are int8 / uint8 (exact in fp16; the bias |x|^2 is rounded once)
};

// Shared memory of the rescoring kernel: the staged query, then candidate ids, approximate and exact keys.
template <int OP> __host__ __device__ inline size_t flat_rescore_qbytes(uint32_t qstride) {
    return OP >= OP_L2I ? qstride : size_t(qstride) * 4;   // (qstride is a multiple of 16)
}
template <int OP> inline size_t flat_rescore_smem(uint32_t qstride) {
    return flat_rescore_qbytes<OP>(qstride) + size_t(FLAT_CMAX) * 4 * 3;
}

template <int ROWT, int OP, int KC>
__global__ void __launch_bounds__(32, 16) flat_rescore_kernel(const __grid_constant__ SearchParams p,
                                                             const __grid_constant__ RescoreParams rp) {
    constexpr bool kInt = (OP >= OP_L2I);   // the integer GEMM's candidates: exact keys, (key, id) lists
    constexpr int G = kInt ? 4 : 16 / Row<ROWT>::LPT;
    constexpr int GROUPS = 32 / G;
    // rows per group and pass: two, but one for integer rows under the float operators (no spills in 128 registers)
    constexpr int NR = (ROWT == SVSB200_I8 || ROWT == SVSB200_U8) && !kInt ? 1 : 2;
    constexpr unsigned FULL = 0xFFFFFFFFu;
    constexpr uint32_t CMAX = FLAT_CMAX;
    extern __shared__ __align__(16) unsigned char smem_raw[];
    float* q_s = reinterpret_cast<float*>(smem_raw);                   // qstride floats (integer: qstride codes)
    uint32_t* cid = reinterpret_cast<uint32_t*>(smem_raw + flat_rescore_qbytes<OP>(p.qstride));   // [CMAX]
    float* akey = reinterpret_cast<float*>(cid + CMAX);               // [CMAX] approximate keys (integer: ordered keys)
    float* ekey = akey + CMAX;                                        // [CMAX] exact keys
    const int lane = threadIdx.x;
    const int g = lane / G, t = lane % G;
    const uint32_t q = blockIdx.x;
    if (q >= rp.nq) return;
    const uint32_t total = rp.nsplit * uint32_t(KC);
    const uint32_t* okey = reinterpret_cast<const uint32_t*>(rp.cand_key);
    // candidates of every base range; T = the smallest per-range list maximum (every excluded row is >= it)
    float T = INFINITY;
    uint64_t Tp = ~uint64_t(0);   // integer: the smallest list-maximum (key, id) pair
    for (uint32_t s = 0; s < rp.nsplit; ++s) {
        if constexpr (kInt) {
            uint64_t mx = 0;
            for (uint32_t e = lane; e < uint32_t(KC); e += 32) {
                const size_t o = (size_t(q) * rp.nsplit + s) * uint32_t(KC) + e;
                mx = max(mx, (uint64_t(okey[o]) << 32) | rp.cand_id[o]);
            }
            Tp = min(Tp, flat_pair_max(mx));
        } else {
            float mx = -INFINITY;
            for (uint32_t e = lane; e < uint32_t(KC); e += 32) mx = fmaxf(mx, rp.cand_key[(size_t(q) * rp.nsplit + s) * uint32_t(KC) + e]);
            for (int o = 16; o; o >>= 1) mx = fmaxf(mx, __shfl_xor_sync(FULL, mx, o));
            T = fminf(T, mx);
        }
    }
    uint32_t C = 0;   // valid candidates, compacted
    for (uint32_t i0 = 0; i0 < total; i0 += 32) {
        const uint32_t i = i0 + lane;
        const uint32_t id = i < total ? rp.cand_id[size_t(q) * total + i] : 0xFFFFFFFFu;
        const bool ok = id < rp.n;
        const unsigned m = __ballot_sync(FULL, ok);
        if (ok) {
            const uint32_t o = C + __popc(m & ((1u << lane) - 1u));
            cid[o] = id;
            if constexpr (kInt) reinterpret_cast<uint32_t*>(akey)[o] = okey[size_t(q) * total + i];
            else akey[o] = rp.cand_key[size_t(q) * total + i];
        }
        C += __popc(m);
    }
    __syncwarp();
    if constexpr (kInt) {
        const uint32_t* src = reinterpret_cast<const uint32_t*>(p.qcodes + size_t(q) * p.qstride);
        for (uint32_t i = lane; i < p.qstride / 4; i += 32) reinterpret_cast<uint32_t*>(q_s)[i] = src[i];
    } else {
        for (uint32_t i = lane; i < p.qstride; i += 32) q_s[i] = p.qf[size_t(q) * p.qstride + i];
    }
    __syncwarp();
    const float aux0 = p.qaux[2 * size_t(q)], aux1 = p.qaux[2 * size_t(q) + 1];
    for (uint32_t base = 0; base < C; base += NR * GROUPS)
        eval_pass<ROWT, OP, 0, NR, 1, true>(p, q_s, reinterpret_cast<const char*>(p.vectors), cid, ekey, base, C, g, t, aux0, aux1,
                                           rp.ksign);
    __syncwarp();
    if constexpr (kInt) {
        // rank of every candidate by (exact key, id); F(K) = float(v(K)), v(K) = |q|^2 + K (L2) or K (header)
        const int64_t qq = OP == OP_L2I ? int64_t(__float_as_int(aux1)) : 0;
        bool mismatch = false;
        float kth_key = -INFINITY;
        uint64_t kth_pair = 0;
        for (uint32_t i = lane; i < C; i += 32) {
            const float ke = ekey[i];
            const uint32_t id = cid[i], ok_i = reinterpret_cast<const uint32_t*>(akey)[i];
            uint32_t re = 0;
            for (uint32_t j = 0; j < C; ++j) {
                const float kj = ekey[j];
                re += (kj < ke) || (kj == ke && cid[j] < id);
            }
            if (re < rp.k) {
                rp.out_ids[size_t(q) * rp.k + re] = id;
                rp.out_dists[size_t(q) * rp.k + re] = ke * rp.ksign;
            }
            // the GEMM's key must give the rescored distance
            mismatch |= __ll2float_rn(qq + int32_t(ok_i ^ 0x80000000u)) != ke;
            if (re == rp.k - 1) {
                kth_key = ke;
                kth_pair = (uint64_t(ok_i) << 32) | id;
            }
        }
        mismatch = __any_sync(FULL, mismatch);
        for (int o = 16; o; o >>= 1) kth_key = fmaxf(kth_key, __shfl_xor_sync(FULL, kth_key, o));
        kth_pair = flat_pair_max(kth_pair);
        const int64_t vT = qq + int32_t(uint32_t(Tp >> 32) ^ 0x80000000u);
        const bool exact_at_T = vT < (int64_t(1) << 24) && vT > -(int64_t(1) << 24);
        const bool verified = C >= rp.k && !mismatch && (__ll2float_rn(vT) > kth_key || (exact_at_T && Tp > kth_pair));
        if (lane == 0 && !verified) rp.unverified[atomicAdd(rp.n_unverified, 1u)] = q;
        return;
    }
    // rank of every candidate by (exact key, id) and by approximate key: C <= FLAT_CMAX
    float kth_approx = INFINITY;
    for (uint32_t i = lane; i < C; i += 32) {
        const float ke = ekey[i], ka = akey[i];
        const uint32_t id = cid[i];
        uint32_t re = 0, ra = 0;
        for (uint32_t j = 0; j < C; ++j) {
            const float kj = ekey[j];
            re += (kj < ke) || (kj == ke && cid[j] < id);
            const float aj = akey[j];
            ra += (aj < ka) || (aj == ka && j < i);
        }
        if (re < rp.k) {
            rp.out_ids[size_t(q) * rp.k + re] = id;
            rp.out_dists[size_t(q) * rp.k + re] = ke * rp.ksign;
        }
        if (ra == rp.k - 1) kth_approx = ka;
    }
    for (int o = 16; o; o >>= 1) kth_approx = fminf(kth_approx, __shfl_xor_sync(FULL, kth_approx, o));
    // |approximate key - key| <= E(q) (header): excluded rows are provably outside the exact top k iff T > kth + 2E
    // Every operation of E and of kth + 2E rounds up, so neither can underflow or fall below the true bound.  A query or
    // base with an element that overflowed fp16 has a norm of +inf (flat_tile_kernel) and is never verified.
    const float qn = rp.qnorm[q], xm = __uint_as_float(*rp.xmax_bits);
    const int q_rounded = int(p.scale) - rp.data_rounded;   // p.scale: operands that were rounded to fp16 (0, 1 or 2)
    const float sd = __fmul_ru(2.98023223876953125e-8f, __fsqrt_ru(float(p.dim)));            // 2^-25 sqrt(dim)
    const float dq = q_rounded ? __fadd_ru(__fmul_ru(4.8828125e-4f, qn), sd) : 0.0f;          // ||q~ - q||
    const float dx = rp.data_rounded ? __fadd_ru(__fmul_ru(4.8828125e-4f, xm), sd) : 0.0f;    // ||x~ - x||
    const float qh = __fadd_ru(qn, dq), xh = __fadd_ru(xm, dx);                                // >= ||q~||, ||x~||
    float E = __fadd_ru(__fadd_ru(__fmul_ru(dq, xh), __fmul_ru(qn, dx)),
                        __fmul_ru(__fmul_ru(float(p.dim) * 2.384185791015625e-7f, qh), xh));   // E_ip, dim 2^-22
    if (!p.greater)
        E = __fadd_ru(__fadd_ru(__fmul_ru(2.0f, E), __fmul_ru(dx, __fadd_ru(xm, xh))),        // + ||x~|^2 - |x|^2|
                      rp.data_int ? __fmul_ru(__fmul_ru(1.1920928955078125e-7f, xm), xm) : 0.0f);   // 2^-23 (header)
    E = __fmul_ru(E, 1.0001f);
    const bool finite = isfinite(qn) && isfinite(xm) && isfinite(E);
    const bool verified = C >= rp.k && finite && T > __fadd_ru(kth_approx, __fmul_ru(2.0f, E));
    if (lane == 0 && !verified) rp.unverified[atomicAdd(rp.n_unverified, 1u)] = q;
}

// copies rows `idx[i]` of a dense [*, row_bytes] array to row i (gather) or row i to rows idx[i] (scatter)
__global__ void flat_move_rows_kernel(const char* __restrict__ src, char* __restrict__ dst, const uint32_t* __restrict__ idx,
                                      const uint32_t* __restrict__ count, uint32_t row_bytes, int scatter) {
    const uint32_t i = blockIdx.x;
    if (i >= *count) return;
    const uint32_t r = idx[i];
    const char* s = src + size_t(scatter ? i : r) * row_bytes;
    char* d = dst + size_t(scatter ? r : i) * row_bytes;
    for (uint32_t b = threadIdx.x; b < row_bytes; b += blockDim.x) d[b] = s[b];
}

// ---- dynamic flat index: upkeep of the base tiles -----------------------------------------------------------------
// Rows i < count of blobs tiled 8 rows to a tile (flat_tile_rows with tile_rows = 8), with their bias and norms, ->
// slots slots[i] (slots NULL: first + i) of base blobs tiled FLAT_BN rows to a tile.  `src` NULL turns the slots into
// padding rows: zero blobs (so that an integer key stays the empty key) and the bias `empty_bias`.  A row is KB blobs
// of four 16-byte chunks in either operand kind; one warp per row.
__global__ void flat_place_rows_kernel(const uint4* __restrict__ src, const uint32_t* __restrict__ src_bias,
                                       const float* __restrict__ src_norms, const uint32_t* __restrict__ slots, uint32_t first,
                                       uint32_t count, uint32_t KB, uint32_t empty_bias, uint4* __restrict__ dst,
                                       uint32_t* __restrict__ bias, float* __restrict__ norms) {
    const uint32_t i = blockIdx.x * (blockDim.x / 32) + threadIdx.x / 32;
    const uint32_t lane = threadIdx.x & 31;
    if (i >= count) return;
    const uint32_t s = slots ? slots[i] : first + i;
    for (uint32_t j = lane; j < 4 * KB; j += 32) {
        const uint4 v = src ? src[flat_blob_offset<16>(i / 8, i % 8, 16 * j, 8, KB) / 16] : make_uint4(0u, 0u, 0u, 0u);
        dst[flat_blob_offset<16>(s / FLAT_BN, s % FLAT_BN, 16 * j, FLAT_BN, KB) / 16] = v;
    }
    if (lane == 0) {
        bias[s] = src ? src_bias[i] : empty_bias;
        if (norms) norms[s] = src ? src_norms[i] : 0.f;
    }
}

// Xmax of a dynamic flat index: the largest norm over its Valid slots (norms are >= 0 or +inf, so their bits order as
// unsigned integers).  *xmax_bits is 0 before the launch.
__global__ void flat_masked_xmax_kernel(const float* __restrict__ norms, const uint8_t* __restrict__ status, uint32_t n,
                                        unsigned int* __restrict__ xmax_bits) {
    unsigned int m = 0;
    for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x)
        if (status[i] == SLOT_VALID) m = max(m, __float_as_uint(norms[i]));
    m = __reduce_max_sync(0xFFFFFFFFu, m);
    if ((threadIdx.x & 31) == 0 && m) atomicMax(xmax_bits, m);
}

// ---- filtered search: the per-call mask (all of it in the scratch) ---------------------------------------------------
// Row i is allowed iff bit i % 32 of bitmap word i / 32 is set, i < n and (a dynamic flat index) its slot is Valid:
// status[i] = Valid / Empty, and the allowed rows again as bitmap words (zero past n).  One warp per word.
__global__ void flat_filter_rows_kernel(const uint32_t* __restrict__ bitmap, const uint8_t* __restrict__ slot_status,
                                        uint32_t n, uint8_t* __restrict__ status, uint32_t* __restrict__ words) {
    const uint32_t w = blockIdx.x * (blockDim.x / 32) + threadIdx.x / 32, lane = threadIdx.x & 31;
    if (w >= (n + 31) / 32) return;
    const uint32_t i = 32 * w + lane;
    const bool ok = i < n && ((__ldg(bitmap + w) >> lane) & 1u) && (!slot_status || slot_status[i] == SLOT_VALID);
    const uint32_t m = __ballot_sync(0xFFFFFFFFu, ok);
    if (i < n) status[i] = ok ? SLOT_VALID : SLOT_EMPTY;
    if (lane == 0) words[w] = m;
}

// The set bits of `words` as ascending row ids: ids[0 .. *count).  One block; each thread takes a run of words.
__global__ void __launch_bounds__(1024) flat_compact_kernel(const uint32_t* __restrict__ words, uint32_t nwords,
                                                            uint32_t* __restrict__ ids, uint32_t* __restrict__ count) {
    __shared__ uint32_t warp_total[32];
    const uint32_t per = (nwords + blockDim.x - 1) / blockDim.x;
    const uint32_t w0 = min(nwords, threadIdx.x * per), w1 = min(nwords, w0 + per);
    const uint32_t lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    uint32_t c = 0;
    for (uint32_t w = w0; w < w1; ++w) c += __popc(words[w]);
    uint32_t x = c;   // inclusive prefix over the warp, then over the warps
    for (uint32_t o = 1; o < 32; o <<= 1) {
        const uint32_t y = __shfl_up_sync(0xFFFFFFFFu, x, o);
        if (lane >= o) x += y;
    }
    if (lane == 31) warp_total[warp] = x;
    __syncthreads();
    if (warp == 0) {
        uint32_t t = lane < blockDim.x / 32 ? warp_total[lane] : 0u;
        for (uint32_t o = 1; o < 32; o <<= 1) {
            const uint32_t y = __shfl_up_sync(0xFFFFFFFFu, t, o);
            if (lane >= o) t += y;
        }
        warp_total[lane] = t;
    }
    __syncthreads();
    uint32_t o = x - c + (warp ? warp_total[warp - 1] : 0u);
    for (uint32_t w = w0; w < w1; ++w)
        for (uint32_t b = words[w]; b; b &= b - 1) ids[o++] = 32 * w + uint32_t(__ffs(int(b)) - 1);
    if (threadIdx.x == blockDim.x - 1) *count = o;
}

// The GEMM's bias for this call: row i keeps bias[i] when it is allowed, every other column gets the empty bias.
__global__ void flat_mask_bias_kernel(const uint32_t* __restrict__ bias, const uint32_t* __restrict__ words, uint32_t n,
                                      uint32_t rows, uint32_t empty_bias, uint32_t* __restrict__ out) {
    for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < rows; i += gridDim.x * blockDim.x)
        out[i] = i < n && ((words[i >> 5] >> (i & 31)) & 1u) ? bias[i] : empty_bias;
}

// Ids of a search over the gathered allowed rows -> row ids (`rows`, the compacted ids) -> external ids (`ext_ids`,
// a dynamic flat index).  Padding ids stay all-ones.
__global__ void flat_unmap_ids_kernel(uint64_t* __restrict__ ids, size_t count, const uint32_t* __restrict__ rows,
                                      const uint64_t* __restrict__ ext_ids) {
    for (size_t i = size_t(blockIdx.x) * blockDim.x + threadIdx.x; i < count; i += size_t(gridDim.x) * blockDim.x) {
        const uint64_t id = ids[i];
        if (id == ~uint64_t(0)) continue;
        const uint32_t r = rows[id];
        ids[i] = ext_ids ? ext_ids[r] : r;
    }
}

// The filtered searches pad with +inf for every metric (the scan pads inner product with -inf).
__global__ void flat_pad_inf_kernel(const uint64_t* __restrict__ ids, float* __restrict__ dists, size_t count) {
    for (size_t i = size_t(blockIdx.x) * blockDim.x + threadIdx.x; i < count; i += size_t(gridDim.x) * blockDim.x)
        if (ids[i] == ~uint64_t(0)) dists[i] = INFINITY;
}

// ---- launchers ------------------------------------------------------------------------------------------------------
// Rows -> the operand blobs of `kind`: flat_tile_kernel (fp16) or flat_tile8_kernel (8-bit, which has no norms).
// `bias` (float, or int32 for 8-bit blobs), `norms` and `max_norm_bits` may be NULL.
static cudaError_t flat_tile_rows(int kind, int srct, const void* src, uint32_t row_stride, uint32_t n, uint32_t dim,
                                  uint32_t tile_rows, int l2, void* dst_tiles, void* bias, float* norms,
                                  unsigned int* max_norm_bits, cudaStream_t stream) {
    const uint32_t KB = flat_kblocks(kind, dim);
    const uint32_t rows_padded = (n + tile_rows - 1) / tile_rows * tile_rows;
    cudaError_t err = cudaMemsetAsync(dst_tiles, 0, size_t(rows_padded) * KB * FLAT_BK * 2, stream);
    if (err != cudaSuccess) return err;
    const LaunchConfig cfg{int((rows_padded + 7) / 8), 8, 0, stream};
    const char* s = static_cast<const char*>(src);
    if (kind == FLAT_F16)
        return dispatch(DataRows{}, srct, [&](auto t) {
            return launch_kernel(flat_tile_kernel<decltype(t)::value>, cfg, cfg.grid, false, s, row_stride, n, dim, tile_rows,
                                 KB, 1.0f, l2, static_cast<__half*>(dst_tiles), static_cast<float*>(bias), norms,
                                 max_norm_bits);
        });
    return dispatch(IntList<SVSB200_I8, SVSB200_U8>{}, srct, [&](auto t) {
        return launch_kernel(flat_tile8_kernel<decltype(t)::value>, cfg, cfg.grid, false, s, row_stride, n, dim, tile_rows, KB,
                             l2, static_cast<uint8_t*>(dst_tiles), static_cast<int*>(bias));
    });
}

// Lists of absent pieces: (empty key, no id).  `key_bits`: +inf (fp16 lists) or 0xFFFFFFFF (integer lists).
__global__ void flat_fill_kernel(uint32_t* __restrict__ key, uint32_t key_bits, uint32_t* __restrict__ id, size_t count) {
    for (size_t i = size_t(blockIdx.x) * blockDim.x + threadIdx.x; i < count; i += size_t(gridDim.x) * blockDim.x) {
        key[i] = key_bits;
        id[i] = 0xFFFFFFFFu;
    }
}

// Grid size, sharing factor and lists per query for a problem with lists of `kc` entries (FLAT_KC: two per piece,
// FLAT_KC_DEEP: one): as many CTAs as SMs in groups of R, fewer segments while a query tile would be cut into more
// pieces than the rescoring kernel holds candidates for (small batches over a large base).
static void flat_plan(uint32_t mtiles, uint32_t ntiles, uint32_t sm_count, uint32_t kc, uint32_t* ctas, uint32_t* share,
                      uint32_t* nlists) {
    const uint32_t per_piece = kc == FLAT_KC ? 2 : 1;
    const uint32_t R = mtiles >= 8 ? 4 : mtiles >= 4 ? 2 : 1;
    const uint32_t ngroups = (mtiles + R - 1) / R;
    const uint64_t total = uint64_t(ngroups) * ntiles;
    uint32_t g = uint32_t(std::min<uint64_t>(std::max(1u, sm_count / R), total));
    for (;; --g) {
        uint32_t pieces = 1;
        for (uint32_t m = 0; m < ngroups; ++m)
            pieces = std::max(pieces, flat_cta_of_tile(uint64_t(m + 1) * ntiles - 1, total, g) -
                                          flat_cta_of_tile(uint64_t(m) * ntiles, total, g) + 1);
        if (per_piece * pieces * kc <= FLAT_CMAX || g == 1) {
            *ctas = g * R;
            *share = R;
            *nlists = per_piece * pieces;
            return;
        }
    }
}

static cudaError_t flat_gemm_topk(int kind, int kc, const void* a_tiles, const void* b_tiles, const void* b_bias, uint32_t KB, uint32_t ntiles,
                                  uint32_t mtiles, uint32_t ctas, uint32_t share, uint32_t nlists, float key_scale, float* cand_key,
                                  uint32_t* cand_id, uint32_t* progress, cudaStream_t stream, bool masked = false) {
    FlatParams fp{};
    fp.a_tiles = static_cast<const __half*>(a_tiles);
    fp.b_tiles = static_cast<const __half*>(b_tiles);
    fp.b_bias = static_cast<const float*>(b_bias);
    fp.KB = KB;
    fp.ntiles = ntiles;
    fp.mtiles = mtiles;
    fp.nlists = nlists;
    fp.share = share;
    fp.progress = progress;
    fp.key_scale = key_scale;
    fp.cand_key = cand_key;
    fp.cand_id = cand_id;
    const size_t entries = size_t(mtiles) * FLAT_BM * nlists * kc;
    const uint32_t empty_key = kind == FLAT_F16 ? 0x7F800000u : 0xFFFFFFFFu;
    flat_fill_kernel<<<unsigned(std::min<size_t>(4096, (entries + 255) / 256)), 256, 0, stream>>>(
        reinterpret_cast<uint32_t*>(cand_key), empty_key, cand_id, entries);
    count_launch();
    return dispatch(IntList<FLAT_KC, FLAT_KC_DEEP>{}, kc, [&](auto c) {
        constexpr int KC = decltype(c)::value;
        const LaunchConfig cfg{int(ctas), int(FLAT_THREADS / 32), FlatShape<KC>::SMEM, stream};
        return dispatch(IntList<FLAT_F16, FLAT_S8, FLAT_U8>{}, kind, [&](auto k) {
            constexpr int KIND = decltype(k)::value;
            // (fp16 keys need no mask: fmaf(scale, s, +inf) is +inf or NaN, which no list is offered)
            if constexpr (KIND != FLAT_F16)
                if (masked) return launch_kernel(flat_gemm_topk_kernel<KIND, uint32_t(KC), true>, cfg, ctas, true, fp);
            return launch_kernel(flat_gemm_topk_kernel<KIND, uint32_t(KC)>, cfg, ctas, true, fp);
        });
    });
}

static cudaError_t flat_rescore(int rowt, int op, int kc, const SearchParams& p, const float* cand_key, const uint32_t* cand_id, uint32_t nsplit,
                                uint32_t nq, uint32_t k, const float* qnorm, const unsigned int* xmax_bits, uint64_t* out_ids,
                                float* out_dists, uint32_t* unverified, uint32_t* n_unverified, cudaStream_t stream) {
    RescoreParams rp{};
    rp.cand_key = cand_key;
    rp.cand_id = cand_id;
    rp.nsplit = nsplit;
    rp.nq = nq;
    rp.k = k;
    rp.n = p.n;
    rp.qnorm = qnorm;
    rp.xmax_bits = xmax_bits;
    rp.out_ids = out_ids;
    rp.out_dists = out_dists;
    rp.unverified = unverified;
    rp.n_unverified = n_unverified;
    rp.ksign = p.greater ? -1.0f : 1.0f;
    rp.data_rounded = rowt == SVSB200_F32;
    rp.data_int = rowt == SVSB200_I8 || rowt == SVSB200_U8;
    // rows wider than about 9 000 elements need more than the default 48 KB of shared memory: the kernel opts in
    return dispatch(IntList<FLAT_KC, FLAT_KC_DEEP>{}, kc, [&](auto c) {
        return dispatch(DataRows{}, rowt, [&](auto t) {
            return dispatch(RescoreOps<decltype(t)::value>{}, op, [&](auto o) {
                const LaunchConfig cfg{int(nq), 1, flat_rescore_smem<decltype(o)::value>(p.qstride), stream};
                return launch_kernel(flat_rescore_kernel<decltype(t)::value, decltype(o)::value, decltype(c)::value>, cfg,
                                     nq, cfg.smem_bytes > 48 * 1024, p, rp);
            });
        });
    });
}

static cudaError_t flat_move_rows(const void* src, void* dst, const uint32_t* idx, const uint32_t* count, uint32_t max_count,
                                  uint32_t row_bytes, int scatter, cudaStream_t stream) {
    if (max_count == 0) return cudaSuccess;
    flat_move_rows_kernel<<<max_count, 128, 0, stream>>>(static_cast<const char*>(src), static_cast<char*>(dst), idx, count,
                                                        row_bytes, scatter);
    count_launch();
    return cudaGetLastError();
}

// The bias of a padding row: +inf (fp16 keys) or INT32_MAX (integer keys).
static uint32_t flat_empty_bias(int kind) { return kind == FLAT_F16 ? 0x7F800000u : 0x7FFFFFFFu; }

// flat_place_rows_kernel into `base` (tiles of operand kind `kind`); src NULL makes the slots padding rows.
static cudaError_t flat_place_rows(int kind, uint32_t dim, const void* src, const void* src_bias, const float* src_norms,
                                   const uint32_t* slots, uint32_t first, uint32_t count, Replica::FlatBase& base,
                                   cudaStream_t stream) {
    if (count == 0) return cudaSuccess;
    flat_place_rows_kernel<<<(count + 7) / 8, 256, 0, stream>>>(
        static_cast<const uint4*>(src), static_cast<const uint32_t*>(src_bias), src_norms, slots, first, count,
        flat_kblocks(kind, dim), flat_empty_bias(kind), reinterpret_cast<uint4*>(base.tiles.ptr),
        reinterpret_cast<uint32_t*>(base.bias.ptr), base.norms.ptr);
    count_launch();
    return cudaGetLastError();
}

// The deep lists of one query tile keep at most FLAT_CMAX / FLAT_KC_DEEP = 7 CTAs busy: batches of one or two tiles
// run faster on the scan (DESIGN.md §9b), so the deep lists need more than 2 FLAT_BM queries.
static bool flat_deep_batch(size_t nq) { return nq > 2 * FLAT_BM; }

// The base tiles and bias of operand kind `kind` (and, for fp16 tiles, flat_xmax), built once per replica.
static int ensure_flat_base(svsb200_index* ix, Replica* rep, int kind, cudaStream_t stream) {
    Replica::FlatBase& base = kind == FLAT_F16 ? rep->flat_f16 : rep->flat_int;
    std::lock_guard<std::mutex> lock(rep->mu);
    if (base.tiles.ptr) return 0;
    const uint32_t n = uint32_t(ix->n), dim = uint32_t(ix->dim), ntiles = (n + FLAT_BN - 1) / FLAT_BN;
    CUDA_TRY(base.tiles.ensure(size_t(ntiles) * FLAT_BN * flat_kblocks(kind, dim) * FLAT_BK * 2));
    CUDA_TRY(base.bias.ensure(size_t(ntiles) * FLAT_BN));
    if (kind == FLAT_F16) {
        CUDA_TRY(rep->flat_xmax.ensure(1));
        CUDA_TRY(cudaMemsetAsync(rep->flat_xmax.ptr, 0, 4, stream));
    }
    // dynamic flat index: the norm of every slot, flat_xmax being taken over the Valid ones (ensure_slots_xmax)
    float* norms = nullptr;
    if (ix->slot_mask && kind == FLAT_F16) {
        CUDA_TRY(base.norms.ensure(size_t(ntiles) * FLAT_BN));
        norms = base.norms.ptr;
        rep->flat_xmax_stale = true;
    }
    CUDA_TRY(flat_tile_rows(kind, ix->dtype, rep->d_vectors.ptr, ix->row_stride, n, dim, FLAT_BN, ix->metric == SVSB200_L2,
                            base.tiles.ptr, base.bias.ptr, norms, kind == FLAT_F16 && !norms ? rep->flat_xmax.ptr : nullptr,
                            stream));
    if (ix->slot_mask) {   // slots that are not Valid become padding rows
        std::vector<uint32_t> empty;
        for (uint32_t s = 0; s < n; ++s)
            if (ix->slots.status[s] != SLOT_VALID) empty.push_back(s);
        DeviceBuffer<uint32_t> d_empty;
        CUDA_TRY(d_empty.ensure(std::max<size_t>(empty.size(), 1)));
        CUDA_TRY(cudaMemcpyAsync(d_empty.ptr, empty.data(), empty.size() * 4, cudaMemcpyHostToDevice, stream));
        CUDA_TRY(flat_place_rows(kind, dim, nullptr, nullptr, nullptr, d_empty.ptr, 0, uint32_t(empty.size()), base, stream));
        CUDA_TRY(cudaStreamSynchronize(stream));   // (before d_empty goes)
    }
    CUDA_TRY(cudaStreamSynchronize(stream));
    return 0;
}

// flat_xmax of a dynamic flat index, retaken over the Valid slots when they changed since it was last taken (a stale
// maximum would still be sound, but it could keep sending every query to the scan after the row that set it is gone).
static int ensure_slots_xmax(svsb200_index* ix, Replica* rep, cudaStream_t stream) {
    std::lock_guard<std::mutex> lock(rep->mu);
    if (!rep->flat_xmax_stale) return 0;
    const uint32_t n = uint32_t(ix->n);
    CUDA_TRY(cudaMemsetAsync(rep->flat_xmax.ptr, 0, 4, stream));
    const unsigned grid = unsigned(std::max<size_t>(1, std::min<size_t>((n + 255) / 256, size_t(rep->sm_count) * 4)));
    flat_masked_xmax_kernel<<<grid, 256, 0, stream>>>(rep->flat_f16.norms.ptr, rep->d_status.ptr, n, rep->flat_xmax.ptr);
    count_launch();
    CUDA_TRY(cudaGetLastError());
    CUDA_TRY(cudaStreamSynchronize(stream));
    rep->flat_xmax_stale = false;
    return 0;
}

// Shared body of the tensor-core flat search: device buffers in, device buffers out, enqueued on sc->stream except
// for one synchronisation (the count of queries that need the exact-scan fallback).  `max_kc` is the deepest list the
// caller allows: k + 8 <= FLAT_KC runs the FLAT_KC lists, k + 8 <= FLAT_KC_DEEP (Flat handles only) the deep ones.
// Ids are row numbers (dynamic flat index: slots; flat_on_device maps them to external ids).
// Filtered (flat_filtered_on_device): `row_bits` / `row_status` mark the allowed rows (a dynamic index's: allowed and
// Valid) as a bitmap and as status bytes, both in the scratch.  The GEMM reads a scratch copy of the bias whose other
// columns are empty, so they are never offered to a list; the scans skip them through the status bytes.
static int flat_rows_on_device(svsb200_index* ix, Replica* rep, Scratch* sc, const void* d_queries, int qdtype, size_t nq,
                               size_t k, uint64_t* d_out_ids, float* d_out_dists, uint32_t* fallback_queries,
                               uint32_t max_kc, const uint32_t* row_bits = nullptr, const uint8_t* row_status = nullptr) {
    if (fallback_queries) *fallback_queries = 0;
    if (nq == 0) return 0;
    cudaStream_t stream = sc->stream;
    const bool int_data = ix->dtype == SVSB200_I8 || ix->dtype == SVSB200_U8;
    const uint32_t kc = k + 8 <= FLAT_KC ? FLAT_KC : FLAT_KC_DEEP;
    const bool shape_ok = ix->storage == SVSB200_PLAIN && ix->metric != SVSB200_COSINE && k + 8 <= max_kc && ix->n >= 512 &&
                          (kc == FLAT_KC || flat_deep_batch(nq));
    // the integer GEMM: (int8, int8) / (uint8, uint8), every int32 sum exact
    const bool int_gemm = shape_ok && int_data && qdtype == ix->dtype && ix->dim <= FLAT_INT_MAX_DIM &&
                          flat_rescore_smem<OP_L2I>(query_stride(ix->dim)) <= kSmemOptInMax;
    // the fp16 GEMM: float32 / float16 data with float32 / float16 queries, integer data with float32 queries; rows
    // whose staged float query does not fit the rescoring kernel's shared memory keep the scan
    const bool f16_gemm = shape_ok && (int_data ? qdtype == SVSB200_F32 : (qdtype == SVSB200_F32 || qdtype == SVSB200_F16)) &&
                          flat_rescore_smem<OP_L2F>(query_stride(ix->dim)) <= kSmemOptInMax;
    if (!int_gemm && !f16_gemm) {   // shapes outside the GEMM paths: the exact scan
        if (fallback_queries) *fallback_queries = uint32_t(nq);
        return search_on_device(ix, rep, sc, d_queries, qdtype, nq, k, k, k, d_out_ids, 8, d_out_dists, stream, true,
                                row_status);
    }
    const uint32_t n = uint32_t(ix->n), dim = uint32_t(ix->dim);
    const int kind = !int_gemm ? FLAT_F16 : ix->dtype == SVSB200_I8 ? FLAT_S8 : FLAT_U8;
    const uint32_t KB = flat_kblocks(kind, dim);
    const uint32_t ntiles = (n + 255) / 256, mtiles = uint32_t((nq + 127) / 128);
    const int l2 = ix->metric == SVSB200_L2;
    if (int rc = ensure_flat_base(ix, rep, kind, stream)) return rc;
    if (ix->slot_mask && kind == FLAT_F16)
        if (int rc = ensure_slots_xmax(ix, rep, stream)) return rc;
    const Replica::FlatBase& base = kind == FLAT_F16 ? rep->flat_f16 : rep->flat_int;
    const void* bias = base.bias.ptr;
    if (row_bits) {
        CUDA_TRY(sc->flt_bias.ensure(size_t(ntiles) * FLAT_BN));
        const unsigned grid = unsigned(std::min<size_t>((size_t(ntiles) * FLAT_BN + 255) / 256, size_t(rep->sm_count) * 8));
        flat_mask_bias_kernel<<<grid, 256, 0, stream>>>(reinterpret_cast<const uint32_t*>(base.bias.ptr), row_bits, n,
                                                         ntiles * FLAT_BN, flat_empty_bias(kind), sc->flt_bias.ptr);
        count_launch();
        CUDA_TRY(cudaGetLastError());
        bias = sc->flt_bias.ptr;
    }
    // one CTA per SM over equal runs of output tiles; `nsplit` = candidate lists per query (flat_plan)
    uint32_t flat_ctas = 1, flat_share = 1, nsplit = 2;
    flat_plan(mtiles, ntiles, uint32_t(rep->sm_count), kc, &flat_ctas, &flat_share, &nsplit);
    const size_t qrow = size_t(dim) * esize(qdtype);
    CUDA_TRY(sc->flat_a.ensure(size_t(mtiles) * 128 * KB * 32 * 2));
    CUDA_TRY(sc->flat_qnorm.ensure(size_t(mtiles) * 128));
    CUDA_TRY(sc->flat_ckey.ensure(size_t(mtiles) * 128 * nsplit * kc));
    CUDA_TRY(sc->flat_cid.ensure(size_t(mtiles) * 128 * nsplit * kc));
    CUDA_TRY(sc->flat_unv.ensure(nq + 1));
    CUDA_TRY(sc->flat_progress.ensure(flat_ctas));
    CUDA_TRY(cudaMemsetAsync(sc->flat_progress.ptr, 0, size_t(flat_ctas) * 4, stream));
    // (query norms: the fp16 path's error bound only)
    CUDA_TRY(flat_tile_rows(kind, qdtype, d_queries, uint32_t(qrow), uint32_t(nq), dim, 128, 0, sc->flat_a.ptr, nullptr,
                            kind == FLAT_F16 ? sc->flat_qnorm.ptr : nullptr, nullptr, stream));
    CUDA_TRY(flat_gemm_topk(kind, kc, sc->flat_a.ptr, base.tiles.ptr, bias, KB, ntiles, mtiles, flat_ctas, flat_share, nsplit,
                            l2 ? -2.0f : -1.0f, sc->flat_ckey.ptr, sc->flat_cid.ptr, sc->flat_progress.ptr, stream,
                            row_bits != nullptr));
    // exact re-scoring with the search path's distance code: prepared queries as for a search
    if (int rc = prepare_queries(ix, rep, sc, d_queries, qdtype, nq, int_gemm ? PREP_INT : PREP_FLOAT, stream)) return rc;
    SearchParams p{};
    p.vectors = rep->d_vectors.ptr;
    p.n = n;
    p.dim = dim;
    p.row_stride = ix->row_stride;
    p.greater = !l2;
    p.qf = sc->q_f32.ptr;
    p.qcodes = sc->q_codes.ptr;
    p.qaux = sc->q_aux.ptr;
    p.qstride = query_stride(dim);
    p.nq = uint32_t(nq);
    p.k = uint32_t(k);
    CUDA_TRY(cudaMemsetAsync(sc->flat_unv.ptr, 0, 4, stream));
    // rounding terms of E(q) (file header, fp16 path): float32 queries and float32 data are rounded to fp16
    p.scale = (qdtype == SVSB200_F32 ? 1.0f : 0.0f) + (ix->dtype == SVSB200_F32 ? 1.0f : 0.0f);   // number of rounded operands
    const int op = int_gemm ? (l2 ? OP_L2I : OP_IPI) : (l2 ? OP_L2F : OP_IPF);
    CUDA_TRY(flat_rescore(ix->dtype, op, kc, p, sc->flat_ckey.ptr, sc->flat_cid.ptr, nsplit, uint32_t(nq), uint32_t(k),
                          sc->flat_qnorm.ptr, rep->flat_xmax.ptr, d_out_ids, d_out_dists, sc->flat_unv.ptr + 1, sc->flat_unv.ptr, stream));
    // queries whose bound did not verify: exact scan, results scattered over the rescored rows
    uint32_t nunv = 0;
    CUDA_TRY(cudaMemcpyAsync(&nunv, sc->flat_unv.ptr, 4, cudaMemcpyDeviceToHost, stream));
    CUDA_TRY(cudaStreamSynchronize(stream));
    if (fallback_queries) *fallback_queries = nunv;
    if (nunv) {
        CUDA_TRY(sc->flat_q2.ensure(size_t(nunv) * qrow));
        CUDA_TRY(sc->flat_i2.ensure(size_t(nunv) * k));
        CUDA_TRY(sc->flat_d2.ensure(size_t(nunv) * k));
        CUDA_TRY(flat_move_rows(d_queries, sc->flat_q2.ptr, sc->flat_unv.ptr + 1, sc->flat_unv.ptr, nunv, uint32_t(qrow), 0, stream));
        int rc = search_on_device(ix, rep, sc, sc->flat_q2.ptr, qdtype, nunv, k, k, k, sc->flat_i2.ptr, 8, sc->flat_d2.ptr, stream, true,
                                  row_status);
        if (rc) return rc;
        CUDA_TRY(flat_move_rows(sc->flat_i2.ptr, d_out_ids, sc->flat_unv.ptr + 1, sc->flat_unv.ptr, nunv, uint32_t(k * 8), 1, stream));
        CUDA_TRY(flat_move_rows(sc->flat_d2.ptr, d_out_dists, sc->flat_unv.ptr + 1, sc->flat_unv.ptr, nunv, uint32_t(k * 4), 1, stream));
    }
    return 0;
}

// flat_rows_on_device, with a dynamic flat index's slots mapped to external ids on every route (GEMM, fallback, scan).
static int flat_on_device(svsb200_index* ix, Replica* rep, Scratch* sc, const void* d_queries, int qdtype, size_t nq, size_t k,
                          uint64_t* d_out_ids, float* d_out_dists, uint32_t* fallback_queries, uint32_t max_kc) {
    if (int rc = flat_rows_on_device(ix, rep, sc, d_queries, qdtype, nq, k, d_out_ids, d_out_dists, fallback_queries, max_kc))
        return rc;
    if (ix->slot_mask) CUDA_TRY(slots_to_external(d_out_ids, nq * k, rep->d_ext_ids.ptr, sc->stream));
    return 0;
}

// ---- filtered search (include/svsb200.h, svsb200_flat_index_search_filtered) ----
// Route of a filtered search with `allowed` of `n` rows allowed (svsb200_flat_filter_plan): at most n / FLAT_SPARSE_DIV
// allowed rows are gathered and scanned alone (the sparse route), more run the index's own routing with the disallowed
// rows masked out (the dense route).  DESIGN.md §9d has the measurement behind the divisor.
constexpr size_t FLAT_SPARSE_DIV = 64;
static int flat_filter_route(size_t n, size_t allowed) {
    return allowed * FLAT_SPARSE_DIV <= n ? SVSB200_FLAT_ROUTE_SPARSE : SVSB200_FLAT_ROUTE_DENSE;
}

// The filtered search on device buffers, enqueued on sc->stream apart from one synchronisation for the count of allowed
// rows (and the dense route's own).  Ids are external ids for a dynamic flat index.
static int flat_filtered_on_device(svsb200_index* ix, Replica* rep, Scratch* sc, const void* d_queries, int qdtype, size_t nq,
                                   size_t k, const uint32_t* d_bitmap, uint64_t* d_out_ids, float* d_out_dists,
                                   size_t* out_allowed, uint32_t* fallback_queries) {
    if (fallback_queries) *fallback_queries = 0;
    cudaStream_t stream = sc->stream;
    const uint32_t n = uint32_t(ix->n), words = (n + 31) / 32;
    CUDA_TRY(sc->flt_status.ensure(std::max<size_t>(n, 1)));
    CUDA_TRY(sc->flt_bits.ensure(std::max<size_t>(words, 1)));
    CUDA_TRY(sc->flt_ids.ensure(size_t(n) + 1));   // [count][ids]
    if (words) {
        flat_filter_rows_kernel<<<(words + 7) / 8, 256, 0, stream>>>(d_bitmap, ix->slot_mask ? rep->d_status.ptr : nullptr, n,
                                                                   sc->flt_status.ptr, sc->flt_bits.ptr);
        count_launch();
    }
    flat_compact_kernel<<<1, 1024, 0, stream>>>(sc->flt_bits.ptr, words, sc->flt_ids.ptr + 1, sc->flt_ids.ptr);
    count_launch();
    CUDA_TRY(cudaGetLastError());
    uint32_t allowed = 0;
    CUDA_TRY(cudaMemcpyAsync(&allowed, sc->flt_ids.ptr, 4, cudaMemcpyDeviceToHost, stream));
    CUDA_TRY(cudaStreamSynchronize(stream));
    if (out_allowed) *out_allowed = allowed;
    if (nq == 0) return 0;
    const uint32_t max_kc = FLAT_KC_DEEP;   // (the Flat handle's and the dynamic flat index's deepest lists)
    const uint64_t* ext_ids = ix->slot_mask ? rep->d_ext_ids.ptr : nullptr;
    const unsigned grid = unsigned(std::min<size_t>((nq * k + 255) / 256, size_t(rep->sm_count) * 8));
    if (allowed == 0) {
        CUDA_TRY(cudaMemsetAsync(d_out_ids, 0xFF, nq * k * 8, stream));
    } else if (flat_filter_route(n, allowed) == SVSB200_FLAT_ROUTE_SPARSE) {
        // the allowed rows, gathered in ascending order, and the exact scan over them alone (ties by position == by
        // row); the scratch lends them to a transient index on the same device for the call
        const uint32_t* rows = sc->flt_ids.ptr + 1;
        CUDA_TRY(sc->flt_rows.ensure(size_t(allowed) * ix->row_stride));
        CUDA_TRY(flat_move_rows(rep->d_vectors.ptr, sc->flt_rows.ptr, rows, sc->flt_ids.ptr, allowed, ix->row_stride, 0, stream));
        svsb200_index sub;
        sub.dtype = ix->dtype;
        sub.metric = ix->metric;
        sub.storage = ix->storage;
        sub.n = allowed;
        sub.dim = ix->dim;
        sub.row_stride = ix->row_stride;
        sub.gstride = 32;
        Replica subrep;
        subrep.device = rep->device;
        subrep.sm_count = rep->sm_count;
        subrep.d_vectors = std::move(sc->flt_rows);
        const int rc = search_on_device(&sub, &subrep, sc, d_queries, qdtype, nq, k, k, k, d_out_ids, 8, d_out_dists, stream,
                                        true);
        sc->flt_rows = std::move(subrep.d_vectors);
        if (rc) return rc;
        if (fallback_queries) *fallback_queries = uint32_t(nq);
        flat_unmap_ids_kernel<<<grid, 256, 0, stream>>>(d_out_ids, nq * k, rows, ext_ids);
        count_launch();
    } else {
        if (int rc = flat_rows_on_device(ix, rep, sc, d_queries, qdtype, nq, k, d_out_ids, d_out_dists, fallback_queries, max_kc,
                                         sc->flt_bits.ptr, sc->flt_status.ptr))
            return rc;
        if (ext_ids) CUDA_TRY(slots_to_external(d_out_ids, nq * k, ext_ids, stream));
    }
    flat_pad_inf_kernel<<<grid, 256, 0, stream>>>(d_out_ids, d_out_dists, nq * k);
    count_launch();
    CUDA_TRY(cudaGetLastError());
    return 0;
}

// ---- dynamic flat index: the tiles follow every mutation (host.cuh) ----
// Each built operand kind of the index's rows: fp16 tiles, and the integer tiles of int8 / uint8 rows.
template <typename F> static int for_each_flat_base(svsb200_index* ix, Replica* rep, F body) {
    if (rep->flat_f16.tiles.ptr)
        if (int rc = body(FLAT_F16, rep->flat_f16)) return rc;
    if (rep->flat_int.tiles.ptr)
        if (int rc = body(ix->dtype == SVSB200_I8 ? FLAT_S8 : FLAT_U8, rep->flat_int)) return rc;
    return 0;
}

uint32_t flat_max_kc_deep() { return FLAT_KC_DEEP; }

int flat_slots_grow(svsb200_index* ix, Replica* rep, size_t old_n, size_t new_n, cudaStream_t stream) {
    const uint32_t dim = uint32_t(ix->dim);
    const size_t old_t = (old_n + FLAT_BN - 1) / FLAT_BN, new_t = (new_n + FLAT_BN - 1) / FLAT_BN;
    const size_t cap_t = (rep->d_status.count + FLAT_BN - 1) / FLAT_BN;   // geometric, with the slot arrays
    if (new_t <= old_t) return 0;
    return for_each_flat_base(ix, rep, [&](int kind, Replica::FlatBase& base) -> int {
        const size_t tile_bytes = size_t(FLAT_BN) * flat_kblocks(kind, dim) * FLAT_BK * 2;
        CUDA_TRY(cudaStreamSynchronize(stream));
        CUDA_TRY(grow(base.tiles, old_t * tile_bytes, cap_t * tile_bytes));
        CUDA_TRY(grow(base.bias, old_t * FLAT_BN, cap_t * FLAT_BN));
        if (base.norms.ptr) CUDA_TRY(grow(base.norms, old_t * FLAT_BN, cap_t * FLAT_BN));
        CUDA_TRY(flat_place_rows(kind, dim, nullptr, nullptr, nullptr, nullptr, uint32_t(old_t * FLAT_BN),
                                 uint32_t((new_t - old_t) * FLAT_BN), base, stream));
        return 0;
    });
}

int flat_slots_place(svsb200_index* ix, Replica* rep, const void* d_rows, const uint32_t* d_slots, uint32_t count,
                     cudaStream_t stream) {
    rep->flat_xmax_stale = true;
    if (count == 0) return 0;
    const uint32_t dim = uint32_t(ix->dim), rows8 = (count + 7) / 8 * 8;
    Replica::SlotStaging& st = rep->staging;
    return for_each_flat_base(ix, rep, [&](int kind, Replica::FlatBase& base) -> int {
        // the full tiling's kernels, 8 rows to a tile, then every row moved to its slot (the kinds run one after the
        // other on `stream`, so they share the staging)
        CUDA_TRY(st.tiles.ensure(size_t(rows8) * flat_kblocks(kind, dim) * FLAT_BK * 2));
        CUDA_TRY(st.bias.ensure(rows8));
        if (base.norms.ptr) CUDA_TRY(st.norms.ensure(rows8));
        float* norms = base.norms.ptr ? st.norms.ptr : nullptr;
        CUDA_TRY(flat_tile_rows(kind, ix->dtype, d_rows, ix->row_stride, count, dim, 8, ix->metric == SVSB200_L2,
                                st.tiles.ptr, st.bias.ptr, norms, nullptr, stream));
        CUDA_TRY(flat_place_rows(kind, dim, st.tiles.ptr, st.bias.ptr, norms, d_slots, 0, count, base, stream));
        return 0;
    });
}

int flat_slots_clear(svsb200_index* ix, Replica* rep, const uint32_t* d_slots, uint32_t count, cudaStream_t stream) {
    rep->flat_xmax_stale = true;
    return for_each_flat_base(ix, rep, [&](int kind, Replica::FlatBase& base) -> int {
        CUDA_TRY(flat_place_rows(kind, uint32_t(ix->dim), nullptr, nullptr, nullptr, d_slots, 0, count, base, stream));
        return 0;
    });
}

void flat_slots_reset(Replica* rep) {
    rep->flat_f16 = Replica::FlatBase{};
    rep->flat_int = Replica::FlatBase{};
    rep->flat_xmax_stale = true;
}

// The plan of flat_on_device for k and a device of `sm_count` SMs (svsb200_flat_plan / svsb200_flat_plan_k).
static void flat_plan_rows(size_t nq, size_t n, uint32_t kc, int sm_count, uint32_t* ctas, uint32_t* share,
                           uint32_t* lists_per_query, uint64_t* segment_begin) {
    const uint32_t mtiles = uint32_t((nq + FLAT_BM - 1) / FLAT_BM), ntiles = uint32_t((n + FLAT_BN - 1) / FLAT_BN);
    flat_plan(mtiles, ntiles, uint32_t(sm_count), kc, ctas, share, lists_per_query);
    if (segment_begin) {
        const uint32_t nseg = *ctas / *share, ngroups = (mtiles + *share - 1) / *share;
        const uint64_t total = uint64_t(ngroups) * ntiles;
        for (uint32_t b = 0; b <= nseg; ++b) segment_begin[b] = flat_seg_begin(total, nseg, b);
    }
}

}  // namespace svsb200

using namespace svsb200;

// The two search bodies behind the four entry points here and the dynamic flat index's two (dynamic_flat.cu): `who`
// names the entry point in errors, `max_kc` is its deepest list (flat_on_device).  A flat handle is never dynamic and
// lives on one device.

// Enqueue-only form on device buffers, on the scratch bound to the caller's stream.
int svsb200::flat_search_device(const char* who, svsb200_index* ix, const void* d_queries, int qdtype, size_t nq, size_t k,
                                uint64_t* d_out_ids, float* d_out_dists, void* stream_, uint32_t* fallback_queries,
                                uint32_t max_kc) {
    const std::string w(who);
    if (!ix) return fail(w + ": NULL index");
    if (nq && (!d_queries || !d_out_ids || !d_out_dists)) return fail(w + ": NULL buffer");
    if (k == 0 || k > 1024) return fail(w + ": k must be in [1, 1024]");
    if (qdtype < SVSB200_F32 || qdtype > SVSB200_U8) return fail("bad query dtype");
    if (ix->reps.size() != 1) return fail(w + ": the index must live on exactly one device");
    if (ix->dynamic) return fail(w + ": flat search is not available on a dynamic index");
    Replica* rep = ix->reps[0].get();
    return run_on_stream(rep, stream_, [&](Scratch* sc) {
        return flat_on_device(ix, rep, sc, d_queries, qdtype, nq, k, d_out_ids, d_out_dists, fallback_queries, max_kc);
    });
}

// Blocking form on host buffers, on a scratch set of the pool (the first replica's).
int svsb200::flat_search_host(const char* who, svsb200_index* ix, const void* queries, int qdtype, size_t nq, size_t k,
                                uint64_t* out_ids, float* out_dists, uint32_t max_kc) {
    const std::string w(who);
    if (!ix) return fail(w + ": NULL index");
    if (k == 0 || k > 1024) return fail(w + ": k must be in [1, 1024]");
    if (nq == 0) return 0;
    if (!queries || !out_ids || !out_dists) return fail(w + ": NULL buffer");
    if (qdtype < SVSB200_F32 || qdtype > SVSB200_U8) return fail("bad query dtype");
    if (ix->dynamic) return fail(w + ": flat search is not available on a dynamic index");
    Replica* rep = ix->reps[0].get();
    return run_host_search(rep, {queries, nullptr, out_ids, out_dists}, nq * ix->dim * esize(qdtype), 0, nq, k,
                           [&](Scratch* sc, const StagedBuffers& d) {
                               return flat_on_device(ix, rep, sc, d.queries, qdtype, nq, k, d.ids, d.dists, nullptr, max_kc);
                           });
}

// The checks of both filtered forms: the arguments, and the query types the unfiltered search takes (an empty mask
// would otherwise let any query type through).
static int flat_filtered_check(const std::string& w, svsb200_index* ix, const void* bitmap, int qdtype, size_t k) {
    if (!ix) return fail(w + ": NULL index");
    if (!bitmap) return fail(w + ": NULL bitmap");
    if (k == 0 || k > 1024) return fail(w + ": k must be in [1, 1024]");
    if (qdtype < SVSB200_F32 || qdtype > SVSB200_U8) return fail("bad query dtype");
    if (ix->dynamic) return fail(w + ": flat search is not available on a dynamic index");
    const bool int_rows = ix->dtype == SVSB200_I8 || ix->dtype == SVSB200_U8;
    if ((qdtype == SVSB200_I8 || qdtype == SVSB200_U8) && qdtype != ix->dtype)
        return fail(w + ": int8/uint8 queries need rows of the same type");
    if (qdtype == SVSB200_F16 && int_rows) return fail(w + ": float16 queries need float32/float16 rows");
    return 0;
}

int svsb200::flat_search_filtered_device(const char* who, svsb200_index* ix, const void* d_queries, int qdtype, size_t nq,
                                         size_t k, const uint32_t* d_bitmap, uint64_t* d_out_ids, float* d_out_dists,
                                         void* stream_, size_t* out_allowed, uint32_t* fallback_queries) {
    const std::string w(who);
    if (int rc = flat_filtered_check(w, ix, d_bitmap, qdtype, k)) return rc;
    if (nq && (!d_queries || !d_out_ids || !d_out_dists)) return fail(w + ": NULL buffer");
    if (ix->reps.size() != 1) return fail(w + ": the index must live on exactly one device");
    Replica* rep = ix->reps[0].get();
    return run_on_stream(rep, stream_, [&](Scratch* sc) {
        return flat_filtered_on_device(ix, rep, sc, d_queries, qdtype, nq, k, d_bitmap, d_out_ids, d_out_dists, out_allowed,
                                       fallback_queries);
    });
}

int svsb200::flat_search_filtered_host(const char* who, svsb200_index* ix, const void* queries, int qdtype, size_t nq, size_t k,
                                       const uint32_t* bitmap, uint64_t* out_ids, float* out_dists, size_t* out_allowed) {
    const std::string w(who);
    if (int rc = flat_filtered_check(w, ix, bitmap, qdtype, k)) return rc;
    if (nq && (!queries || !out_ids || !out_dists)) return fail(w + ": NULL buffer");
    Replica* rep = ix->reps[0].get();
    return run_host_search(rep, {queries, bitmap, out_ids, out_dists}, nq * ix->dim * esize(qdtype), (ix->n + 31) / 32, nq, k,
                           [&](Scratch* sc, const StagedBuffers& d) {
                               return flat_filtered_on_device(ix, rep, sc, d.queries, qdtype, nq, k, d.bitmap, d.ids, d.dists,
                                                              out_allowed, nullptr);
                           });
}

extern "C" {

int svsb200_flat_filter_plan(size_t n, size_t allowed, int* route) {
    if (!route) return fail("svsb200_flat_filter_plan: NULL output");
    if (allowed > n) return fail("svsb200_flat_filter_plan: more allowed rows than rows");
    *route = flat_filter_route(n, allowed);
    return 0;
}

int svsb200_flat_index_search_filtered_device(svsb200_flat* index, const void* d_queries, int qdtype, size_t nq, size_t k,
                                              const uint32_t* d_id_bitmap, uint64_t* d_out_ids, float* d_out_dists,
                                              void* stream, size_t* out_allowed, uint32_t* fallback_queries) {
    return flat_search_filtered_device("svsb200_flat_index_search_filtered_device", index ? index->ix.get() : nullptr,
                                       d_queries, qdtype, nq, k, d_id_bitmap, d_out_ids, d_out_dists, stream, out_allowed,
                                       fallback_queries);
}

int svsb200_flat_index_search_filtered(svsb200_flat* index, const void* queries, int qdtype, size_t nq, size_t k,
                                       const uint32_t* id_bitmap, uint64_t* out_ids, float* out_dists, size_t* out_allowed) {
    return flat_search_filtered_host("svsb200_flat_index_search_filtered", index ? index->ix.get() : nullptr, queries, qdtype,
                                     nq, k, id_bitmap, out_ids, out_dists, out_allowed);
}

// How svsb200_flat_search* splits a problem (include/svsb200.h): host arithmetic only, so that the work split -- which the
// kernel recomputes from the same inline functions -- can be checked without a device (tests/test_flat_plan.py).
int svsb200_flat_plan(size_t nq, size_t n, int sm_count, uint32_t* ctas, uint32_t* share, uint32_t* lists_per_query,
                      uint64_t* segment_begin) {
    if (nq == 0 || n == 0 || sm_count <= 0 || !ctas || !share || !lists_per_query)
        return fail("svsb200_flat_plan: nq, n, sm_count must be positive and the outputs non-NULL");
    if (nq > (size_t(1) << 31) || n > (size_t(1) << 31)) return fail("svsb200_flat_plan: problem too large");
    flat_plan_rows(nq, n, FLAT_KC, sm_count, ctas, share, lists_per_query, segment_begin);
    return 0;
}

int svsb200_flat_plan_k(size_t nq, size_t n, size_t k, int sm_count, uint32_t* ctas, uint32_t* share, uint32_t* lists_per_query,
                        uint32_t* list_entries, uint64_t* segment_begin) {
    if (nq == 0 || n == 0 || sm_count <= 0 || !ctas || !share || !lists_per_query || !list_entries)
        return fail("svsb200_flat_plan_k: nq, n, sm_count must be positive and the outputs non-NULL");
    if (k == 0 || k + 8 > FLAT_KC_DEEP) return fail("svsb200_flat_plan_k: k must be in [1, 121]");
    if (nq > (size_t(1) << 31) || n > (size_t(1) << 31)) return fail("svsb200_flat_plan_k: problem too large");
    *list_entries = k + 8 <= FLAT_KC ? FLAT_KC : FLAT_KC_DEEP;
    if (*list_entries == FLAT_KC_DEEP && !flat_deep_batch(nq)) {   // the scan route: no GEMM
        *ctas = *share = *lists_per_query = *list_entries = 0;
        return 0;
    }
    flat_plan_rows(nq, n, *list_entries, sm_count, ctas, share, lists_per_query, segment_begin);
    return 0;
}

int svsb200_flat_search_device(svsb200_index* ix, const void* d_queries, int qdtype, size_t nq, size_t k, uint64_t* d_out_ids,
                               float* d_out_dists, void* stream_, uint32_t* fallback_queries) {
    return flat_search_device("svsb200_flat_search_device", ix, d_queries, qdtype, nq, k, d_out_ids, d_out_dists, stream_,
                              fallback_queries, FLAT_KC);
}

int svsb200_flat_search(svsb200_index* ix, const void* queries, int qdtype, size_t nq, size_t k, uint64_t* out_ids,
                        float* out_dists) {
    if (ix && nq == 0) return 0;   // an empty batch succeeds whatever k (the Flat handle checks k first)
    return flat_search_host("svsb200_flat_search", ix, queries, qdtype, nq, k, out_ids, out_dists, FLAT_KC);
}

int svsb200_flat_index_create(const void* vectors, int dtype, size_t n, size_t dim, size_t row_stride_bytes, int metric,
                              int device, svsb200_flat** out) {
    const char* who = "svsb200_flat_index_create";
    if (!out) return fail("svsb200_flat_index_create: out is NULL");
    *out = nullptr;
    if (!vectors) return fail("svsb200_flat_index_create: NULL input");
    if (dtype < SVSB200_F32 || dtype > SVSB200_U8) return fail("svsb200_flat_index_create: bad dtype");
    if (metric < SVSB200_L2 || metric > SVSB200_COSINE) return fail("svsb200_flat_index_create: bad metric");
    if (n == 0 || dim == 0) return fail("svsb200_flat_index_create: empty dataset");
    if (n >= (size_t(1) << 31)) return fail("svsb200_flat_index_create: more than 2^31-1 vectors per index");
    const size_t row_bytes = dim * esize(dtype);
    if (row_stride_bytes && row_stride_bytes < row_bytes) return fail("svsb200_flat_index_create: row stride below the row size");
    cudaDeviceProp prop;
    if (int rc = check_device(who, device, &prop)) return rc;
    auto flat = std::make_unique<svsb200_flat>();
    flat->ix = std::make_unique<svsb200_index>();
    svsb200_index* ix = flat->ix.get();
    ix->dtype = dtype;
    ix->metric = metric;
    ix->storage = SVSB200_PLAIN;
    ix->n = n;
    ix->dim = dim;
    ix->row_stride = data_row_stride(SVSB200_PLAIN, dtype, dim);
    ix->gstride = 32;   // the scan's block of rows (struct svsb200_flat); there is no adjacency
    ix->reps.push_back(std::make_unique<Replica>());
    Replica* rep = ix->reps.back().get();
    rep->device = device;
    rep->sm_count = prop.multiProcessorCount;
    CUDA_TRY(cudaSetDevice(device));
    const size_t vbytes = n * size_t(ix->row_stride);
    CUDA_TRY(rep->d_vectors.ensure(vbytes));
    CUDA_TRY(cudaMemset(rep->d_vectors.ptr, 0, vbytes));
    CUDA_TRY(cudaMemcpy2D(rep->d_vectors.ptr, ix->row_stride, vectors, row_stride_bytes ? row_stride_bytes : row_bytes, row_bytes,
                          n, cudaMemcpyHostToDevice));
    ix->device_bytes = vbytes;
    *out = flat.release();
    return 0;
}

int svsb200_flat_index_destroy(svsb200_flat* index) {
    delete index;   // Replica / Scratch destructors release the device memory
    return 0;
}

size_t svsb200_flat_index_size(const svsb200_flat* index) { return index ? index->ix->n : 0; }
size_t svsb200_flat_index_dimensions(const svsb200_flat* index) { return index ? index->ix->dim : 0; }
size_t svsb200_flat_index_device_bytes(const svsb200_flat* index) { return index ? index->ix->device_bytes : 0; }

int svsb200_flat_index_search_device(svsb200_flat* index, const void* d_queries, int qdtype, size_t nq, size_t k,
                                     uint64_t* d_out_ids, float* d_out_dists, void* stream_, uint32_t* fallback_queries) {
    return flat_search_device("svsb200_flat_index_search_device", index ? index->ix.get() : nullptr, d_queries, qdtype, nq, k,
                              d_out_ids, d_out_dists, stream_, fallback_queries, FLAT_KC_DEEP);
}

int svsb200_flat_index_search(svsb200_flat* index, const void* queries, int qdtype, size_t nq, size_t k, uint64_t* out_ids,
                              float* out_dists) {
    return flat_search_host("svsb200_flat_index_search", index ? index->ix.get() : nullptr, queries, qdtype, nq, k, out_ids,
                            out_dists, FLAT_KC_DEEP);
}

}  // extern "C"
