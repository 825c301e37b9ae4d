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
//      inner product) and keep, per query, the KC smallest keys seen in this CTA's base range.
//   2. flat_rescore_kernel: every candidate of a query (all ranges) is re-scored with the search path's own
//      bit-exact distance code (eval_pass) and the k best by (key, id) are written out.
//   3. verification: fp16 rounding moves a key by at most E(q) (derived below); a base row that is NOT a
//      candidate has an approximate key >= T, the smallest per-range list maximum.  If T > kth-smallest approximate
//      key + 2 E(q), no excluded row can belong to the exact top k, so the rescored result IS the exact result.
//      Queries that fail the test (rare) are searched again with the exact scan kernel -- the result is exact
//      in every case.
//
// Error bound: with q~, x~ the fp16-rounded operands (relative rounding 2^-11 per element; float16 inputs are
// not rounded at all), r = the number of rounded operands (0..2):
//   |q~.x~ - q.x| <= ||q~ - q|| ||x~|| + ||q|| ||x~ - x|| <= r 2^-11 ||q|| ||x|| (1 + 2^-11),
// the products are exact in fp32 and the tensor-core accumulation of `dim` of them adds at most dim 2^-22 ||q|| ||x||;
// for L2 the bias |x~|^2 differs from |x|^2 by at most 2^-10 ||x||^2 when the data was rounded.  So
//   E_ip(q) = (r 2^-11 + dim 2^-22) ||q|| Xmax,      E_l2(q) = 2 E_ip(q) + [data rounded] 2^-10 Xmax^2.
#include "search_kernel.cuh"

#include <cuda_fp16.h>

namespace svsb200 {

constexpr uint32_t FLAT_BM = 128, FLAT_BN = 256, FLAT_BK = 32;      // tile sizes (rows, rows, k elements per blob)
constexpr uint32_t FLAT_A_BYTES = FLAT_BM * FLAT_BK * 2, FLAT_B_BYTES = FLAT_BN * FLAT_BK * 2;
constexpr uint32_t FLAT_STAGE_BYTES = FLAT_A_BYTES + FLAT_B_BYTES;
constexpr uint32_t FLAT_STAGES = 6;
constexpr uint32_t FLAT_KC = 33;                                     // list entries per (query, base range)
constexpr uint32_t FLAT_LEAD = 4;                                    // tiles a CTA may run ahead of its segment's slowest CTA
constexpr uint32_t FLAT_CMAX = 1024;                                 // candidates per query the rescoring kernel holds

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
// keeps the compiler from moving reads of an accumulator register across the wait that completes it
__device__ __forceinline__ void reg_fence(float& r) { asm volatile("" : "+f"(r)::"memory"); }
// Warpgroup-MMA shared-memory matrix descriptor, K-major, no swizzle (layout type 0): 8x8-element core matrices of
// 128 contiguous bytes; LBO = byte distance between the two 8-element k-chunks of one K=16 MMA, SBO = byte distance
// between 8-row groups.
__device__ __forceinline__ uint64_t wgmma_desc(uint32_t smem_addr, uint32_t lbo_bytes, uint32_t sbo_bytes) {
    return uint64_t((smem_addr >> 4) & 0x3FFFu) | (uint64_t((lbo_bytes >> 4) & 0x3FFFu) << 16) |
           (uint64_t((sbo_bytes >> 4) & 0x3FFFu) << 32);
}
// D (64 x 256, fp32, in registers) [+]= A (64 x 16) . B (256 x 16)^T, both fp16 K-major in shared memory.
__device__ __forceinline__ void wgmma_m64n256k16(float (&d)[128], uint64_t adesc, uint64_t bdesc, uint32_t accumulate) {
    asm volatile(
        "{\n\t"
        ".reg .pred p;\n\t"
        "setp.ne.b32 p, %130, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n256k16.f32.f16.f16 "
        "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
        "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, "
        "%32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, "
        "%48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63, "
        "%64, %65, %66, %67, %68, %69, %70, %71, %72, %73, %74, %75, %76, %77, %78, %79, "
        "%80, %81, %82, %83, %84, %85, %86, %87, %88, %89, %90, %91, %92, %93, %94, %95, "
        "%96, %97, %98, %99, %100, %101, %102, %103, %104, %105, %106, %107, %108, %109, %110, %111, "
        "%112, %113, %114, %115, %116, %117, %118, %119, %120, %121, %122, %123, %124, %125, %126, %127}, "
        "%128, %129, p, 1, 1, 0, 0;\n\t"
        "}\n"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
          "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
          "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
          "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]),
          "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]),
          "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]),
          "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]),
          "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63]),
          "+f"(d[64]), "+f"(d[65]), "+f"(d[66]), "+f"(d[67]), "+f"(d[68]), "+f"(d[69]), "+f"(d[70]), "+f"(d[71]),
          "+f"(d[72]), "+f"(d[73]), "+f"(d[74]), "+f"(d[75]), "+f"(d[76]), "+f"(d[77]), "+f"(d[78]), "+f"(d[79]),
          "+f"(d[80]), "+f"(d[81]), "+f"(d[82]), "+f"(d[83]), "+f"(d[84]), "+f"(d[85]), "+f"(d[86]), "+f"(d[87]),
          "+f"(d[88]), "+f"(d[89]), "+f"(d[90]), "+f"(d[91]), "+f"(d[92]), "+f"(d[93]), "+f"(d[94]), "+f"(d[95]),
          "+f"(d[96]), "+f"(d[97]), "+f"(d[98]), "+f"(d[99]), "+f"(d[100]), "+f"(d[101]), "+f"(d[102]), "+f"(d[103]),
          "+f"(d[104]), "+f"(d[105]), "+f"(d[106]), "+f"(d[107]), "+f"(d[108]), "+f"(d[109]), "+f"(d[110]), "+f"(d[111]),
          "+f"(d[112]), "+f"(d[113]), "+f"(d[114]), "+f"(d[115]), "+f"(d[116]), "+f"(d[117]), "+f"(d[118]), "+f"(d[119]),
          "+f"(d[120]), "+f"(d[121]), "+f"(d[122]), "+f"(d[123]), "+f"(d[124]), "+f"(d[125]), "+f"(d[126]), "+f"(d[127])
        : "l"(adesc), "l"(bdesc), "r"(accumulate));
}
// Per-query list of the FLAT_KC smallest keys: shared memory, [query row][FLAT_KC] with FLAT_KC odd, so that a warp
// reading one row side by side is bank-conflict free.  Keys are stored as order-preserving unsigned integers
// (REDUX.MAX works on them); a list starts full of +inf / no-id entries, so there is no fill count -- an update always
// replaces the current maximum, and the row's threshold is the new maximum.
static_assert(FLAT_KC % 2 == 1 && FLAT_KC > 32 && FLAT_KC <= 64, "list layout");
__device__ __forceinline__ uint32_t flat_ord(float f) {
    const uint32_t u = __float_as_uint(f);
    return u ^ (uint32_t(int32_t(u) >> 31) | 0x80000000u);
}
__device__ __forceinline__ float flat_unord(uint32_t o) {
    return __uint_as_float(o ^ ((o >> 31) ? 0x80000000u : 0xFFFFFFFFu));
}
// The whole warp updates the list of row `list_row` with (key, id); returns the row's new threshold (warp-uniform).
__device__ __forceinline__ float flat_list_replace_max(uint32_t* lkey, uint32_t* lid, uint32_t list_row, uint32_t lane,
                                                      float key, uint32_t id) {
    uint32_t* rk = lkey + list_row * FLAT_KC;
    uint32_t v0 = rk[lane];
    uint32_t v1 = lane + 32 < FLAT_KC ? rk[lane + 32] : 0u;
    const uint32_t mx = __reduce_max_sync(0xFFFFFFFFu, max(v0, v1));
    const uint32_t in0 = __ballot_sync(0xFFFFFFFFu, v0 == mx);
    const uint32_t in1 = __ballot_sync(0xFFFFFFFFu, v1 == mx && lane + 32 < FLAT_KC);
    const uint32_t slot = in0 ? uint32_t(__ffs(int(in0)) - 1) : uint32_t(__ffs(int(in1)) + 31);
    const uint32_t nk = flat_ord(key);
    if (lane == (slot & 31u)) {
        rk[slot] = nk;
        lid[list_row * FLAT_KC + slot] = id;
        if (slot < 32) v0 = nk; else v1 = nk;
    }
    return flat_unord(__reduce_max_sync(0xFFFFFFFFu, max(v0, v1)));
}

struct FlatParams {
    const __half* a_tiles;    // [mtiles][KB] blobs of FLAT_A_BYTES
    const __half* b_tiles;    // [ntiles][KB] blobs of FLAT_B_BYTES
    const float* b_bias;      // [ntiles * FLAT_BN]: |x~|^2 (L2) / 0 (inner product), +inf for padding rows
    uint32_t KB, ntiles, mtiles, nlists;
    uint32_t share;           // R: CTAs that walk the same base tiles at the same time, on R consecutive query tiles
    uint32_t* progress;       // [gridDim.x] tiles started by each CTA (zeroed before the launch)
    float key_scale;          // key = bias + key_scale * s
    float* cand_key;          // [mtiles * FLAT_BM][nlists][FLAT_KC], pre-filled with (+inf, no id)
    uint32_t* cand_id;
};

// Work split: query tiles are taken R at a time ("row groups"); the (row group, base tile) pairs form one row-major
// sequence, cut into G = gridDim.x / R contiguous, equal segments -- every SM gets the same number of tiles whatever
// the batch size.  Segment g is walked by R CTAs (blockIdx g, g + G, ...: all resident at once, started together, doing
// identical work), one per query tile of the row group: they ask for the same base tile within microseconds of each
// other, so all but the first request are served by L2 -- without this, one CTA per SM streams as many different
// places of a base that is many times the L2, and every operand byte comes from DRAM.  A segment may run over a
// row-group boundary (the lists are flushed there), and a query tile is covered by a few consecutive segments
// ("pieces"); each piece keeps two lists per query, one per half of the 256 tile columns.
__host__ __device__ inline uint64_t flat_seg_begin(uint64_t total, uint32_t ctas, uint32_t b) { return total * b / ctas; }
__host__ __device__ inline uint32_t flat_cta_of_tile(uint64_t t, uint64_t total, uint32_t ctas) {
    uint32_t b = uint32_t(t * ctas / total);
    while (b + 1 < ctas && flat_seg_begin(total, ctas, b + 1) <= t) ++b;
    while (b > 0 && flat_seg_begin(total, ctas, b) > t) --b;
    return b;
}

// Threads: warps 0-7 are the two consumer warpgroups (a warpgroup is four consecutive warps starting at a multiple of
// four), warp 8 the producer.  Shared memory: stages | list keys [2][128][KC] | list ids [2][128][KC] | barriers.
constexpr uint32_t FLAT_CONSUMER_WARPS = 8, FLAT_THREADS = 32 * FLAT_CONSUMER_WARPS + 32;
constexpr size_t kFlatSmem = size_t(FLAT_STAGES) * FLAT_STAGE_BYTES + 2 * 2 * size_t(FLAT_KC) * FLAT_BM * 4 + 128;
static_assert(kFlatSmem <= 227 * 1024, "flat GEMM shared memory exceeds the 227 KB a block may use");

__global__ void __launch_bounds__(FLAT_THREADS, 1) flat_gemm_topk_kernel(const __grid_constant__ FlatParams fp) {
    extern __shared__ __align__(1024) uint8_t smem[];
    uint8_t* stages = smem;
    uint32_t* lkey = reinterpret_cast<uint32_t*>(smem + size_t(FLAT_STAGES) * FLAT_STAGE_BYTES);   // [2][128][KC] ordered keys
    uint32_t* lid = lkey + 2 * size_t(FLAT_KC) * FLAT_BM;
    uint64_t* bars = reinterpret_cast<uint64_t*>(lid + 2 * size_t(FLAT_KC) * FLAT_BM);
    uint64_t* full = bars;                       // [STAGES] bytes of a stage have landed
    uint64_t* empty = bars + FLAT_STAGES;        // [STAGES] the MMAs of every consumer warp reading a stage have completed

    const uint32_t warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const uint32_t nseg = gridDim.x / fp.share, seg = blockIdx.x % nseg, member = blockIdx.x / nseg;
    const uint32_t ngroups = (fp.mtiles + fp.share - 1) / fp.share;
    const uint64_t total = uint64_t(ngroups) * fp.ntiles;
    const uint64_t t_lo = flat_seg_begin(total, nseg, seg), t_hi = flat_seg_begin(total, nseg, seg + 1);
    // (a CTA's query tile advances by `share` at a row-group boundary; tiles of a query tile past the last one are skipped
    // by every role alike)
    const uint32_t mtile0 = uint32_t(t_lo / fp.ntiles) * fp.share + member, nt0 = uint32_t(t_lo % fp.ntiles);

    if (threadIdx.x == 0) {
        for (uint32_t i = 0; i < FLAT_STAGES; ++i) {
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
                    if (++s == FLAT_STAGES) {
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
    // half, updated by the whole warp (all lanes of a quad see the new threshold) =====
    const uint32_t wg = warp >> 2;
    const uint32_t row0 = wg * 64 + (warp & 3u) * 16 + (lane >> 2);   // the thread's rows: row0, row0 + 8
    const uint32_t frow = wg * 64 + (warp & 3u) * 16 + (lane >> 1), fhalf = lane & 1u;   // the (row, half) list this lane clears / writes out
    float d[128];
#pragma unroll
    for (uint32_t i = 0; i < 128; ++i) d[i] = 0.f;
    float thr[2][2];   // [row i][column half]: the largest key of that list
#pragma unroll
    for (uint32_t i = 0; i < 4; ++i) thr[i >> 1][i & 1] = INFINITY;
    for (uint32_t e = 0; e < FLAT_KC; ++e) {
        lkey[(fhalf * FLAT_BM + frow) * FLAT_KC + e] = flat_ord(INFINITY);
        lid[(fhalf * FLAT_BM + frow) * FLAT_KC + e] = 0xFFFFFFFFu;
    }
    __syncwarp();
    uint32_t s = 0, ph = 0, mtile = mtile0, nt = nt0;
    for (uint64_t t = t_lo; t < t_hi; ++t) {
        if (mtile >= fp.mtiles) {
            if (++nt == fp.ntiles) {
                nt = 0;
                mtile += fp.share;
            }
            continue;
        }
        // ---- mainloop: one k-block per stage, two K=16 MMAs each; a stage is released once the MMAs of the next one
        // have been issued and its own have completed ----
        uint32_t prev = 0;
        for (uint32_t kb = 0; kb < fp.KB; ++kb) {
            mbar_wait(full + s, ph);
            const uint32_t a_addr = smem_u32(stages + size_t(s) * FLAT_STAGE_BYTES) + wg * 1024u;   // 8 row groups of 128 B
            const uint32_t b_addr = smem_u32(stages + size_t(s) * FLAT_STAGE_BYTES + FLAT_A_BYTES);
            wgmma_fence();
#pragma unroll
            for (uint32_t j = 0; j < FLAT_BK / 16; ++j) {
                // k-chunks 2j and 2j+1 of the blob: [kc][rows/8][8][8] halves
                const uint64_t adesc = wgmma_desc(a_addr + 2 * j * (FLAT_BM * 16), FLAT_BM * 16, 128);
                const uint64_t bdesc = wgmma_desc(b_addr + 2 * j * (FLAT_BN * 16), FLAT_BN * 16, 128);
                wgmma_m64n256k16(d, adesc, bdesc, (kb | j) != 0 ? 1u : 0u);
            }
            wgmma_commit();
            wgmma_wait<1>();
            if (kb > 0 && lane == 0) mbar_arrive(empty + prev);
            prev = s;
            if (++s == FLAT_STAGES) {
                s = 0;
                ph ^= 1u;
            }
        }
        wgmma_wait<0>();
#pragma unroll
        for (uint32_t i = 0; i < 128; ++i) reg_fence(d[i]);
        if (lane == 0) mbar_arrive(empty + prev);

        // ---- epilogue: keys of the thread's 128 elements; only columns whose keys beat a row's threshold (rare once
        // the lists have settled) are looked at key by key, the lanes with such a key served in turn by the whole warp ----
        const float* bias = fp.b_bias + size_t(nt) * FLAT_BN + 2 * (lane & 3u);
#pragma unroll
        for (uint32_t c = 0; c < FLAT_BN / 8; ++c) {
            const uint32_t h = c / (FLAT_BN / 16);
            const float2 b2 = __ldg(reinterpret_cast<const float2*>(bias + 8 * c));
            float key[4];
            key[0] = fmaf(fp.key_scale, d[4 * c + 0], b2.x);
            key[1] = fmaf(fp.key_scale, d[4 * c + 1], b2.y);
            key[2] = fmaf(fp.key_scale, d[4 * c + 2], b2.x);
            key[3] = fmaf(fp.key_scale, d[4 * c + 3], b2.y);
            const bool any = fminf(key[0], key[1]) < thr[0][h] || fminf(key[2], key[3]) < thr[1][h];
            if (!__any_sync(0xFFFFFFFFu, any)) continue;
            uint32_t* my_key = lkey + size_t(h) * FLAT_BM * FLAT_KC;
            uint32_t* my_id = lid + size_t(h) * FLAT_BM * FLAT_KC;
#pragma unroll
            for (uint32_t v = 0; v < 4; ++v) {
                const uint32_t i = v >> 1;
                bool pending = key[v] < thr[i][h];
                uint32_t hits = __ballot_sync(0xFFFFFFFFu, pending);
                while (hits) {
                    const uint32_t src = uint32_t(__ffs(int(hits)) - 1);
                    const float k_src = __shfl_sync(0xFFFFFFFFu, key[v], src);
                    const uint32_t id = nt * FLAT_BN + 8 * c + 2 * (src & 3u) + (v & 1u);
                    const float tnew = flat_list_replace_max(my_key, my_id, row0 - (lane >> 2) + (src >> 2) + 8 * i, lane,
                                                             k_src, id);
                    if ((lane >> 2) == (src >> 2)) thr[i][h] = tnew;
                    // another lane of the quad may hold a key of the same row that no longer beats the new threshold
                    pending = pending && lane != src && key[v] < thr[i][h];
                    hits = __ballot_sync(0xFFFFFFFFu, pending);
                }
            }
        }
        if (++nt == fp.ntiles || t + 1 == t_hi) {
            // the query tile (or this CTA's part of it) is finished: lists out, lists reset
            const uint32_t piece = seg - flat_cta_of_tile(uint64_t(mtile / fp.share) * fp.ntiles, total, nseg);
            const size_t q = size_t(mtile) * FLAT_BM + frow;
            float* ok = fp.cand_key + (q * fp.nlists + piece * 2 + fhalf) * FLAT_KC;
            uint32_t* oi = fp.cand_id + (q * fp.nlists + piece * 2 + fhalf) * FLAT_KC;
            uint32_t* rk = lkey + (fhalf * FLAT_BM + frow) * FLAT_KC;
            uint32_t* ri = lid + (fhalf * FLAT_BM + frow) * FLAT_KC;
            __syncwarp();
            for (uint32_t e = 0; e < FLAT_KC; ++e) {
                ok[e] = flat_unord(rk[e]);
                oi[e] = ri[e];
                rk[e] = flat_ord(INFINITY);
                ri[e] = 0xFFFFFFFFu;
            }
            __syncwarp();
#pragma unroll
            for (uint32_t i = 0; i < 4; ++i) thr[i >> 1][i & 1] = INFINITY;
            nt = 0;
            mtile += fp.share;
        }
    }
}

// ---- operand tiling: rows -> fp16 blobs in the canonical K-major layout of the warpgroup MMA ----------------------
// element (row r, k e) of tile t = r / TR lives at  ((t*KB + e/32) * 4 + (e%32)/8) * TR*8 + ((r%TR)/8)*64 + (r%8)*8 + e%8
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
    for (uint32_t e = lane; e < dim; e += 32) {
        float x;
        if constexpr (SRCT == SVSB200_F32) x = reinterpret_cast<const float*>(row)[e];
        else x = __half2float(reinterpret_cast<const __half*>(row)[e]);
        const __half h = __float2half_rn(x * scale);
        const float xr = __half2float(h) / scale;
        sq_rounded = fmaf(xr, xr, sq_rounded);
        sq_exact = fmaf(x, x, sq_exact);
        const size_t o = ((size_t(t) * KB + e / 32) * 4 + (e % 32) / 8) * (size_t(TR) * 8) + (rr / 8) * 64 + (rr % 8) * 8 + e % 8;
        dst[o] = h;
    }
    for (int o = 16; o; o >>= 1) {
        sq_rounded += __shfl_xor_sync(0xFFFFFFFFu, sq_rounded, o);
        sq_exact += __shfl_xor_sync(0xFFFFFFFFu, sq_exact, o);
    }
    if (lane == 0) {
        if (bias) bias[r] = l2 ? sq_rounded : 0.f;
        const float nrm = sqrtf(sq_exact) * 1.000001f;
        if (norms) norms[r] = nrm;
        if (max_norm_bits) atomicMax(max_norm_bits, __float_as_uint(nrm));
    }
}

// ---- exact re-scoring + verification: one warp per query ----------------------------------------------------------
struct RescoreParams {
    const float* cand_key;    // [nq_padded][nsplit][KC]
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
};

template <int ROWT, int OP>
__global__ void __launch_bounds__(32, 16) flat_rescore_kernel(const __grid_constant__ SearchParams p,
                                                             const __grid_constant__ RescoreParams rp) {
    constexpr int G = 16 / Row<ROWT>::LPT;
    constexpr int GROUPS = 32 / G;
    constexpr unsigned FULL = 0xFFFFFFFFu;
    constexpr uint32_t CMAX = FLAT_CMAX;
    extern __shared__ __align__(16) unsigned char smem_raw[];
    float* q_s = reinterpret_cast<float*>(smem_raw);
    uint32_t* cid = reinterpret_cast<uint32_t*>(q_s + p.qstride);   // [CMAX]
    float* akey = reinterpret_cast<float*>(cid + CMAX);               // [CMAX] approximate keys
    float* ekey = akey + CMAX;                                        // [CMAX] exact keys
    const int lane = threadIdx.x;
    const int g = lane / G, t = lane % G;
    const uint32_t q = blockIdx.x;
    if (q >= rp.nq) return;
    const uint32_t total = rp.nsplit * FLAT_KC;
    // candidates of every base range; T = the smallest per-range list maximum (every excluded row is >= it)
    float T = INFINITY;
    for (uint32_t s = 0; s < rp.nsplit; ++s) {
        float mx = -INFINITY;
        for (uint32_t e = lane; e < FLAT_KC; e += 32) mx = fmaxf(mx, rp.cand_key[(size_t(q) * rp.nsplit + s) * FLAT_KC + e]);
        for (int o = 16; o; o >>= 1) mx = fmaxf(mx, __shfl_xor_sync(FULL, mx, o));
        T = fminf(T, mx);
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
            akey[o] = rp.cand_key[size_t(q) * total + i];
        }
        C += __popc(m);
    }
    __syncwarp();
    for (uint32_t i = lane; i < p.qstride; i += 32) q_s[i] = p.qf[size_t(q) * p.qstride + i];
    __syncwarp();
    const float aux0 = p.qaux[2 * size_t(q)], aux1 = p.qaux[2 * size_t(q) + 1];
    for (uint32_t base = 0; base < C; base += 2 * GROUPS)
        eval_pass<ROWT, OP, 0, 2, 1, true>(p, q_s, reinterpret_cast<const char*>(p.vectors), cid, ekey, base, C, g, t, aux0, aux1,
                                           rp.ksign);
    __syncwarp();
    // rank of every candidate by (exact key, id) and by approximate key: k is small, C <= 512
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
    const float qn = rp.qnorm[q], xm = __uint_as_float(*rp.xmax_bits);
    const float rounded = p.scale;   // operands that were rounded to fp16 (0, 1 or 2)
    const float e_ip = (rounded * 4.8828125e-4f + float(p.dim) * 2.384185791015625e-7f) * qn * xm * 1.0001f;   // 2^-11 each, dim 2^-22
    const float E = p.greater ? e_ip : 2.0f * e_ip + (rounded > 1.5f || rp.data_rounded ? 9.765625e-4f * xm * xm : 0.0f);
    const bool verified = C >= rp.k && T > kth_approx + 2.0f * E;
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

// ---- launchers (called from svsb200.cu) ------------------------------------------------------------------------------
cudaError_t flat_tile_rows(int srct, const void* src, uint32_t row_stride, uint32_t n, uint32_t dim, uint32_t tile_rows,
                           float scale, int l2, void* dst_tiles, float* bias, float* norms, unsigned int* max_norm_bits,
                           cudaStream_t stream) {
    const uint32_t KB = (dim + FLAT_BK - 1) / FLAT_BK;
    const uint32_t rows_padded = (n + tile_rows - 1) / tile_rows * tile_rows;
    cudaError_t err = cudaMemsetAsync(dst_tiles, 0, size_t(rows_padded) * KB * FLAT_BK * 2, stream);
    if (err != cudaSuccess) return err;
    const unsigned grid = (rows_padded + 7) / 8;
    if (srct == SVSB200_F32)
        flat_tile_kernel<SVSB200_F32><<<grid, 256, 0, stream>>>(static_cast<const char*>(src), row_stride, n, dim, tile_rows, KB, scale,
                                                               l2, static_cast<__half*>(dst_tiles), bias, norms, max_norm_bits);
    else
        flat_tile_kernel<SVSB200_F16><<<grid, 256, 0, stream>>>(static_cast<const char*>(src), row_stride, n, dim, tile_rows, KB, scale,
                                                               l2, static_cast<__half*>(dst_tiles), bias, norms, max_norm_bits);
    count_launch();
    return cudaGetLastError();
}

__global__ void flat_fill_kernel(float* __restrict__ key, uint32_t* __restrict__ id, size_t count) {
    for (size_t i = size_t(blockIdx.x) * blockDim.x + threadIdx.x; i < count; i += size_t(gridDim.x) * blockDim.x) {
        key[i] = INFINITY;
        id[i] = 0xFFFFFFFFu;
    }
}

// Grid size, sharing factor and lists per query for a problem: as many CTAs as SMs in groups of R, fewer segments
// while a query tile would be cut into more pieces than the rescoring kernel holds candidates for (small batches
// over a large base).
void flat_plan(uint32_t mtiles, uint32_t ntiles, uint32_t sm_count, uint32_t* ctas, uint32_t* share, uint32_t* nlists) {
    const uint32_t R = mtiles >= 8 ? 4 : mtiles >= 4 ? 2 : 1;
    const uint32_t ngroups = (mtiles + R - 1) / R;
    const uint64_t total = uint64_t(ngroups) * ntiles;
    uint32_t g = uint32_t(std::min<uint64_t>(std::max(1u, sm_count / R), total));
    for (;; --g) {
        uint32_t pieces = 1;
        for (uint32_t m = 0; m < ngroups; ++m)
            pieces = std::max(pieces, flat_cta_of_tile(uint64_t(m + 1) * ntiles - 1, total, g) -
                                          flat_cta_of_tile(uint64_t(m) * ntiles, total, g) + 1);
        if (2 * pieces * FLAT_KC <= FLAT_CMAX || g == 1) {
            *ctas = g * R;
            *share = R;
            *nlists = 2 * pieces;
            return;
        }
    }
}

cudaError_t flat_gemm_topk(const void* a_tiles, const void* b_tiles, const float* b_bias, uint32_t KB, uint32_t ntiles,
                           uint32_t mtiles, uint32_t ctas, uint32_t share, uint32_t nlists, float key_scale, float* cand_key,
                           uint32_t* cand_id, uint32_t* progress, cudaStream_t stream) {
    FlatParams fp{};
    fp.a_tiles = static_cast<const __half*>(a_tiles);
    fp.b_tiles = static_cast<const __half*>(b_tiles);
    fp.b_bias = b_bias;
    fp.KB = KB;
    fp.ntiles = ntiles;
    fp.mtiles = mtiles;
    fp.nlists = nlists;
    fp.share = share;
    fp.progress = progress;
    fp.key_scale = key_scale;
    fp.cand_key = cand_key;
    fp.cand_id = cand_id;
    cudaError_t err = cudaFuncSetAttribute(flat_gemm_topk_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, int(kFlatSmem));
    if (err != cudaSuccess) return err;
    const size_t entries = size_t(mtiles) * FLAT_BM * nlists * FLAT_KC;
    flat_fill_kernel<<<unsigned(std::min<size_t>(4096, (entries + 255) / 256)), 256, 0, stream>>>(cand_key, cand_id, entries);
    count_launch();
    flat_gemm_topk_kernel<<<ctas, FLAT_THREADS, kFlatSmem, stream>>>(fp);
    count_launch();
    return cudaGetLastError();
}

template <int ROWT> static cudaError_t rescore_rowt(int op, const SearchParams& p, const RescoreParams& rp, cudaStream_t stream) {
    const size_t smem = size_t(p.qstride) * 4 + size_t(FLAT_CMAX) * 4 * 3;
    if (op == OP_L2F) flat_rescore_kernel<ROWT, OP_L2F><<<rp.nq, 32, smem, stream>>>(p, rp);
    else if (op == OP_IPF) flat_rescore_kernel<ROWT, OP_IPF><<<rp.nq, 32, smem, stream>>>(p, rp);
    else return cudaErrorInvalidValue;
    count_launch();
    return cudaGetLastError();
}

cudaError_t flat_rescore(int rowt, int op, const SearchParams& p, const float* cand_key, const uint32_t* cand_id, uint32_t nsplit,
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
    return rowt == SVSB200_F32 ? rescore_rowt<SVSB200_F32>(op, p, rp, stream) : rescore_rowt<SVSB200_F16>(op, p, rp, stream);
}

cudaError_t flat_move_rows(const void* src, void* dst, const uint32_t* idx, const uint32_t* count, uint32_t max_count,
                           uint32_t row_bytes, int scatter, cudaStream_t stream) {
    if (max_count == 0) return cudaSuccess;
    flat_move_rows_kernel<<<max_count, 128, 0, stream>>>(static_cast<const char*>(src), static_cast<char*>(dst), idx, count,
                                                        row_bytes, scatter);
    count_launch();
    return cudaGetLastError();
}

uint32_t flat_kc() { return FLAT_KC; }

}  // namespace svsb200

// How svsb200_flat_search* splits a problem (include/svsb200.h): host arithmetic only, so that the work split -- which the
// kernel recomputes from the same inline functions -- can be checked without a device (tests/test_flat_plan.py).
extern "C" int svsb200_flat_plan(size_t nq, size_t n, int sm_count, uint32_t* ctas, uint32_t* share, uint32_t* lists_per_query,
                                 uint64_t* segment_begin) {
    using namespace svsb200;
    if (nq == 0 || n == 0 || sm_count <= 0 || !ctas || !share || !lists_per_query)
        return set_error("svsb200_flat_plan: nq, n, sm_count must be positive and the outputs non-NULL");
    if (nq > (size_t(1) << 31) || n > (size_t(1) << 31)) return set_error("svsb200_flat_plan: problem too large");
    const uint32_t mtiles = uint32_t((nq + FLAT_BM - 1) / FLAT_BM), ntiles = uint32_t((n + FLAT_BN - 1) / FLAT_BN);
    flat_plan(mtiles, ntiles, uint32_t(sm_count), ctas, share, lists_per_query);
    if (segment_begin) {
        const uint32_t nseg = *ctas / *share, ngroups = (mtiles + *share - 1) / *share;
        const uint64_t total = uint64_t(ngroups) * ntiles;
        for (uint32_t b = 0; b <= nseg; ++b) segment_begin[b] = flat_seg_begin(total, nseg, b);
    }
    return 0;
}
