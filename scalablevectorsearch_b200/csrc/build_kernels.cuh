// build_kernels.cuh -- GPU Vamana graph construction (SURVEY.md §8 f1): the reference's VamanaBuilder
// (index/vamana/vamana_build.h:169-599) restated as rounds of whole-batch kernels.
//
// Per round over a batch of nodes (vamana_build.h:221-310 `construct`):
//   1. generate_neighbors (:320-470): greedy search from the medoid for every batch node -- the lean search
//      kernel in HIST mode (search_fast.cuh) with the visited filter on and the full search history kept (up to
//      kHistMax entries; a longer history fails the build) -- then candidate pool = history + the node's current
//      neighbours, sorted by TotalOrder, truncated to max_candidate_pool_size, and alpha-robust pruning to
//      graph_max_degree (prune.h: Progressive strategy for L2 :183-240, Iterative for inner product :107-170):
//      `build_prune_kernel`, mode FORWARD;
//   2. add_reverse_edges (:475-580): every new edge v->u is mirrored as u->v when u has room
//      (`reverse_insert_kernel`), otherwise recorded in a per-vertex overflow list; vertices with overflow are
//      re-pruned over (overflow + adjacency) to prune_to: `build_prune_kernel`, mode REVERSE.
// Two passes (index.h:436-439): reverse pruning with alpha = 1 first, then with the configured alpha; the
// forward pruning always uses the configured alpha (vamana_build.h:268-272).
// A candidate set larger than the kPoolMax-entry shared pool is streamed through it in sorted chunks, each merged
// into the best max_candidate_pool_size so far, so the pool is the best of the whole set by TotalOrder.
//
// The reference's result depends on thread timing only through rounds of several nodes (add_reverse_edges walks a
// node's row while its peers append to it).  So the parity bar is (tests/test_gpu_build_exact.py): exact rows where
// every round holds one node (static builds of n <= 40, dynamic adds of at most 40 points); equal neighbour sets
// for large adds into an existing graph; recall equivalence of whole static builds, the reference's own bar
// (tests/integration/vamana/index_build.cpp:96,139).
// Distances inside the builder use the search path's bit-exact code (eval_pass), keys = sign * distance: the float tree
// for float32 / float16 rows, the exact integer ops (OP_*I) for int8 / uint8 rows, whose datum is its own query.
// SQ rows (int8 / uint8 codes with one global scale and bias, SQ = true) follow the reference's VamanaBuildAdaptor for
// SQ data (extensions/vamana/scalar.h:47-86): the datum is decompressed and prepared as the SQ search prepares an fp32
// query (stage_sq_datum), then measured with the SQ search's operators (OP_L2I scaled by scale^2, OP_IPF, OP_COSF).
//
// The dynamic index reuses these kernels: add_points runs `construct` over a list of slots (BuildParams::slots),
// and consolidate (consolidate.h) selects each node's candidate pool with `consolidate_pool_kernel` and prunes it
// with `build_prune_kernel` in mode CONSOLIDATE.
#pragma once

#include "query_prep.cuh"
#include "search_fast.cuh"

#include <cfloat>

namespace svsb200 {

constexpr uint32_t kPoolMax = 512;   // candidate pool entries per node held in shared memory
constexpr uint32_t kHistMax = 4096;  // search history entries recorded per node; a longer history fails the build

enum BuildPruneMode : int {
    PRUNE_FORWARD = 0,       // pool = search history + adjacency
    PRUNE_REVERSE = 1,       // pool = overflow edges + adjacency
    PRUNE_CONSOLIDATE = 2,   // pool = hist[w] as given (consolidate_pool_kernel's selection)
};

struct BuildParams {
    int reverse;                 // BuildPruneMode
    uint32_t first;              // forward: first entry of the batch (node = first + i, or slots[first + i]; query row i)
    uint32_t count;              // forward / consolidate: batch size
    const uint32_t* count_ptr;   // reverse: number of touched vertices (device)
    const uint32_t* nodes;       // reverse: the touched vertices; consolidate: the batch's nodes
    uint2* hist;                 // forward, consolidate: [count][hist_cap] {key bits, id}
    uint32_t* hist_count;
    uint32_t hist_cap;
    const int* head;             // reverse: overflow linked lists (head per vertex, -1 = empty)
    const int* next;
    const uint32_t* pair_v;
    uint32_t* graph;             // [n][gstride], neighbours first, kNoNeighbor padding
    uint32_t* deg;               // [n]
    uint32_t gstride;
    uint32_t max_degree;         // R
    uint32_t limit;              // size of the pruned list: R (forward) / prune_to (reverse)
    uint32_t max_candidates;
    float alpha;
    int iterative;               // prune strategy: 0 = Progressive (L2), 1 = Iterative (inner product, cosine)
    unsigned int* work_counter;
    const uint32_t* slots;       // forward: the batch's nodes are slots[first + i] (NULL: first + i)
    const uint8_t* status;       // consolidate_pool_kernel: SlotStatus per slot
    uint32_t* scratch_ids;       // consolidate_pool_kernel: [grid][scratch_len] per warp
    float* scratch_keys;
    uint32_t scratch_len;        // a power of two >= max_degree^2
    unsigned int* hist_overflow; // forward: set to 1 when a search history reached hist_cap entries
};

// Per-CTA (one warp) shared memory of build_prune_kernel.
__host__ __device__ inline size_t build_smem_bytes(uint32_t qstride) {
    // query | candidate ids | candidate keys | prune state | compact list ids, keys, pool positions | result
    return size_t(qstride) * 4 + size_t(kPoolMax) * 4 * 6 + 256 * 4;
}

// An int8 / uint8 row's codes as the integer distance code expects its operand (what prepare_queries_kernel writes in
// PREP_INT mode): the raw bytes, zero-padded to qstride (a multiple of 16) bytes, to `dst`.  Returns the exact sum x*x.
template <int ROWT>
__device__ __forceinline__ int stage_codes(const char* row, uint32_t dim, uint32_t qstride, uint32_t* dst, int lane) {
    int xx = 0;
    for (uint32_t i = lane; i < qstride / 4; i += 32) {
        uint32_t w = 0;
        if (4 * i < dim) {
            w = reinterpret_cast<const uint32_t*>(row)[i];
            if (4 * i + 4 > dim) w &= (1u << (8 * (dim - 4 * i))) - 1u;
        }
        dst[i] = w;
        if constexpr (ROWT == SVSB200_I8) xx = __dp4a(int(w), int(w), xx);
        else xx = int(__dp4a(w, w, unsigned(xx)));
    }
    for (int o = 16; o; o >>= 1) xx += __shfl_xor_sync(0xFFFFFFFFu, xx, o);
    return xx;
}

// The cosine `a_norm` of an int8 / uint8 row (CosineSimilarity::fix_argument -> distance::norm, distance_core.h:45-66):
// sqrt of a sequential fp32 `accum += x*x`.  Every partial sum is a non-negative integer no larger than xx, so while
// xx <= 2^24 they are all exact and the result is float(xx); above that the order rounds, and lane 0 repeats the sum in
// the reference's order.
template <int ROWT>
__device__ __forceinline__ float codes_norm(const char* row, uint32_t dim, int xx, int lane) {
    float acc = float(xx);
    if (xx > (1 << 24)) {
        if (lane == 0) {
            acc = 0.f;
            for (uint32_t i = 0; i < dim; ++i) {
                const int v = ROWT == SVSB200_I8 ? int(int8_t(row[i])) : int(uint8_t(row[i]));
                acc = __fadd_rn(acc, float(v * v));
            }
        }
        acc = __shfl_sync(0xFFFFFFFFu, acc, 0);
    }
    return __fsqrt_rn(acc);
}

// An SQ datum as its own query: DecompressionAdaptor::fix_argument (quantization/scalar/scalar.h:583-589) decompresses
// the codes to fp32 and hands them to the compressed distance's fix_argument, which is what prepare_queries_kernel
// does for an fp32 query of the SQ search (query_prep.cuh).  OP_L2I (EuclideanCompressed): the fp32 row compressed
// again -- the round trip need not return the datum's codes -- to qstride bytes at `dst`, `aux1` = the int32 bits of
// their sum x*x.  OP_IPF / OP_COSF: the fp32 row, zero-padded to qstride floats at `dst`; returns the MIP offset or the
// cosine norm.  One warp; `dst` in shared or global memory.
template <int ROWT, int OP>
__device__ __forceinline__ float stage_sq_datum(const SearchParams& p, const char* row, void* dst, int lane, float& aux1) {
    auto code = [&](uint32_t i) { return ROWT == SVSB200_I8 ? int(int8_t(row[i])) : int(uint8_t(row[i])); };
    if constexpr (OP == OP_L2I) {
        uint8_t* c = static_cast<uint8_t*>(dst);
        int xx = 0;
        for (uint32_t i = lane; i < p.qstride; i += 32) {
            uint8_t cv = 0;
            if (i < p.dim) {
                cv = sq_compress_code(sq_decompress(code(i), p.scale, p.bias), ROWT, p.scale, p.bias);
                const int v = ROWT == SVSB200_I8 ? int(int8_t(cv)) : int(cv);
                xx += v * v;
            }
            c[i] = cv;
        }
        for (int o = 16; o; o >>= 1) xx += __shfl_xor_sync(0xFFFFFFFFu, xx, o);
        aux1 = __int_as_float(xx);
        __syncwarp();
        return 0.f;
    } else {
        static_assert(OP == OP_IPF || OP == OP_COSF, "SQ builds measure with OP_L2I, OP_IPF or OP_COSF");
        float* f = static_cast<float*>(dst);
        for (uint32_t i = lane; i < p.qstride; i += 32) f[i] = i < p.dim ? sq_decompress(code(i), p.scale, p.bias) : 0.f;
        __syncwarp();
        float aux0 = 0.f;
        if (lane == 0) {
            if constexpr (OP == OP_IPF) aux0 = sq_ip_offset(f, p.dim, p.bias);
            else aux0 = sequential_norm(p.dim, [&](uint32_t i) { return __fmul_rn(f[i], f[i]); });
        }
        return __shfl_sync(0xFFFFFFFFu, aux0, 0);
    }
}

// Row `id` of the dataset as the operand the distance code expects in q_s (what prepare_queries_kernel does for a
// query): for the float ops the exact fp32 conversion, zero padding; for the integer ops the raw codes (stage_codes),
// with `aux1` = the int32 bits of sum x*x that OP_L2I needs; for SQ rows stage_sq_datum.
// Returns the row's Euclidean norm (the `a_norm` of CosineSimilarity::fix_argument, cosine.h:117-119), or for SQ rows
// stage_sq_datum's value.
template <int ROWT, int OP, bool SQ = false>
__device__ __forceinline__ float stage_row(const SearchParams& p, uint32_t id, float* q_s, int lane, float& aux1) {
    const char* row = reinterpret_cast<const char*>(p.vectors) + size_t(id) * p.row_stride;
    if constexpr (SQ) {
        return stage_sq_datum<ROWT, OP>(p, row, q_s, lane, aux1);
    } else if constexpr (OP >= OP_L2I) {
        const int xx = stage_codes<ROWT>(row, p.dim, p.qstride, reinterpret_cast<uint32_t*>(q_s), lane);
        aux1 = __int_as_float(xx);
        return codes_norm<ROWT>(row, p.dim, xx, lane);
    } else {
        float sq = 0.f;
        for (uint32_t i = lane; i < p.qstride; i += 32) {
            float v = 0.f;
            if (i < p.dim) {
                if constexpr (ROWT == SVSB200_F32) v = reinterpret_cast<const float*>(row)[i];
                else v = __half2float(reinterpret_cast<const __half*>(row)[i]);
            }
            q_s[i] = v;
            sq = fmaf(v, v, sq);
        }
        for (int o = 16; o; o >>= 1) sq += __shfl_xor_sync(0xFFFFFFFFu, sq, o);
        return sqrtf(sq);
    }
}

// Sorts the first `count` (key, id) pairs by TotalOrder (key, then id), one warp: bitonic over the next power of two
// >= 32, the tail padded with (+inf, 0xFFFFFFFF).  The arrays (shared or global) need room for that power of two.
__device__ __forceinline__ void warp_sort_pairs(float* key, uint32_t* id, uint32_t count, int lane) {
    uint32_t N = 32;
    while (N < count) N <<= 1;
    for (uint32_t i = count + lane; i < N; i += 32) {
        key[i] = INFINITY;
        id[i] = 0xFFFFFFFFu;
    }
    __syncwarp();
    for (uint32_t k = 2; k <= N; k <<= 1) {
        for (uint32_t j = k >> 1; j > 0; j >>= 1) {
            for (uint32_t i = lane; i < N / 2; i += 32) {
                const uint32_t a = ((i & ~(j - 1)) << 1) | (i & (j - 1));
                const uint32_t b = a | j;
                const bool up = (a & k) == 0;
                const float ka = key[a], kb = key[b];
                const uint32_t ia = id[a], ib = id[b];
                const bool a_gt_b = (kb < ka) || (!(ka < kb) && ib < ia);
                if (a_gt_b == up) {
                    key[a] = kb; key[b] = ka;
                    id[a] = ib; id[b] = ia;
                }
            }
            __syncwarp();
        }
    }
}

// Merges the sorted chunk (lkey, lid)[0, Q) into the sorted pool (ckey, cid)[0, P) and keeps the first `cap` entries by
// TotalOrder (merge path: output k takes A[i] or B[k - i], i found by binary search).  (tkey, tid) hold kPoolMax
// entries of scratch.  Returns the new pool size.  One warp; ids are distinct.
__device__ __forceinline__ uint32_t merge_into_pool(float* ckey, uint32_t* cid, uint32_t P, const float* lkey,
                                                    const uint32_t* lid, uint32_t Q, uint32_t cap, float* tkey,
                                                    uint32_t* tid, int lane) {
    const uint32_t out = min(P + Q, cap);
    auto a_first = [&](uint32_t i, uint32_t j) {   // pool entry i before chunk entry j
        return ckey[i] < lkey[j] || (!(lkey[j] < ckey[i]) && cid[i] < lid[j]);
    };
    for (uint32_t k = lane; k < out; k += 32) {
        uint32_t lo = k > Q ? k - Q : 0, hi = min(k, P);
        while (lo < hi) {
            const uint32_t mid = (lo + hi) >> 1;
            if (a_first(mid, k - 1 - mid)) lo = mid + 1;
            else hi = mid;
        }
        const uint32_t j = k - lo;
        const bool take_a = j >= Q || (lo < P && a_first(lo, j));
        tkey[k] = take_a ? ckey[lo] : lkey[j];
        tid[k] = take_a ? cid[lo] : lid[j];
    }
    __syncwarp();
    for (uint32_t k = lane; k < out; k += 32) {
        ckey[k] = tkey[k];
        cid[k] = tid[k];
    }
    __syncwarp();
    return out;
}

template <int ROWT, int OP, int DS, int KS, bool SQ = false>
__global__ void __launch_bounds__(32, SQ ? kSqBuildMinBlocks : 16) build_prune_kernel(const __grid_constant__ SearchParams p,
                                                            const __grid_constant__ BuildParams bp) {
    constexpr int G = OP >= OP_L2I ? 4 : KS * 16 / Row<ROWT>::LPT;   // threads per row, as in eval_pass
    constexpr int GROUPS = 32 / G;
    constexpr unsigned FULL = 0xFFFFFFFFu;
    extern __shared__ __align__(16) unsigned char smem_raw[];
    const int lane = threadIdx.x;
    const int g = lane / G, t = lane % G;
    const unsigned lt_mask = (1u << lane) - 1u;
    float* q_s = reinterpret_cast<float*>(smem_raw);
    uint32_t* cid = reinterpret_cast<uint32_t*>(q_s + p.qstride);   // [kPoolMax] pool ids
    float* ckey = reinterpret_cast<float*>(cid + kPoolMax);           // [kPoolMax] key of (node, candidate)
    float* state = ckey + kPoolMax;                                   // [kPoolMax] prune state
    uint32_t* lid = reinterpret_cast<uint32_t*>(state + kPoolMax);    // [kPoolMax] compact list: ids
    float* lkey = reinterpret_cast<float*>(lid + kPoolMax);           // [kPoolMax] compact list: keys
    uint32_t* lpos = reinterpret_cast<uint32_t*>(lkey + kPoolMax);    // [kPoolMax] compact list: pool positions
    uint32_t* res = lpos + kPoolMax;                                  // [256] result
    const char* vectors = reinterpret_cast<const char*>(p.vectors);
    const float ksign = p.greater ? -1.0f : 1.0f;
    const uint32_t total = bp.reverse == PRUNE_REVERSE ? *bp.count_ptr : bp.count;

    for (;;) {
        uint32_t w = 0;
        if (lane == 0) w = atomicAdd(bp.work_counter, 1u);
        w = __shfl_sync(FULL, w, 0);
        if (w >= total) break;
        const uint32_t node = bp.reverse ? bp.nodes[w] : bp.slots ? bp.slots[bp.first + w] : bp.first + w;
        const uint32_t deg0 = min(bp.deg[node], bp.max_degree);
        uint32_t* row = bp.graph + size_t(node) * bp.gstride;

        // ---- candidate pool ----
        uint32_t P = 0;       // entries whose key is known
        uint32_t M = 0;       // entries of lid[] whose distance to `node` still has to be computed
        float qnorm = 1.0f;   // cosine: norm of the vector currently staged as the query
        float qaux1 = 0.f;    // OP_L2I: int32 bits of sum x*x of the vector currently staged as the query
        if (bp.reverse == PRUNE_CONSOLIDATE) {
            // the whole pool, keys included, as consolidate_pool_kernel selected it
            qnorm = stage_row<ROWT, OP, SQ>(p, node, q_s, lane, qaux1);
            P = min(bp.hist_count[w], min(bp.hist_cap, kPoolMax));
            for (uint32_t i = lane; i < P; i += 32) {
                const uint2 e = bp.hist[size_t(w) * bp.hist_cap + i];
                ckey[i] = __uint_as_float(e.x);
                cid[i] = e.y;
            }
        } else if (!bp.reverse) {
            // the node as a query: prepared by the search launch of this round
            if constexpr (OP >= OP_L2I) {
                const uint32_t* src = reinterpret_cast<const uint32_t*>(p.qcodes + size_t(w) * p.qstride);
                for (uint32_t i = lane; i < p.qstride / 4; i += 32) reinterpret_cast<uint32_t*>(q_s)[i] = src[i];
                qaux1 = p.qaux[2 * size_t(w) + 1];
            } else {
                for (uint32_t i = lane; i < p.qstride; i += 32) q_s[i] = p.qf[size_t(w) * p.qstride + i];
            }
            qnorm = p.qaux[2 * size_t(w)];
            const uint32_t H = bp.hist_count[w];
            // the search stops recording at hist_cap entries: the history may be incomplete, so the build fails
            if (H >= bp.hist_cap && lane == 0) atomicExch(bp.hist_overflow, 1u);
            if (H + deg0 > kPoolMax) {
                // more than the shared pool holds: the unexpanded neighbours, then the history in chunks, each merged
                // into the best max_candidates so far
                const uint2* hist = bp.hist + size_t(w) * bp.hist_cap;
                uint32_t Q = 0;
                for (uint32_t j0 = 0; j0 < deg0; j0 += 32) {
                    const uint32_t j = j0 + lane;
                    const uint32_t id = j < deg0 ? row[j] : kNoNeighbor;
                    bool fresh = id != kNoNeighbor && id != node;
                    for (uint32_t i = 0; fresh && i < H; ++i) fresh = hist[i].y != id;
                    const unsigned m = __ballot_sync(FULL, fresh);
                    if (fresh) lid[Q + __popc(m & lt_mask)] = id;
                    Q += __popc(m);
                }
                __syncwarp();
                for (uint32_t base = 0; base < Q; base += 2 * GROUPS)
                    eval_pass<ROWT, OP, DS, 2, KS, true>(p, q_s, vectors, lid, lkey, base, Q, g, t, qnorm, qaux1, ksign);
                __syncwarp();
                warp_sort_pairs(lkey, lid, Q, lane);
                P = merge_into_pool(ckey, cid, 0, lkey, lid, Q, bp.max_candidates, state, lpos, lane);
                for (uint32_t h0 = 0; h0 < H; h0 += kPoolMax) {
                    Q = min(kPoolMax, H - h0);
                    for (uint32_t i = lane; i < Q; i += 32) {
                        const uint2 e = hist[h0 + i];
                        lkey[i] = __uint_as_float(e.x);
                        lid[i] = e.y;
                    }
                    __syncwarp();
                    warp_sort_pairs(lkey, lid, Q, lane);
                    P = merge_into_pool(ckey, cid, P, lkey, lid, Q, bp.max_candidates, state, lpos, lane);
                }
            } else {
                P = H;
                for (uint32_t i = lane; i < P; i += 32) {
                    const uint2 e = bp.hist[size_t(w) * bp.hist_cap + i];
                    ckey[i] = __uint_as_float(e.x);
                    cid[i] = e.y;
                }
                __syncwarp();
                // neighbours of the node that the search did not visit (vamana_build.h:424-441)
                for (uint32_t j0 = 0; j0 < deg0; j0 += 32) {
                    const uint32_t j = j0 + lane;
                    const uint32_t id = j < deg0 ? row[j] : kNoNeighbor;
                    bool fresh = id != kNoNeighbor && id != node;
                    for (uint32_t i = 0; fresh && i < P; ++i) fresh = cid[i] != id;
                    const unsigned m = __ballot_sync(FULL, fresh);
                    if (fresh) lid[M + __popc(m & lt_mask)] = id;
                    M += __popc(m);
                }
            }
        } else {
            qnorm = stage_row<ROWT, OP, SQ>(p, node, q_s, lane, qaux1);
            // overflow edges of this round (vamana_build.h:528-531): one per node of the round that links here, so
            // they are distinct and none is the node itself
            uint32_t nover = 0;
            if (lane == 0)
                for (int i = bp.head[node]; i >= 0; i = bp.next[i]) ++nover;
            nover = __shfl_sync(FULL, nover, 0);
            if (nover + deg0 > kPoolMax) {
                // more than the shared pool holds: the old adjacency list, then the overflow edges that are not in it
                // in chunks, each merged into the best max_candidates so far.  res[] keeps a copy of the list.
                uint32_t Q = 0;
                for (uint32_t j0 = 0; j0 < deg0; j0 += 32) {
                    const uint32_t j = j0 + lane;
                    const uint32_t id = j < deg0 ? row[j] : kNoNeighbor;
                    const bool ok = id != kNoNeighbor && id != node;
                    const unsigned m = __ballot_sync(FULL, ok);
                    if (ok) lid[Q + __popc(m & lt_mask)] = res[Q + __popc(m & lt_mask)] = id;
                    Q += __popc(m);
                }
                const uint32_t nrow = Q;
                __syncwarp();
                for (uint32_t base = 0; base < Q; base += 2 * GROUPS)
                    eval_pass<ROWT, OP, DS, 2, KS, true>(p, q_s, vectors, lid, lkey, base, Q, g, t, qnorm, qaux1, ksign);
                __syncwarp();
                warp_sort_pairs(lkey, lid, Q, lane);
                P = merge_into_pool(ckey, cid, 0, lkey, lid, Q, bp.max_candidates, state, lpos, lane);
                int cur = bp.head[node];
                while (cur >= 0) {
                    if (lane == 0)
                        for (Q = 0; cur >= 0 && Q < kPoolMax; cur = bp.next[cur]) lid[Q++] = bp.pair_v[cur];
                    Q = __shfl_sync(FULL, Q, 0);
                    cur = __shfl_sync(FULL, cur, 0);
                    __syncwarp();
                    uint32_t U = 0;
                    for (uint32_t j0 = 0; j0 < Q; j0 += 32) {
                        const uint32_t j = j0 + lane;
                        const uint32_t id = j < Q ? lid[j] : kNoNeighbor;
                        bool fresh = j < Q;
                        for (uint32_t z = 0; fresh && z < nrow; ++z) fresh = res[z] != id;
                        const unsigned m = __ballot_sync(FULL, fresh);
                        if (fresh) lid[U + __popc(m & lt_mask)] = id;
                        U += __popc(m);
                    }
                    __syncwarp();
                    for (uint32_t base = 0; base < U; base += 2 * GROUPS)
                        eval_pass<ROWT, OP, DS, 2, KS, true>(p, q_s, vectors, lid, lkey, base, U, g, t, qnorm, qaux1, ksign);
                    __syncwarp();
                    warp_sort_pairs(lkey, lid, U, lane);
                    P = merge_into_pool(ckey, cid, P, lkey, lid, U, bp.max_candidates, state, lpos, lane);
                }
            } else {
                if (lane == 0) {
                    uint32_t c = 0;
                    for (int i = bp.head[node]; i >= 0; i = bp.next[i]) lid[c++] = bp.pair_v[i];
                }
                M = nover;
                __syncwarp();
                // the old adjacency list, minus what the overflow already holds (:534-538)
                for (uint32_t j0 = 0; j0 < deg0; j0 += 32) {
                    const uint32_t j = j0 + lane;
                    const uint32_t id = j < deg0 ? row[j] : kNoNeighbor;
                    bool fresh = id != kNoNeighbor && id != node;
                    for (uint32_t i = 0; fresh && i < nover; ++i) fresh = lid[i] != id;
                    const unsigned m = __ballot_sync(FULL, fresh);
                    if (fresh) lid[M + __popc(m & lt_mask)] = id;
                    M += __popc(m);
                }
            }
        }
        __syncwarp();
        // distances node -> lid[0..M), appended to the pool
        for (uint32_t base = 0; base < M; base += 2 * GROUPS)
            eval_pass<ROWT, OP, DS, 2, KS, true>(p, q_s, vectors, lid, lkey, base, M, g, t, qnorm, qaux1, ksign);
        __syncwarp();
        for (uint32_t i = lane; i < M; i += 32) {
            cid[P + i] = lid[i];
            ckey[P + i] = lkey[i];
        }
        P += M;
        __syncwarp();

        warp_sort_pairs(ckey, cid, P, lane);
        P = min(P, bp.max_candidates);

        // ---- heuristic_prune_neighbors (prune.h): state[] is the Progressive strategy's `pruned` ratio
        // (tombstone = lowest, sentinel = max) or the Iterative strategy's state (0 available, 1 added, 2 pruned)
        for (uint32_t i = lane; i < P; i += 32) state[i] = bp.iterative ? 0.0f : -FLT_MAX;
        __syncwarp();
        uint32_t nres = 0;
        float cur_alpha = 1.0f;
        // while (result.size() < max && !cmp(alpha, current_alpha)): cmp is < for L2, > for inner product
        while (nres < bp.limit && !(p.greater ? bp.alpha > cur_alpha : bp.alpha < cur_alpha)) {
            uint32_t start = 0;
            while (nres < bp.limit && start < P) {
                // next pool entry that is not excluded at this alpha level
                uint32_t j = start + lane;
                bool ok = false;
                if (j < P) {
                    const float st = state[j];
                    const bool excluded = bp.iterative ? st != 0.0f : cur_alpha < st;
                    ok = !excluded && cid[j] != node;
                }
                const unsigned m = __ballot_sync(FULL, ok);
                if (m == 0) {
                    start += 32;
                    continue;
                }
                j = start + __ffs(m) - 1;
                start = j + 1;
                if (lane == 0) {
                    state[j] = bp.iterative ? 1.0f : FLT_MAX;
                    res[nres] = cid[j];
                }
                ++nres;
                qnorm = stage_row<ROWT, OP, SQ>(p, cid[j], q_s, lane, qaux1);
                __syncwarp();
                // the later entries still available at this level, compacted
                uint32_t L = 0;
                for (uint32_t t0 = start; t0 < P; t0 += 32) {
                    const uint32_t tt = t0 + lane;
                    bool av = false;
                    if (tt < P) {
                        const float st = state[tt];
                        av = bp.iterative ? st == 0.0f : !(cur_alpha < st);
                    }
                    const unsigned mm = __ballot_sync(FULL, av);
                    if (av) {
                        lid[L + __popc(mm & lt_mask)] = cid[tt];
                        lpos[L + __popc(mm & lt_mask)] = tt;
                    }
                    L += __popc(mm);
                }
                __syncwarp();
                if (L == 0) continue;
                // djk for every listed entry: key(selected, candidate)
                for (uint32_t base = 0; base < L; base += 2 * GROUPS)
                    eval_pass<ROWT, OP, DS, 2, KS, true>(p, q_s, vectors, lid, lkey, base, L, g, t, qnorm, qaux1, ksign);
                __syncwarp();
                for (uint32_t i = lane; i < L; i += 32) {
                    const uint32_t tt = lpos[i];
                    const float djk = lkey[i] * ksign;          // distance(selected, candidate)
                    const float dvt = ckey[tt] * ksign;         // distance(node, candidate)
                    if (bp.iterative) {
                        // if (cmp(current_alpha * djk, candidate.distance())) pruned   (prune.h:150)
                        const float lhs = cur_alpha * djk;
                        if (p.greater ? lhs > dvt : lhs < dvt) state[tt] = 2.0f;
                    } else {
                        // pruned[t] = std::max(pruned[t], candidate.distance() / djk, cmp)   (prune.h:227)
                        const float r = dvt / djk;
                        if (state[tt] < r) state[tt] = r;
                    }
                }
                __syncwarp();
            }
            if (bp.alpha == 1.0f) break;
            if (bp.iterative)
                for (uint32_t i = lane; i < P; i += 32)
                    if (state[i] == 2.0f) state[i] = 0.0f;   // reenable (prune.h:160-163)
            cur_alpha *= bp.alpha;
            __syncwarp();
        }
        __syncwarp();
        // ---- graph.replace_node(node, result) ----
        for (uint32_t j = lane; j < bp.gstride; j += 32) row[j] = j < nres ? res[j] : kNoNeighbor;
        if (lane == 0) bp.deg[node] = nres;
        __syncwarp();
    }
}

// Candidate pools of consolidation (GraphConsolidator::generate_updates, consolidate.h:191-288), one warp per Valid
// node that has a neighbour which is not Valid, persistent over bp.nodes[0 .. bp.count):
//   populate_candidates: the node's Valid neighbours and the adjacency rows of the others;
//   filter_candidates: repeats and ids that are not Valid dropped, distances from the node (cosine: fix_argument on the
//   node), sorted;  the first max_candidate_pool_size are kept.
// The whole set (up to max_degree^2 ids) lives in this warp's slice of global scratch; it is sorted by id to drop the
// repeats, then by TotalOrder (key, id) -- the reference sorts by distance alone, so its order among exactly equal
// distances is unspecified -- and the best max_candidates go to hist[w] for build_prune_kernel (PRUNE_CONSOLIDATE).
// The node itself stays in the pool when a deleted neighbour links back to it, as in the reference; the prune skips
// it.  The kernel reads the node's own row and the rows of slots that are not Valid only.  Over SQ codes (SQ = true) the
// node is staged as the SQ build stages a datum (stage_sq_datum) and the candidates are measured with the SQ search's
// operators: the general distance of the reference's build adaptor (consolidate.h:241-244).
template <int ROWT, int OP, int DS, int KS, bool SQ = false>
__global__ void __launch_bounds__(32, SQ && OP < OP_L2I ? kSqBuildMinBlocks : 16) consolidate_pool_kernel(const __grid_constant__ SearchParams p,
                                                                 const __grid_constant__ BuildParams bp) {
    constexpr int G = OP >= OP_L2I ? 4 : KS * 16 / Row<ROWT>::LPT;   // threads per row, as in eval_pass
    constexpr int GROUPS = 32 / G;
    constexpr unsigned FULL = 0xFFFFFFFFu;
    extern __shared__ __align__(16) unsigned char smem_raw[];
    float* q_s = reinterpret_cast<float*>(smem_raw);
    const int lane = threadIdx.x;
    const int g = lane / G, t = lane % G;
    const unsigned lt_mask = (1u << lane) - 1u;
    uint32_t* sid = bp.scratch_ids + size_t(blockIdx.x) * bp.scratch_len;
    float* skey = bp.scratch_keys + size_t(blockIdx.x) * bp.scratch_len;
    const char* vectors = reinterpret_cast<const char*>(p.vectors);
    const float ksign = p.greater ? -1.0f : 1.0f;

    for (;;) {
        uint32_t w = 0;
        if (lane == 0) w = atomicAdd(bp.work_counter, 1u);
        w = __shfl_sync(FULL, w, 0);
        if (w >= bp.count) break;
        const uint32_t node = bp.nodes[w];
        const uint32_t* row = bp.graph + size_t(node) * bp.gstride;
        const uint32_t deg0 = min(bp.deg[node], bp.max_degree);
        // ---- populate_candidates + the Valid filter ----
        uint32_t M = 0;
        for (uint32_t j = 0; j < deg0; ++j) {
            const uint32_t dst = row[j];
            if (bp.status[dst] == SLOT_VALID) {
                if (lane == 0) sid[M] = dst;
                ++M;
                continue;
            }
            const uint32_t* orow = bp.graph + size_t(dst) * bp.gstride;
            const uint32_t od = min(bp.deg[dst], bp.max_degree);
            for (uint32_t j0 = 0; j0 < od; j0 += 32) {
                const uint32_t jj = j0 + lane;
                const uint32_t id = jj < od ? orow[jj] : kNoNeighbor;
                const bool keep = id != kNoNeighbor && bp.status[id] == SLOT_VALID;
                const unsigned m = __ballot_sync(FULL, keep);
                if (keep) sid[M + __popc(m & lt_mask)] = id;
                M += __popc(m);
            }
        }
        __syncwarp();
        // ---- repeats: sort by id, keep the first of every run ----
        for (uint32_t i = lane; i < M; i += 32) skey[i] = 0.0f;
        warp_sort_pairs(skey, sid, M, lane);
        uint32_t U = 0, carry = 0xFFFFFFFFu;
        for (uint32_t i0 = 0; i0 < M; i0 += 32) {
            const uint32_t i = i0 + lane;
            const uint32_t id = i < M ? sid[i] : 0xFFFFFFFFu;
            uint32_t prev = __shfl_up_sync(FULL, id, 1);
            if (lane == 0) prev = carry;
            carry = __shfl_sync(FULL, id, 31);
            const bool keep = i < M && id != prev;
            const unsigned m = __ballot_sync(FULL, keep);
            __syncwarp();
            if (keep) sid[U + __popc(m & lt_mask)] = id;
            U += __popc(m);
        }
        __syncwarp();
        // ---- filter_candidates: distances from the node, TotalOrder ----
        float qaux1 = 0.f;
        const float qnorm = stage_row<ROWT, OP, SQ>(p, node, q_s, lane, qaux1);
        __syncwarp();
        for (uint32_t base = 0; base < U; base += 2 * GROUPS)
            eval_pass<ROWT, OP, DS, 2, KS, true>(p, q_s, vectors, sid, skey, base, U, g, t, qnorm, qaux1, ksign);
        __syncwarp();
        warp_sort_pairs(skey, sid, U, lane);
        const uint32_t P = min(U, bp.max_candidates);
        for (uint32_t i = lane; i < P; i += 32)
            bp.hist[size_t(w) * bp.hist_cap + i] = make_uint2(__float_as_uint(skey[i]), sid[i]);
        if (lane == 0) bp.hist_count[w] = P;
        __syncwarp();
    }
}

// The builder's launchers, instantiated once per row type in build_<type>.cu.  Its lean search (HIST) and prune take
// BuildOps; consolidation's candidate pools are for DynamicRows (and over SQ codes DynamicSqRows, build_sq_<type>.cu).  The prune and the pool run on the caller's grid:
// `grid` warps, for the pool each with its own scratch slice (bp.scratch_len entries).
template <int ROWT> cudaError_t launch_build_search(int op, const SearchParams& p, const LaunchConfig& cfg) {
    return dispatch(BuildOps<ROWT>{}, op, [&](auto o) { return launch_fast<ROWT, decltype(o)::value, true, false>(p, cfg); });
}
template <int ROWT>
cudaError_t launch_build_prune_op(int op, const SearchParams& p, const BuildParams& bp, int grid, cudaStream_t stream) {
    const LaunchConfig cfg{grid, 1, build_smem_bytes(p.qstride), stream};
    return dispatch(BuildOps<ROWT>{}, op, [&](auto o) {
        constexpr int OP = decltype(o)::value;
        return with_shape<OP, false>(p.dim, true, [&](auto ds, auto ks) {
            return launch_kernel(build_prune_kernel<ROWT, OP, decltype(ds)::value, decltype(ks)::value>, cfg, grid, true,
                                 p, bp);
        });
    });
}
// SQ rows: batch rows [first, first+count) (or slots[first + q]) prepared as their own queries (stage_sq_datum) into
// qcodes (OP_L2I) or qf, and qaux = {aux0, aux1}.  One warp per row.
template <int ROWT, int OP>
__global__ void batch_sq_kernel(const __grid_constant__ SearchParams p, uint32_t first, uint32_t count,
                                const uint32_t* __restrict__ slots, float* __restrict__ qf, uint8_t* __restrict__ qcodes,
                                float* __restrict__ qaux) {
    const uint32_t q = blockIdx.x * (blockDim.x / 32) + threadIdx.x / 32;
    const int lane = threadIdx.x & 31;
    if (q >= count) return;
    const char* row = reinterpret_cast<const char*>(p.vectors) + size_t(slots ? slots[first + q] : first + q) * p.row_stride;
    void* dst = OP == OP_L2I ? static_cast<void*>(qcodes + size_t(q) * p.qstride) : static_cast<void*>(qf + size_t(q) * p.qstride);
    float aux1 = 0.f;
    const float aux0 = stage_sq_datum<ROWT, OP>(p, row, dst, lane, aux1);
    if (lane == 0) {
        qaux[2 * size_t(q)] = aux0;
        qaux[2 * size_t(q) + 1] = aux1;
    }
}

// The SQ builder's launchers (BuildSqOps), instantiated once per code type in build_sq_<type>.cu.  The lean search's
// OP_L2I form reads SearchParams::sq at run time, so the integer builder's launch_build_search serves SQ L2; this one
// takes OP_IPF and OP_COSF.
template <int ROWT> cudaError_t launch_build_search_sq(int op, const SearchParams& p, const LaunchConfig& cfg) {
    return dispatch(IntList<OP_IPF, OP_COSF>{}, op, [&](auto o) { return launch_fast<ROWT, decltype(o)::value, true, false>(p, cfg); });
}
template <int ROWT>
cudaError_t launch_build_prune_sq(int op, const SearchParams& p, const BuildParams& bp, int grid, cudaStream_t stream) {
    const LaunchConfig cfg{grid, 1, build_smem_bytes(p.qstride), stream};
    return dispatch(BuildSqOps{}, op, [&](auto o) {
        constexpr int OP = decltype(o)::value;
        return with_shape<OP, false>(p.dim, true, [&](auto ds, auto ks) {
            return launch_kernel(build_prune_kernel<ROWT, OP, decltype(ds)::value, decltype(ks)::value, true>, cfg, grid,
                                 true, p, bp);
        });
    });
}
template <int ROWT>
cudaError_t launch_build_batch_sq(int op, const SearchParams& p, uint32_t first, uint32_t count, const uint32_t* slots,
                                  float* qf, uint8_t* qcodes, float* qaux, cudaStream_t stream) {
    const LaunchConfig cfg{int((count + 7) / 8), 8, 0, stream};
    return dispatch(BuildSqOps{}, op, [&](auto o) {
        return launch_kernel(batch_sq_kernel<ROWT, decltype(o)::value>, cfg, size_t(cfg.grid), false, p, first, count,
                             slots, qf, qcodes, qaux);
    });
}

template <int ROWT>
cudaError_t launch_consolidate_pool_op(int op, const SearchParams& p, const BuildParams& bp, int grid, cudaStream_t stream) {
    const LaunchConfig cfg{grid, 1, size_t(p.qstride) * 4, stream};
    return dispatch(DynamicOps{}, op, [&](auto o) {
        constexpr int OP = decltype(o)::value;
        return with_shape<OP, false>(p.dim, true, [&](auto ds, auto ks) {
            return launch_kernel(consolidate_pool_kernel<ROWT, OP, decltype(ds)::value, decltype(ks)::value>, cfg, grid, false,
                                 p, bp);
        });
    });
}
template <int ROWT>
cudaError_t launch_consolidate_pool_sq(int op, const SearchParams& p, const BuildParams& bp, int grid, cudaStream_t stream) {
    const LaunchConfig cfg{grid, 1, size_t(p.qstride) * 4, stream};
    return dispatch(DynamicSqOps{}, op, [&](auto o) {
        constexpr int OP = decltype(o)::value;
        return with_shape<OP, false>(p.dim, true, [&](auto ds, auto ks) {
            return launch_kernel(consolidate_pool_kernel<ROWT, OP, decltype(ds)::value, decltype(ks)::value, true>, cfg, grid,
                                 false, p, bp);
        });
    });
}

extern template cudaError_t launch_build_search<SVSB200_F32>(int, const SearchParams&, const LaunchConfig&);
extern template cudaError_t launch_build_search<SVSB200_F16>(int, const SearchParams&, const LaunchConfig&);
extern template cudaError_t launch_build_search<SVSB200_I8>(int, const SearchParams&, const LaunchConfig&);
extern template cudaError_t launch_build_search<SVSB200_U8>(int, const SearchParams&, const LaunchConfig&);
extern template cudaError_t launch_build_prune_op<SVSB200_F32>(int, const SearchParams&, const BuildParams&, int, cudaStream_t);
extern template cudaError_t launch_build_prune_op<SVSB200_F16>(int, const SearchParams&, const BuildParams&, int, cudaStream_t);
extern template cudaError_t launch_build_prune_op<SVSB200_I8>(int, const SearchParams&, const BuildParams&, int, cudaStream_t);
extern template cudaError_t launch_build_prune_op<SVSB200_U8>(int, const SearchParams&, const BuildParams&, int, cudaStream_t);
extern template cudaError_t launch_build_search_sq<SVSB200_I8>(int, const SearchParams&, const LaunchConfig&);
extern template cudaError_t launch_build_search_sq<SVSB200_U8>(int, const SearchParams&, const LaunchConfig&);
extern template cudaError_t launch_build_prune_sq<SVSB200_I8>(int, const SearchParams&, const BuildParams&, int, cudaStream_t);
extern template cudaError_t launch_build_prune_sq<SVSB200_U8>(int, const SearchParams&, const BuildParams&, int, cudaStream_t);
extern template cudaError_t launch_build_batch_sq<SVSB200_I8>(int, const SearchParams&, uint32_t, uint32_t, const uint32_t*,
                                                             float*, uint8_t*, float*, cudaStream_t);
extern template cudaError_t launch_build_batch_sq<SVSB200_U8>(int, const SearchParams&, uint32_t, uint32_t, const uint32_t*,
                                                             float*, uint8_t*, float*, cudaStream_t);
extern template cudaError_t launch_consolidate_pool_op<SVSB200_F32>(int, const SearchParams&, const BuildParams&, int, cudaStream_t);
extern template cudaError_t launch_consolidate_pool_op<SVSB200_F16>(int, const SearchParams&, const BuildParams&, int, cudaStream_t);
extern template cudaError_t launch_consolidate_pool_sq<SVSB200_I8>(int, const SearchParams&, const BuildParams&, int, cudaStream_t);
extern template cudaError_t launch_consolidate_pool_sq<SVSB200_U8>(int, const SearchParams&, const BuildParams&, int, cudaStream_t);

}  // namespace svsb200
