// ivf_kernel.cuh -- kernels of the IVF index (ivf.cu): the cluster-major leaf scan, the k-means update and the grouped
// assignment and update of the hierarchical k-means.
//
// Replaces, for float32 / float16 rows (file:line under the reference's include/svs):
//   index/ivf/index.h  IVFIndex::search's leaf scan (one thread per query walks each probed cluster)
//   index/ivf/common.h:446-490 centroid_adjustment (the k-means update)
//
// ivf_scan_kernel: one work item is (cluster, chunk of up to Q queries probing it).  Persistent CTAs pull work items
// from a counter; a CTA streams the cluster's rows through a two-slot shared-memory ring (cp.async, 16 bytes per
// copy), so a probed cluster's rows leave HBM once per query chunk instead of once per query.  Each warp scores its
// queries against every staged tile with the search path's own distance code (float_rows in its shared-memory form,
// finish_distance), bit for bit, and keeps one sorted top-k list per (query, probe) in shared memory.  A cluster's rows
// are stored in ascending original id, and a new row goes after an equal old key, so every list is ordered by
// (distance, original id): the TotalOrder of the merge that follows (merge_topk_kernel).
#pragma once

#include "query_prep.cuh"
#include "search_kernel.cuh"

namespace svsb200 {

constexpr int IVF_WARPS = 8;              // warps per CTA of the scan
constexpr uint32_t IVF_TILE_ROWS = 32;    // rows per ring slot (fewer for very wide rows: ivf.cu)
constexpr uint32_t IVF_QMAX = 64;         // queries per work item

struct IvfScanParams {
    SearchParams p;                 // dim, row_stride, qf / qaux / qstride, greater (the distance code's fields)
    const char* rows;               // cluster-major rows, each cluster starting on a 32-row boundary
    const uint32_t* row_ids;        // original id of every stored row
    const uint32_t* cl_start;       // [C] first stored row of each cluster
    const uint32_t* cl_count;       // [C] rows of each cluster
    const uint32_t* list_off;       // [C+1] per-cluster query lists: entries list_off[c] .. list_off[c+1]
    const uint32_t* list;           // entry = query * P + probe, ascending within a list
    const uint32_t* item_off;       // [C+1] work items of each cluster (ceil(list length / Q)); item_off[C] = total
    uint32_t C, P, nq, k, Q, tile_rows;
    uint64_t* out_ids;              // [P][nq][k] per (probe, query) lists, original ids
    float* out_dists;
    unsigned int* work_counter;
};

// Shared memory of one CTA: the ring, then per query slot {query, keys, ids}, then per warp {candidate keys, positions}.
__host__ __device__ inline size_t ivf_slot_bytes(uint32_t qstride, uint32_t k) {
    return size_t(qstride) * 4 + (size_t(k) * 8 + 15) / 16 * 16;
}
__host__ __device__ inline size_t ivf_smem_bytes(uint32_t row_stride, uint32_t tile_rows, uint32_t qstride, uint32_t k,
                                                 uint32_t Q) {
    return 2 * size_t(tile_rows) * row_stride + size_t(Q) * ivf_slot_bytes(qstride, k) + size_t(IVF_WARPS) * 32 * 8;
}

// Merges the `count` scored rows of a tile (keys in ckey[0..count), ids ids[0..count), ascending) into the sorted list
// (bkey, bid) of `size` <= k entries: the result of inserting them one by one, each after the equal keys already there,
// truncated at k.  Warp-collective.
// DYN (the dynamic IVF index, dynamic_ivf.cu): the ids are slots in no particular order, all-ones marking a tombstone,
// which is not a candidate; the list is ordered by (key, slot), so both the upper bound and the rank among the tile's
// survivors compare (key, id) lexicographically.
template <bool DYN = false>
__device__ __forceinline__ void ivf_merge(float* bkey, uint32_t* bid, uint32_t& size, uint32_t k, const float* ckey,
                                          const uint32_t* ids, uint32_t count, uint32_t* spos, int lane) {
    constexpr unsigned FULL = 0xFFFFFFFFu;
    if constexpr (DYN) {
        const uint32_t id = uint32_t(lane) < count ? ids[lane] : 0xFFFFFFFFu;
        const bool valid = id != 0xFFFFFFFFu;
        const float d = valid ? ckey[lane] : 0.0f;
        // (d, id) before (e, j): distinct ids, so no pair is equal
        auto before = [](float d, uint32_t id, float e, uint32_t j) { return d < e || (!(e < d) && id < j); };
        const bool surv = valid && (size < k || before(d, id, bkey[size - 1], bid[size - 1]));
        const unsigned m = __ballot_sync(FULL, surv);
        if (!m) return;
        uint32_t ipos = 0;   // entries before (d, id): upper bound
        if (surv) {
            uint32_t lo = 0, hi = size;
            while (lo < hi) {
                const uint32_t mid = (lo + hi) >> 1;
                if (before(d, id, bkey[mid], bid[mid])) hi = mid; else lo = mid + 1;
            }
            ipos = lo;
        }
        uint32_t rank = 0;   // survivors before this one
        for (int s = 0; s < 32; ++s) {
            const float ds = __shfl_sync(FULL, d, s);
            const uint32_t is = __shfl_sync(FULL, id, s);
            if (surv && ((m >> s) & 1u)) rank += before(ds, is, d, id);
        }
        const uint32_t S = __popc(m);
        if (surv) spos[__popc(m & ((1u << lane) - 1u))] = ipos;
        const uint32_t minpos = __reduce_min_sync(FULL, surv ? ipos : 0xFFFFFFFFu);
        __syncwarp();
        if (minpos < size) {   // (as below)
            for (int ch = int((size - 1) >> 5); ch >= int(minpos >> 5); --ch) {
                const uint32_t j = uint32_t(ch) * 32 + lane;
                const bool have = j < size;
                const float kk = have ? bkey[j] : 0.0f;
                const uint32_t ii = have ? bid[j] : 0u;
                uint32_t shift = 0;
                for (uint32_t s = 0; s < S; ++s) shift += spos[s] <= j;
                __syncwarp();
                if (have && j + shift < k) {
                    bkey[j + shift] = kk;
                    bid[j + shift] = ii;
                }
                __syncwarp();
            }
        }
        const uint32_t fp = ipos + rank;
        if (surv && fp < k) {
            bkey[fp] = d;
            bid[fp] = id;
        }
        size = min(size + S, k);
        __syncwarp();
        return;
    }
    const bool valid = uint32_t(lane) < count;
    const float d = valid ? ckey[lane] : 0.0f;
    const bool surv = valid && (size < k || d < bkey[size - 1]);
    const unsigned m = __ballot_sync(FULL, surv);
    if (!m) return;
    uint32_t ipos = 0;   // entries with a key <= d: upper bound
    if (surv) {
        uint32_t lo = 0, hi = size;
        while (lo < hi) {
            const uint32_t mid = (lo + hi) >> 1;
            if (d < bkey[mid]) hi = mid; else lo = mid + 1;
        }
        ipos = lo;
    }
    uint32_t rank = 0;   // survivors before this one: smaller keys, or equal keys on lower lanes
    for (int s = 0; s < 32; ++s) {
        const float ds = __shfl_sync(FULL, d, s);
        if (surv && ((m >> s) & 1u)) rank += (ds < d) || (!(d < ds) && s < lane);
    }
    const uint32_t S = __popc(m);
    if (surv) spos[__popc(m & ((1u << lane) - 1u))] = ipos;
    const uint32_t minpos = __reduce_min_sync(FULL, surv ? ipos : 0xFFFFFFFFu);
    const uint32_t id = valid ? ids[lane] : 0u;
    __syncwarp();
    if (minpos < size) {   // old entries move up by the number of survivors inserted at or before them, top first
        for (int ch = int((size - 1) >> 5); ch >= int(minpos >> 5); --ch) {
            const uint32_t j = uint32_t(ch) * 32 + lane;
            const bool have = j < size;
            const float kk = have ? bkey[j] : 0.0f;
            const uint32_t ii = have ? bid[j] : 0u;
            uint32_t shift = 0;
            for (uint32_t s = 0; s < S; ++s) shift += spos[s] <= j;
            __syncwarp();
            if (have && j + shift < k) {
                bkey[j + shift] = kk;
                bid[j + shift] = ii;
            }
            __syncwarp();
        }
    }
    const uint32_t fp = ipos + rank;
    if (surv && fp < k) {
        bkey[fp] = d;
        bid[fp] = id;
    }
    size = min(size + S, k);
    __syncwarp();
}

// DYN: the dynamic IVF index (ivf_merge<true>): row_ids holds slots, all-ones for a tombstone; lists by (distance, slot).
template <int ROWT, int OP, int DS, int NR, bool DYN = false>
__global__ void __launch_bounds__(IVF_WARPS * 32, 2) ivf_scan_kernel(const __grid_constant__ IvfScanParams ip) {
    constexpr int G = 16 / Row<ROWT>::LPT;   // threads per row
    constexpr int GROUPS = 32 / G;            // rows per warp and pass
    extern __shared__ __align__(16) unsigned char smem_raw[];
    const SearchParams& p = ip.p;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int g = lane / G, t = lane % G;
    const uint32_t tile_bytes = ip.tile_rows * p.row_stride;
    unsigned char* ring = smem_raw;
    unsigned char* slots = smem_raw + 2 * size_t(tile_bytes);
    const size_t slot_bytes = ivf_slot_bytes(p.qstride, ip.k);
    float* ckey = reinterpret_cast<float*>(slots + size_t(ip.Q) * slot_bytes) + warp * 64;
    uint32_t* spos = reinterpret_cast<uint32_t*>(ckey + 32);
    const float ksign = p.greater ? -1.0f : 1.0f;
    __shared__ uint32_t s_item;
    __shared__ uint32_t s_size[IVF_QMAX];   // list length of every slot
    const uint32_t total = ip.item_off[ip.C];

    for (;;) {
        if (threadIdx.x == 0) s_item = atomicAdd(ip.work_counter, 1u);
        __syncthreads();
        const uint32_t item = s_item;
        __syncthreads();
        if (item >= total) break;
        // the cluster of this item: last c with item_off[c] <= item
        uint32_t lo = 0, hi = ip.C;
        while (hi - lo > 1) {
            const uint32_t mid = (lo + hi) >> 1;
            if (ip.item_off[mid] <= item) lo = mid; else hi = mid;
        }
        const uint32_t c = lo;
        const uint32_t first = ip.list_off[c] + (item - ip.item_off[c]) * ip.Q;
        const uint32_t nslots = min(ip.Q, ip.list_off[c + 1] - first);
        const uint32_t count = ip.cl_count[c];
        const char* crows = ip.rows + size_t(ip.cl_start[c]) * p.row_stride;
        const uint32_t* cids = ip.row_ids + ip.cl_start[c];
        const uint32_t ntiles = (count + ip.tile_rows - 1) / ip.tile_rows;
        auto stage = [&](uint32_t tile) {   // whole tile, padding rows included (the cluster's storage is 32-row aligned)
            const char* src = crows + size_t(tile) * tile_bytes;
            unsigned char* dst = ring + (tile & 1u) * tile_bytes;
            for (uint32_t o = threadIdx.x * 16; o < tile_bytes; o += IVF_WARPS * 32 * 16) cp_async16(dst + o, src + o);
            cp_async_commit();
        };
        if (ntiles) stage(0);
        // the slots' queries (prepared as for the scan) and empty lists
        for (uint32_t s = 0; s < nslots; ++s) {
            const uint32_t q = ip.list[first + s] / ip.P;
            float* q_s = reinterpret_cast<float*>(slots + s * slot_bytes);
            for (uint32_t i = threadIdx.x; i < p.qstride; i += IVF_WARPS * 32) q_s[i] = p.qf[size_t(q) * p.qstride + i];
        }
        if (threadIdx.x < IVF_QMAX) s_size[threadIdx.x] = 0;
        __syncthreads();
        for (uint32_t tile = 0; tile < ntiles; ++tile) {
            if (tile + 1 < ntiles) {
                stage(tile + 1);
                asm volatile("cp.async.wait_group 1;" ::: "memory");
            } else {
                cp_async_wait_all();
            }
            __syncthreads();
            const char* trow = reinterpret_cast<const char*>(ring + (tile & 1u) * tile_bytes);
            const uint32_t rows = min(ip.tile_rows, count - tile * ip.tile_rows);
#pragma unroll 1
            for (uint32_t i = 0; i < IVF_QMAX / IVF_WARPS; ++i) {
                const uint32_t s = warp + IVF_WARPS * i;
                if (s >= nslots) break;
                const float* q_s = reinterpret_cast<const float*>(slots + s * slot_bytes);
                float* bkey = const_cast<float*>(q_s) + p.qstride;
                uint32_t* bid = reinterpret_cast<uint32_t*>(bkey + ip.k);
                const uint32_t q = ip.list[first + s] / ip.P;
                const float aux0 = p.qaux[2 * size_t(q)];
                for (uint32_t base = 0; base < rows; base += NR * GROUPS) {
                    const char* rowp[NR];
                    uint32_t idx[NR];
#pragma unroll
                    for (int r = 0; r < NR; ++r) {
                        idx[r] = base + r * GROUPS + g;
                        rowp[r] = idx[r] < rows ? trow + size_t(idx[r]) * p.row_stride : nullptr;
                    }
                    float sum[NR], nrm[NR];
                    float_rows<ROWT, OP, DS, NR, false, true>(p, q_s, rowp, t, sum, nrm);
#pragma unroll
                    for (int r = 0; r < NR; ++r) {
                        const float d = finish_distance<OP>(p, sum[r], nrm[r], 0, 0, aux0, 0.0f);
                        if (t == 0 && rowp[r]) ckey[idx[r]] = __fmul_rn(d, ksign);
                    }
                }
                __syncwarp();
                uint32_t size = s_size[s];
                ivf_merge<DYN>(bkey, bid, size, ip.k, ckey, cids + tile * ip.tile_rows, rows, spos, lane);
                if (lane == 0) s_size[s] = size;
            }
            __syncthreads();   // (the slot is staged again two tiles on)
        }
        // the lists out, padded with all-ones ids and the worst distance
#pragma unroll 1
        for (uint32_t i = 0; i < IVF_QMAX / IVF_WARPS; ++i) {
            const uint32_t s = warp + IVF_WARPS * i;
            if (s >= nslots) break;
            const float* bkey = reinterpret_cast<const float*>(slots + s * slot_bytes) + p.qstride;
            const uint32_t* bid = reinterpret_cast<const uint32_t*>(bkey + ip.k);
            const uint32_t e = ip.list[first + s], q = e / ip.P, probe = e - q * ip.P;
            const size_t o = (size_t(probe) * ip.nq + q) * ip.k;
            for (uint32_t j = lane; j < ip.k; j += 32) {
                const bool v = j < s_size[s];
                ip.out_ids[o + j] = v ? uint64_t(bid[j]) : ~uint64_t(0);
                ip.out_dists[o + j] = v ? __fmul_rn(bkey[j], ksign) : (p.greater ? -INFINITY : INFINITY);
            }
        }
        __syncthreads();   // (the slots and s_size are refilled by the next item)
    }
}

// ---- SQ rows under L2: the leaf on the integer tensor cores ----
// EuclideanCompressed (quantization/scalar/scalar.h:58-105) is scale^2 * float(sum (qc - x)^2) with an exact integer
// sum, so qq + xx - 2 <qc, x> from int8 / uint8 MMAs gives the same bits in any order.  The arithmetic is int32 and
// wraps as the search path's dp4a sums do, so even past the reference's own bound (dim * 255^2 < 2^31) the keys equal
// finish_distance<OP_L2I>'s.
// Shared memory of one CTA: the ring; per query slot {query codes zero-padded to kpad = dim rounded up to 32 bytes, keys,
// ids}; per warp {candidate keys, positions}; per query slot the 32 dot products of a tile; the 32 rows' xx.
__host__ __device__ inline size_t ivf_sq_slot_bytes(uint32_t dim, uint32_t k) {
    return size_t((dim + 31) & ~31u) + (size_t(k) * 8 + 15) / 16 * 16;
}
__host__ __device__ inline size_t ivf_sq_l2_smem_bytes(uint32_t row_stride, uint32_t tile_rows, uint32_t dim, uint32_t k,
                                                       uint32_t Q) {
    return 2 * size_t(tile_rows) * row_stride + size_t(Q) * (ivf_sq_slot_bytes(dim, k) + 32 * 4) + size_t(IVF_WARPS) * 32 * 8 +
           32 * 4;
}

template <int ROWT>
__device__ __forceinline__ void mma_m16n8k32_int(int (&c)[4], const uint32_t (&a)[4], const uint32_t (&b)[2]) {
    if constexpr (ROWT == SVSB200_I8) {
        asm volatile("mma.sync.aligned.m16n8k32.row.col.s32.s8.s8.s32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
                     : "+r"(c[0]), "+r"(c[1]), "+r"(c[2]), "+r"(c[3])
                     : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b[0]), "r"(b[1]));
    } else {
        asm volatile("mma.sync.aligned.m16n8k32.row.col.s32.u8.u8.s32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
                     : "+r"(c[0]), "+r"(c[1]), "+r"(c[2]), "+r"(c[3])
                     : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b[0]), "r"(b[1]));
    }
}

// Work items, ring, lists and output are ivf_scan_kernel's.  Per staged tile: the slots' query codes (the A operand,
// zero-padded to a multiple of 32 bytes) times the tile's codes (the B operand) on mma.m16n8k32, warp w taking the
// queries 16 (w / 2) .. + 16 and the rows 16 (w % 2) .. + 16; warp 0 also sums each row's xx with dp4a.  Code bytes
// past a row's stride, rows past the tile and queries past the work item's slots count as zero, so Q and the tile
// need not fill whole MMA blocks.  Then every slot's 32 keys go through ivf_merge<DYN>.
template <int ROWT, bool DYN>
__global__ void __launch_bounds__(IVF_WARPS * 32, 2) ivf_scan_sq_l2_kernel(const __grid_constant__ IvfScanParams ip) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    const SearchParams& p = ip.p;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int grp = lane >> 2, tig = lane & 3;
    const uint32_t tile_bytes = ip.tile_rows * p.row_stride;
    const uint32_t kpad = (p.dim + 31) & ~31u;
    unsigned char* ring = smem_raw;
    unsigned char* slots = smem_raw + 2 * size_t(tile_bytes);
    const size_t slot_bytes = ivf_sq_slot_bytes(p.dim, ip.k);
    float* ckey = reinterpret_cast<float*>(slots + size_t(ip.Q) * slot_bytes) + warp * 64;
    uint32_t* spos = reinterpret_cast<uint32_t*>(ckey + 32);
    int* dots = reinterpret_cast<int*>(slots + size_t(ip.Q) * slot_bytes + size_t(IVF_WARPS) * 32 * 8);   // [Q][32]
    int* xxs = dots + size_t(ip.Q) * 32;                                                                  // [32]
    __shared__ uint32_t s_item;
    __shared__ uint32_t s_size[IVF_QMAX];
    const uint32_t total = ip.item_off[ip.C];

    for (;;) {
        if (threadIdx.x == 0) s_item = atomicAdd(ip.work_counter, 1u);
        __syncthreads();
        const uint32_t item = s_item;
        __syncthreads();
        if (item >= total) break;
        uint32_t lo = 0, hi = ip.C;
        while (hi - lo > 1) {
            const uint32_t mid = (lo + hi) >> 1;
            if (ip.item_off[mid] <= item) lo = mid; else hi = mid;
        }
        const uint32_t c = lo;
        const uint32_t first = ip.list_off[c] + (item - ip.item_off[c]) * ip.Q;
        const uint32_t nslots = min(ip.Q, ip.list_off[c + 1] - first);
        const uint32_t count = ip.cl_count[c];
        const char* crows = ip.rows + size_t(ip.cl_start[c]) * p.row_stride;
        const uint32_t* cids = ip.row_ids + ip.cl_start[c];
        const uint32_t ntiles = (count + ip.tile_rows - 1) / ip.tile_rows;
        auto stage = [&](uint32_t tile) {
            const char* src = crows + size_t(tile) * tile_bytes;
            unsigned char* dst = ring + (tile & 1u) * tile_bytes;
            for (uint32_t o = threadIdx.x * 16; o < tile_bytes; o += IVF_WARPS * 32 * 16) cp_async16(dst + o, src + o);
            cp_async_commit();
        };
        if (ntiles) stage(0);
        // the slots' query codes (prepared as for the SQ search: PREP_SQ_L2), zero past qstride up to kpad
        for (uint32_t s = 0; s < nslots; ++s) {
            uint32_t* q_s = reinterpret_cast<uint32_t*>(slots + s * slot_bytes);
            const uint32_t* src = reinterpret_cast<const uint32_t*>(p.qcodes + size_t(ip.list[first + s] / ip.P) * p.qstride);
            for (uint32_t i = threadIdx.x; i < kpad / 4; i += IVF_WARPS * 32) q_s[i] = 4 * i < p.qstride ? src[i] : 0u;
        }
        if (threadIdx.x < IVF_QMAX) s_size[threadIdx.x] = 0;
        __syncthreads();
        for (uint32_t tile = 0; tile < ntiles; ++tile) {
            if (tile + 1 < ntiles) {
                stage(tile + 1);
                asm volatile("cp.async.wait_group 1;" ::: "memory");
            } else {
                cp_async_wait_all();
            }
            __syncthreads();
            const unsigned char* trow = ring + (tile & 1u) * tile_bytes;
            const uint32_t rows = min(ip.tile_rows, count - tile * ip.tile_rows);
            // dot products: A block m = warp / 2, row blocks n0 = 16 (warp % 2) and n0 + 8
            const uint32_t m0 = uint32_t(warp >> 1) * 16, r0 = uint32_t(warp & 1) * 16;
            if (m0 < nslots && r0 < rows) {
                int acc[2][4] = {};
                const unsigned char* qa = slots + size_t(m0 + grp) * slot_bytes;
                const unsigned char* qb = qa + 8 * slot_bytes;
                const bool qlive0 = m0 + grp < nslots, qlive1 = m0 + grp + 8 < nslots;   // (slots past Q do not exist)
                const bool live0 = r0 + grp < rows, live1 = r0 + 8 + grp < rows;
                const unsigned char* b0row = trow + size_t(r0 + grp) * p.row_stride;
                const unsigned char* b1row = b0row + 8 * size_t(p.row_stride);
#pragma unroll 1
                for (uint32_t k0 = 0; k0 < kpad; k0 += 32) {
                    const uint32_t o0 = k0 + 4 * tig, o1 = o0 + 16;
                    const uint32_t a[4] = {qlive0 ? *reinterpret_cast<const uint32_t*>(qa + o0) : 0u,
                                           qlive1 ? *reinterpret_cast<const uint32_t*>(qb + o0) : 0u,
                                           qlive0 ? *reinterpret_cast<const uint32_t*>(qa + o1) : 0u,
                                           qlive1 ? *reinterpret_cast<const uint32_t*>(qb + o1) : 0u};
                    const uint32_t b0[2] = {live0 && o0 < p.row_stride ? *reinterpret_cast<const uint32_t*>(b0row + o0) : 0u,
                                            live0 && o1 < p.row_stride ? *reinterpret_cast<const uint32_t*>(b0row + o1) : 0u};
                    const uint32_t b1[2] = {live1 && o0 < p.row_stride ? *reinterpret_cast<const uint32_t*>(b1row + o0) : 0u,
                                            live1 && o1 < p.row_stride ? *reinterpret_cast<const uint32_t*>(b1row + o1) : 0u};
                    mma_m16n8k32_int<ROWT>(acc[0], a, b0);
                    mma_m16n8k32_int<ROWT>(acc[1], a, b1);
                }
#pragma unroll
                for (int h = 0; h < 2; ++h) {
                    const uint32_t col = r0 + 8 * h + 2 * tig;
                    if (qlive0) {
                        dots[(m0 + grp) * 32 + col] = acc[h][0];
                        dots[(m0 + grp) * 32 + col + 1] = acc[h][1];
                    }
                    if (qlive1) {
                        dots[(m0 + grp + 8) * 32 + col] = acc[h][2];
                        dots[(m0 + grp + 8) * 32 + col + 1] = acc[h][3];
                    }
                }
            }
            if (warp == 0) {   // xx of every row of the tile
                int xx = 0;
                if (uint32_t(lane) < rows) {
                    const uint32_t* w = reinterpret_cast<const uint32_t*>(trow + size_t(lane) * p.row_stride);
                    for (uint32_t i = 0; i < p.row_stride / 4; ++i) {
                        if constexpr (ROWT == SVSB200_I8) xx = __dp4a(int(w[i]), int(w[i]), xx);
                        else xx = int(__dp4a(w[i], w[i], unsigned(xx)));
                    }
                }
                xxs[lane] = xx;
            }
            __syncthreads();
#pragma unroll 1
            for (uint32_t i = 0; i < IVF_QMAX / IVF_WARPS; ++i) {
                const uint32_t s = warp + IVF_WARPS * i;
                if (s >= nslots) break;
                float* bkey = reinterpret_cast<float*>(slots + s * slot_bytes + kpad);
                uint32_t* bid = reinterpret_cast<uint32_t*>(bkey + ip.k);
                const uint32_t q = ip.list[first + s] / ip.P;
                const uint32_t qq = __float_as_uint(p.qaux[2 * size_t(q) + 1]);   // int32 bits of sum qc^2
                if (uint32_t(lane) < rows) {
                    const uint32_t l2 = qq + uint32_t(xxs[lane]) - 2u * uint32_t(dots[s * 32 + lane]);
                    ckey[lane] = __fmul_rn(p.scale_sq, float(int(l2)));
                }
                __syncwarp();
                uint32_t size = s_size[s];
                ivf_merge<DYN>(bkey, bid, size, ip.k, ckey, cids + tile * ip.tile_rows, rows, spos, lane);
                if (lane == 0) s_size[s] = size;
            }
            __syncthreads();
        }
#pragma unroll 1
        for (uint32_t i = 0; i < IVF_QMAX / IVF_WARPS; ++i) {
            const uint32_t s = warp + IVF_WARPS * i;
            if (s >= nslots) break;
            const float* bkey = reinterpret_cast<const float*>(slots + s * slot_bytes + kpad);
            const uint32_t* bid = reinterpret_cast<const uint32_t*>(bkey + ip.k);
            const uint32_t e = ip.list[first + s], q = e / ip.P, probe = e - q * ip.P;
            const size_t o = (size_t(probe) * ip.nq + q) * ip.k;
            for (uint32_t j = lane; j < ip.k; j += 32) {
                const bool v = j < s_size[s];
                ip.out_ids[o + j] = v ? uint64_t(bid[j]) : ~uint64_t(0);
                ip.out_dists[o + j] = v ? bkey[j] : INFINITY;
            }
        }
        __syncthreads();
    }
}

// ---- SQ compression (SQDataset::compress, quantization/scalar/scalar.h:447-469) ----
// out[0] = min and out[1] = max as order-preserving keys (atomicMin / atomicMax), out[2] = non-zero when a value is not
// finite, out[3] = the first index holding a zero (the reference's sequential min keeps the sign of the first zero).
__device__ __forceinline__ uint32_t sq_order_key(float v) {
    const uint32_t u = __float_as_uint(__fadd_rn(v, 0.0f));   // -0 -> +0: both zeros are one key
    return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}
__global__ void sq_minmax_kernel(const float* __restrict__ x, size_t count, uint64_t base, uint32_t* __restrict__ out,
                                 unsigned long long* __restrict__ first_zero) {
    uint32_t mn = 0xFFFFFFFFu, mx = 0u, bad = 0u;
    unsigned long long fz = ~0ull;
    for (size_t i = size_t(blockIdx.x) * blockDim.x + threadIdx.x; i < count; i += size_t(gridDim.x) * blockDim.x) {
        const float v = x[i];
        if (!isfinite(v)) bad = 1u;
        const uint32_t key = sq_order_key(v);
        mn = min(mn, key);
        mx = max(mx, key);
        if (v == 0.0f && fz == ~0ull) fz = base + i;
    }
    for (int o = 16; o; o >>= 1) {
        mn = min(mn, __shfl_xor_sync(0xFFFFFFFFu, mn, o));
        mx = max(mx, __shfl_xor_sync(0xFFFFFFFFu, mx, o));
        bad |= __shfl_xor_sync(0xFFFFFFFFu, bad, o);
        fz = min(fz, __shfl_xor_sync(0xFFFFFFFFu, fz, o));
    }
    if ((threadIdx.x & 31) == 0) {
        atomicMin(out, mn);
        atomicMax(out + 1, mx);
        if (bad) atomicOr(out + 2, 1u);
        if (fz != ~0ull) atomicMin(first_zero, fz);
    }
}
// detail::compress (scalar.h:38-42): clamp(round((x - bias) / scale), MIN, MAX), halves away from zero.
template <int CODE>
__global__ void sq_encode_kernel(const float* __restrict__ x, size_t count, float scale, float bias, uint8_t* __restrict__ out) {
    constexpr float lo = CODE == SVSB200_I8 ? -128.f : 0.f, hi = CODE == SVSB200_I8 ? 127.f : 255.f;
    for (size_t i = size_t(blockIdx.x) * blockDim.x + threadIdx.x; i < count; i += size_t(gridDim.x) * blockDim.x) {
        const float r = fminf(fmaxf(roundf(__fdiv_rn(__fsub_rn(x[i], bias), scale)), lo), hi);
        out[i] = CODE == SVSB200_I8 ? uint8_t(int8_t(int(r))) : uint8_t(int(r));
    }
}

// ---- inversion of the probes: per-cluster lists of (query, probe), ascending ----
// counts[c] += 1 for every probe of c.
__global__ void ivf_count_kernel(const uint64_t* __restrict__ probes, size_t total, uint32_t* __restrict__ counts) {
    const size_t i = size_t(blockIdx.x) * blockDim.x + threadIdx.x;
    if (i < total) atomicAdd(counts + probes[i], 1u);
}
// One CTA: list_off = exclusive scan of counts, item_off = exclusive scan of ceil(counts / Q); cursor = list_off.
__global__ void ivf_scan_offsets_kernel(const uint32_t* __restrict__ counts, uint32_t C, uint32_t Q, uint32_t* __restrict__ list_off,
                                        uint32_t* __restrict__ item_off, uint32_t* __restrict__ cursor) {
    __shared__ uint32_t part_l[1024], part_i[1024];
    const uint32_t per = (C + blockDim.x - 1) / blockDim.x, lo = min(C, threadIdx.x * per), hi = min(C, lo + per);
    uint32_t sl = 0, si = 0;
    for (uint32_t c = lo; c < hi; ++c) {
        sl += counts[c];
        si += (counts[c] + Q - 1) / Q;
    }
    part_l[threadIdx.x] = sl;
    part_i[threadIdx.x] = si;
    __syncthreads();
    if (threadIdx.x == 0) {
        uint32_t al = 0, ai = 0;
        for (uint32_t i = 0; i < blockDim.x; ++i) {
            const uint32_t vl = part_l[i], vi = part_i[i];
            part_l[i] = al;
            part_i[i] = ai;
            al += vl;
            ai += vi;
        }
        list_off[C] = al;
        item_off[C] = ai;
    }
    __syncthreads();
    sl = part_l[threadIdx.x];
    si = part_i[threadIdx.x];
    for (uint32_t c = lo; c < hi; ++c) {
        list_off[c] = sl;
        cursor[c] = sl;
        item_off[c] = si;
        sl += counts[c];
        si += (counts[c] + Q - 1) / Q;
    }
}
// Every (query, probe) into its cluster's list (in arbitrary order; ivf_sort_lists_kernel orders them).
__global__ void ivf_fill_kernel(const uint64_t* __restrict__ probes, size_t total, uint32_t* __restrict__ cursor,
                                uint32_t* __restrict__ list) {
    const size_t i = size_t(blockIdx.x) * blockDim.x + threadIdx.x;
    if (i < total) list[atomicAdd(cursor + probes[i], 1u)] = uint32_t(i);   // i = query * P + probe
}
// One CTA per cluster: bitonic sort of its list in shared memory (lists hold distinct entries, so the order is unique).
__global__ void ivf_sort_lists_kernel(const uint32_t* __restrict__ list_off, uint32_t* __restrict__ list) {
    extern __shared__ uint32_t buf[];
    const uint32_t lo = list_off[blockIdx.x], len = list_off[blockIdx.x + 1] - lo;
    if (len < 2) return;
    uint32_t n2 = 1;
    while (n2 < len) n2 <<= 1;
    for (uint32_t i = threadIdx.x; i < n2; i += blockDim.x) buf[i] = i < len ? list[lo + i] : 0xFFFFFFFFu;
    __syncthreads();
    for (uint32_t size = 2; size <= n2; size <<= 1) {
        for (uint32_t stride = size >> 1; stride; stride >>= 1) {
            for (uint32_t i = threadIdx.x; i < n2; i += blockDim.x) {
                const uint32_t j = i ^ stride;
                if (j > i) {
                    const bool up = (i & size) == 0;
                    const uint32_t a = buf[i], b = buf[j];
                    if ((a > b) == up) {
                        buf[i] = b;
                        buf[j] = a;
                    }
                }
            }
            __syncthreads();
        }
    }
    for (uint32_t i = threadIdx.x; i < len; i += blockDim.x) list[lo + i] = buf[i];
}

// ---- k-means ----
// The update of centroid_adjustment (common.h:446-490): one warp per centroid, lanes over the dimensions.  The members
// are the training rows assigned to it, summed in float32 in ascending row order onto the old centroid; a centroid
// with members becomes that sum times float(1.0 / (count + 1)) (the old centroid counts as one point); counts[c] is the
// number of members.
template <int ROWT>
__global__ void ivf_kmeans_update_kernel(const char* __restrict__ train, uint32_t row_bytes, uint32_t ntrain, uint32_t dim,
                                         const uint32_t* __restrict__ assign, uint32_t C, float* __restrict__ cent,
                                         uint32_t* __restrict__ counts) {
    const uint32_t c = blockIdx.x * (blockDim.x / 32) + threadIdx.x / 32;
    const int lane = threadIdx.x & 31;
    if (c >= C) return;
    float* row = cent + size_t(c) * dim;
    uint32_t cnt = 0;
    for (uint32_t i0 = 0; i0 < ntrain; i0 += 32) {
        const uint32_t i = i0 + lane;
        unsigned m = __ballot_sync(0xFFFFFFFFu, i < ntrain && assign[i] == c);
        cnt += __popc(m);
        while (m) {
            const uint32_t r = i0 + __ffs(m) - 1;
            m &= m - 1;
            const char* x = train + size_t(r) * row_bytes;
            for (uint32_t d = lane; d < dim; d += 32) {
                const float v = ROWT == SVSB200_F32 ? reinterpret_cast<const float*>(x)[d]
                                                    : __half2float(reinterpret_cast<const __half*>(x)[d]);
                row[d] = __fadd_rn(row[d], v);
            }
        }
    }
    if (cnt) {
        const float inv = __double2float_rn(__ddiv_rn(1.0, double(cnt) + 1.0));
        for (uint32_t d = lane; d < dim; d += 32) row[d] = __fmul_rn(row[d], inv);
    }
    if (lane == 0) counts[c] = cnt;
}

// ---- hierarchical k-means: the level-2 problems of every level-1 group at once (ivf.cu, ivf_group_assign) ----
// Rows are reached through a group-major permutation `perm` (ascending row id inside a group); a position is an index
// into it.  One work item is a tile of at most `tile` positions of one group with that group's centroid range.
struct IvfGroupAssignParams {
    SearchParams p;           // dim, qstride, greater (the distance code's fields)
    const char* rows;         // dense rows of the row type, row_bytes apart
    uint32_t row_bytes;
    const uint32_t* perm;     // position -> row id
    const uint4* items;       // {first position, end position, first centroid, centroids}
    const float* cent;        // [C][dim] dense float32 centroids
    uint32_t tile, chunk;     // positions per item, centroids staged per round
    uint32_t* out;            // global centroid of every position (by_row: of every row id)
    int by_row;
};

// Shared memory of one CTA: the tile's prepared rows and the staged centroids (qstride floats each), then per row of the
// tile the query's a_norm and its best (key, centroid).
__host__ __device__ inline size_t ivf_group_smem_bytes(uint32_t qstride, uint32_t tile, uint32_t chunk) {
    return (size_t(tile) + chunk) * qstride * 4 + size_t(tile) * 12;
}

// (key, centroid) a before b: NaN keys last, then key, then the lower centroid (the order of the model's lexsort).
__device__ __forceinline__ bool ivf_nearer(float ka, uint32_t ia, float kb, uint32_t ib) {
    const bool na = isnan(ka), nb = isnan(kb);
    if (na != nb) return nb;
    if (!na && (ka < kb || kb < ka)) return ka < kb;
    return ia < ib;
}

// Nearest centroid of every position of an item among its group's centroids: each row of the tile is prepared in shared
// memory as prepare_queries_kernel prepares a query (PREP_FLOAT), the group's centroids pass through shared memory
// `chunk` at a time (each read once per tile), and a warp scores one row against the staged centroids with the scan's
// distance code (float_rows over float32 rows in its shared-memory form, finish_distance) -- the bits of a search of the
// row against the centroids.  Ties go to the lower centroid.
template <int QT, int OP, int DS>
__global__ void __launch_bounds__(IVF_WARPS * 32, 2) ivf_group_assign_kernel(const __grid_constant__ IvfGroupAssignParams gp) {
    constexpr int NR = OP == OP_COSF || DS == 0 ? 1 : 2;   // (two centroids per pass spill at the generic dimension)
    constexpr int G = 16 / Row<SVSB200_F32>::LPT;   // threads per centroid
    constexpr int GROUPS = 32 / G;                  // centroids per warp and pass
    constexpr unsigned FULL = 0xFFFFFFFFu;
    extern __shared__ __align__(16) unsigned char smem_raw[];
    const SearchParams& p = gp.p;
    const uint32_t qs = p.qstride, dim = p.dim;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int g = lane / G, t = lane % G;
    float* qv = reinterpret_cast<float*>(smem_raw);   // [tile][qs]
    float* cv = qv + size_t(gp.tile) * qs;             // [chunk][qs]
    float* aux = cv + size_t(gp.chunk) * qs;           // [tile]
    float* bkey = aux + gp.tile;                       // [tile]
    uint32_t* bidx = reinterpret_cast<uint32_t*>(bkey + gp.tile);
    const float ksign = p.greater ? -1.0f : 1.0f;
    const uint4 it = gp.items[blockIdx.x];
    const uint32_t nrows = it.y - it.x;
    for (uint32_t i = threadIdx.x; i < gp.tile * qs; i += IVF_WARPS * 32) {
        const uint32_t r = i / qs, e = i - r * qs;
        float v = 0.f;
        if (r < nrows && e < dim) v = q_simd<QT>(gp.rows + size_t(gp.perm[it.x + r]) * gp.row_bytes, e);
        qv[i] = v;
    }
    for (uint32_t i = threadIdx.x; i < gp.chunk * qs; i += IVF_WARPS * 32) cv[i] = 0.f;   // (the padding stays zero)
    if (threadIdx.x < gp.tile) {
        float a = 0.f;
        if (OP == OP_COSF && threadIdx.x < nrows) {
            const char* src = gp.rows + size_t(gp.perm[it.x + threadIdx.x]) * gp.row_bytes;
            a = sequential_norm(dim, [&](uint32_t i) {
                const float v = q_scalar<QT>(src, i);
                return __fmul_rn(v, v);
            });
        }
        aux[threadIdx.x] = a;
        bkey[threadIdx.x] = __int_as_float(0x7FC00000);
        bidx[threadIdx.x] = 0xFFFFFFFFu;
    }
    for (uint32_t c0 = 0; c0 < it.w; c0 += gp.chunk) {
        const uint32_t cn = min(gp.chunk, it.w - c0);
        __syncthreads();   // (the previous chunk is consumed; the first time: the preparation is done)
        const float* src = gp.cent + size_t(it.z + c0) * dim;
        for (uint32_t i = threadIdx.x; i < cn * dim; i += IVF_WARPS * 32) {
            const uint32_t r = i / dim;
            cv[r * qs + (i - r * dim)] = src[i];
        }
        __syncthreads();
#pragma unroll 1
        for (uint32_t r = warp; r < nrows; r += IVF_WARPS) {
            const float* q_s = qv + size_t(r) * qs;
            const float a = aux[r];
            float best = __int_as_float(0x7FC00000);
            uint32_t bi = 0xFFFFFFFFu;
#pragma unroll 1
            for (uint32_t base = 0; base < cn; base += NR * GROUPS) {
                const char* rowp[NR];
                uint32_t idx[NR];
#pragma unroll
                for (int k = 0; k < NR; ++k) {
                    idx[k] = base + k * GROUPS + g;
                    rowp[k] = idx[k] < cn ? reinterpret_cast<const char*>(cv + size_t(idx[k]) * qs) : nullptr;
                }
                float sum[NR], nrm[NR];
                float_rows<SVSB200_F32, OP, DS, NR, false, true>(p, q_s, rowp, t, sum, nrm);
#pragma unroll
                for (int k = 0; k < NR; ++k) {
                    const float key = __fmul_rn(finish_distance<OP>(p, sum[k], nrm[k], 0, 0, a, 0.0f), ksign);
                    if (rowp[k] && ivf_nearer(key, c0 + idx[k], best, bi)) {
                        best = key;
                        bi = c0 + idx[k];
                    }
                }
            }
            for (int off = 16; off; off >>= 1) {
                const float ok = __shfl_xor_sync(FULL, best, off);
                const uint32_t oi = __shfl_xor_sync(FULL, bi, off);
                if (ivf_nearer(ok, oi, best, bi)) {
                    best = ok;
                    bi = oi;
                }
            }
            if (lane == 0 && ivf_nearer(best, bi, bkey[r], bidx[r])) {
                bkey[r] = best;
                bidx[r] = bi;
            }
        }
    }
    __syncthreads();
    for (uint32_t r = threadIdx.x; r < nrows; r += IVF_WARPS * 32)
        gp.out[gp.by_row ? gp.perm[it.x + r] : it.x + r] = it.z + bidx[r];
}

// ivf_kmeans_update_kernel's rule for the level-2 centroids: one warp per centroid c, whose members are the positions
// of its group's range [range[c].x, range[c].y) assigned to it (assign is by position), summed in ascending position
// (= ascending training row) order onto the old centroid.
template <int ROWT>
__global__ void ivf_kmeans_group_update_kernel(const char* __restrict__ train, uint32_t row_bytes, const uint32_t* __restrict__ perm,
                                               const uint2* __restrict__ range, uint32_t dim, const uint32_t* __restrict__ assign,
                                               uint32_t C, float* __restrict__ cent, uint32_t* __restrict__ counts) {
    const uint32_t c = blockIdx.x * (blockDim.x / 32) + threadIdx.x / 32;
    const int lane = threadIdx.x & 31;
    if (c >= C) return;
    float* row = cent + size_t(c) * dim;
    const uint32_t lo = range[c].x, hi = range[c].y;
    uint32_t cnt = 0;
    for (uint32_t i0 = lo; i0 < hi; i0 += 32) {
        const uint32_t i = i0 + lane;
        unsigned m = __ballot_sync(0xFFFFFFFFu, i < hi && assign[i] == c);
        cnt += __popc(m);
        while (m) {
            const uint32_t r = i0 + __ffs(m) - 1;
            m &= m - 1;
            const char* x = train + size_t(perm[r]) * row_bytes;
            for (uint32_t d = lane; d < dim; d += 32) {
                const float v = ROWT == SVSB200_F32 ? reinterpret_cast<const float*>(x)[d]
                                                    : __half2float(reinterpret_cast<const __half*>(x)[d]);
                row[d] = __fadd_rn(row[d], v);
            }
        }
    }
    if (cnt) {
        const float inv = __double2float_rn(__ddiv_rn(1.0, double(cnt) + 1.0));
        for (uint32_t d = lane; d < dim; d += 32) row[d] = __fmul_rn(row[d], inv);
    }
    if (lane == 0) counts[c] = cnt;
}

// out[i] = i: the row ids a stable sort by group permutes.
__global__ void ivf_iota_kernel(uint32_t* __restrict__ out, size_t count) {
    const size_t i = size_t(blockIdx.x) * blockDim.x + threadIdx.x;
    if (i < count) out[i] = uint32_t(i);
}

// ---- filtered search (ivf.cu, ivf_search_filtered_on_device) ----
// One CTA per cluster: masked[r] = row_ids[r] where that id's bit of `bitmap` is set, all-ones otherwise (a tombstone or
// padding entry already is), for the cluster's stored rows [cl_start, cl_start + cl_count); cl_allowed[c] counts the
// entries kept, cl_rows[c] the entries that are not all-ones.  The ids index the bitmap: original ids of the static
// index, slots of the dynamic one.
__global__ void ivf_filter_mask_kernel(const uint32_t* __restrict__ row_ids, const uint32_t* __restrict__ cl_start,
                                       const uint32_t* __restrict__ cl_count, const uint32_t* __restrict__ bitmap,
                                       uint32_t* __restrict__ masked, uint32_t* __restrict__ cl_allowed,
                                       uint32_t* __restrict__ cl_rows) {
    const uint32_t c = blockIdx.x, start = cl_start[c], count = cl_count[c];
    uint32_t allowed = 0, rows = 0;
    for (uint32_t base = 0; base < count; base += blockDim.x) {   // (uniform trip count: __syncthreads_count inside)
        const uint32_t i = base + threadIdx.x;
        const uint32_t id = i < count ? row_ids[start + i] : 0xFFFFFFFFu;
        const bool valid = id != 0xFFFFFFFFu;
        const bool keep = valid && ((bitmap[id >> 5] >> (id & 31u)) & 1u);
        if (i < count) masked[start + i] = keep ? id : 0xFFFFFFFFu;
        allowed += __syncthreads_count(keep);
        rows += __syncthreads_count(valid);
    }
    if (threadIdx.x == 0) {
        cl_allowed[c] = allowed;
        cl_rows[c] = rows;
    }
}
// One warp per query of a probe round: the allowed and Valid rows of its first P probes (probes [nq][P]) summed and
// written, with P, to query qidx[i] (qidx NULL: i) of the per-query outputs.
__global__ void ivf_filter_count_kernel(const uint64_t* __restrict__ probes, uint32_t nq, uint32_t P,
                                        const uint32_t* __restrict__ qidx, const uint32_t* __restrict__ cl_allowed,
                                        const uint32_t* __restrict__ cl_rows, uint32_t* __restrict__ q_probes,
                                        uint32_t* __restrict__ q_allowed, uint32_t* __restrict__ q_rows) {
    const uint32_t i = blockIdx.x * (blockDim.x / 32) + threadIdx.x / 32;
    const int lane = threadIdx.x & 31;
    if (i >= nq) return;
    uint32_t a = 0, r = 0;
    for (uint32_t j = lane; j < P; j += 32) {
        const uint64_t c = probes[size_t(i) * P + j];
        a += cl_allowed[c];
        r += cl_rows[c];
    }
    a = __reduce_add_sync(0xFFFFFFFFu, a);
    r = __reduce_add_sync(0xFFFFFFFFu, r);
    if (lane == 0) {
        const uint32_t q = qidx ? qidx[i] : i;
        q_probes[q] = P;
        q_allowed[q] = a;
        q_rows[q] = r;
    }
}
// dst row i <- src row idx[i], rows of `row_bytes` bytes.
__global__ void ivf_gather_rows_kernel(const unsigned char* __restrict__ src, const uint32_t* __restrict__ idx, size_t count,
                                       size_t row_bytes, unsigned char* __restrict__ dst) {
    for (size_t e = size_t(blockIdx.x) * blockDim.x + threadIdx.x; e < count * row_bytes; e += size_t(gridDim.x) * blockDim.x) {
        const size_t i = e / row_bytes;
        dst[e] = src[size_t(idx[i]) * row_bytes + (e - i * row_bytes)];
    }
}
// Result row i of a query group -> row idx[i] of the batch's result (idx NULL: i), `k` entries a row; a padding entry
// (all-ones id) gets distance +inf, whatever the metric.
// (In place when idx is NULL: each entry is read and written by one thread.)
__global__ void ivf_filter_scatter_kernel(const uint64_t* ids, const float* dists, const uint32_t* __restrict__ idx,
                                          size_t count, uint32_t k, uint64_t* out_ids, float* out_dists) {
    const size_t e = size_t(blockIdx.x) * blockDim.x + threadIdx.x;
    if (e >= count * k) return;
    const size_t i = e / k, o = (idx ? size_t(idx[i]) : i) * k + (e - i * k);
    const uint64_t id = ids[e];
    out_ids[o] = id;
    out_dists[o] = id == ~uint64_t(0) ? INFINITY : dists[e];
}

// probes / assignments: 64-bit search ids -> 32-bit cluster numbers
__global__ void ivf_narrow_ids_kernel(const uint64_t* __restrict__ in, size_t count, uint32_t* __restrict__ out) {
    const size_t i = size_t(blockIdx.x) * blockDim.x + threadIdx.x;
    if (i < count) out[i] = uint32_t(in[i]);
}

}  // namespace svsb200
