// ivf.cu -- the IVF index of the C ABI (include/svsb200.h, svsb200_ivf_*): flat and hierarchical k-means clustering,
// the cluster-major layout and the search (DESIGN.md §15).
//
// Search, per chunk of queries:
//   1. probe: the flat search (flat.cu) over the centroids with k = n_probes -- exact distances of the search path,
//      ties to the lower centroid (the reference ranks centroids from an sgemm, ivf/common.h:641-684, 854-888);
//   2. the queries prepared as for the scan (prepare_queries);
//   3. inversion: the probes [nq][P] become per-cluster lists of (query, probe), ascending (count, scan, fill, sort);
//   4. ivf_scan_kernel (ivf_kernel.cuh): one work item per (cluster, chunk of up to Q queries), writing the top k of
//      every (query, probe) as [P][nq][k];
//   5. merge_topk_kernel (search.cu) merges the P lists of a query with TotalOrder into [nq][k].
// The per-(query, probe) lists are kept under IVF_LIST_BUDGET bytes by cutting the batch into query chunks.
#include "ivf.cuh"
#include "ivf_kernel.cuh"

#include <cub/device/device_radix_sort.cuh>

#include <algorithm>
#include <cmath>
#include <cstring>
#include <map>
#include <numeric>
#include <vector>

namespace svsb200 {

constexpr size_t IVF_LIST_BUDGET = size_t(256) << 20;   // bytes of per-(query, probe) lists per query chunk
constexpr size_t IVF_MAX_CHUNK = 8192;                  // queries per chunk (a cluster's list is sorted in shared memory)
constexpr size_t IVF_MIN_TRAINING_SAMPLE_MULTIPLIER = 2;   // common.h:66
constexpr double IVF_EPSILON = 1.0 / 1024.0;               // common.h:59

// ---- the documented random sequence (splitmix64) ----
static uint64_t ivf_next(uint64_t& s) {
    uint64_t z = (s += 0x9E3779B97F4A7C15ull);
    z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
    z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
    return z ^ (z >> 31);
}
static float ivf_uniform(uint64_t& s) { return float(ivf_next(s) >> 40) * 0x1p-24f; }
// The first m of a Fisher-Yates shuffle of [0, n).
static std::vector<uint32_t> ivf_shuffle_prefix(uint64_t& s, size_t n, size_t m) {
    std::vector<uint32_t> perm(n);
    std::iota(perm.begin(), perm.end(), 0u);
    for (size_t i = 0; i < m; ++i) std::swap(perm[i], perm[i + ivf_next(s) % (n - i)]);
    perm.resize(m);
    return perm;
}

// normalize_centroids (common.h:342-363): x * (1 / norm), the norm a sequential float32 sum of squares.
static void ivf_normalize(float* cent, size_t C, size_t dim) {
    for (size_t c = 0; c < C; ++c) {
        float* x = cent + c * dim;
        float acc = 0.0f;
        for (size_t d = 0; d < dim; ++d) {
            const float sq = x[d] * x[d];
            acc = acc + sq;
        }
        const float norm = std::sqrt(acc);
        if (norm != 0.0f) {
            const float inv = 1.0f / norm;
            for (size_t d = 0; d < dim; ++d) x[d] = x[d] * inv;
        }
    }
}

// centroid_split (common.h:493-537) with the documented sequence, over C centroids trained on m rows.
static void ivf_split(float* cent, uint32_t* counts, size_t C, size_t dim, size_t m, uint64_t& s) {
    for (size_t i = 0; i < C; ++i) {
        if (counts[i] != 0) continue;
        size_t j = 0;
        for (;; j = (j + 1) % C) {
            if (counts[j] == 0) continue;
            const float p = float(counts[j]) / float(m);
            if (ivf_uniform(s) < p) break;
        }
        float* ci = cent + i * dim;
        float* cj = cent + j * dim;
        std::copy(cj, cj + dim, ci);
        for (size_t d = 0; d < dim; ++d) {
            const double up = 1.0 + IVF_EPSILON, down = 1.0 - IVF_EPSILON;
            ci[d] = float(double(ci[d]) * (d % 2 == 0 ? up : down));
            cj[d] = float(double(cj[d]) * (d % 2 == 0 ? down : up));
        }
        counts[i] = counts[j] / 2;
        counts[j] -= counts[i];
    }
}

int ivf_centroid_index(const float* centroids, size_t C, size_t dim, int metric, int device, std::unique_ptr<svsb200_flat>* out) {
    svsb200_flat* f = nullptr;
    if (int rc = svsb200_flat_index_create(centroids, SVSB200_F32, C, dim, 0, metric, device, &f)) return rc;
    out->reset(f);
    return 0;
}

int ivf_assign(svsb200_flat* cent, const char* d_rows, int dtype, size_t count, size_t row_bytes, size_t batch,
               uint32_t* d_assign, cudaStream_t stream) {
    DeviceBuffer<uint64_t> ids;
    DeviceBuffer<float> dists;
    const size_t b = std::min(batch, count);
    CUDA_TRY(ids.ensure(std::max<size_t>(b, 1)));
    CUDA_TRY(dists.ensure(std::max<size_t>(b, 1)));
    for (size_t lo = 0; lo < count; lo += b) {
        const size_t nb = std::min(b, count - lo);
        if (int rc = flat_search_device("svsb200_ivf: assignment", cent->ix.get(), d_rows + lo * row_bytes, dtype, nb, 1,
                                        ids.ptr, dists.ptr, stream, nullptr, flat_max_kc_deep()))
            return rc;
        ivf_narrow_ids_kernel<<<unsigned((nb + 255) / 256), 256, 0, stream>>>(ids.ptr, nb, d_assign + lo);
        count_launch();
        CUDA_TRY(cudaGetLastError());
    }
    CUDA_TRY(cudaStreamSynchronize(stream));   // (before ids and dists go)
    return 0;
}

// The checks and the training-set size of both k-means (kmeans.h:54-66): m training rows, refused when m < C.
static int ivf_training_size(const char* who, size_t n, size_t C, size_t minibatch_size, float training_fraction, size_t* m) {
    const std::string w(who);
    if (C == 0) return fail(w + ": num_centroids must be positive");
    if (minibatch_size == 0) return fail(w + ": minibatch_size must be positive");
    if (!(training_fraction >= 0.0f) || !std::isfinite(training_fraction))
        return fail(w + ": training_fraction must be a finite non-negative number");
    const size_t min_training = std::min(C * IVF_MIN_TRAINING_SAMPLE_MULTIPLIER, n);
    *m = std::min(n, std::max(min_training, size_t(std::ceil(float(n) * training_fraction))));
    if (*m < C)
        return fail(w + ": insufficient data for clustering: " + std::to_string(*m) + " training rows, " + std::to_string(C) +
                    " centroids required");
    return 0;
}

// Step 1 of both k-means: the training sample, the first m of a shuffle of [0, n) in ascending order, gathered.
static std::vector<char> ivf_training_rows(uint64_t& s, const void* vectors, size_t n, size_t m, size_t row_bytes) {
    std::vector<uint32_t> sample = ivf_shuffle_prefix(s, n, m);
    std::sort(sample.begin(), sample.end());
    const char* src = static_cast<const char*>(vectors);
    std::vector<char> train(m * row_bytes);
    for (size_t i = 0; i < m; ++i)
        std::copy(src + size_t(sample[i]) * row_bytes, src + size_t(sample[i] + 1) * row_bytes, train.data() + i * row_bytes);
    return train;
}

// Row `i` of dense rows as float32.
static void ivf_row_f32(const char* rows, int dtype, size_t row_bytes, size_t i, size_t dim, float* out) {
    const char* x = rows + i * row_bytes;
    for (size_t d = 0; d < dim; ++d)
        out[d] = dtype == SVSB200_F32 ? reinterpret_cast<const float*>(x)[d] : __half2float(reinterpret_cast<const __half*>(x)[d]);
}

// Step 3 of the flat k-means: num_iterations rounds of assignment (the centroid index `cix`, which holds `cent`), update,
// split and normalisation of the C centroids `cent` over the m training rows d_train; `cix` follows the centroids.
// d_assign holds at least m entries.
static int ivf_kmeans_iterate(svsb200_flat* cix, std::vector<float>& cent, size_t C, size_t dim, const char* d_train, int dtype,
                              size_t m, size_t minibatch_size, size_t num_iterations, bool ip_like, uint64_t& s,
                              uint32_t* d_assign, cudaStream_t stream) {
    const size_t row_bytes = dim * esize(dtype);
    Replica* crep = cix->ix->reps[0].get();
    DeviceBuffer<uint32_t> d_counts;
    DeviceBuffer<float> d_cent;
    CUDA_TRY(d_counts.ensure(C));
    CUDA_TRY(d_cent.ensure(C * dim));
    std::vector<uint32_t> counts(C);
    for (size_t it = 0; it < num_iterations; ++it) {
        if (int rc = ivf_assign(cix, d_train, dtype, m, row_bytes, minibatch_size, d_assign, stream)) return rc;
        CUDA_TRY(cudaMemcpyAsync(d_cent.ptr, cent.data(), C * dim * 4, cudaMemcpyHostToDevice, stream));
        const unsigned warps = 8;
        const LaunchConfig cfg{int((C + warps - 1) / warps), int(warps), 0, stream};
        CUDA_TRY(dispatch(IvfRows{}, dtype, [&](auto row) {
            return launch_kernel(ivf_kmeans_update_kernel<decltype(row)::value>, cfg, size_t(cfg.grid), false, d_train,
                                 uint32_t(row_bytes), uint32_t(m), uint32_t(dim), static_cast<const uint32_t*>(d_assign),
                                 uint32_t(C), d_cent.ptr, d_counts.ptr);
        }));
        CUDA_TRY(cudaMemcpyAsync(cent.data(), d_cent.ptr, C * dim * 4, cudaMemcpyDeviceToHost, stream));
        CUDA_TRY(cudaMemcpyAsync(counts.data(), d_counts.ptr, C * 4, cudaMemcpyDeviceToHost, stream));
        CUDA_TRY(cudaStreamSynchronize(stream));
        ivf_split(cent.data(), counts.data(), C, dim, m, s);
        if (ip_like) ivf_normalize(cent.data(), C, dim);
        // the centroid index takes the new rows; its GEMM operands are rebuilt by the next search
        CUDA_TRY(cudaMemcpy2D(crep->d_vectors.ptr, cix->ix->row_stride, cent.data(), dim * 4, dim * 4, C, cudaMemcpyHostToDevice));
        flat_slots_reset(crep);
    }
    return 0;
}

// The group-major permutation of `count` rows by their group keys (each < ngroups): a stable radix sort of (key, row id),
// so that the rows of a group stay in ascending id.  Synchronises `stream`.
static int ivf_group_rows(const uint32_t* d_keys, size_t count, size_t ngroups, uint32_t* d_perm, cudaStream_t stream) {
    DeviceBuffer<uint32_t> ids, keys;
    DeviceBuffer<char> temp;
    CUDA_TRY(ids.ensure(count));
    CUDA_TRY(keys.ensure(count));
    ivf_iota_kernel<<<unsigned((count + 255) / 256), 256, 0, stream>>>(ids.ptr, count);
    count_launch();
    CUDA_TRY(cudaGetLastError());
    int end_bit = 1;
    while (end_bit < 32 && (size_t(1) << end_bit) < ngroups) ++end_bit;
    size_t bytes = 0;
    CUDA_TRY(cub::DeviceRadixSort::SortPairs(nullptr, bytes, d_keys, keys.ptr, ids.ptr, d_perm, int(count), 0, end_bit, stream));
    CUDA_TRY(temp.ensure(std::max<size_t>(bytes, 1)));
    CUDA_TRY(cub::DeviceRadixSort::SortPairs(temp.ptr, bytes, d_keys, keys.ptr, ids.ptr, d_perm, int(count), 0, end_bit, stream));
    CUDA_TRY(cudaStreamSynchronize(stream));   // (before the buffers go)
    return 0;
}

// A level-1 group as the grouped kernels see it: its positions in a group-major permutation and its centroids.
struct IvfGroup {
    size_t pos, rows, cent, cents;
};

// The shape of ivf_group_assign_kernel for `dim`-element rows (svsb200_ivf_group_plan): `tile` positions per work item,
// 64 halved while two tiles of prepared rows would pass 96 KB, the centroids staged `tile` at a time.
struct IvfGroupPlan {
    uint32_t tile, chunk;
    size_t smem;
};
static int ivf_group_plan(size_t dim, IvfGroupPlan* plan) {
    const uint32_t qs = query_stride(dim);
    uint32_t tile = 64;
    while (tile > 1 && ivf_group_smem_bytes(qs, 2 * tile, 0) > (size_t(96) << 10)) tile >>= 1;
    *plan = {tile, tile, ivf_group_smem_bytes(qs, tile, tile)};
    if (plan->smem > kSmemOptInMax - 1024) return fail("svsb200_ivf_cluster_hierarchical: rows too wide for the grouped kernels");
    return 0;
}

// Nearest centroid of every position of the groups (each row among its own group's centroids d_cent [C][dim]),
// ivf_group_assign_kernel over work items of at most `tile` positions, launched over `batch` positions at a time (which
// changes no result).  out: global centroid per position, or per row id with by_row.  Synchronises `stream`.
static int ivf_group_assign(const char* d_rows, int dtype, size_t dim, int metric, const uint32_t* d_perm,
                            const std::vector<IvfGroup>& groups, size_t batch, const float* d_cent, uint32_t* d_out, bool by_row,
                            cudaStream_t stream) {
    const uint32_t qs = query_stride(dim);
    IvfGroupPlan plan;
    if (int rc = ivf_group_plan(dim, &plan)) return rc;
    const uint32_t tile = plan.tile;
    const size_t smem = plan.smem;
    size_t total = 0;
    for (const IvfGroup& g : groups) total = std::max(total, g.pos + g.rows);
    // the work items of every batch, in order, and where each batch's items start
    std::vector<uint4> items;
    std::vector<size_t> first;
    for (size_t lo = 0; lo < total; lo += batch) {
        const size_t hi = std::min(total, lo + batch);
        first.push_back(items.size());
        for (const IvfGroup& g : groups) {
            if (g.cents == 0) continue;
            const size_t a = std::max(lo, g.pos), b = std::min(hi, g.pos + g.rows);
            for (size_t x = a; x < b; x += tile)
                items.push_back(make_uint4(uint32_t(x), uint32_t(std::min(b, x + tile)), uint32_t(g.cent), uint32_t(g.cents)));
        }
    }
    first.push_back(items.size());
    if (items.empty()) return 0;
    DeviceBuffer<uint4> d_items;
    CUDA_TRY(d_items.ensure(items.size()));
    CUDA_TRY(cudaMemcpyAsync(d_items.ptr, items.data(), items.size() * sizeof(uint4), cudaMemcpyHostToDevice, stream));
    IvfGroupAssignParams gp{};
    gp.p.dim = uint32_t(dim);
    gp.p.qstride = qs;
    gp.p.greater = metric != SVSB200_L2;
    gp.rows = d_rows;
    gp.row_bytes = uint32_t(dim * esize(dtype));
    gp.perm = d_perm;
    gp.cent = d_cent;
    gp.tile = tile;
    gp.chunk = plan.chunk;
    gp.out = d_out;
    gp.by_row = by_row;
    const int op = metric == SVSB200_L2 ? OP_L2F : metric == SVSB200_IP ? OP_IPF : OP_COSF;
    for (size_t b = 0; b + 1 < first.size(); ++b) {
        const size_t count = first[b + 1] - first[b];
        if (count == 0) continue;
        gp.items = d_items.ptr + first[b];
        const LaunchConfig cfg{int(count), IVF_WARPS, smem, stream};
        CUDA_TRY(dispatch(IvfRows{}, dtype, [&](auto qt) {
            return dispatch(IvfOps{}, op, [&](auto o) {
                constexpr int OP = decltype(o)::value;
                return with_shape<OP, true>(uint32_t(dim), false, [&](auto ds, auto) {
                    return launch_kernel(ivf_group_assign_kernel<decltype(qt)::value, OP, decltype(ds)::value>, cfg, count,
                                         true, gp);
                });
            });
        }));
    }
    CUDA_TRY(cudaStreamSynchronize(stream));   // (before the items go)
    return 0;
}

// Rows per group and pass of ivf_scan_kernel: two where they fit the register bound without spilling, one for float16
// rows, SQ codes and cosine (as for the masked scan) and for the dynamic form's generic dimension.
constexpr int ivf_scan_rows_per_pass(int rowt, int op, int ds, bool dyn) {
    return rowt == SVSB200_F16 || rowt == SVSB200_I8 || rowt == SVSB200_U8 || op == OP_COSF || (dyn && ds == 0) ? 1 : 2;
}

template <int ROWT, bool DYN, typename Ops = IvfOps>
static cudaError_t launch_ivf_scan(int op, const IvfScanParams& ip, const LaunchConfig& cfg) {
    return dispatch(Ops{}, op, [&](auto o) {
        constexpr int OP = decltype(o)::value;
        return with_shape<OP, true>(ip.p.dim, false, [&](auto ds, auto) {
            constexpr int DS = decltype(ds)::value;
            constexpr int NR = ivf_scan_rows_per_pass(ROWT, OP, DS, DYN);
            return launch_kernel(ivf_scan_kernel<ROWT, OP, DS, NR, DYN>, cfg, size_t(1) << 20, true, ip);
        });
    });
}

// Queries per chunk: the per-(query, probe) lists under IVF_LIST_BUDGET.
static size_t ivf_chunk(size_t P, size_t k) {
    return std::max<size_t>(1, std::min(IVF_MAX_CHUNK, IVF_LIST_BUDGET / (P * k * 12)));
}

// The shape of one search (svsb200_ivf_plan): the ring tile, Q and the CTAs per SM it implies, the query chunk, the
// leaf kernel and, for the float tree, its static dimension and rows per pass.
struct IvfPlan {
    uint32_t tile_rows, Q, ctas, leaf, ds, nr;
    size_t chunk, smem;
};
static int ivf_plan(size_t dim, int dtype, int storage, int metric, size_t k, size_t P, bool dyn, IvfPlan* plan) {
    const uint32_t row_stride = data_row_stride(storage, dtype, dim), qstride = query_stride(dim);
    // SQ rows: MIP and cosine run ivf_scan_kernel on the decompressed float tree, L2 the tensor-core leaf
    const bool sq_l2 = storage == SVSB200_SQ && metric == SVSB200_L2;
    // ring tiles: 32 rows, fewer for rows so wide that two tiles would pass 96 KB
    uint32_t tile_rows = IVF_TILE_ROWS;
    while (tile_rows > 1 && 2 * size_t(tile_rows) * row_stride > (size_t(96) << 10)) tile_rows >>= 1;
    auto smem = [&](size_t q) {
        return sq_l2 ? ivf_sq_l2_smem_bytes(row_stride, tile_rows, uint32_t(dim), uint32_t(k), uint32_t(q))
                     : ivf_smem_bytes(row_stride, tile_rows, qstride, uint32_t(k), uint32_t(q));
    };
    // queries per work item: two CTAs per SM where they fit, else one
    const size_t fixed = smem(0);
    const size_t slot = smem(1) - fixed;
    const size_t limit = kSmemOptInMax - 1024;   // (the kernel's static shared memory)
    auto fit = [&](size_t room) { return fixed < room ? std::min<size_t>(IVF_QMAX, (room - fixed) / slot) : 0; };
    size_t Q = fit(limit / 2);
    const uint32_t ctas = Q ? 2 : 1;
    if (Q == 0) Q = fit(limit);
    if (Q == 0) return fail("svsb200_ivf_search: k and the row size need more shared memory than a CTA has");
    *plan = {tile_rows, uint32_t(Q), ctas, sq_l2 ? 1u : 0u, 0, 0, ivf_chunk(P, k), smem(Q)};
    if (sq_l2) return 0;
    const int op = metric == SVSB200_L2 ? OP_L2F : metric == SVSB200_IP ? OP_IPF : OP_COSF;
    CUDA_TRY(dispatch(IvfOps{}, op, [&](auto o) {
        constexpr int OP = decltype(o)::value;
        return with_shape<OP, true>(uint32_t(dim), false, [&](auto ds, auto) {
            constexpr int DS = decltype(ds)::value;
            plan->ds = DS;
            plan->nr = ivf_scan_rows_per_pass(dtype, OP, DS, dyn);
            return cudaSuccess;
        });
    }));
    return 0;
}

static IvfScratch* ivf_scratch(svsb200_ivf* iv, Scratch* sc) {
    std::lock_guard<std::mutex> lock(iv->mu);
    auto& slot = iv->scratch[sc];
    if (!slot) slot = std::make_unique<IvfScratch>();
    return slot.get();
}

int ivf_search_on_device(svsb200_ivf* iv, Scratch* sc, const void* d_queries, int qdtype, size_t nq, size_t k, size_t P,
                         uint64_t* d_out_ids, float* d_out_dists, const uint64_t* d_ext_ids, const uint32_t* d_masked_ids) {
    svsb200_index* ix = iv->ix.get();
    Replica* rep = ix->reps[0].get();
    cudaStream_t stream = sc->stream;
    IvfScratch* is = ivf_scratch(iv, sc);
    const uint32_t C = uint32_t(iv->C), dim = uint32_t(ix->dim), qstride = query_stride(dim);
    const bool sq = ix->storage == SVSB200_SQ;
    const bool sq_l2 = sq && ix->metric == SVSB200_L2;
    const bool dyn = d_ext_ids || d_masked_ids;   // the scan's DYN form: all-ones ids are not candidates
    IvfPlan plan;
    if (int rc = ivf_plan(dim, ix->dtype, ix->storage, ix->metric, k, P, dyn, &plan)) return rc;
    const uint32_t tile_rows = plan.tile_rows;
    const size_t Q = plan.Q, chunk = plan.chunk;
    const size_t qrow = size_t(dim) * esize(qdtype);
    const size_t cmax = std::min(chunk, nq);
    CUDA_TRY(is->probe_ids.ensure(cmax * P));
    CUDA_TRY(is->probe_dists.ensure(cmax * P));
    CUDA_TRY(is->list_ids.ensure(cmax * P * k));
    CUDA_TRY(is->list_dists.ensure(cmax * P * k));
    CUDA_TRY(is->counts.ensure(C));
    CUDA_TRY(is->list_off.ensure(C + 1));
    CUDA_TRY(is->item_off.ensure(C + 1));
    CUDA_TRY(is->cursor.ensure(C));
    CUDA_TRY(is->list.ensure(cmax * P));
    const int op = sq_l2 ? OP_L2I : ix->metric == SVSB200_L2 ? OP_L2F : ix->metric == SVSB200_IP ? OP_IPF : OP_COSF;
    const int prep = !sq ? PREP_FLOAT : sq_l2 ? PREP_SQ_L2 : ix->metric == SVSB200_IP ? PREP_SQ_IP : PREP_SQ_COS;
    for (size_t q0 = 0; q0 < nq; q0 += chunk) {
        const size_t nqc = std::min(chunk, nq - q0);
        const char* qp = static_cast<const char*>(d_queries) + q0 * qrow;
        // 1. probe
        if (int rc = flat_search_device("svsb200_ivf_search: probe", iv->cent->ix.get(), qp, qdtype, nqc, P,
                                        is->probe_ids.ptr, is->probe_dists.ptr, stream, nullptr, flat_max_kc_deep()))
            return rc;
        // 2. the scan's query operands
        if (int rc = prepare_queries(ix, rep, sc, qp, qdtype, nqc, prep, stream)) return rc;
        // 3. inversion
        const size_t total = nqc * P;
        const unsigned tb = unsigned((total + 255) / 256);
        CUDA_TRY(cudaMemsetAsync(is->counts.ptr, 0, size_t(C) * 4, stream));
        ivf_count_kernel<<<tb, 256, 0, stream>>>(is->probe_ids.ptr, total, is->counts.ptr);
        ivf_scan_offsets_kernel<<<1, 1024, 0, stream>>>(is->counts.ptr, C, uint32_t(Q), is->list_off.ptr, is->item_off.ptr,
                                                         is->cursor.ptr);
        ivf_fill_kernel<<<tb, 256, 0, stream>>>(is->probe_ids.ptr, total, is->cursor.ptr, is->list.ptr);
        size_t n2 = 1;
        while (n2 < nqc) n2 <<= 1;
        ivf_sort_lists_kernel<<<C, 512, n2 * 4, stream>>>(is->list_off.ptr, is->list.ptr);
        for (int i = 0; i < 4; ++i) count_launch();
        CUDA_TRY(cudaGetLastError());
        // 4. the cluster-major scan
        IvfScanParams ip{};
        ip.p.dim = dim;
        ip.p.row_stride = ix->row_stride;
        ip.p.greater = ix->metric != SVSB200_L2;
        ip.p.sq = sq;
        ip.p.scale = sq ? ix->scale : 1.0f;
        ip.p.bias = ix->bias;
        ip.p.scale_sq = ix->scale * ix->scale;   // EuclideanCompressed ctor (scalar.h:68-72)
        ip.p.qf = sc->q_f32.ptr;
        ip.p.qcodes = sc->q_codes.ptr;
        ip.p.qaux = sc->q_aux.ptr;
        ip.p.qstride = qstride;
        ip.p.nq = uint32_t(nqc);
        ip.p.k = uint32_t(k);
        ip.rows = reinterpret_cast<const char*>(rep->d_vectors.ptr);
        ip.row_ids = d_masked_ids ? d_masked_ids : iv->d_row_ids.ptr;
        ip.cl_start = iv->d_start.ptr;
        ip.cl_count = iv->d_count.ptr;
        ip.list_off = is->list_off.ptr;
        ip.list = is->list.ptr;
        ip.item_off = is->item_off.ptr;
        ip.C = C;
        ip.P = uint32_t(P);
        ip.nq = uint32_t(nqc);
        ip.k = uint32_t(k);
        ip.Q = uint32_t(Q);
        ip.tile_rows = tile_rows;
        ip.out_ids = is->list_ids.ptr;
        ip.out_dists = is->list_dists.ptr;
        ip.work_counter = sc->d_counter.ptr;
        CUDA_TRY(cudaMemsetAsync(sc->d_counter.ptr, 0, sizeof(unsigned int), stream));
        const LaunchConfig cfg{-rep->sm_count, IVF_WARPS, plan.smem, stream};
        if (sq_l2) {
            CUDA_TRY(dispatch(IvfSqRows{}, ix->dtype, [&](auto row) {
                constexpr int R = decltype(row)::value;
                return dyn ? launch_kernel(ivf_scan_sq_l2_kernel<R, true>, cfg, size_t(1) << 20, true, ip)
                                 : launch_kernel(ivf_scan_sq_l2_kernel<R, false>, cfg, size_t(1) << 20, true, ip);
            }));
        } else if (sq) {
            CUDA_TRY(dispatch(IvfSqRows{}, ix->dtype, [&](auto row) {
                return dyn ? launch_ivf_scan<decltype(row)::value, true, IvfSqOps>(op, ip, cfg)
                                 : launch_ivf_scan<decltype(row)::value, false, IvfSqOps>(op, ip, cfg);
            }));
        } else {
            CUDA_TRY(dispatch(IvfRows{}, ix->dtype, [&](auto row) {
                return dyn ? launch_ivf_scan<decltype(row)::value, true>(op, ip, cfg)
                                 : launch_ivf_scan<decltype(row)::value, false>(op, ip, cfg);
            }));
        }
        // 5. merge
        if (int rc = svsb200_merge_topk_device(is->list_ids.ptr, is->list_dists.ptr, P, nqc, k, ix->metric, d_out_ids + q0 * k,
                                               d_out_dists + q0 * k, rep->device, stream))
            return rc;
    }
    if (d_ext_ids) CUDA_TRY(slots_to_external(d_out_ids, nq * k, d_ext_ids, stream));   // slots -> external ids
    return 0;
}

// Filtered search, per call:
//   1. ivf_filter_mask_kernel: the row ids with every disallowed row all-ones, and per cluster the allowed and Valid rows;
//   2. growth: the probe at P, ivf_filter_count_kernel sums the counts over each query's P clusters; the queries short of
//      k allowed rows go on to min(4 P, P_max), and only they are probed again;
//   3. the queries grouped by their final P: the plain body over the masked ids (the scan's DYN form, which skips
//      all-ones ids and orders by (distance, id)) on the gathered queries, its rows scattered back with +inf padding.
int ivf_search_filtered_on_device(svsb200_ivf* iv, Scratch* sc, const void* d_queries, int qdtype, size_t nq, size_t k,
                                  size_t n_probes, const uint32_t* d_bitmap, uint64_t* d_out_ids, float* d_out_dists,
                                  uint32_t* d_probes, uint32_t* d_allowed, uint32_t* d_rows, const uint64_t* d_ext_ids) {
    const char* who = "svsb200_ivf_search_filtered";
    svsb200_index* ix = iv->ix.get();
    cudaStream_t stream = sc->stream;
    IvfScratch* is = ivf_scratch(iv, sc);
    const uint32_t C = uint32_t(iv->C);
    const size_t p_max = std::min<size_t>(C, 1024);
    const size_t qrow = ix->dim * esize(qdtype);
    const auto* queries = static_cast<const unsigned char*>(d_queries);
    // 1. the masked ids
    CUDA_TRY(is->masked.ensure(iv->d_row_ids.count));
    CUDA_TRY(is->cl_allowed.ensure(C));
    CUDA_TRY(is->cl_rows.ensure(C));
    ivf_filter_mask_kernel<<<C, 256, 0, stream>>>(iv->d_row_ids.ptr, iv->d_start.ptr, iv->d_count.ptr, d_bitmap,
                                                  is->masked.ptr, is->cl_allowed.ptr, is->cl_rows.ptr);
    count_launch();
    CUDA_TRY(cudaGetLastError());
    CUDA_TRY(is->q_probes.ensure(nq));
    CUDA_TRY(is->q_allowed.ensure(nq));
    CUDA_TRY(is->q_rows.ensure(nq));
    CUDA_TRY(is->qidx.ensure(nq));
    // `count` queries at positions idx into is->gq (the batch itself when they are all of it, in order)
    auto gather = [&](const std::vector<uint32_t>& idx) -> const unsigned char* {
        if (idx.size() == nq) return queries;
        if (is->gq.ensure(idx.size() * qrow) != cudaSuccess) return nullptr;
        const size_t bytes = idx.size() * qrow;
        ivf_gather_rows_kernel<<<unsigned(std::min<size_t>((bytes + 255) / 256, 4096)), 256, 0, stream>>>(
            queries, is->qidx.ptr, idx.size(), qrow, is->gq.ptr);
        count_launch();
        return cudaGetLastError() == cudaSuccess ? is->gq.ptr : nullptr;
    };
    // 2. growth
    std::vector<uint32_t> active(nq), allowed(nq);
    std::iota(active.begin(), active.end(), 0u);
    std::map<size_t, std::vector<uint32_t>> groups;   // final P -> its queries, ascending
    for (size_t P = n_probes;; P = std::min(4 * P, p_max)) {
        const size_t na = active.size();
        CUDA_TRY(cudaMemcpyAsync(is->qidx.ptr, active.data(), na * 4, cudaMemcpyHostToDevice, stream));
        const unsigned char* qp = gather(active);
        if (!qp) return fail(std::string(who) + ": gathering the queries failed");
        const size_t pc = std::max<size_t>(1, std::min(na, IVF_LIST_BUDGET / (P * 12)));
        CUDA_TRY(is->f_probe_ids.ensure(pc * P));
        CUDA_TRY(is->f_probe_dists.ensure(pc * P));
        for (size_t a0 = 0; a0 < na; a0 += pc) {
            const size_t m = std::min(pc, na - a0);
            if (int rc = flat_search_device("svsb200_ivf_search_filtered: probe", iv->cent->ix.get(), qp + a0 * qrow, qdtype,
                                            m, P, is->f_probe_ids.ptr, is->f_probe_dists.ptr, stream, nullptr,
                                            flat_max_kc_deep()))
                return rc;
            ivf_filter_count_kernel<<<unsigned((m + 7) / 8), 256, 0, stream>>>(
                is->f_probe_ids.ptr, uint32_t(m), uint32_t(P), is->qidx.ptr + a0, is->cl_allowed.ptr, is->cl_rows.ptr,
                is->q_probes.ptr, is->q_allowed.ptr, is->q_rows.ptr);
            count_launch();
            CUDA_TRY(cudaGetLastError());
        }
        if (P == p_max) {
            groups[P] = std::move(active);
            break;
        }
        CUDA_TRY(cudaMemcpyAsync(allowed.data(), is->q_allowed.ptr, nq * 4, cudaMemcpyDeviceToHost, stream));
        CUDA_TRY(cudaStreamSynchronize(stream));
        std::vector<uint32_t> short_of_k;
        for (uint32_t q : active) (allowed[q] >= k ? groups[P] : short_of_k).push_back(q);
        if (short_of_k.empty()) break;
        active = std::move(short_of_k);
    }
    // 3. the scan per group
    for (auto& [P, idx] : groups) {
        const size_t ng = idx.size();
        CUDA_TRY(cudaMemcpyAsync(is->qidx.ptr, idx.data(), ng * 4, cudaMemcpyHostToDevice, stream));
        const unsigned char* qp = gather(idx);
        if (!qp) return fail(std::string(who) + ": gathering the queries failed");
        const bool whole = ng == nq;   // the batch in order: the body writes the outputs, padded +inf in place
        if (!whole) {
            CUDA_TRY(is->g_ids.ensure(ng * k));
            CUDA_TRY(is->g_dists.ensure(ng * k));
        }
        uint64_t* gi = whole ? d_out_ids : is->g_ids.ptr;
        float* gd = whole ? d_out_dists : is->g_dists.ptr;
        if (int rc = ivf_search_on_device(iv, sc, qp, qdtype, ng, k, P, gi, gd, nullptr, is->masked.ptr)) return rc;
        ivf_filter_scatter_kernel<<<unsigned((ng * k + 255) / 256), 256, 0, stream>>>(
            gi, gd, whole ? nullptr : is->qidx.ptr, ng, uint32_t(k), d_out_ids, d_out_dists);
        count_launch();
        CUDA_TRY(cudaGetLastError());
    }
    if (d_probes) CUDA_TRY(cudaMemcpyAsync(d_probes, is->q_probes.ptr, nq * 4, cudaMemcpyDeviceToDevice, stream));
    if (d_allowed) CUDA_TRY(cudaMemcpyAsync(d_allowed, is->q_allowed.ptr, nq * 4, cudaMemcpyDeviceToDevice, stream));
    if (d_rows) CUDA_TRY(cudaMemcpyAsync(d_rows, is->q_rows.ptr, nq * 4, cudaMemcpyDeviceToDevice, stream));
    if (d_ext_ids) CUDA_TRY(slots_to_external(d_out_ids, nq * k, d_ext_ids, stream));   // slots -> external ids
    return 0;
}

int ivf_check_search(const char* who, const svsb200_ivf* iv, int qdtype, size_t k, size_t n_probes) {
    const std::string w(who);
    if (!iv) return fail(w + ": NULL index");
    if (k == 0 || k > 1024) return fail(w + ": k must be in [1, 1024]");
    if (n_probes == 0 || n_probes > std::min<size_t>(iv->C, 1024))
        return fail(w + ": n_probes must be in [1, min(num_clusters, 1024)] = [1, " +
                    std::to_string(std::min<size_t>(iv->C, 1024)) + "]");
    if (qdtype != SVSB200_F32 && qdtype != SVSB200_F16) return fail(w + ": queries must be float32 or float16");
    return 0;
}

static int ivf_check_rows(const char* who, const void* vectors, int dtype, size_t n, size_t dim, int metric, bool sq = false) {
    const std::string w(who);
    if (!vectors) return fail(w + ": NULL input");
    if (sq) {
        if (dtype != SVSB200_I8 && dtype != SVSB200_U8) return fail(w + ": SQ codes must be int8 or uint8");
    } else if (dtype != SVSB200_F32 && dtype != SVSB200_F16) {
        return fail(w + ": rows must be float32 or float16 (integer, SQ and LVQ rows are not supported)");
    }
    if (metric < SVSB200_L2 || metric > SVSB200_COSINE) return fail(w + ": bad metric");
    if (n == 0 || dim == 0) return fail(w + ": empty dataset");
    if (n >= (size_t(1) << 31)) return fail(w + ": more than 2^31-1 vectors");
    return 0;
}

cudaError_t sq_encode(const float* d_x, size_t count, int code_type, float scale, float bias, uint8_t* d_codes, unsigned grid,
                      cudaStream_t stream) {
    if (code_type == SVSB200_I8)
        sq_encode_kernel<SVSB200_I8><<<grid, 256, 0, stream>>>(d_x, count, scale, bias, d_codes);
    else
        sq_encode_kernel<SVSB200_U8><<<grid, 256, 0, stream>>>(d_x, count, scale, bias, d_codes);
    count_launch();
    return cudaGetLastError();
}

// IVFIndex::assemble_from_clustering over checked rows (SQ codes when `storage` is SVSB200_SQ): the cluster-major layout,
// each cluster from a 32-row boundary, its rows in ascending id, zero padding.
static int ivf_assemble(const char* who, const void* vectors, int dtype, int storage, float scale, float bias, size_t n,
                        size_t dim, int metric, const float* centroids, size_t num_centroids, const uint32_t* assignments,
                        int device, svsb200_ivf** out) {
    const std::string w(who);
    const size_t C = num_centroids;
    if (!centroids) return fail(w + ": NULL centroids");
    if (C == 0 || C >= (size_t(1) << 31)) return fail(w + ": num_centroids must be in [1, 2^31)");
    if (assignments)
        for (size_t i = 0; i < n; ++i)
            if (assignments[i] >= C) return fail(w + ": assignment " + std::to_string(i) + " is not a cluster");
    cudaDeviceProp prop;
    if (int rc = check_device(who, device, &prop)) return rc;
    CUDA_TRY(cudaSetDevice(device));
    auto iv = std::make_unique<svsb200_ivf>();
    iv->n = n;
    iv->C = C;
    iv->centroids.assign(centroids, centroids + C * dim);
    if (int rc = ivf_centroid_index(centroids, C, dim, metric, device, &iv->cent)) return rc;
    const size_t row_bytes = dim * esize(dtype);
    std::vector<uint32_t> assign(n);
    if (assignments) {
        std::copy(assignments, assignments + n, assign.begin());
    } else {
        OwnStream own;
        CUDA_TRY(cudaStreamCreateWithFlags(&own.s, cudaStreamNonBlocking));
        DeviceBuffer<char> d_rows;
        DeviceBuffer<uint32_t> d_assign;
        CUDA_TRY(d_rows.ensure(n * row_bytes));
        CUDA_TRY(d_assign.ensure(n));
        CUDA_TRY(cudaMemcpy(d_rows.ptr, vectors, n * row_bytes, cudaMemcpyHostToDevice));
        if (int rc = ivf_assign(iv->cent.get(), d_rows.ptr, dtype, n, row_bytes, 65536, d_assign.ptr, own.s)) return rc;
        CUDA_TRY(cudaMemcpy(assign.data(), d_assign.ptr, n * 4, cudaMemcpyDeviceToHost));
    }
    // cluster-major layout: clusters in order, each from a 32-row boundary, its rows in ascending id
    iv->sizes.assign(C, 0);
    for (uint32_t a : assign) ++iv->sizes[a];
    std::vector<uint32_t> start(C), fill(C);
    size_t stored = 0;
    for (size_t c = 0; c < C; ++c) {
        start[c] = uint32_t(stored);
        fill[c] = uint32_t(stored);
        stored += round_up(iv->sizes[c], 32);
    }
    if (stored >= (size_t(1) << 32)) return fail(w + ": too many rows");
    auto ix = std::make_unique<svsb200_index>();
    ix->dtype = dtype;
    ix->metric = metric;
    ix->storage = storage;
    ix->scale = scale;
    ix->bias = bias;
    ix->n = std::max<size_t>(stored, 1);
    ix->dim = dim;
    ix->row_stride = data_row_stride(storage, dtype, dim);
    ix->gstride = 32;
    std::vector<uint32_t> row_ids(ix->n, 0xFFFFFFFFu);
    std::vector<char> rows(ix->n * size_t(ix->row_stride), 0);
    const char* src = static_cast<const char*>(vectors);
    for (size_t i = 0; i < n; ++i) {
        const uint32_t r = fill[assign[i]]++;
        row_ids[r] = uint32_t(i);
        std::copy(src + i * row_bytes, src + (i + 1) * row_bytes, rows.data() + size_t(r) * ix->row_stride);
    }
    ix->reps.push_back(std::make_unique<Replica>());
    Replica* rep = ix->reps.back().get();
    rep->device = device;
    rep->sm_count = prop.multiProcessorCount;
    CUDA_TRY(rep->d_vectors.ensure(rows.size()));
    CUDA_TRY(cudaMemcpy(rep->d_vectors.ptr, rows.data(), rows.size(), cudaMemcpyHostToDevice));
    CUDA_TRY(iv->d_row_ids.ensure(row_ids.size()));
    CUDA_TRY(cudaMemcpy(iv->d_row_ids.ptr, row_ids.data(), row_ids.size() * 4, cudaMemcpyHostToDevice));
    CUDA_TRY(iv->d_start.ensure(C));
    CUDA_TRY(cudaMemcpy(iv->d_start.ptr, start.data(), C * 4, cudaMemcpyHostToDevice));
    CUDA_TRY(iv->d_count.ensure(C));
    CUDA_TRY(cudaMemcpy(iv->d_count.ptr, iv->sizes.data(), C * 4, cudaMemcpyHostToDevice));
    ix->device_bytes = rows.size() + row_ids.size() * 4 + C * 8 + iv->cent->ix->device_bytes;
    iv->ix = std::move(ix);
    *out = iv.release();
    return 0;
}


}  // namespace svsb200

using namespace svsb200;

extern "C" {

int svsb200_ivf_random(uint64_t seed, size_t count, uint64_t* out) {
    if (count && !out) return fail("svsb200_ivf_random: NULL output");
    for (size_t i = 0; i < count; ++i) out[i] = ivf_next(seed);
    return 0;
}

// Host arithmetic only: the plan ivf_search_on_device runs, so that every shape can be checked without a device
// (tests/test_ivf_plan.py).
int svsb200_ivf_plan(size_t dim, int dtype, int storage, int metric, size_t k, size_t n_probes, size_t nq, int dynamic,
                     uint32_t* tile_rows, uint32_t* queries_per_item, uint32_t* ctas_per_sm, uint32_t* query_chunk,
                     uint32_t* leaf, uint32_t* static_dim, uint32_t* rows_per_pass, uint64_t* smem_bytes) {
    const std::string w = "svsb200_ivf_plan";
    if (!tile_rows || !queries_per_item || !ctas_per_sm || !query_chunk || !leaf || !static_dim || !rows_per_pass ||
        !smem_bytes)
        return fail(w + ": NULL output");
    const bool plain = storage == SVSB200_PLAIN && (dtype == SVSB200_F32 || dtype == SVSB200_F16);
    const bool sq = storage == SVSB200_SQ && (dtype == SVSB200_I8 || dtype == SVSB200_U8);
    if (!plain && !sq) return fail(w + ": rows are float32 / float16 (plain) or int8 / uint8 (SQ)");
    if (metric < SVSB200_L2 || metric > SVSB200_COSINE) return fail(w + ": bad metric");
    if (dim == 0 || dim > (size_t(1) << 24)) return fail(w + ": dim must be in [1, 2^24]");
    if (k == 0 || k > 1024) return fail(w + ": k must be in [1, 1024]");
    if (n_probes == 0 || n_probes > 1024) return fail(w + ": n_probes must be in [1, 1024]");
    if (nq == 0) return fail(w + ": nq must be positive");
    IvfPlan plan;
    if (int rc = ivf_plan(dim, dtype, storage, metric, k, n_probes, dynamic != 0, &plan)) return rc;
    *tile_rows = plan.tile_rows;
    *queries_per_item = plan.Q;
    *ctas_per_sm = plan.ctas;
    *query_chunk = uint32_t(std::min(plan.chunk, nq));
    *leaf = plan.leaf;
    *static_dim = plan.ds;
    *rows_per_pass = plan.nr;
    *smem_bytes = plan.smem;
    return 0;
}

int svsb200_ivf_group_plan(size_t dim, uint32_t* tile, uint32_t* chunk, uint64_t* smem_bytes) {
    if (!tile || !chunk || !smem_bytes) return fail("svsb200_ivf_group_plan: NULL output");
    if (dim == 0 || dim > (size_t(1) << 24)) return fail("svsb200_ivf_group_plan: dim must be in [1, 2^24]");
    IvfGroupPlan plan;
    if (int rc = ivf_group_plan(dim, &plan)) return rc;
    *tile = plan.tile;
    *chunk = plan.chunk;
    *smem_bytes = plan.smem;
    return 0;
}

int svsb200_ivf_cluster(const void* vectors, int dtype, size_t n, size_t dim, int metric, size_t num_centroids,
                        size_t minibatch_size, size_t num_iterations, int is_hierarchical, float training_fraction,
                        uint64_t seed, int device, float* out_centroids, uint32_t* out_assignments) {
    const char* who = "svsb200_ivf_cluster";
    if (int rc = ivf_check_rows(who, vectors, dtype, n, dim, metric)) return rc;
    if (is_hierarchical)
        return fail("svsb200_ivf_cluster: is_hierarchical = true: this entry point is the flat k-means; hierarchical k-means "
                    "is svsb200_ivf_cluster_hierarchical");
    if (!out_centroids || !out_assignments) return fail("svsb200_ivf_cluster: NULL output");
    const size_t C = num_centroids;
    size_t m = 0;
    if (int rc = ivf_training_size(who, n, C, minibatch_size, training_fraction, &m)) return rc;
    cudaDeviceProp prop;
    if (int rc = check_device(who, device, &prop)) return rc;
    CUDA_TRY(cudaSetDevice(device));
    const size_t row_bytes = dim * esize(dtype);
    // 1-2. training sample and initial centroids
    uint64_t s = seed;
    const std::vector<char> train = ivf_training_rows(s, vectors, n, m, row_bytes);
    const std::vector<uint32_t> init = ivf_shuffle_prefix(s, m, C);
    std::vector<float> cent(C * dim);
    for (size_t c = 0; c < C; ++c) ivf_row_f32(train.data(), dtype, row_bytes, init[c], dim, cent.data() + c * dim);
    const bool ip_like = metric != SVSB200_L2;
    if (ip_like) ivf_normalize(cent.data(), C, dim);
    OwnStream own;
    CUDA_TRY(cudaStreamCreateWithFlags(&own.s, cudaStreamNonBlocking));
    std::unique_ptr<svsb200_flat> cix;
    if (int rc = ivf_centroid_index(cent.data(), C, dim, metric, device, &cix)) return rc;
    DeviceBuffer<char> d_train;
    DeviceBuffer<uint32_t> d_assign;
    CUDA_TRY(d_train.ensure(m * row_bytes));
    CUDA_TRY(d_assign.ensure(std::max(m, n)));
    CUDA_TRY(cudaMemcpy(d_train.ptr, train.data(), m * row_bytes, cudaMemcpyHostToDevice));
    // 3. iterations
    if (int rc = ivf_kmeans_iterate(cix.get(), cent, C, dim, d_train.ptr, dtype, m, minibatch_size, num_iterations, ip_like, s,
                                    d_assign.ptr, own.s))
        return rc;
    // 4. final assignment of every row
    DeviceBuffer<char> d_rows;
    CUDA_TRY(d_rows.ensure(n * row_bytes));
    CUDA_TRY(cudaMemcpy(d_rows.ptr, vectors, n * row_bytes, cudaMemcpyHostToDevice));
    if (int rc = ivf_assign(cix.get(), d_rows.ptr, dtype, n, row_bytes, minibatch_size, d_assign.ptr, own.s)) return rc;
    CUDA_TRY(cudaMemcpy(out_assignments, d_assign.ptr, n * 4, cudaMemcpyDeviceToHost));
    std::copy(cent.begin(), cent.end(), out_centroids);
    return 0;
}

int svsb200_ivf_cluster_hierarchical(const void* vectors, int dtype, size_t n, size_t dim, int metric, size_t num_centroids,
                                     size_t level1_clusters, size_t minibatch_size, size_t num_iterations,
                                     float training_fraction, uint64_t seed, int device, float* out_centroids,
                                     uint32_t* out_assignments, uint32_t* out_level2_counts) {
    const char* who = "svsb200_ivf_cluster_hierarchical";
    if (int rc = ivf_check_rows(who, vectors, dtype, n, dim, metric)) return rc;
    if (!out_centroids || !out_assignments) return fail("svsb200_ivf_cluster_hierarchical: NULL output");
    const size_t C = num_centroids;
    size_t m = 0;
    if (int rc = ivf_training_size(who, n, C, minibatch_size, training_fraction, &m)) return rc;
    const size_t L1 = level1_clusters ? level1_clusters : size_t(std::sqrt(double(C)));
    if (L1 > C)
        return fail("svsb200_ivf_cluster_hierarchical: level1_clusters (" + std::to_string(L1) +
                    ") must be at most num_centroids (" + std::to_string(C) + ")");
    cudaDeviceProp prop;
    if (int rc = check_device(who, device, &prop)) return rc;
    CUDA_TRY(cudaSetDevice(device));
    const size_t row_bytes = dim * esize(dtype);
    const bool ip_like = metric != SVSB200_L2;
    // 1. training sample
    uint64_t s = seed;
    const std::vector<char> train = ivf_training_rows(s, vectors, n, m, row_bytes);
    // 2-3. level 1: the flat k-means with L1 centroids on the sample
    const std::vector<uint32_t> init1 = ivf_shuffle_prefix(s, m, L1);
    std::vector<float> cent1(L1 * dim);
    for (size_t c = 0; c < L1; ++c) ivf_row_f32(train.data(), dtype, row_bytes, init1[c], dim, cent1.data() + c * dim);
    if (ip_like) ivf_normalize(cent1.data(), L1, dim);
    OwnStream own;
    CUDA_TRY(cudaStreamCreateWithFlags(&own.s, cudaStreamNonBlocking));
    std::unique_ptr<svsb200_flat> cix1;
    if (int rc = ivf_centroid_index(cent1.data(), L1, dim, metric, device, &cix1)) return rc;
    DeviceBuffer<char> d_train;
    DeviceBuffer<uint32_t> d_tl1, d_tperm, d_tassign, d_counts;
    CUDA_TRY(d_train.ensure(m * row_bytes));
    CUDA_TRY(d_tl1.ensure(m));
    CUDA_TRY(cudaMemcpy(d_train.ptr, train.data(), m * row_bytes, cudaMemcpyHostToDevice));
    if (int rc = ivf_kmeans_iterate(cix1.get(), cent1, L1, dim, d_train.ptr, dtype, m, minibatch_size, num_iterations, ip_like, s,
                                    d_tl1.ptr, own.s))
        return rc;
    // 4. the sample against the final level-1 centroids: t_g training rows per group
    if (int rc = ivf_assign(cix1.get(), d_train.ptr, dtype, m, row_bytes, minibatch_size, d_tl1.ptr, own.s)) return rc;
    std::vector<uint32_t> tl1(m);
    CUDA_TRY(cudaMemcpy(tl1.data(), d_tl1.ptr, m * 4, cudaMemcpyDeviceToHost));
    std::vector<size_t> t(L1, 0), c(L1), tstart(L1), cstart(L1);
    for (uint32_t g : tl1) ++t[g];
    // 5. level-2 centroids per group: the proportional floor, then remainder draws (a draw on a group without training
    // rows, or with as many centroids as training rows, is discarded)
    size_t total = 0;
    for (size_t g = 0; g < L1; ++g) total += c[g] = size_t(double(t[g]) / double(m) * double(C));
    while (total < C) {
        const size_t j = ivf_next(s) % L1;
        if (t[j] == 0 || c[j] == t[j]) continue;
        ++c[j];
        ++total;
    }
    std::vector<uint64_t> gs(L1);   // the groups' own streams
    for (size_t g = 0; g < L1; ++g) gs[g] = ivf_next(s);
    for (size_t g = 0, tp = 0, cp = 0; g < L1; tp += t[g], cp += c[g], ++g) {
        tstart[g] = tp;
        cstart[g] = cp;
    }
    // 7. level 2, every group in lockstep: the training rows group-major, each group's centroids from its own rows
    CUDA_TRY(d_tperm.ensure(m));
    if (int rc = ivf_group_rows(d_tl1.ptr, m, L1, d_tperm.ptr, own.s)) return rc;
    std::vector<uint32_t> tperm(m);   // (the same permutation on the host, for the initial centroids)
    {
        std::vector<size_t> fill(tstart);
        for (size_t i = 0; i < m; ++i) tperm[fill[tl1[i]]++] = uint32_t(i);
    }
    std::vector<float> cent(C * dim);
    std::vector<IvfGroup> tgroups(L1);
    std::vector<uint2> range(C);
    for (size_t g = 0; g < L1; ++g) {
        tgroups[g] = {tstart[g], t[g], cstart[g], c[g]};
        if (c[g] == 0) continue;
        const std::vector<uint32_t> init = ivf_shuffle_prefix(gs[g], t[g], c[g]);
        for (size_t j = 0; j < c[g]; ++j) {
            ivf_row_f32(train.data(), dtype, row_bytes, tperm[tstart[g] + init[j]], dim, cent.data() + (cstart[g] + j) * dim);
            range[cstart[g] + j] = make_uint2(uint32_t(tstart[g]), uint32_t(tstart[g] + t[g]));
        }
    }
    if (ip_like) ivf_normalize(cent.data(), C, dim);
    DeviceBuffer<float> d_cent;
    DeviceBuffer<uint2> d_range;
    CUDA_TRY(d_cent.ensure(C * dim));
    CUDA_TRY(d_range.ensure(C));
    CUDA_TRY(d_tassign.ensure(m));
    CUDA_TRY(d_counts.ensure(C));
    CUDA_TRY(cudaMemcpy(d_range.ptr, range.data(), C * sizeof(uint2), cudaMemcpyHostToDevice));
    std::vector<uint32_t> counts(C);
    for (size_t it = 0; it < num_iterations; ++it) {
        CUDA_TRY(cudaMemcpyAsync(d_cent.ptr, cent.data(), C * dim * 4, cudaMemcpyHostToDevice, own.s));
        if (int rc = ivf_group_assign(d_train.ptr, dtype, dim, metric, d_tperm.ptr, tgroups, minibatch_size, d_cent.ptr,
                                      d_tassign.ptr, false, own.s))
            return rc;
        const unsigned warps = 8;
        const LaunchConfig cfg{int((C + warps - 1) / warps), int(warps), 0, own.s};
        CUDA_TRY(dispatch(IvfRows{}, dtype, [&](auto row) {
            return launch_kernel(ivf_kmeans_group_update_kernel<decltype(row)::value>, cfg, size_t(cfg.grid), false,
                                 static_cast<const char*>(d_train.ptr), uint32_t(row_bytes),
                                 static_cast<const uint32_t*>(d_tperm.ptr), static_cast<const uint2*>(d_range.ptr),
                                 uint32_t(dim), static_cast<const uint32_t*>(d_tassign.ptr), uint32_t(C), d_cent.ptr,
                                 d_counts.ptr);
        }));
        CUDA_TRY(cudaMemcpyAsync(cent.data(), d_cent.ptr, C * dim * 4, cudaMemcpyDeviceToHost, own.s));
        CUDA_TRY(cudaMemcpyAsync(counts.data(), d_counts.ptr, C * 4, cudaMemcpyDeviceToHost, own.s));
        CUDA_TRY(cudaStreamSynchronize(own.s));
        for (size_t g = 0; g < L1; ++g)
            if (c[g]) ivf_split(cent.data() + cstart[g] * dim, counts.data() + cstart[g], c[g], dim, t[g], gs[g]);
        if (ip_like) ivf_normalize(cent.data(), C, dim);
    }
    // 6. every row to its nearest level-1 centroid among the groups with level-2 centroids
    std::vector<uint32_t> pop;
    for (size_t g = 0; g < L1; ++g)
        if (c[g]) pop.push_back(uint32_t(g));
    std::unique_ptr<svsb200_flat> cixp;
    if (pop.size() < L1) {
        std::vector<float> cp(pop.size() * dim);
        for (size_t i = 0; i < pop.size(); ++i)
            std::copy(cent1.begin() + pop[i] * dim, cent1.begin() + (pop[i] + 1) * dim, cp.begin() + i * dim);
        if (int rc = ivf_centroid_index(cp.data(), pop.size(), dim, metric, device, &cixp)) return rc;
    }
    DeviceBuffer<char> d_rows;
    DeviceBuffer<uint32_t> d_assign, d_perm;
    CUDA_TRY(d_rows.ensure(n * row_bytes));
    CUDA_TRY(d_assign.ensure(n));
    CUDA_TRY(d_perm.ensure(n));
    CUDA_TRY(cudaMemcpy(d_rows.ptr, vectors, n * row_bytes, cudaMemcpyHostToDevice));
    if (int rc = ivf_assign(cixp ? cixp.get() : cix1.get(), d_rows.ptr, dtype, n, row_bytes, minibatch_size, d_assign.ptr, own.s))
        return rc;
    std::vector<uint32_t> al1(n);   // the index of the row's group in `pop`
    CUDA_TRY(cudaMemcpy(al1.data(), d_assign.ptr, n * 4, cudaMemcpyDeviceToHost));
    std::vector<size_t> a(pop.size(), 0);
    for (uint32_t p : al1) ++a[p];
    if (int rc = ivf_group_rows(d_assign.ptr, n, pop.size(), d_perm.ptr, own.s)) return rc;
    std::vector<IvfGroup> agroups(pop.size());
    for (size_t i = 0, ap = 0; i < pop.size(); ap += a[i], ++i) agroups[i] = {ap, a[i], cstart[pop[i]], c[pop[i]]};
    // 7. every row to the nearest of its own group's level-2 centroids
    CUDA_TRY(cudaMemcpy(d_cent.ptr, cent.data(), C * dim * 4, cudaMemcpyHostToDevice));
    if (int rc = ivf_group_assign(d_rows.ptr, dtype, dim, metric, d_perm.ptr, agroups, minibatch_size, d_cent.ptr, d_assign.ptr,
                                  true, own.s))
        return rc;
    CUDA_TRY(cudaMemcpy(out_assignments, d_assign.ptr, n * 4, cudaMemcpyDeviceToHost));
    std::copy(cent.begin(), cent.end(), out_centroids);
    if (out_level2_counts)
        for (size_t g = 0; g < L1; ++g) out_level2_counts[g] = uint32_t(c[g]);
    return 0;
}

int svsb200_ivf_create(const void* vectors, int dtype, size_t n, size_t dim, int metric, const float* centroids,
                       size_t num_centroids, const uint32_t* assignments, int device, svsb200_ivf** out) {
    const char* who = "svsb200_ivf_create";
    if (!out) return fail("svsb200_ivf_create: out is NULL");
    *out = nullptr;
    if (int rc = ivf_check_rows(who, vectors, dtype, n, dim, metric)) return rc;
    return ivf_assemble(who, vectors, dtype, SVSB200_PLAIN, 0.0f, 0.0f, n, dim, metric, centroids, num_centroids, assignments,
                        device, out);
}

int svsb200_ivf_create_sq(const void* codes, int code_type, size_t n, size_t dim, int metric, float scale, float bias,
                          const float* centroids, size_t num_centroids, const uint32_t* assignments, int device,
                          svsb200_ivf** out) {
    const char* who = "svsb200_ivf_create_sq";
    if (!out) return fail("svsb200_ivf_create_sq: out is NULL");
    *out = nullptr;
    if (int rc = ivf_check_rows(who, codes, code_type, n, dim, metric, true)) return rc;
    if (int rc = sq_check_params(who, scale, bias)) return rc;
    if (!assignments) return fail("svsb200_ivf_create_sq: SQ rows need assignments (there is no float row to rank)");
    return ivf_assemble(who, codes, code_type, SVSB200_SQ, scale, bias, n, dim, metric, centroids, num_centroids, assignments,
                        device, out);
}

int svsb200_sq_compress(const float* data, size_t n, size_t dim, int code_type, int device, void* out_codes, float* out_scale,
                        float* out_bias) {
    const char* who = "svsb200_sq_compress";
    if (!data || !out_codes || !out_scale || !out_bias) return fail("svsb200_sq_compress: NULL argument");
    if (code_type != SVSB200_I8 && code_type != SVSB200_U8) return fail("svsb200_sq_compress: codes must be int8 or uint8");
    const size_t count = n * dim;
    if (count == 0) return fail("svsb200_sq_compress: empty dataset");
    cudaDeviceProp prop;
    if (int rc = check_device(who, device, &prop)) return rc;
    CUDA_TRY(cudaSetDevice(device));
    OwnStream own;
    CUDA_TRY(cudaStreamCreateWithFlags(&own.s, cudaStreamNonBlocking));
    // the values pass through the device in pieces of at most 2^26, twice: min and max, then the codes
    const size_t piece = std::min(count, size_t(1) << 26);
    DeviceBuffer<float> d_x;
    DeviceBuffer<uint8_t> d_codes;
    DeviceBuffer<uint32_t> d_red;
    DeviceBuffer<unsigned long long> d_zero;
    CUDA_TRY(d_x.ensure(piece));
    CUDA_TRY(d_codes.ensure(piece));
    CUDA_TRY(d_red.ensure(3));
    CUDA_TRY(d_zero.ensure(1));
    const uint32_t init[3] = {0xFFFFFFFFu, 0u, 0u};
    CUDA_TRY(cudaMemcpyAsync(d_red.ptr, init, sizeof(init), cudaMemcpyHostToDevice, own.s));
    CUDA_TRY(cudaMemsetAsync(d_zero.ptr, 0xFF, sizeof(unsigned long long), own.s));
    const unsigned grid = unsigned(std::min<size_t>((piece + 255) / 256, size_t(prop.multiProcessorCount) * 8));
    for (size_t lo = 0; lo < count; lo += piece) {
        const size_t m = std::min(piece, count - lo);
        CUDA_TRY(cudaMemcpyAsync(d_x.ptr, data + lo, m * 4, cudaMemcpyHostToDevice, own.s));
        sq_minmax_kernel<<<grid, 256, 0, own.s>>>(d_x.ptr, m, lo, d_red.ptr, d_zero.ptr);
        count_launch();
        CUDA_TRY(cudaGetLastError());
        CUDA_TRY(cudaStreamSynchronize(own.s));   // (d_x is reused)
    }
    uint32_t red[3];
    unsigned long long first_zero = 0;
    CUDA_TRY(cudaMemcpy(red, d_red.ptr, sizeof(red), cudaMemcpyDeviceToHost));
    CUDA_TRY(cudaMemcpy(&first_zero, d_zero.ptr, sizeof(first_zero), cudaMemcpyDeviceToHost));
    if (red[2]) return fail("svsb200_sq_compress: the data hold a NaN or an infinity");
    auto from_key = [](uint32_t k) {
        const uint32_t u = (k & 0x80000000u) ? (k & 0x7FFFFFFFu) : ~k;
        float f;
        std::memcpy(&f, &u, 4);
        return f;
    };
    float mn = from_key(red[0]);
    const float mx = from_key(red[1]);
    if (mn == 0.0f) mn = data[first_zero];   // the sign of the first zero, as the reference's sequential min keeps it
    if (!(mx > mn)) return fail("svsb200_sq_compress: constant data (max == min) have no SQ scale");
    // scale = (max - min) / (MAX - MIN), bias = min - MIN * scale: every operation rounded on its own, no contraction
    const float MIN = code_type == SVSB200_I8 ? -128.0f : 0.0f, MAX = code_type == SVSB200_I8 ? 127.0f : 255.0f;
    volatile float range = mx - mn;
    const float scale = range / (MAX - MIN);
    volatile float t = MIN * scale;
    const float bias = mn - t;
    for (size_t lo = 0; lo < count; lo += piece) {
        const size_t m = std::min(piece, count - lo);
        CUDA_TRY(cudaMemcpyAsync(d_x.ptr, data + lo, m * 4, cudaMemcpyHostToDevice, own.s));
        CUDA_TRY(sq_encode(d_x.ptr, m, code_type, scale, bias, d_codes.ptr, grid, own.s));
        CUDA_TRY(cudaMemcpyAsync(static_cast<uint8_t*>(out_codes) + lo, d_codes.ptr, m, cudaMemcpyDeviceToHost, own.s));
        CUDA_TRY(cudaStreamSynchronize(own.s));   // (d_x and d_codes are reused)
    }
    *out_scale = scale;
    *out_bias = bias;
    return 0;
}

int svsb200_ivf_destroy(svsb200_ivf* index) {
    delete index;
    return 0;
}

size_t svsb200_ivf_size(const svsb200_ivf* index) { return index ? index->n : 0; }
size_t svsb200_ivf_dimensions(const svsb200_ivf* index) { return index ? index->ix->dim : 0; }
size_t svsb200_ivf_num_clusters(const svsb200_ivf* index) { return index ? index->C : 0; }
size_t svsb200_ivf_device_bytes(const svsb200_ivf* index) { return index ? index->ix->device_bytes : 0; }

int svsb200_ivf_cluster_sizes(const svsb200_ivf* index, uint32_t* out) {
    if (!index || !out) return fail("svsb200_ivf_cluster_sizes: NULL argument");
    std::copy(index->sizes.begin(), index->sizes.end(), out);
    return 0;
}

int svsb200_ivf_centroids(const svsb200_ivf* index, float* out) {
    if (!index || !out) return fail("svsb200_ivf_centroids: NULL argument");
    std::copy(index->centroids.begin(), index->centroids.end(), out);
    return 0;
}

int svsb200_ivf_search_device(svsb200_ivf* index, const void* d_queries, int qdtype, size_t nq, size_t k, size_t n_probes,
                              uint64_t* d_out_ids, float* d_out_dists, void* stream_) {
    if (int rc = ivf_check_search("svsb200_ivf_search_device", index, qdtype, k, n_probes)) return rc;
    if (nq == 0) return 0;
    if (!d_queries || !d_out_ids || !d_out_dists) return fail("svsb200_ivf_search_device: NULL buffer");
    return run_on_stream(index->ix->reps[0].get(), stream_, [&](Scratch* sc) {
        return ivf_search_on_device(index, sc, d_queries, qdtype, nq, k, n_probes, d_out_ids, d_out_dists, nullptr);
    });
}

int svsb200_ivf_search(svsb200_ivf* index, const void* queries, int qdtype, size_t nq, size_t k, size_t n_probes,
                       uint64_t* out_ids, float* out_dists) {
    if (int rc = ivf_check_search("svsb200_ivf_search", index, qdtype, k, n_probes)) return rc;
    if (nq == 0) return 0;
    if (!queries || !out_ids || !out_dists) return fail("svsb200_ivf_search: NULL buffer");
    return run_host_search(index->ix->reps[0].get(), {queries, nullptr, out_ids, out_dists}, nq * index->ix->dim * esize(qdtype),
                           0, nq, k, [&](Scratch* sc, const StagedBuffers& d) {
                               return ivf_search_on_device(index, sc, d.queries, qdtype, nq, k, n_probes, d.ids, d.dists, nullptr);
                           });
}

int svsb200_ivf_search_filtered_device(svsb200_ivf* index, const void* d_queries, int qdtype, size_t nq, size_t k,
                                       size_t n_probes, const uint32_t* d_id_bitmap, uint64_t* d_out_ids, float* d_out_dists,
                                       uint32_t* d_out_probes, uint32_t* d_out_allowed, uint32_t* d_out_rows, void* stream_) {
    const char* who = "svsb200_ivf_search_filtered_device";
    if (int rc = ivf_check_search(who, index, qdtype, k, n_probes)) return rc;
    if (!d_id_bitmap) return fail("svsb200_ivf_search_filtered_device: NULL bitmap");
    if (nq == 0) return 0;
    if (!d_queries || !d_out_ids || !d_out_dists) return fail("svsb200_ivf_search_filtered_device: NULL buffer");
    return run_on_stream(index->ix->reps[0].get(), stream_, [&](Scratch* sc) {
        return ivf_search_filtered_on_device(index, sc, d_queries, qdtype, nq, k, n_probes, d_id_bitmap, d_out_ids, d_out_dists,
                                             d_out_probes, d_out_allowed, d_out_rows, nullptr);
    });
}

int svsb200_ivf_search_filtered(svsb200_ivf* index, const void* queries, int qdtype, size_t nq, size_t k, size_t n_probes,
                                const uint32_t* id_bitmap, uint64_t* out_ids, float* out_dists, uint32_t* out_probes,
                                uint32_t* out_allowed, uint32_t* out_rows) {
    if (int rc = ivf_check_search("svsb200_ivf_search_filtered", index, qdtype, k, n_probes)) return rc;
    if (!id_bitmap) return fail("svsb200_ivf_search_filtered: NULL bitmap");
    if (nq == 0) return 0;
    if (!queries || !out_ids || !out_dists) return fail("svsb200_ivf_search_filtered: NULL buffer");
    return run_host_search(index->ix->reps[0].get(), {queries, id_bitmap, out_ids, out_dists, {out_probes, out_allowed, out_rows}},
                           nq * index->ix->dim * esize(qdtype), (index->n + 31) / 32, nq, k,
                           [&](Scratch* sc, const StagedBuffers& d) {
                               return ivf_search_filtered_on_device(index, sc, d.queries, qdtype, nq, k, n_probes, d.bitmap, d.ids,
                                                                    d.dists, d.per_query[0], d.per_query[1], d.per_query[2],
                                                                    nullptr);
                           });
}

}  // extern "C"
