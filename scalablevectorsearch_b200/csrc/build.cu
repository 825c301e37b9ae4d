// build.cu -- host side of the GPU Vamana graph builder (SURVEY.md §8 f1) + its small helper kernels.
// Replaces index::vamana::auto_build / VamanaBuilder::construct (index/vamana/index.h:404-440,968-994,
// vamana_build.h:221-310) for float32 / float16 / int8 / uint8 data with L2, inner-product or cosine distance.  Integer
// rows are built with exact int x int distances, float rows with the fp32 expression tree of the search, SQ codes with
// the SQ search's distances from each decompressed datum (svsb200_build_vamana_sq).
#include "build_kernels.cuh"
#include "host.cuh"
#include "ivf.cuh"   // sq_check_params

#include <type_traits>
#include <vector>

namespace svsb200 {

// add_reverse_edges, first half (vamana_build.h:484-501): one thread per new edge v -> u.
// The batch's nodes are first + i, or slots[first + i] when `slots` is given.
__global__ void reverse_insert_kernel(uint32_t first, uint32_t count, const uint32_t* __restrict__ slots,
                                      uint32_t* __restrict__ graph, uint32_t* __restrict__ deg,
                                      uint32_t gstride, uint32_t max_degree, int* __restrict__ head, int* __restrict__ next,
                                      uint32_t* __restrict__ pair_v, uint32_t* __restrict__ pair_count,
                                      uint32_t* __restrict__ touched, uint32_t* __restrict__ touched_count,
                                      uint32_t pair_cap) {
    const uint32_t idx = blockIdx.x * blockDim.x + threadIdx.x;
    const uint32_t i = idx / max_degree, j = idx % max_degree;
    if (i >= count) return;
    const uint32_t v = slots ? slots[first + i] : first + i;
    if (j >= min(deg[v], max_degree)) return;
    const uint32_t u = graph[size_t(v) * gstride + j];
    if (u == kNoNeighbor || u == v) return;
    // graph.add_edge(u, v) keeps rows free of repeats (core/graph/graph.h:211-260)
    // The reference tests the degree first (vamana_build.h:494-500): a full row takes the edge into the overflow even
    // when it already holds v, so that row is pruned again.
    uint32_t* urow = graph + size_t(u) * gstride;
    const uint32_t du = min(deg[u], max_degree);
    bool present = false;
    for (uint32_t z = 0; z < du && !present; ++z) present = urow[z] == v;
    if (present) {
        if (du < max_degree) return;
    } else {
        const uint32_t slot = atomicAdd(deg + u, 1u);
        if (slot < max_degree) {
            urow[slot] = v;
            return;
        }
        atomicSub(deg + u, 1u);
    }
    const uint32_t e = atomicAdd(pair_count, 1u);
    if (e >= pair_cap) return;
    pair_v[e] = v;
    const int old = atomicExch(head + u, int(e));
    next[e] = old;
    if (old < 0) touched[atomicAdd(touched_count, 1u)] = u;
}

__global__ void reset_heads_kernel(const uint32_t* __restrict__ touched, const uint32_t* __restrict__ touched_count,
                                   int* __restrict__ head) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < *touched_count) head[touched[i]] = -1;
}

// ---- medoid (core/medioid.h:232-350): mean in double, then the row closest to it in double; with `status`, over the
// Valid rows only (find_medioid's predicate) ----
template <int ROWT>
__global__ void column_sum_kernel(const char* __restrict__ vectors, uint32_t n, uint32_t dim, uint32_t row_stride,
                                  const uint8_t* __restrict__ status, double* __restrict__ sums) {
    const uint32_t rows_per_block = 256;
    const uint32_t r0 = blockIdx.x * rows_per_block;
    for (uint32_t d = threadIdx.x; d < dim; d += blockDim.x) {
        double acc = 0.0;
        for (uint32_t r = r0; r < min(n, r0 + rows_per_block); ++r) {
            if (status && status[r] != SLOT_VALID) continue;
            const char* row = vectors + size_t(r) * row_stride;
            if constexpr (ROWT == SVSB200_F32) acc += double(reinterpret_cast<const float*>(row)[d]);
            else if constexpr (ROWT == SVSB200_F16) acc += double(__half2float(reinterpret_cast<const __half*>(row)[d]));
            else if constexpr (ROWT == SVSB200_I8) acc += double(reinterpret_cast<const int8_t*>(row)[d]);
            else acc += double(reinterpret_cast<const uint8_t*>(row)[d]);
        }
        atomicAdd(sums + d, acc);
    }
}

// `count` rows enter the mean.  narrow = 1 compares the distances after narrowing to float, ties by id (find_medioid
// keeps Neighbor<size_t>{i, narrow_cast<float>(distance)}), narrow = 0 compares the doubles (the static builder).
template <int ROWT>
__global__ void medoid_distance_kernel(const char* __restrict__ vectors, uint32_t n, uint32_t dim, uint32_t row_stride,
                                       const uint8_t* __restrict__ status, double count, int narrow,
                                       const double* __restrict__ sums, double* __restrict__ best_d,
                                       uint32_t* __restrict__ best_i) {
    // one warp per row; block-level argmin, one (distance, id) pair per block
    __shared__ double sd[8];
    __shared__ uint32_t si[8];
    const uint32_t warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const uint32_t r = blockIdx.x * 8 + warp;
    const bool use = r < n && !(status && status[r] != SLOT_VALID);
    double acc = 0.0;
    if (use) {
        const char* row = vectors + size_t(r) * row_stride;
        for (uint32_t d = lane; d < dim; d += 32) {
            double x;
            if constexpr (ROWT == SVSB200_F32) x = double(reinterpret_cast<const float*>(row)[d]);
            else if constexpr (ROWT == SVSB200_F16) x = double(__half2float(reinterpret_cast<const __half*>(row)[d]));
            else if constexpr (ROWT == SVSB200_I8) x = double(reinterpret_cast<const int8_t*>(row)[d]);
            else x = double(reinterpret_cast<const uint8_t*>(row)[d]);
            const double diff = sums[d] / count - x;
            acc += diff * diff;
        }
    }
    for (int o = 16; o; o >>= 1) acc += __shfl_xor_sync(0xFFFFFFFFu, acc, o);
    if (lane == 0) {
        sd[warp] = !use ? 1e300 : narrow ? double(float(acc)) : acc;
        si[warp] = r;
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        double bd = sd[0];
        uint32_t bi = si[0];
        for (int w2 = 1; w2 < 8; ++w2)
            if (sd[w2] < bd) {
                bd = sd[w2];
                bi = si[w2];
            }
        best_d[blockIdx.x] = bd;
        best_i[blockIdx.x] = bi;
    }
}

// neighbours-first device rows -> the reference's in-memory layout (degree first, core/graph/graph.h:103-114)
__global__ void export_graph_kernel(const uint32_t* __restrict__ graph, const uint32_t* __restrict__ deg, uint32_t n,
                                    uint32_t gstride, uint32_t max_degree, uint32_t* __restrict__ out) {
    const uint32_t row = blockIdx.x * (blockDim.x / 32) + threadIdx.x / 32;
    const uint32_t lane = threadIdx.x & 31;
    if (row >= n) return;
    const uint32_t d = min(deg[row], max_degree);
    uint32_t* o = out + size_t(row) * (max_degree + 1);
    if (lane == 0) o[0] = d;
    for (uint32_t j = lane; j < max_degree; j += 32) o[1 + j] = j < d ? graph[size_t(row) * gstride + j] : 0u;
}

// batch rows [first, first+count) (or slots[first + q]) as prepared fp32 queries (exact conversion, zero padding)
template <int ROWT>
__global__ void batch_queries_kernel(const char* __restrict__ vectors, uint32_t row_stride, uint32_t dim, uint32_t qstride,
                                     uint32_t first, uint32_t count, const uint32_t* __restrict__ slots,
                                     float* __restrict__ qf, float* __restrict__ qaux) {
    const uint32_t q = blockIdx.x * (blockDim.x / 32) + threadIdx.x / 32;
    const uint32_t lane = threadIdx.x & 31;
    if (q >= count) return;
    const char* row = vectors + size_t(slots ? slots[first + q] : first + q) * row_stride;
    float sq = 0.f;
    for (uint32_t i = lane; i < qstride; i += 32) {
        float v = 0.f;
        if (i < dim) {
            if constexpr (ROWT == SVSB200_F32) v = reinterpret_cast<const float*>(row)[i];
            else v = __half2float(reinterpret_cast<const __half*>(row)[i]);
        }
        qf[size_t(q) * qstride + i] = v;
        sq = fmaf(v, v, sq);
    }
    for (int o = 16; o; o >>= 1) sq += __shfl_xor_sync(0xFFFFFFFFu, sq, o);
    if (lane == 0) {   // {a_norm, unused}: the cosine query norm (cosine.h:117-119)
        qaux[2 * size_t(q)] = sqrtf(sq);
        qaux[2 * size_t(q) + 1] = 0.f;
    }
}

// int8 / uint8 batch rows as prepared integer queries (prepare_queries_kernel's PREP_INT mode): the raw codes
// zero-padded to qstride bytes, {a_norm in distance::norm's order, int32 bits of sum x*x}
template <int ROWT>
__global__ void batch_codes_kernel(const char* __restrict__ vectors, uint32_t row_stride, uint32_t dim, uint32_t qstride,
                                   uint32_t first, uint32_t count, const uint32_t* __restrict__ slots,
                                   uint8_t* __restrict__ qcodes, float* __restrict__ qaux) {
    const uint32_t q = blockIdx.x * (blockDim.x / 32) + threadIdx.x / 32;
    const int lane = threadIdx.x & 31;
    if (q >= count) return;
    const char* row = vectors + size_t(slots ? slots[first + q] : first + q) * row_stride;
    const int xx = stage_codes<ROWT>(row, dim, qstride, reinterpret_cast<uint32_t*>(qcodes + size_t(q) * qstride), lane);
    const float a_norm = codes_norm<ROWT>(row, dim, xx, lane);
    if (lane == 0) {
        qaux[2 * size_t(q)] = a_norm;
        qaux[2 * size_t(q) + 1] = __int_as_float(xx);
    }
}

static bool int_dtype(int dtype) { return dtype == SVSB200_I8 || dtype == SVSB200_U8; }

__global__ void fill_u32_kernel(uint32_t* p, size_t n, uint32_t v) {
    const size_t i = size_t(blockIdx.x) * blockDim.x + threadIdx.x;
    if (i < n) p[i] = v;
}

// deg[v] = length of row v (neighbours first, kNoNeighbor padding)
__global__ void row_degrees_kernel(const uint32_t* __restrict__ graph, uint32_t n, uint32_t gstride, uint32_t max_degree,
                                   uint32_t* __restrict__ deg) {
    const uint32_t v = blockIdx.x * blockDim.x + threadIdx.x;
    if (v >= n) return;
    const uint32_t* row = graph + size_t(v) * gstride;
    uint32_t d = 0;
    while (d < max_degree && row[d] != kNoNeighbor) ++d;
    deg[v] = d;
}

int row_degrees(const GraphBuild& b) {
    row_degrees_kernel<<<unsigned((b.n + 255) / 256), 256, 0, b.stream>>>(b.graph, uint32_t(b.n), b.gstride, b.R, b.deg);
    count_launch();
    CUDA_TRY(cudaGetLastError());
    return 0;
}

int medoid(const GraphBuild& b, const uint8_t* d_status, size_t count, uint32_t* out) {
    const size_t n = b.n, dim = b.dim;
    const unsigned nblk = unsigned((n + 7) / 8);
    DeviceBuffer<double> d_sums, d_best_d;
    DeviceBuffer<uint32_t> d_best_i;
    CUDA_TRY(d_sums.ensure(dim));
    CUDA_TRY(d_best_d.ensure(nblk));
    CUDA_TRY(d_best_i.ensure(nblk));
    CUDA_TRY(cudaMemsetAsync(d_sums.ptr, 0, dim * 8, b.stream));
    const char* v = static_cast<const char*>(b.vectors);
    const int narrow = d_status ? 1 : 0;
    CUDA_TRY(dispatch(DataRows{}, b.dtype, [&](auto t) {
        constexpr int T = decltype(t)::value;
        column_sum_kernel<T><<<unsigned((n + 255) / 256), 128, 0, b.stream>>>(v, uint32_t(n), uint32_t(dim), b.row_stride, d_status, d_sums.ptr);
        medoid_distance_kernel<T><<<nblk, 256, 0, b.stream>>>(v, uint32_t(n), uint32_t(dim), b.row_stride, d_status, double(count), narrow, d_sums.ptr, d_best_d.ptr, d_best_i.ptr);
        return cudaSuccess;
    }));
    count_launch();
    count_launch();
    CUDA_TRY(cudaGetLastError());
    std::vector<double> bd(nblk);
    std::vector<uint32_t> bi(nblk);
    CUDA_TRY(cudaMemcpyAsync(bd.data(), d_best_d.ptr, size_t(nblk) * 8, cudaMemcpyDeviceToHost, b.stream));
    CUDA_TRY(cudaMemcpyAsync(bi.data(), d_best_i.ptr, size_t(nblk) * 4, cudaMemcpyDeviceToHost, b.stream));
    CUDA_TRY(cudaStreamSynchronize(b.stream));
    size_t best = 0;
    for (size_t k = 1; k < nblk; ++k)
        if (bd[k] < bd[best]) best = k;
    *out = bi[best];
    return 0;
}

// The lean search kernel in HIST mode over this graph: parameters and launch configuration (visited filter sized for
// b.n).  Errors read "<who>: ...".
static int build_search_config(const char* who, const GraphBuild& b, SearchParams* p, LaunchConfig* cfg) {
    if (b.window == 0) return fail(std::string(who) + ": window_size must be positive");
    if (b.window + 32 > kPoolMax - b.gstride) return fail(std::string(who) + ": window_size too large for the candidate pool");
    *p = SearchParams{};
    p->vectors = b.vectors;
    p->graph = b.graph;
    p->ref_degree = nullptr;
    p->n = uint32_t(b.n);
    p->dim = uint32_t(b.dim);
    p->row_stride = b.row_stride;
    p->gstride = b.gstride;
    p->greater = b.metric != SVSB200_L2;
    p->sq = b.sq;
    p->scale = b.sq ? b.scale : 1.f;
    p->bias = b.bias;
    p->scale_sq = b.scale * b.scale;   // EuclideanCompressed ctor (scalar.h:68-72)
    p->qcodes = nullptr;
    p->qstride = query_stride(b.dim);
    p->k = 0;
    p->window = uint32_t(b.window);
    p->capacity = uint32_t(b.window);
    p->cap_pad = uint32_t((b.window + 31) / 32 * 32);
    p->deg_pad = b.gstride;
    p->id_bytes = 4;
    // the whole history is kept; build_prune_kernel selects the pool from it in chunks when it outgrows shared memory
    p->hist_cap = kHistMax;
    // visited filter of the lean kernel, at its default size
    const LeanFilter lean = lean_filter(b.n, 2048);
    p->filter_slots = lean.slots;
    p->filter_shift = lean.shift;
    p->filter_tag16 = 1;
    *cfg = LaunchConfig{};
    cfg->warps_per_cta = 1;
    cfg->smem_bytes = fast_smem_bytes(p->qstride, p->cap_pad, p->deg_pad, lean.slots * 2u);
    cfg->stream = b.stream;
    cfg->grid = -b.sm_count;
    if (cfg->smem_bytes > kSmemOptInMax) return fail(std::string(who) + ": window_size too large for shared memory");
    return 0;
}

int check_construct(const char* who, const GraphBuild& b) {
    SearchParams p;
    LaunchConfig cfg;
    return build_search_config(who, b, &p, &cfg);
}

int construct_graph(const char* who, const GraphBuild& b, float reverse_alpha, uint32_t entry_point, const uint32_t* d_slots,
                    size_t count) {
    SearchParams p;
    LaunchConfig cfg;
    if (int rc = build_search_config(who, b, &p, &cfg)) return rc;
    if (count == 0) return 0;
    const uint32_t R = b.R, qstride = p.qstride, row_stride = b.row_stride;
    const cudaStream_t stream = b.stream;
    const int dtype = b.dtype;
    // batches (vamana_build.h:229-240)
    size_t num_batches = std::max<size_t>(40, (count + 4095) / 4096);
    if (num_batches > count) num_batches = count;
    const size_t batchsize = (count + num_batches - 1) / num_batches;
    const size_t pair_cap = batchsize * R;

    DeviceBuffer<uint32_t> d_hist_count, d_pair_v, d_counts, d_touched;
    DeviceBuffer<int> d_head, d_next;
    DeviceBuffer<uint2> d_hist;
    DeviceBuffer<float> d_qf, d_qaux;
    DeviceBuffer<uint8_t> d_qcodes;
    DeviceBuffer<unsigned int> d_work;
    CUDA_TRY(d_head.ensure(b.n));
    CUDA_TRY(cudaMemsetAsync(d_head.ptr, 0xFF, b.n * 4, stream));
    CUDA_TRY(d_next.ensure(pair_cap));
    CUDA_TRY(d_pair_v.ensure(pair_cap));
    CUDA_TRY(d_touched.ensure(pair_cap));
    CUDA_TRY(d_counts.ensure(3));   // pair count, touched count, history overflow flag
    CUDA_TRY(cudaMemsetAsync(d_counts.ptr + 2, 0, 4, stream));
    CUDA_TRY(d_hist.ensure(batchsize * size_t(p.hist_cap)));
    CUDA_TRY(d_hist_count.ensure(batchsize));
    // integer rows: int x int distances throughout, as the reference's default build adaptor uses the datum itself as
    // the query (extensions.h:114-282); SQ codes: the SQ search's operators over the decompressed datum
    const int op = b.sq ? (b.metric == SVSB200_L2 ? OP_L2I : b.metric == SVSB200_IP ? OP_IPF : OP_COSF)
                 : int_dtype(dtype) ? (b.metric == SVSB200_L2 ? OP_L2I : b.metric == SVSB200_IP ? OP_IPI : OP_COSI)
                                    : (b.metric == SVSB200_L2 ? OP_L2F : b.metric == SVSB200_IP ? OP_IPF : OP_COSF);
    const bool ints = op >= OP_L2I;
    if (ints) CUDA_TRY(d_qcodes.ensure(batchsize * size_t(qstride)));
    else CUDA_TRY(d_qf.ensure(batchsize * size_t(qstride)));
    CUDA_TRY(d_qaux.ensure(batchsize * 2));
    CUDA_TRY(cudaMemsetAsync(d_qaux.ptr, 0, batchsize * 2 * 4, stream));
    CUDA_TRY(d_work.ensure(1));
    p.entry_point = entry_point;
    p.qf = d_qf.ptr;
    p.qcodes = d_qcodes.ptr;
    p.qaux = d_qaux.ptr;
    p.work_counter = d_work.ptr;
    p.hist = d_hist.ptr;
    p.hist_count = d_hist_count.ptr;

    BuildParams bp{};
    bp.hist = d_hist.ptr;
    bp.hist_count = d_hist_count.ptr;
    bp.hist_cap = p.hist_cap;
    bp.head = d_head.ptr;
    bp.next = d_next.ptr;
    bp.pair_v = d_pair_v.ptr;
    bp.graph = b.graph;
    bp.deg = b.deg;
    bp.gstride = b.gstride;
    bp.max_degree = R;
    bp.max_candidates = uint32_t(b.max_candidates);
    bp.hist_overflow = d_counts.ptr + 2;
    bp.iterative = b.metric != SVSB200_L2;
    bp.work_counter = d_work.ptr;
    bp.count_ptr = d_counts.ptr + 1;
    bp.nodes = d_touched.ptr;
    bp.slots = d_slots;
    const int prune_grid = b.sm_count * 16;
    const char* vectors = static_cast<const char*>(b.vectors);
    auto prune = [&](int grid) {
        if (b.sq) return dispatch(BuildSqRows{}, dtype, [&](auto t) { return launch_build_prune_sq<decltype(t)::value>(op, p, bp, grid, stream); });
        return dispatch(DataRows{}, dtype, [&](auto t) { return launch_build_prune_op<decltype(t)::value>(op, p, bp, grid, stream); });
    };

    for (size_t bi = 0; bi < num_batches; ++bi) {
        const size_t start = std::min(count, batchsize * bi), stop = std::min(count, batchsize * (bi + 1));
        if (stop == start) continue;
        const uint32_t B = uint32_t(stop - start);
        // 1. generate_neighbors: search ...
        if (b.sq) {
            CUDA_TRY(dispatch(BuildSqRows{}, dtype, [&](auto t) {
                return launch_build_batch_sq<decltype(t)::value>(op, p, uint32_t(start), B, d_slots, d_qf.ptr, d_qcodes.ptr,
                                                                 d_qaux.ptr, stream);
            }));
        } else {
            CUDA_TRY(dispatch(DataRows{}, dtype, [&](auto t) {
                constexpr int T = decltype(t)::value;
                if constexpr (T == SVSB200_I8 || T == SVSB200_U8)
                    batch_codes_kernel<T><<<(B + 7) / 8, 256, 0, stream>>>(vectors, row_stride, uint32_t(b.dim), qstride, uint32_t(start), B, d_slots, d_qcodes.ptr, d_qaux.ptr);
                else
                    batch_queries_kernel<T><<<(B + 7) / 8, 256, 0, stream>>>(vectors, row_stride, uint32_t(b.dim), qstride, uint32_t(start), B, d_slots, d_qf.ptr, d_qaux.ptr);
                return cudaSuccess;
            }));
            count_launch();
        }
        CUDA_TRY(cudaMemsetAsync(d_work.ptr, 0, 4, stream));
        p.nq = B;
        // SQ L2: the integer builder's OP_L2I search, which reads SearchParams::sq
        CUDA_TRY(b.sq && op != OP_L2I
                     ? dispatch(BuildSqRows{}, dtype, [&](auto t) { return launch_build_search_sq<decltype(t)::value>(op, p, cfg); })
                     : dispatch(DataRows{}, dtype, [&](auto t) { return launch_build_search<decltype(t)::value>(op, p, cfg); }));
        // ... pool + prune (always with the configured alpha, vamana_build.h:268-272)
        CUDA_TRY(cudaMemsetAsync(d_work.ptr, 0, 4, stream));
        bp.reverse = PRUNE_FORWARD;
        bp.first = uint32_t(start);
        bp.count = B;
        bp.limit = R;
        bp.alpha = b.alpha;
        CUDA_TRY(prune(std::min<int>(prune_grid, int(B))));
        // 2. add_reverse_edges
        CUDA_TRY(cudaMemsetAsync(d_counts.ptr, 0, 8, stream));
        reverse_insert_kernel<<<unsigned((size_t(B) * R + 255) / 256), 256, 0, stream>>>(
            uint32_t(start), B, d_slots, b.graph, b.deg, b.gstride, R, d_head.ptr, d_next.ptr, d_pair_v.ptr, d_counts.ptr,
            d_touched.ptr, d_counts.ptr + 1, uint32_t(pair_cap));
        count_launch();
        CUDA_TRY(cudaMemsetAsync(d_work.ptr, 0, 4, stream));
        bp.reverse = PRUNE_REVERSE;
        bp.limit = uint32_t(b.prune_to);
        bp.alpha = reverse_alpha;
        CUDA_TRY(prune(prune_grid));
        reset_heads_kernel<<<unsigned((pair_cap + 255) / 256), 256, 0, stream>>>(d_touched.ptr, d_counts.ptr + 1, d_head.ptr);
        count_launch();
        CUDA_TRY(cudaGetLastError());
    }
    uint32_t hist_overflow = 0;
    CUDA_TRY(cudaMemcpyAsync(&hist_overflow, d_counts.ptr + 2, 4, cudaMemcpyDeviceToHost, stream));
    CUDA_TRY(cudaStreamSynchronize(stream));
    if (hist_overflow)
        return fail(std::string(who) + ": a construction search expanded more than " + std::to_string(kHistMax) +
                    " nodes; its history would be incomplete");
    return 0;
}

}  // namespace svsb200

using namespace svsb200;

// The static build of both entry points; `sq` marks int8 / uint8 rows as SQ codes of `scale` and `bias`.  Errors read
// "<who>: ...".
static int build_static(const char* who, const void* vectors, int dtype, size_t n, size_t dim, size_t row_stride_bytes,
                        int metric, bool sq, float scale, float bias, float alpha, size_t graph_max_degree,
                        size_t window_size, size_t max_candidate_pool_size, size_t prune_to, int device,
                        uint32_t* graph_rows_out, uint32_t* entry_point_out) {
    const std::string w = who;
    if (!vectors || !graph_rows_out || !entry_point_out) return fail(w + ": NULL argument");
    if (dtype < SVSB200_F32 || dtype > SVSB200_U8) return fail(w + ": bad dtype");
    if (metric < SVSB200_L2 || metric > SVSB200_COSINE) return fail(w + ": bad metric");
    if (n < 2 || dim == 0 || n >= (size_t(1) << 31)) return fail(w + ": bad shape");
    if (graph_max_degree == 0 || graph_max_degree > 32u * kFastMaxGW) return fail(w + ": graph_max_degree must be in [1, 128]");
    if (window_size == 0) return fail(w + ": window_size must be positive");
    // verify_and_set_default_index_parameters (index/vamana/index.h:1079-1110)
    // The candidate pool holds kPoolMax entries: the default is clamped to it, a larger value refused.
    if (max_candidate_pool_size == 0) max_candidate_pool_size = std::min<size_t>(3 * window_size, kPoolMax);
    if (max_candidate_pool_size > kPoolMax)
        return fail(w + ": max_candidate_pool_size above 512, the GPU builder's candidate pool");
    if (prune_to == 0) prune_to = graph_max_degree >= 16 ? graph_max_degree - 4 : graph_max_degree;
    if (prune_to > graph_max_degree) return fail(w + ": prune_to must be <= graph_max_degree");
    if (alpha == 0.f) alpha = metric == SVSB200_L2 ? 1.2f : 0.95f;
    if (metric == SVSB200_L2 ? alpha < 1.0f : alpha > 1.0f) return fail(w + ": alpha on the wrong side of 1 for this metric");
    const uint32_t R = uint32_t(graph_max_degree);
    cudaDeviceProp prop;
    if (int rc = check_device(who, device, &prop)) return rc;
    CUDA_TRY(cudaSetDevice(device));

    const size_t row_bytes = dim * esize(dtype);
    const size_t src_stride = row_stride_bytes ? row_stride_bytes : row_bytes;
    GraphBuild b;
    b.dtype = dtype;
    b.metric = metric;
    b.n = n;
    b.dim = dim;
    b.R = R;
    b.gstride = graph_stride(R);
    b.row_stride = data_row_stride(SVSB200_PLAIN, dtype, dim);
    b.window = window_size;
    b.max_candidates = max_candidate_pool_size;
    b.prune_to = prune_to;
    b.alpha = alpha;
    b.sq = sq;
    b.scale = scale;
    b.bias = bias;
    b.sm_count = prop.multiProcessorCount;
    if (int rc = check_construct(who, b)) return rc;

    DeviceBuffer<char> d_vectors;
    DeviceBuffer<uint32_t> d_graph, d_deg, d_export;
    cudaStream_t stream;
    CUDA_TRY(cudaStreamCreateWithFlags(&stream, cudaStreamNonBlocking));
    std::unique_ptr<CUstream_st, cudaError_t (*)(cudaStream_t)> stream_owner(stream, cudaStreamDestroy);
    b.stream = stream;
    CUDA_TRY(d_vectors.ensure(n * size_t(b.row_stride)));
    CUDA_TRY(cudaMemset(d_vectors.ptr, 0, n * size_t(b.row_stride)));
    CUDA_TRY(cudaMemcpy2D(d_vectors.ptr, b.row_stride, vectors, src_stride, row_bytes, n, cudaMemcpyHostToDevice));
    CUDA_TRY(d_graph.ensure(n * size_t(b.gstride)));
    CUDA_TRY(d_deg.ensure(n));
    CUDA_TRY(cudaMemset(d_deg.ptr, 0, n * 4));
    b.vectors = d_vectors.ptr;
    b.graph = d_graph.ptr;
    b.deg = d_deg.ptr;
    {
        const size_t cnt = n * size_t(b.gstride);
        fill_u32_kernel<<<unsigned((cnt + 255) / 256), 256, 0, stream>>>(d_graph.ptr, cnt, kNoNeighbor);
        count_launch();
    }
    // ---- entry point = medoid (index.h:986-990, core/medioid.h:292-330) ----
    uint32_t entry_point = 0;
    if (int rc = medoid(b, nullptr, n, &entry_point)) return rc;
    // ---- two passes (index.h:436-439): reverse pruning with alpha 1, then with the configured alpha ----
    for (int pass = 0; pass < 2; ++pass)
        if (int rc = construct_graph(who, b, pass == 0 ? 1.0f : alpha, entry_point, nullptr, n)) return rc;
    // ---- export in the reference's layout ----
    CUDA_TRY(d_export.ensure(n * size_t(R + 1)));
    export_graph_kernel<<<unsigned((n + 7) / 8), 256, 0, stream>>>(d_graph.ptr, d_deg.ptr, uint32_t(n), b.gstride, R, d_export.ptr);
    count_launch();
    CUDA_TRY(cudaGetLastError());
    CUDA_TRY(cudaMemcpyAsync(graph_rows_out, d_export.ptr, n * size_t(R + 1) * 4, cudaMemcpyDeviceToHost, stream));
    CUDA_TRY(cudaStreamSynchronize(stream));
    *entry_point_out = entry_point;
    return 0;
}

extern "C" int svsb200_build_vamana(const void* vectors, int dtype, size_t n, size_t dim, size_t row_stride_bytes, int metric,
                                    float alpha, size_t graph_max_degree, size_t window_size,
                                    size_t max_candidate_pool_size, size_t prune_to, int device, uint32_t* graph_rows_out,
                                    uint32_t* entry_point_out) {
    return build_static("svsb200_build_vamana", vectors, dtype, n, dim, row_stride_bytes, metric, false, 1.f, 0.f, alpha,
                        graph_max_degree, window_size, max_candidate_pool_size, prune_to, device, graph_rows_out,
                        entry_point_out);
}

extern "C" int svsb200_build_vamana_sq(const void* codes, int code_type, size_t n, size_t dim, int metric, float scale,
                                       float bias, float alpha, size_t graph_max_degree, size_t window_size,
                                       size_t max_candidate_pool_size, size_t prune_to, int device, uint32_t* graph_rows_out,
                                       uint32_t* entry_point_out) {
    const char* who = "svsb200_build_vamana_sq";
    if (code_type != SVSB200_I8 && code_type != SVSB200_U8) return fail("svsb200_build_vamana_sq: codes must be int8 or uint8");
    if (int rc = sq_check_params(who, scale, bias)) return rc;
    return build_static(who, codes, code_type, n, dim, 0, metric, true, scale, bias, alpha, graph_max_degree, window_size,
                        max_candidate_pool_size, prune_to, device, graph_rows_out, entry_point_out);
}
