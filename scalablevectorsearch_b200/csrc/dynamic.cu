// dynamic.cu -- the dynamic (mutable) Vamana index of the C ABI: MutableVamanaIndex
// (index/vamana/dynamic_index.h) built or assembled from a graph, data and external ids, with insertion, soft
// deletion, consolidation and compaction.  Every slot has a status (Valid / Deleted / Empty) and an external id in
// HBM; the external -> slot translator (core/translation.h) lives on the host, and the slot rules are slots.h's.
// Searches go through svsb200_search* and run the lean kernel's MutableBuffer form (search_fast.cuh, MUT = true);
// insertion runs the graph builder over the new slots (build.cu), consolidation its prune kernel over pools selected by
// consolidate_pool_kernel.
// SQ storage (svsb200_dynamic_create_sq): the rows are int8 / uint8 codes under one scale and bias fixed at creation.
// Searches, insertion and consolidation measure them with the SQ search's operators, as the SQ builder does (build.cu);
// added float32 rows are encoded on the device (sq_encode) before they are placed; compact moves codes as it moves rows.
#include "build_kernels.cuh"
#include "host.cuh"
#include "ivf.cuh"   // sq_check_params, sq_encode

#include <algorithm>
#include <cmath>

namespace svsb200 {

static int check_dynamic(const svsb200_index* ix, const char* who) {
    if (!ix) return fail(std::string(who) + ": NULL index");
    if (!ix->dynamic) return fail(std::string(who) + ": not a dynamic index (create it with svsb200_dynamic_create)");
    return 0;
}

// Row slots[i] of the data <- row i of `src` (row_stride bytes, a multiple of 16); adjacency row slots[i] emptied
// (copy_points + clear_lists, dynamic_index.h:714-716).  One warp per row.
__global__ void place_rows_kernel(const uint4* __restrict__ src, const uint32_t* __restrict__ slots, uint32_t count,
                                  uint32_t row_stride, uint4* __restrict__ vectors, uint32_t* __restrict__ graph,
                                  uint32_t gstride) {
    const uint32_t i = blockIdx.x * (blockDim.x / 32) + threadIdx.x / 32;
    const uint32_t lane = threadIdx.x & 31;
    if (i >= count) return;
    const size_t s = slots[i], words = row_stride / 16;
    for (size_t j = lane; j < words; j += 32) vectors[s * words + j] = src[i * words + j];
    for (uint32_t j = lane; j < gstride; j += 32) graph[s * gstride + j] = kNoNeighbor;
}

__global__ void deleted_to_empty_kernel(uint8_t* __restrict__ status, uint32_t n) {
    const uint32_t v = blockIdx.x * blockDim.x + threadIdx.x;
    if (v < n && status[v] == SLOT_DELETED) status[v] = SLOT_EMPTY;
}

// The rows consolidation rewrites: Valid nodes with at least one neighbour that is not Valid (is_deleted is
// status != Valid, so Empty counts; consolidate.h:249-257).  Listed in no particular order.
__global__ void consolidation_nodes_kernel(const uint32_t* __restrict__ graph, const uint32_t* __restrict__ deg,
                                           const uint8_t* __restrict__ status, uint32_t n, uint32_t gstride,
                                           uint32_t* __restrict__ list, uint32_t* __restrict__ count) {
    const uint32_t v = blockIdx.x * blockDim.x + threadIdx.x;
    if (v >= n || status[v] != SLOT_VALID) return;
    const uint32_t* row = graph + size_t(v) * gstride;
    for (uint32_t j = 0; j < deg[v]; ++j)
        if (status[row[j]] != SLOT_VALID) {
            list[atomicAdd(count, 1u)] = v;
            return;
        }
}

// ref_degree[v] = deg[v]: rows written by a mutation hold no repeats, so their stored length is the reference's degree
__global__ void ref_degree_kernel(const uint32_t* __restrict__ deg, uint32_t n, uint16_t* __restrict__ ref_degree) {
    const uint32_t v = blockIdx.x * blockDim.x + threadIdx.x;
    if (v < n) ref_degree[v] = uint16_t(deg[v]);
}

// compact (dynamic_index.h:817-916): new slot i <- old slot new_to_old[i]; data row, adjacency row with every id mapped
// through old_to_new, stored degree.  One warp per new slot.
__global__ void compact_kernel(const uint32_t* __restrict__ new_to_old, const uint32_t* __restrict__ old_to_new, uint32_t m,
                               uint32_t row_stride, uint32_t gstride, const uint4* __restrict__ vec_in,
                               const uint32_t* __restrict__ graph_in, const uint16_t* __restrict__ refdeg_in,
                               uint4* __restrict__ vec_out, uint32_t* __restrict__ graph_out, uint16_t* __restrict__ refdeg_out) {
    const uint32_t i = blockIdx.x * (blockDim.x / 32) + threadIdx.x / 32;
    const uint32_t lane = threadIdx.x & 31;
    if (i >= m) return;
    const size_t o = new_to_old[i], words = row_stride / 16;
    for (size_t j = lane; j < words; j += 32) vec_out[i * words + j] = vec_in[o * words + j];
    for (uint32_t j = lane; j < gstride; j += 32) {
        const uint32_t id = graph_in[o * gstride + j];
        graph_out[size_t(i) * gstride + j] = id == kNoNeighbor ? kNoNeighbor : old_to_new[id];
    }
    if (lane == 0) refdeg_out[i] = refdeg_in[o];
}

// Bytes of device memory a dynamic index with room for `slots` slots holds.
static size_t dynamic_bytes(const svsb200_index* ix, size_t slots) {
    return slots * (size_t(ix->row_stride) + size_t(ix->gstride) * sizeof(uint32_t) + sizeof(uint16_t) + 1 + sizeof(uint64_t));
}

// Mutation parameters, 0 selecting the default (verify_and_set_default_index_parameters, index.h:1079-1110, and the
// from-graph constructor's window 2R, dynamic_index.h:198).  Rejects what the GPU builder cannot honour exactly: its
// candidate pool holds kPoolMax entries, so max_candidates <= 512 (the default 3 * window is clamped to 512).
static int resolve_mutation_parameters(const char* who, int metric, size_t R, float* alpha, size_t* window,
                                       size_t* max_candidates, size_t* prune_to) {
    const std::string w(who);
    if (*alpha == 0.f) *alpha = metric == SVSB200_L2 ? 1.2f : 0.95f;
    if (!(*alpha > 0.f) || !std::isfinite(*alpha) || (metric == SVSB200_L2 ? *alpha < 1.0f : *alpha > 1.0f))
        return fail(w + ": alpha on the wrong side of 1 for this metric");
    if (*window == 0) *window = 2 * R;
    if (*window + 32 > kPoolMax - graph_stride(R)) return fail(w + ": window_size too large for the candidate pool");
    if (*max_candidates == 0) *max_candidates = std::min<size_t>(3 * *window, kPoolMax);
    if (*max_candidates > kPoolMax) return fail(w + ": max_candidates above 512, the GPU builder's candidate pool");
    if (*prune_to == 0) *prune_to = R >= 16 ? R - 4 : R;
    if (*prune_to > R) return fail(w + ": prune_to must be <= graph_max_degree");
    return 0;
}

// The graph of a dynamic index as the builder sees it (deg = the caller's [n] scratch), on rep's device.
static GraphBuild graph_build(const svsb200_index* ix, Replica* rep, uint32_t* deg, cudaStream_t stream) {
    GraphBuild b;
    b.dtype = ix->dtype;
    b.metric = ix->metric;
    b.n = ix->n;
    b.dim = ix->dim;
    b.R = uint32_t(ix->max_degree);
    b.gstride = ix->gstride;
    b.row_stride = ix->row_stride;
    b.vectors = rep->d_vectors.ptr;
    b.graph = rep->d_graph.ptr;
    b.deg = deg;
    b.window = ix->dyn_window;
    b.max_candidates = ix->dyn_max_candidates;
    b.prune_to = ix->dyn_prune_to;
    b.alpha = ix->dyn_alpha;
    b.sq = ix->storage == SVSB200_SQ;
    b.scale = b.sq ? ix->scale : 1.f;
    b.bias = b.sq ? ix->bias : 0.f;
    b.sm_count = rep->sm_count;
    b.stream = stream;
    return b;
}

}  // namespace svsb200

using namespace svsb200;

// The body of svsb200_dynamic_create and svsb200_dynamic_create_sq, after their row checks: `storage` SVSB200_PLAIN, or
// SVSB200_SQ with aux = {scale, bias}.  Errors read "<who>: ...".
static int dynamic_create(const char* who, const void* vectors, int dtype, int storage, const float* aux, size_t n,
                          size_t dim, const uint32_t* graph_rows, size_t graph_row_len, uint32_t entry_point, int metric,
                          const uint64_t* external_ids, int device, svsb200_index** out) {
    const std::string w(who);
    if (!out) return fail(w + ": NULL output");
    *out = nullptr;
    if (n && !external_ids) return fail(w + ": NULL external ids");
    if (graph_row_len < 2 || graph_row_len - 1 > 32u * kFastMaxGW) return fail(w + ": graph_max_degree must be in [1, 128]");
    if (n >= (size_t(1) << 30)) return fail(w + ": at most 2^30 - 1 slots");
    SlotTable slots;
    if (int rc = slots.assign(who, external_ids, n)) return rc;
    svsb200_index* ix = nullptr;
    if (int rc = svsb200_index_create(vectors, dtype, n, dim, 0, graph_rows, graph_row_len, entry_point, metric, storage, aux,
                                      device, &ix))
        return rc;
    std::unique_ptr<svsb200_index, int (*)(svsb200_index*)> owner(ix, svsb200_index_destroy);
    ix->slots = std::move(slots);
    Replica* rep = ix->reps[0].get();
    CUDA_TRY(cudaSetDevice(rep->device));
    if (int rc = upload_slots(rep, ix->slots)) return rc;
    ix->device_bytes += n * (1 + sizeof(uint64_t));
    ix->dynamic = true;
    if (int rc = resolve_mutation_parameters(who, metric, ix->max_degree, &ix->dyn_alpha, &ix->dyn_window,
                                             &ix->dyn_max_candidates, &ix->dyn_prune_to))
        return rc;
    *out = owner.release();
    return 0;
}

extern "C" {

int svsb200_dynamic_create(const void* vectors, int dtype, size_t n, size_t dim, const uint32_t* graph_rows,
                           size_t graph_row_len, uint32_t entry_point, int metric, const uint64_t* external_ids, int device,
                           svsb200_index** out) {
    if (out) *out = nullptr;
    if (dtype != SVSB200_F32 && dtype != SVSB200_F16) return fail("svsb200_dynamic_create: float32 / float16 data only");
    return dynamic_create("svsb200_dynamic_create", vectors, dtype, SVSB200_PLAIN, nullptr, n, dim, graph_rows, graph_row_len,
                          entry_point, metric, external_ids, device, out);
}

int svsb200_dynamic_create_sq(const void* codes, int code_type, size_t n, size_t dim, float scale, float bias,
                              const uint32_t* graph_rows, size_t graph_row_len, uint32_t entry_point, int metric,
                              const uint64_t* external_ids, int device, svsb200_index** out) {
    const char* who = "svsb200_dynamic_create_sq";
    if (out) *out = nullptr;
    if (code_type != SVSB200_I8 && code_type != SVSB200_U8) return fail("svsb200_dynamic_create_sq: codes must be int8 or uint8");
    if (int rc = sq_check_params(who, scale, bias)) return rc;
    const float aux[2] = {scale, bias};
    return dynamic_create(who, codes, code_type, SVSB200_SQ, aux, n, dim, graph_rows, graph_row_len, entry_point, metric,
                          external_ids, device, out);
}

int svsb200_dynamic_delete(svsb200_index* ix, const uint64_t* ids, size_t count) {
    if (int rc = check_dynamic(ix, "svsb200_dynamic_delete")) return rc;
    if (count && !ids) return fail("svsb200_dynamic_delete: NULL ids");
    std::vector<uint32_t> slots;
    if (int rc = ix->slots.find("svsb200_dynamic_delete", ids, count, &slots)) return rc;
    if (count == 0) return 0;
    // (once this stream is drained the new status is visible to every later search of the index, whatever its stream)
    int rc = after_searches(ix, [&](Replica* rep, cudaStream_t stream) -> int {
        Replica::SlotStaging& st = rep->staging;
        CUDA_TRY(st.slots.ensure(count));
        CUDA_TRY(cudaMemcpyAsync(st.slots.ptr, slots.data(), count * sizeof(uint32_t), cudaMemcpyHostToDevice, stream));
        CUDA_TRY(mark_slots(st.slots.ptr, nullptr, count, SLOT_DELETED, rep, stream));
        CUDA_TRY(cudaStreamSynchronize(stream));
        return 0;
    });
    if (rc) return rc;
    // delete_entry + translator_.delete_external (dynamic_index.h:773-788)
    ix->slots.commit_delete(slots, ids, SLOT_DELETED);
    return 0;
}

int svsb200_dynamic_ids(const svsb200_index* ix, uint64_t* out_ids, size_t* count) {
    if (int rc = check_dynamic(ix, "svsb200_dynamic_ids")) return rc;
    return ix->slots.ids("svsb200_dynamic_ids", out_ids, count);
}

int svsb200_dynamic_has_id(const svsb200_index* ix, uint64_t id, int* out) {
    if (int rc = check_dynamic(ix, "svsb200_dynamic_has_id")) return rc;
    return ix->slots.has_id("svsb200_dynamic_has_id", id, out);
}

int svsb200_dynamic_export(const svsb200_index* ix, uint32_t* graph_rows_out, uint8_t* status_out, uint64_t* ext_ids_out,
                           uint32_t* entry_point_out) {
    if (int rc = check_dynamic(ix, "svsb200_dynamic_export")) return rc;
    const size_t n = ix->n, R = ix->max_degree;
    if (graph_rows_out) {
        const Replica* rep = ix->reps[0].get();
        CUDA_TRY(cudaSetDevice(rep->device));
        std::vector<uint32_t> rows(n * size_t(ix->gstride));
        CUDA_TRY(cudaMemcpy(rows.data(), rep->d_graph.ptr, rows.size() * sizeof(uint32_t), cudaMemcpyDeviceToHost));
        // neighbours-first device rows -> the reference's in-memory layout (degree first, core/graph/graph.h:103-114)
        for (size_t v = 0; v < n; ++v) {
            const uint32_t* in = rows.data() + v * ix->gstride;
            uint32_t* o = graph_rows_out + v * (R + 1);
            size_t d = 0;
            while (d < R && in[d] != kNoNeighbor) ++d;
            o[0] = uint32_t(d);
            for (size_t j = 0; j < R; ++j) o[1 + j] = j < d ? in[j] : 0u;
        }
    }
    ix->slots.export_to(status_out, ext_ids_out);
    if (entry_point_out) *entry_point_out = ix->entry_point;
    return 0;
}

int svsb200_dynamic_set_build_parameters(svsb200_index* ix, float alpha, size_t window_size, size_t max_candidates,
                                         size_t prune_to) {
    const char* who = "svsb200_dynamic_set_build_parameters";
    if (int rc = check_dynamic(ix, who)) return rc;
    if (int rc = resolve_mutation_parameters(who, ix->metric, ix->max_degree, &alpha, &window_size, &max_candidates, &prune_to))
        return rc;
    ix->dyn_alpha = alpha;
    ix->dyn_window = window_size;
    ix->dyn_max_candidates = max_candidates;
    ix->dyn_prune_to = prune_to;
    return 0;
}

int svsb200_dynamic_get_build_parameters(const svsb200_index* ix, float* alpha, size_t* window_size, size_t* max_candidates,
                                         size_t* prune_to) {
    if (int rc = check_dynamic(ix, "svsb200_dynamic_get_build_parameters")) return rc;
    if (alpha) *alpha = ix->dyn_alpha;
    if (window_size) *window_size = ix->dyn_window;
    if (max_candidates) *max_candidates = ix->dyn_max_candidates;
    if (prune_to) *prune_to = ix->dyn_prune_to;
    return 0;
}

int svsb200_dynamic_add(svsb200_index* ix, const void* vectors, int dtype, size_t count, const uint64_t* ids, int reuse_empty,
                        uint64_t* slots_out) {
    const char* who = "svsb200_dynamic_add";
    if (int rc = check_dynamic(ix, who)) return rc;
    if (count == 0) return 0;
    if (!vectors || !ids) return fail("svsb200_dynamic_add: NULL argument");
    // an SQ index takes float32 rows and encodes them with its fixed scale and bias (SQDataset::set_datum)
    const bool sq = ix->storage == SVSB200_SQ;
    if (sq) {
        if (dtype != SVSB200_F32) return fail("svsb200_dynamic_add: an SQ index takes float32 points");
        const float* x = static_cast<const float*>(vectors);
        for (size_t i = 0; i < count * ix->dim; ++i)
            if (!std::isfinite(x[i])) return fail("svsb200_dynamic_add: the points hold a NaN or an infinity");
    } else if (dtype != ix->dtype) {
        return fail("svsb200_dynamic_add: the points' dtype differs from the index's");
    }
    if (int rc = ix->slots.check_new(who, ids, count)) return rc;
    // slots (add_points, dynamic_index.h:670-706): Empty ones from first_empty_ (from 0 with reuse_empty), then appended
    std::vector<uint32_t> slots;
    const size_t old_n = ix->n, new_n = ix->slots.choose(count, reuse_empty ? 0 : ix->slots.first_empty, &slots);
    if (new_n >= (size_t(1) << 30)) return fail("svsb200_dynamic_add: at most 2^30 - 1 slots");
    {
        GraphBuild b;
        b = graph_build(ix, ix->reps[0].get(), nullptr, nullptr);
        b.n = new_n;
        if (int rc = check_construct(who, b)) return rc;
    }
    int rc = after_searches(ix, [&](Replica* rep, cudaStream_t stream) -> int {
        if (const size_t cap = slot_capacity(rep, new_n)) {   // (these first: d_status's size is the capacity)
            CUDA_TRY(cudaStreamSynchronize(stream));
            CUDA_TRY(grow(rep->d_vectors, old_n * ix->row_stride, cap * ix->row_stride));
            CUDA_TRY(grow(rep->d_graph, old_n * ix->gstride, cap * ix->gstride));
            CUDA_TRY(grow(rep->d_ref_degree, old_n, cap));
            if (int rc2 = grow_slots(rep, old_n, cap, stream)) return rc2;
            ix->device_bytes = dynamic_bytes(ix, cap);
        }
        // (the mirror grows before the graph is built: a failed construct_graph leaves edges to the new slots)
        ix->n = new_n;
        ix->slots.status.resize(new_n, SLOT_EMPTY);
        ix->slots.ext_ids.resize(new_n, 0);
        Replica::SlotStaging& st = rep->staging;
        DeviceBuffer<uint32_t> d_deg;
        CUDA_TRY(st.rows.ensure(count * ix->row_stride));
        CUDA_TRY(st.slots.ensure(count));
        CUDA_TRY(st.ids.ensure(count));
        CUDA_TRY(d_deg.ensure(new_n));
        CUDA_TRY(cudaMemsetAsync(st.rows.ptr, 0, count * ix->row_stride, stream));
        const size_t row_bytes = ix->dim * esize(ix->dtype);
        const void* from = vectors;   // the dense rows as stored, `row_bytes` apart
        cudaMemcpyKind kind = cudaMemcpyHostToDevice;
        DeviceBuffer<float> d_points;
        DeviceBuffer<uint8_t> d_codes;
        if (sq) {
            const size_t values = count * ix->dim;
            const unsigned grid = unsigned(std::min<size_t>((values + 255) / 256, size_t(rep->sm_count) * 8));
            CUDA_TRY(d_points.ensure(values));
            CUDA_TRY(d_codes.ensure(values));
            CUDA_TRY(cudaMemcpyAsync(d_points.ptr, vectors, values * sizeof(float), cudaMemcpyHostToDevice, stream));
            CUDA_TRY(sq_encode(d_points.ptr, values, ix->dtype, ix->scale, ix->bias, d_codes.ptr, grid, stream));
            from = d_codes.ptr;
            kind = cudaMemcpyDeviceToDevice;
        }
        CUDA_TRY(cudaMemcpy2DAsync(st.rows.ptr, ix->row_stride, from, row_bytes, row_bytes, count, kind, stream));
        CUDA_TRY(cudaMemcpyAsync(st.slots.ptr, slots.data(), count * sizeof(uint32_t), cudaMemcpyHostToDevice, stream));
        CUDA_TRY(cudaMemcpyAsync(st.ids.ptr, ids, count * sizeof(uint64_t), cudaMemcpyHostToDevice, stream));
        place_rows_kernel<<<unsigned((count + 7) / 8), 256, 0, stream>>>(
            reinterpret_cast<const uint4*>(st.rows.ptr), st.slots.ptr, uint32_t(count), ix->row_stride,
            reinterpret_cast<uint4*>(rep->d_vectors.ptr), rep->d_graph.ptr, ix->gstride);
        count_launch();
        CUDA_TRY(cudaGetLastError());
        const GraphBuild b = graph_build(ix, rep, d_deg.ptr, stream);
        if (int rc2 = row_degrees(b)) return rc2;
        // builder.construct(alpha_, entry_point(), slots) (dynamic_index.h:719-739): its greedy search ignores the slot
        // status, so Deleted slots are walked and may become neighbours of the new points, as in the reference
        if (int rc2 = construct_graph(who, b, ix->dyn_alpha, ix->entry_point, st.slots.ptr, count)) return rc2;
        ref_degree_kernel<<<unsigned((new_n + 255) / 256), 256, 0, stream>>>(d_deg.ptr, uint32_t(new_n), rep->d_ref_degree.ptr);
        count_launch();
        CUDA_TRY(cudaGetLastError());
        CUDA_TRY(mark_slots(st.slots.ptr, st.ids.ptr, count, SLOT_VALID, rep, stream));
        CUDA_TRY(cudaStreamSynchronize(stream));
        return 0;
    });
    if (rc) return rc;
    ix->slots.commit_add(slots, ids, slots_out);
    return 0;
}

int svsb200_dynamic_consolidate(svsb200_index* ix) {
    const char* who = "svsb200_dynamic_consolidate";
    if (int rc = check_dynamic(ix, who)) return rc;
    const size_t n = ix->n, R = ix->max_degree;
    const size_t valid = ix->slots.size();
    const bool replace_entry = ix->slots.status[ix->entry_point] == SLOT_DELETED;
    // (the reference would silently pick slot 0)
    if (replace_entry && valid == 0) return fail("svsb200_dynamic_consolidate: no Valid slot left for the entry point");
    uint32_t entry_point = ix->entry_point;
    int rc = after_searches(ix, [&](Replica* rep, cudaStream_t stream) -> int {
        DeviceBuffer<uint32_t> d_deg, d_nodes, d_count;
        CUDA_TRY(d_deg.ensure(n));
        CUDA_TRY(d_nodes.ensure(n));
        CUDA_TRY(d_count.ensure(1));
        const GraphBuild b = graph_build(ix, rep, d_deg.ptr, stream);
        // the entry point: compute_entry_point(data_, threadpool_, valid) (dynamic_index.h:982-993)
        if (replace_entry)
            if (int rc2 = medoid(b, rep->d_status.ptr, valid, &entry_point)) return rc2;
        if (int rc2 = row_degrees(b)) return rc2;
        CUDA_TRY(cudaMemsetAsync(d_count.ptr, 0, sizeof(uint32_t), stream));
        consolidation_nodes_kernel<<<unsigned((n + 255) / 256), 256, 0, stream>>>(rep->d_graph.ptr, d_deg.ptr, rep->d_status.ptr,
                                                                                 uint32_t(n), ix->gstride, d_nodes.ptr, d_count.ptr);
        count_launch();
        CUDA_TRY(cudaGetLastError());
        uint32_t total = 0;
        CUDA_TRY(cudaMemcpyAsync(&total, d_count.ptr, sizeof(uint32_t), cudaMemcpyDeviceToHost, stream));
        CUDA_TRY(cudaStreamSynchronize(stream));
        if (total) {
            // A node's new row depends only on its own row and on the rows of slots that are not Valid; neither changes
            // while consolidation runs (only Valid rows are rewritten, each by its own node).  So one pass over all
            // nodes, rows rewritten in place batch by batch, equals the reference's batches of 200 000 with updates
            // applied after each batch (consolidate.h).
            const size_t chunk = std::min<size_t>(total, 32768);
            const int grid = int(std::min<size_t>(size_t(rep->sm_count) * 16, chunk));
            uint32_t scratch_len = 32;
            while (scratch_len < R * R) scratch_len <<= 1;
            DeviceBuffer<uint2> d_hist;
            DeviceBuffer<uint32_t> d_hist_count, d_sid;
            DeviceBuffer<float> d_skey;
            DeviceBuffer<unsigned int> d_work;
            CUDA_TRY(d_hist.ensure(chunk * kPoolMax));
            CUDA_TRY(d_hist_count.ensure(chunk));
            CUDA_TRY(d_sid.ensure(size_t(grid) * scratch_len));
            CUDA_TRY(d_skey.ensure(size_t(grid) * scratch_len));
            CUDA_TRY(d_work.ensure(1));
            SearchParams p{};
            p.vectors = rep->d_vectors.ptr;
            p.graph = rep->d_graph.ptr;
            p.n = uint32_t(n);
            p.dim = uint32_t(ix->dim);
            p.row_stride = ix->row_stride;
            p.gstride = ix->gstride;
            p.greater = ix->metric != SVSB200_L2;
            p.sq = b.sq;
            p.scale = b.scale;
            p.bias = b.bias;
            p.scale_sq = b.scale * b.scale;   // EuclideanCompressed ctor (scalar.h:68-72)
            p.qstride = query_stride(ix->dim);
            BuildParams bp{};
            bp.hist = d_hist.ptr;
            bp.hist_count = d_hist_count.ptr;
            bp.hist_cap = kPoolMax;
            bp.graph = rep->d_graph.ptr;
            bp.deg = d_deg.ptr;
            bp.gstride = ix->gstride;
            bp.max_degree = uint32_t(R);
            bp.limit = uint32_t(ix->dyn_prune_to);
            bp.max_candidates = uint32_t(ix->dyn_max_candidates);
            bp.alpha = ix->dyn_alpha;
            bp.iterative = ix->metric != SVSB200_L2;
            bp.work_counter = d_work.ptr;
            bp.status = rep->d_status.ptr;
            bp.scratch_ids = d_sid.ptr;
            bp.scratch_keys = d_skey.ptr;
            bp.scratch_len = scratch_len;
            // over SQ codes the build adaptor's general distance (consolidate.h:241-244): the SQ search's operators
            const int op = ix->metric == SVSB200_L2 ? (b.sq ? OP_L2I : OP_L2F) : ix->metric == SVSB200_IP ? OP_IPF : OP_COSF;
            for (size_t start = 0; start < total; start += chunk) {
                bp.nodes = d_nodes.ptr + start;
                bp.count = uint32_t(std::min<size_t>(chunk, total - start));
                CUDA_TRY(cudaMemsetAsync(d_work.ptr, 0, 4, stream));
                CUDA_TRY(b.sq ? dispatch(DynamicSqRows{}, ix->dtype, [&](auto t) {
                                    return launch_consolidate_pool_sq<decltype(t)::value>(op, p, bp, grid, stream);
                                })
                              : dispatch(DynamicRows{}, ix->dtype, [&](auto t) {
                                    return launch_consolidate_pool_op<decltype(t)::value>(op, p, bp, grid, stream);
                                }));
                CUDA_TRY(cudaMemsetAsync(d_work.ptr, 0, 4, stream));
                bp.reverse = PRUNE_CONSOLIDATE;
                const int prune_grid = int(std::min<size_t>(size_t(rep->sm_count) * 16, bp.count));
                CUDA_TRY(b.sq ? dispatch(DynamicSqRows{}, ix->dtype, [&](auto t) {
                                    return launch_build_prune_sq<decltype(t)::value>(op, p, bp, prune_grid, stream);
                                })
                              : dispatch(DynamicRows{}, ix->dtype, [&](auto t) {
                                    return launch_build_prune_op<decltype(t)::value>(op, p, bp, prune_grid, stream);
                                }));
            }
            ref_degree_kernel<<<unsigned((n + 255) / 256), 256, 0, stream>>>(d_deg.ptr, uint32_t(n), rep->d_ref_degree.ptr);
            count_launch();
        }
        deleted_to_empty_kernel<<<unsigned((n + 255) / 256), 256, 0, stream>>>(rep->d_status.ptr, uint32_t(n));
        count_launch();
        CUDA_TRY(cudaGetLastError());
        CUDA_TRY(cudaStreamSynchronize(stream));
        return 0;
    });
    if (rc) return rc;
    ix->entry_point = entry_point;
    for (auto& st : ix->slots.status)
        if (st == SLOT_DELETED) st = SLOT_EMPTY;
    return 0;
}

int svsb200_dynamic_compact(svsb200_index* ix) {
    const char* who = "svsb200_dynamic_compact";
    if (int rc = check_dynamic(ix, who)) return rc;
    // (the reference throws from robin_map::at after it has already moved the data)
    if (std::find(ix->slots.status.begin(), ix->slots.status.end(), uint8_t(SLOT_DELETED)) != ix->slots.status.end())
        return fail("svsb200_dynamic_compact: the index holds Deleted slots; consolidate first");
    // nonmissing_indices (dynamic_index.h:800-809): the Valid slots, ascending
    const size_t n = ix->n;
    std::vector<uint64_t> ext;
    const std::vector<uint32_t> new_to_old = ix->slots.valid_slots(&ext);
    std::vector<uint32_t> old_to_new(n, kNoNeighbor);
    for (size_t i = 0; i < new_to_old.size(); ++i) old_to_new[new_to_old[i]] = uint32_t(i);
    const size_t m = new_to_old.size();
    if (m == 0 || old_to_new[ix->entry_point] == kNoNeighbor)
        return fail("svsb200_dynamic_compact: the entry point is not Valid; consolidate first");
    int rc = after_searches(ix, [&](Replica* rep, cudaStream_t stream) -> int {
        DeviceBuffer<uint32_t> d_n2o, d_o2n, graph;
        DeviceBuffer<unsigned char> vectors;
        DeviceBuffer<uint16_t> refdeg;
        DeviceBuffer<uint8_t> status;
        DeviceBuffer<uint64_t> ext_ids;
        CUDA_TRY(d_n2o.ensure(m));
        CUDA_TRY(d_o2n.ensure(n));
        CUDA_TRY(vectors.ensure(m * ix->row_stride));
        CUDA_TRY(graph.ensure(m * ix->gstride));
        CUDA_TRY(refdeg.ensure(m));
        CUDA_TRY(cudaMemcpyAsync(d_n2o.ptr, new_to_old.data(), m * 4, cudaMemcpyHostToDevice, stream));
        CUDA_TRY(cudaMemcpyAsync(d_o2n.ptr, old_to_new.data(), n * 4, cudaMemcpyHostToDevice, stream));
        if (int rc2 = compacted_slots(ext, m, &status, &ext_ids, stream)) return rc2;
        compact_kernel<<<unsigned((m + 7) / 8), 256, 0, stream>>>(
            d_n2o.ptr, d_o2n.ptr, uint32_t(m), ix->row_stride, ix->gstride, reinterpret_cast<const uint4*>(rep->d_vectors.ptr),
            rep->d_graph.ptr, rep->d_ref_degree.ptr, reinterpret_cast<uint4*>(vectors.ptr), graph.ptr, refdeg.ptr);
        count_launch();
        CUDA_TRY(cudaGetLastError());
        CUDA_TRY(cudaStreamSynchronize(stream));
        rep->d_vectors = std::move(vectors);   // (the old blocks are freed with the locals)
        rep->d_graph = std::move(graph);
        rep->d_ref_degree = std::move(refdeg);
        rep->d_status = std::move(status);
        rep->d_ext_ids = std::move(ext_ids);
        return 0;
    });
    if (rc) return rc;
    ix->n = m;
    ix->device_bytes = dynamic_bytes(ix, m);
    ix->slots.commit_compact(std::move(ext));
    ix->entry_point = old_to_new[ix->entry_point];
    return 0;
}

}  // extern "C"

// The body of svsb200_dynamic_build and svsb200_dynamic_build_sq, after their row checks: `sq` marks int8 / uint8 rows
// as SQ codes of `scale` and `bias`.  Errors read "<who>: ...".
static int dynamic_build(const char* who, const void* vectors, int dtype, bool sq, float scale, float bias, size_t n,
                         size_t dim, int metric, float alpha, size_t graph_max_degree, size_t window_size,
                         size_t max_candidates, size_t prune_to, const uint64_t* external_ids, int device,
                         svsb200_index** out) {
    const std::string w(who);
    if (!out) return fail(w + ": NULL output");
    *out = nullptr;
    if (metric < SVSB200_L2 || metric > SVSB200_COSINE) return fail(w + ": bad metric");
    if (graph_max_degree == 0 || graph_max_degree > 32u * kFastMaxGW) return fail(w + ": graph_max_degree must be in [1, 128]");
    if (window_size == 0) return fail(w + ": window_size must be positive");
    if (int rc = resolve_mutation_parameters(who, metric, graph_max_degree, &alpha, &window_size, &max_candidates, &prune_to))
        return rc;
    // the ids are checked as the create step checks them, before the build runs
    const char* create = sq ? "svsb200_dynamic_create_sq" : "svsb200_dynamic_create";
    if (n && !external_ids) return fail(std::string(create) + ": NULL external ids");
    {
        SlotTable probe;
        if (int rc = probe.assign(create, external_ids, n)) return rc;
    }
    std::vector<uint32_t> graph(n * (graph_max_degree + 1));
    uint32_t entry_point = 0;
    if (int rc = sq ? svsb200_build_vamana_sq(vectors, dtype, n, dim, metric, scale, bias, alpha, graph_max_degree, window_size,
                                              max_candidates, prune_to, device, graph.data(), &entry_point)
                    : svsb200_build_vamana(vectors, dtype, n, dim, 0, metric, alpha, graph_max_degree, window_size,
                                           max_candidates, prune_to, device, graph.data(), &entry_point))
        return rc;
    svsb200_index* ix = nullptr;
    const float aux[2] = {scale, bias};
    if (int rc = dynamic_create(create, vectors, dtype, sq ? SVSB200_SQ : SVSB200_PLAIN, sq ? aux : nullptr, n, dim, graph.data(),
                                graph_max_degree + 1, entry_point, metric, external_ids, device, &ix))
        return rc;
    ix->dyn_alpha = alpha;
    ix->dyn_window = window_size;
    ix->dyn_max_candidates = max_candidates;
    ix->dyn_prune_to = prune_to;
    *out = ix;
    return 0;
}

extern "C" {

int svsb200_dynamic_build(const void* vectors, int dtype, size_t n, size_t dim, int metric, float alpha,
                          size_t graph_max_degree, size_t window_size, size_t max_candidates, size_t prune_to,
                          const uint64_t* external_ids, int device, svsb200_index** out) {
    if (out) *out = nullptr;
    if (dtype != SVSB200_F32 && dtype != SVSB200_F16) return fail("svsb200_dynamic_build: float32 / float16 data only");
    return dynamic_build("svsb200_dynamic_build", vectors, dtype, false, 1.f, 0.f, n, dim, metric, alpha, graph_max_degree,
                         window_size, max_candidates, prune_to, external_ids, device, out);
}

int svsb200_dynamic_build_sq(const void* codes, int code_type, size_t n, size_t dim, int metric, float scale, float bias,
                             float alpha, size_t graph_max_degree, size_t window_size, size_t max_candidates,
                             size_t prune_to, const uint64_t* external_ids, int device, svsb200_index** out) {
    const char* who = "svsb200_dynamic_build_sq";
    if (out) *out = nullptr;
    if (code_type != SVSB200_I8 && code_type != SVSB200_U8) return fail("svsb200_dynamic_build_sq: codes must be int8 or uint8");
    if (int rc = sq_check_params(who, scale, bias)) return rc;
    return dynamic_build(who, codes, code_type, true, scale, bias, n, dim, metric, alpha, graph_max_degree, window_size,
                         max_candidates, prune_to, external_ids, device, out);
}

}  // extern "C"
