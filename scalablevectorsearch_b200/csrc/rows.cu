// rows.cu -- point access to the stored rows of a graph index (svsb200_index_distances, svsb200_index_reconstruct): the
// search's own distance between a query and a named row, and the rows themselves as float32.  The reference's
// MutableVamanaIndex::get_distance / reconstruct_at (index/vamana/dynamic_index.h:1152-1190, 1306-1322) and
// VamanaIndex::get_distance (index/vamana/index.h:915-933).
//
// The ids are what the handle's searches return: external ids of Valid slots on a dynamic index (through the slot
// table), row ids plus the id offset otherwise.  Every id is checked on the host before any device work.
#include "host.cuh"
#include "query_prep.cuh"
#include "search_kernel.cuh"

#include <algorithm>
#include <string>
#include <vector>

namespace svsb200 {

// One warp per (query, row) pair.  Every thread group of the warp evaluates the pair's row with the search's distance
// code (float_rows / int_rows and finish_distance, as eval_pass runs them), so the result has the search's bits; lane
// 0 writes it.  (With one CTA per SM as the register bound, the float32 cosine form holds its sums in 90 registers; a
// bound of 256 threads alone made ptxas stop at 64 and spill.)
template <int ROWT, int OP>
__global__ void __launch_bounds__(256, 1) row_distance_kernel(const __grid_constant__ SearchParams p,
                                                           const uint32_t* __restrict__ rows, uint32_t count,
                                                           float* __restrict__ out) {
    constexpr bool kInt = OP >= OP_L2I;
    constexpr int G = kInt ? 4 : 16 / Row<ROWT>::LPT;   // threads per row
    const uint32_t i = blockIdx.x * (blockDim.x / 32) + threadIdx.x / 32;
    const int lane = threadIdx.x & 31;
    if (i >= count) return;   // (a whole warp leaves together)
    const int t = lane % G;
    const char* const rowp[1] = {static_cast<const char*>(p.vectors) + size_t(rows[i]) * p.row_stride};
    const float aux0 = p.qaux[2 * size_t(i)], aux1 = p.qaux[2 * size_t(i) + 1];
    float sum[1] = {0.f}, nrm[1] = {0.f};
    int ixy[1] = {0}, iyy[1] = {0};
    if constexpr (kInt) {
        int_rows<ROWT, 1, true>(p, p.qcodes + size_t(i) * p.qstride, rowp, t, ixy, iyy);
    } else {
        float_rows<ROWT, OP, 0, 1, true>(p, p.qf + size_t(i) * p.qstride, rowp, t, sum, nrm);
    }
    const float d = finish_distance<OP>(p, sum[0], nrm[0], ixy[0], iyy[0], aux0, aux1);
    if (lane == 0) out[i] = d;
}

// Row element e of rows[i] as float32, one thread per element: plain float32 as stored, float16 the way the
// reference's Float16 converts to float (f16_scalar), int8 / uint8 exactly, SQ codes as scale * c + bias with two
// roundings (DecompressionAccessor, quantization/scalar/scalar.h:606-620).
__global__ void reconstruct_rows_kernel(const void* __restrict__ vectors, uint32_t row_stride, int dtype, int sq, float scale,
                                        float bias, const uint32_t* __restrict__ rows, uint32_t count, uint32_t dim,
                                        float* __restrict__ out) {
    const size_t e = size_t(blockIdx.x) * blockDim.x + threadIdx.x;
    if (e >= size_t(count) * dim) return;
    const size_t i = e / dim, d = e - i * dim;
    const char* row = static_cast<const char*>(vectors) + size_t(rows[i]) * row_stride;
    float v;
    if (dtype == SVSB200_F32) {
        v = reinterpret_cast<const float*>(row)[d];
    } else if (dtype == SVSB200_F16) {
        v = f16_scalar(reinterpret_cast<const uint16_t*>(row)[d]);
    } else {
        const int c = dtype == SVSB200_I8 ? int(reinterpret_cast<const int8_t*>(row)[d]) : int(reinterpret_cast<const uint8_t*>(row)[d]);
        v = sq ? sq_decompress(c, scale, bias) : float(c);
    }
    out[e] = v;
}

// The row (slot) of every id, or a failure naming the first id the handle does not hold.
static int rows_of(const char* who, const svsb200_index* ix, const uint64_t* ids, size_t count, std::vector<uint32_t>* rows) {
    rows->resize(count);
    for (size_t i = 0; i < count; ++i) {
        const uint64_t id = ids[i];
        if (ix->dynamic) {
            auto it = ix->slots.translator.find(id);   // Valid slots only: a Deleted slot's id is no longer known
            if (it == ix->slots.translator.end())
                return fail(std::string(who) + ": external id " + std::to_string(id) + " is not in the index");
            (*rows)[i] = it->second;
        } else {
            if (id < ix->id_offset || id - ix->id_offset >= ix->n)
                return fail(std::string(who) + ": id " + std::to_string(id) + " is out of range");
            (*rows)[i] = uint32_t(id - ix->id_offset);
        }
    }
    return 0;
}

// The argument checks both entry points share: a graph index of plain or SQ rows, non-null buffers when count > 0.
static int check_rows_call(const char* who, const svsb200_index* ix, size_t count, bool buffers) {
    if (!ix) return fail(std::string(who) + ": NULL index");
    if (count && !buffers) return fail(std::string(who) + ": NULL buffer");
    if (ix->storage == SVSB200_LVQ8) return fail(std::string(who) + ": LVQ-8 rows are not supported");
    if (ix->slot_mask) return fail(std::string(who) + ": not a graph index");
    if (count >= (size_t(1) << 31)) return fail(std::string(who) + ": too many ids in one call");
    return 0;
}

}  // namespace svsb200

using namespace svsb200;

extern "C" {

int svsb200_index_distances(svsb200_index* ix, const void* queries, int qdtype, size_t count, const uint64_t* ids, float* out) {
    const char* who = "svsb200_index_distances";
    if (qdtype < SVSB200_F32 || qdtype > SVSB200_U8) return fail(std::string(who) + ": bad query dtype");
    if (int rc = check_rows_call(who, ix, count, queries && ids && out)) return rc;
    int op = 0, mode = 0;
    if (int rc = choose_op(ix, qdtype, &op, &mode)) return fail(std::string(who) + ": " + svsb200_last_error());
    std::vector<uint32_t> rows;
    if (int rc = rows_of(who, ix, ids, count, &rows)) return rc;
    if (count == 0) return 0;
    Replica* rep = ix->reps[0].get();
    ScratchLease lease;
    if (int rc = lease.checkout(rep)) return rc;
    return lease.run([&](Scratch* sc) -> int {
        const cudaStream_t s = sc->stream;
        const size_t qbytes = count * ix->dim * esize(qdtype);
        CUDA_TRY(sc->q_raw.ensure(qbytes));
        CUDA_TRY(sc->point_rows.ensure(count));
        CUDA_TRY(sc->stage_dists.ensure(count));
        CUDA_TRY(cudaMemcpyAsync(sc->q_raw.ptr, queries, qbytes, cudaMemcpyHostToDevice, s));
        CUDA_TRY(cudaMemcpyAsync(sc->point_rows.ptr, rows.data(), count * 4, cudaMemcpyHostToDevice, s));
        if (int rc = prepare_queries(ix, rep, sc, sc->q_raw.ptr, qdtype, count, mode, s)) return rc;
        SearchParams p{};
        p.vectors = rep->d_vectors.ptr;
        p.n = uint32_t(ix->n);
        p.dim = uint32_t(ix->dim);
        p.row_stride = ix->row_stride;
        p.sq = ix->storage == SVSB200_SQ;
        p.scale = ix->scale;
        p.bias = ix->bias;
        p.scale_sq = ix->scale * ix->scale;   // as search_params sets it
        p.qf = sc->q_f32.ptr;
        p.qcodes = sc->q_codes.ptr;
        p.qaux = sc->q_aux.ptr;
        p.qstride = query_stride(ix->dim);
        p.nq = uint32_t(count);
        const int warps = 8;
        const LaunchConfig cfg{int((count + warps - 1) / warps), warps, 0, s};
        CUDA_TRY(dispatch(DataRows{}, ix->dtype, [&](auto row) {
            constexpr int ROWT = decltype(row)::value;
            return dispatch(SearchOps<ROWT>{}, op, [&](auto o) {
                return launch_kernel(row_distance_kernel<ROWT, decltype(o)::value>, cfg, cfg.grid, false, p,
                                     sc->point_rows.ptr, uint32_t(count), sc->stage_dists.ptr);
            });
        }));
        CUDA_TRY(cudaMemcpyAsync(out, sc->stage_dists.ptr, count * 4, cudaMemcpyDeviceToHost, s));
        CUDA_TRY(cudaStreamSynchronize(s));
        return 0;
    });
}

int svsb200_index_reconstruct(svsb200_index* ix, const uint64_t* ids, size_t count, float* out) {
    const char* who = "svsb200_index_reconstruct";
    if (int rc = check_rows_call(who, ix, count, ids && out)) return rc;
    std::vector<uint32_t> rows;
    if (int rc = rows_of(who, ix, ids, count, &rows)) return rc;
    if (count == 0) return 0;
    if (count * ix->dim >= (size_t(1) << 40)) return fail(std::string(who) + ": output too large");
    Replica* rep = ix->reps[0].get();
    ScratchLease lease;
    if (int rc = lease.checkout(rep)) return rc;
    return lease.run([&](Scratch* sc) -> int {
        const cudaStream_t s = sc->stream;
        const size_t elems = count * ix->dim;
        CUDA_TRY(sc->point_rows.ensure(count));
        CUDA_TRY(sc->dists.ensure(elems));
        CUDA_TRY(cudaMemcpyAsync(sc->point_rows.ptr, rows.data(), count * 4, cudaMemcpyHostToDevice, s));
        reconstruct_rows_kernel<<<unsigned((elems + 255) / 256), 256, 0, s>>>(
            rep->d_vectors.ptr, ix->row_stride, ix->dtype, ix->storage == SVSB200_SQ, ix->scale, ix->bias, sc->point_rows.ptr,
            uint32_t(count), uint32_t(ix->dim), sc->dists.ptr);
        count_launch();
        CUDA_TRY(cudaGetLastError());
        CUDA_TRY(cudaMemcpyAsync(out, sc->dists.ptr, elems * 4, cudaMemcpyDeviceToHost, s));
        CUDA_TRY(cudaStreamSynchronize(s));
        return 0;
    });
}

}  // extern "C"
