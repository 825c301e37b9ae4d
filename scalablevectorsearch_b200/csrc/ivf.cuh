// ivf.cuh -- host-side structures of the IVF index (ivf.cu) shared with the dynamic IVF index (dynamic_ivf.cu).
#pragma once

#include "host.cuh"

#include <cmath>

namespace svsb200 {

// An own stream for the blocking entry points, destroyed on scope exit.
struct OwnStream {
    cudaStream_t s = nullptr;
    ~OwnStream() {
        if (s) cudaStreamDestroy(s);
    }
};

struct IvfScratch {
    DeviceBuffer<uint64_t> probe_ids, list_ids;
    DeviceBuffer<float> probe_dists, list_dists;
    DeviceBuffer<uint32_t> counts, list_off, item_off, cursor, list;
    // filtered search: the masked row ids, per-cluster counts, per-query P / allowed / Valid rows, a query group's
    // positions in the batch, its queries and its results, and the probes of a growth round
    DeviceBuffer<uint32_t> masked, cl_allowed, cl_rows, q_probes, q_allowed, q_rows, qidx;
    DeviceBuffer<unsigned char> gq;
    DeviceBuffer<uint64_t> g_ids, f_probe_ids;
    DeviceBuffer<float> g_dists, f_probe_dists;
};

}  // namespace svsb200

struct svsb200_ivf {
    std::unique_ptr<svsb200_index> ix;      // the cluster-major rows (each cluster from a 32-row boundary, zero padding)
    std::unique_ptr<svsb200_flat> cent;     // the centroids
    size_t n = 0, C = 0;
    std::vector<uint32_t> sizes;
    std::vector<float> centroids;
    svsb200::DeviceBuffer<uint32_t> d_row_ids, d_start, d_count;
    std::mutex mu;
    std::map<svsb200::Scratch*, std::unique_ptr<svsb200::IvfScratch>> scratch;   // per search scratch of ix's replica
    ~svsb200_ivf() {
        if (ix) cudaSetDevice(ix->reps[0]->device);
    }
};

namespace svsb200 {

// The centroids as a graph-free flat index (float32 rows), so that probing and assignment are one flat search.
int ivf_centroid_index(const float* centroids, size_t C, size_t dim, int metric, int device, std::unique_ptr<svsb200_flat>* out);
// Nearest centroid of `count` dense rows (device, row_bytes apart) in batches of `batch`, written to d_assign (uint32).
// Synchronises `stream`.
int ivf_assign(svsb200_flat* cent, const char* d_rows, int dtype, size_t count, size_t row_bytes, size_t batch,
               uint32_t* d_assign, cudaStream_t stream);
int ivf_check_search(const char* who, const svsb200_ivf* iv, int qdtype, size_t k, size_t n_probes);
// The search body on device buffers, enqueued on sc->stream (the centroid search synchronises it).  With d_ext_ids (the
// dynamic index) the row ids are slots, all-ones for a tombstone: the scan runs its DYN form, and the slots of the
// result are mapped to d_ext_ids.  With d_masked_ids the scan reads those row ids instead of the index's (a filtered
// search: disallowed rows all-ones) in its DYN form, and the ids are returned as they are.
int ivf_search_on_device(svsb200_ivf* iv, Scratch* sc, const void* d_queries, int qdtype, size_t nq, size_t k, size_t P,
                         uint64_t* d_out_ids, float* d_out_dists, const uint64_t* d_ext_ids,
                         const uint32_t* d_masked_ids = nullptr);
// The filtered search (include/svsb200.h, svsb200_ivf_search_filtered) on device buffers: `d_bitmap` over the row ids
// (original ids, or slots of the dynamic index, whose results are mapped to d_ext_ids); per-query outputs may be NULL.
// Enqueued on sc->stream apart from the probes and the growth decisions, which synchronise it.
int ivf_search_filtered_on_device(svsb200_ivf* iv, Scratch* sc, const void* d_queries, int qdtype, size_t nq, size_t k,
                                  size_t n_probes, const uint32_t* d_bitmap, uint64_t* d_out_ids, float* d_out_dists,
                                  uint32_t* d_probes, uint32_t* d_allowed, uint32_t* d_rows, const uint64_t* d_ext_ids);

// An SQ index's scale and bias: the scale finite and positive, the bias finite.
inline int sq_check_params(const char* who, float scale, float bias) {
    if (!(scale > 0.0f) || !std::isfinite(scale) || !std::isfinite(bias))
        return fail(std::string(who) + ": the SQ scale must be finite and positive and the bias finite");
    return 0;
}
// `count` float32 values (DEVICE) -> int8 / uint8 codes (`code_type`, DEVICE) with a fixed scale and bias, as
// SQDataset::set_datum encodes (detail::compress); enqueued on `stream` over `grid` blocks.
cudaError_t sq_encode(const float* d_x, size_t count, int code_type, float scale, float bias, uint8_t* d_codes, unsigned grid,
                      cudaStream_t stream);

}  // namespace svsb200
