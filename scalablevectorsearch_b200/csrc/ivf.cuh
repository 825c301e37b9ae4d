// ivf.cuh -- host-side structures of the IVF index (ivf.cu) shared with the dynamic IVF index (dynamic_ivf.cu).
#pragma once

#include "host.cuh"

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
// result are mapped to d_ext_ids.
int ivf_search_on_device(svsb200_ivf* iv, Scratch* sc, const void* d_queries, int qdtype, size_t nq, size_t k, size_t P,
                         uint64_t* d_out_ids, float* d_out_dists, const uint64_t* d_ext_ids);
// The blocking form over HOST buffers.
int ivf_search_host(svsb200_ivf* iv, const void* queries, int qdtype, size_t nq, size_t k, size_t P, uint64_t* out_ids,
                    float* out_dists, const uint64_t* d_ext_ids);

}  // namespace svsb200
