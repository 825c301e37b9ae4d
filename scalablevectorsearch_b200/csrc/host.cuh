// host.cuh -- host-side structures of libsvsb200 shared by index.cu, search.cu, flat.cu and build.cu.
//
// Host-side structure (the reference's thread pool -> CUDA streams, index/vamana/index.h:455-470,564-611):
//   * an index owns one Replica per device (graph + vectors in that device's HBM);
//   * every search call checks a Scratch (stream + prepared-query buffers + work counter + cancel flag) out
//     of the replica's pool, so concurrent host threads search concurrently on their own streams;
//   * a multi-replica index splits a batch with threads::balance (lib/threads/types.h:311-329), one slice per
//     device, results landing in disjoint rows of the caller's arrays (SURVEY.md 8e mode A);
//   * svsb200_search_sharded runs every query on every shard index and merges G*k -> k on one device with
//     the reference's TotalOrder (mode B); with NVLink peer access the shards' search kernels write their
//     rows straight into the merging device's buffer.
//
// No CPU fallback lives here: every entry point either runs CUDA kernels on an sm_90 device or fails.
#pragma once

#include "common.cuh"

#include <map>
#include <memory>
#include <mutex>
#include <string>
#include <vector>

namespace svsb200 {

int fail(const std::string& msg);   // records the calling thread's svsb200_last_error(); returns 1
#define CUDA_TRY(expr)                                                                         \
    do {                                                                                       \
        cudaError_t err__ = (expr);                                                            \
        if (err__ != cudaSuccess) {                                                            \
            return fail(std::string(#expr) + ": " + cudaGetErrorString(err__));                \
        }                                                                                      \
    } while (0)

// The one device check of every entry point that places data on a GPU: `device` is a valid ordinal of an sm_90
// device (this library holds sm_90a code only).  Errors read "<who>: ...".
int check_device(const char* who, int device, cudaDeviceProp* prop);

inline size_t esize(int dtype) { return dtype == SVSB200_F32 ? 4 : dtype == SVSB200_F16 ? 2 : 1; }
inline size_t round_up(size_t x, size_t m) { return (x + m - 1) / m * m; }

// ---- layout rules ----
// Bytes between dataset rows in HBM: 16-byte aligned; LVQ-8 rows as svsb200_lvq8_row_stride.
inline uint32_t data_row_stride(int storage, int dtype, size_t dim) {
    return uint32_t(storage == SVSB200_LVQ8 ? svsb200_lvq8_row_stride(dim) : round_up(dim * esize(dtype), 16));
}
// Words between adjacency rows in HBM.  Rows of up to 128 neighbours are padded to whole 32-word groups (one coalesced
// load per group and lane in the lean kernel, no per-lane bounds checks); wider rows stay 16-byte aligned only.
inline uint32_t graph_stride(size_t max_degree) {
    return uint32_t(round_up(max_degree, max_degree <= 32u * kFastMaxGW ? 32 : 4));
}
// Elements between prepared queries.
inline uint32_t query_stride(size_t dim) { return uint32_t(round_up(dim, 16)); }
// Visited filter of the lean kernel: sets of eight 16-bit tags, at least 64 slots (0 = off).  Sets are added until
// every id >> log2(sets) fits below the 0xFFFF "empty" mark, so the tags stay exact for any n.
struct LeanFilter {
    uint32_t slots, shift;   // shift = log2(sets)
};
inline LeanFilter lean_filter(size_t n, uint32_t slots) {
    if (slots && slots < 64) slots = 64;
    uint32_t shift = 0;
    while ((8u << shift) < slots) ++shift;
    while (slots && (uint64_t(n - 1) >> shift) >= 0xFFFFull) {
        ++shift;
        slots <<= 1;
    }
    return {slots, shift};
}

// Device memory owned by its holder: freed when the holder goes away.  The device it was allocated on must be
// current at that point (Scratch and Replica select it in their destructors, before their members are destroyed).
template <typename T> struct DeviceBuffer {
    T* ptr = nullptr;
    size_t count = 0;
    DeviceBuffer() = default;
    DeviceBuffer(const DeviceBuffer&) = delete;
    DeviceBuffer& operator=(const DeviceBuffer&) = delete;
    DeviceBuffer(DeviceBuffer&& o) noexcept : ptr(o.ptr), count(o.count) {
        o.ptr = nullptr;
        o.count = 0;
    }
    DeviceBuffer& operator=(DeviceBuffer&& o) noexcept {
        std::swap(ptr, o.ptr);
        std::swap(count, o.count);
        return *this;
    }
    ~DeviceBuffer() {
        if (ptr) cudaFree(ptr);
    }
    cudaError_t ensure(size_t n) {
        if (n <= count) return cudaSuccess;
        if (ptr) cudaFree(ptr);   // (synchronises the device: safe against work still using the old block)
        ptr = nullptr;
        count = 0;
        cudaError_t err = cudaMalloc(&ptr, n * sizeof(T));
        if (err == cudaSuccess) count = n;
        return err;
    }
};

// Everything one in-flight search needs on one device: the analogue of the reference's per-thread scratch
// space (index/vamana/index.h:455-470).
struct Scratch {
    int device = 0;
    cudaStream_t stream = nullptr;   // own non-blocking stream (blocking API) or the caller's (device API)
    cudaStream_t ctl = nullptr;      // side stream that raises the cancel flag while `stream` is busy
    bool owns_stream = false;
    DeviceBuffer<unsigned char> q_raw, q_codes, ids;
    DeviceBuffer<float> q_f32, q_aux, dists;
    DeviceBuffer<uint32_t> hops, evals, fetched;
    DeviceBuffer<uint64_t> exh_ids;                    // exhaustive scan split over base ranges: per-range top-k
    DeviceBuffer<float> exh_dists;
    DeviceBuffer<unsigned char> flat_a, flat_q2;       // tensor-core flat search: query tiles, gathered queries
    DeviceBuffer<float> flat_qnorm, flat_ckey, flat_d2;
    DeviceBuffer<uint32_t> flat_cid, flat_unv;         // candidates, unverified list (+ its counter in slot 0)
    DeviceBuffer<uint32_t> flat_progress;              // per CTA of the flat GEMM: tiles started (keeps row groups in step)
    DeviceBuffer<uint64_t> flat_i2;
    DeviceBuffer<uint64_t> gather_ids, merged_ids;     // sharded search (on the merging device)
    DeviceBuffer<float> gather_dists, merged_dists;
    DeviceBuffer<unsigned int> d_counter;
    DeviceBuffer<int> d_cancel;
    cudaEvent_t ev_start = nullptr, ev_stop = nullptr, ev_done = nullptr;
    bool timed = false;
    bool poll_cancel = false;        // this search was given a cancellation predicate: the kernels poll the flag
    size_t counted_nq = 0;
    int last_kernel = 0;
    ~Scratch() {
        cudaSetDevice(device);
        if (ev_start) cudaEventDestroy(ev_start);
        if (ev_stop) cudaEventDestroy(ev_stop);
        if (ev_done) cudaEventDestroy(ev_done);
        if (ctl) cudaStreamDestroy(ctl);
        if (owns_stream && stream) cudaStreamDestroy(stream);
    }
};

// One copy of the index in one device's HBM.
struct Replica {
    int device = 0;
    int sm_count = 0;
    DeviceBuffer<unsigned char> d_vectors;
    DeviceBuffer<uint32_t> d_graph;
    DeviceBuffer<uint16_t> d_ref_degree;
    DeviceBuffer<float> d_mean;          // LVQ-8: dataset mean
    DeviceBuffer<uint32_t> d_entry;      // entry points when there are several
    // tensor-core flat search: the base vectors as fp16 warpgroup-MMA tiles + per-row bias, built on first use
    DeviceBuffer<unsigned char> flat_b;
    DeviceBuffer<float> flat_bias;
    DeviceBuffer<unsigned int> flat_xmax;
    std::mutex mu;
    std::vector<Scratch*> idle;                      // pool for the blocking API
    std::map<cudaStream_t, Scratch*> by_stream;      // one per caller stream for the enqueue-only API
    std::vector<std::unique_ptr<Scratch>> all;       // (declared last: destroyed before the buffers above)
    ~Replica() { cudaSetDevice(device); }
};

// ---- scratch pool ----
inline Scratch* new_scratch(Replica* rep, cudaStream_t caller_stream, std::string* err) {
    auto sc = std::make_unique<Scratch>();
    sc->device = rep->device;
    cudaError_t e = cudaSuccess;
    if (caller_stream) {
        sc->stream = caller_stream;
    } else {
        e = cudaStreamCreateWithFlags(&sc->stream, cudaStreamNonBlocking);
        sc->owns_stream = true;
    }
    if (e == cudaSuccess) e = cudaStreamCreateWithFlags(&sc->ctl, cudaStreamNonBlocking);
    if (e == cudaSuccess) e = sc->d_counter.ensure(1);
    if (e == cudaSuccess) e = sc->d_cancel.ensure(1);
    if (e == cudaSuccess) e = cudaMemset(sc->d_cancel.ptr, 0, sizeof(int));
    if (e == cudaSuccess) e = cudaEventCreate(&sc->ev_start);
    if (e == cudaSuccess) e = cudaEventCreate(&sc->ev_stop);
    if (e == cudaSuccess) e = cudaEventCreateWithFlags(&sc->ev_done, cudaEventDisableTiming);
    if (e != cudaSuccess) {
        *err = std::string("scratch allocation: ") + cudaGetErrorString(e);
        return nullptr;
    }
    Scratch* raw = sc.get();
    rep->all.push_back(std::move(sc));
    return raw;
}

// Blocking API: any idle scratch of the replica (a new one if all are busy -- one per concurrent caller).
inline Scratch* acquire(Replica* rep, std::string* err) {
    std::lock_guard<std::mutex> lock(rep->mu);
    if (!rep->idle.empty()) {
        Scratch* sc = rep->idle.back();
        rep->idle.pop_back();
        return sc;
    }
    return new_scratch(rep, nullptr, err);
}
inline void release(Replica* rep, Scratch* sc) {
    std::lock_guard<std::mutex> lock(rep->mu);
    rep->idle.push_back(sc);
}
// Enqueue-only API: the scratch bound to the caller's stream (work on one stream is ordered, so it is reusable).
inline Scratch* scratch_for_stream(Replica* rep, cudaStream_t stream, std::string* err) {
    std::lock_guard<std::mutex> lock(rep->mu);
    auto it = rep->by_stream.find(stream);
    if (it != rep->by_stream.end()) return it->second;
    Scratch* sc = new_scratch(rep, stream, err);
    if (sc) rep->by_stream[stream] = sc;
    return sc;
}

}  // namespace svsb200

struct svsb200_index {
    int dtype = 0, metric = 0, storage = 0;
    size_t n = 0, dim = 0, max_degree = 0;
    uint32_t row_stride = 0, gstride = 0, entry_point = 0;
    float scale = 1.f, bias = 0.f;
    uint32_t lvq_const_offset = 0;
    size_t device_bytes = 0;          // per replica
    uint64_t id_offset = 0;           // added to every 64-bit output id (shard of a larger index)
    uint32_t n_entry = 1;             // entry points (the first one is `entry_point`)
    long cfg_window = 0, cfg_capacity = 0, cfg_visited = 0;   // search parameters of the TOML an index was assembled from
    std::vector<std::unique_ptr<svsb200::Replica>> reps;
    int counting = 0;
    // options
    long warps_per_cta = 0, ctas_per_sm = 0, rows_in_flight = 0, filter_slots = -1, filter_tag16 = 1, no_split = 0;
    long generic_kernel = 0;          // 1: force the generic (round-1) kernel instead of the lean one
    long host_chunks = 0;             // host-buffer searches: pieces per device whose copies overlap the kernels (0 = auto)
    std::mutex mu;
    svsb200::Scratch* last = nullptr; // scratch of the most recent search: counters, kernel time, kernel kind
};

namespace svsb200 {

// Query preparation == distance::maybe_fix_argument for the whole batch (concepts/distance.h:90-130).
enum PrepMode : int {
    PREP_FLOAT = 0,   // float tree: operands converted exactly like the SIMD loads
    PREP_INT = 1,     // exact integer kernels: raw int8/uint8 query
    PREP_SQ_L2 = 2,   // EuclideanCompressed::fix_argument  (scalar.h:75-82)
    PREP_SQ_IP = 3,   // InnerProductCompressed::fix_argument (scalar.h:123-131)
    PREP_SQ_COS = 4,  // CosineSimilarityCompressed::fix_argument (scalar.h:168-171)
    PREP_LVQ_L2 = 5,  // LVQ-8, L2: query with the dataset mean removed (own spec, DESIGN.md §10)
    PREP_LVQ_IP = 6,  // LVQ-8, IP: raw query + <q, mean>
};

// Converts `nq` queries of type `qdtype` on the device into the search kernels' operands: sc->q_f32, sc->q_codes
// (query_stride(dim) apart) and sc->q_aux, enqueued on `stream`.
int prepare_queries(const svsb200_index* ix, const Replica* rep, Scratch* sc, const void* d_queries, int qdtype, size_t nq,
                    int mode, cudaStream_t stream);

// Shared body of every graph-search entry point: everything on one device, enqueued on `stream`.  `exhaustive`
// scans every base row instead of walking the graph.
int search_on_device(svsb200_index* ix, Replica* rep, Scratch* sc, const void* d_queries, int qdtype, size_t nq, size_t k,
                     size_t window, size_t capacity, void* d_out_ids, int id_bytes, float* d_out_dists, cudaStream_t stream,
                     bool exhaustive = false);

}  // namespace svsb200
