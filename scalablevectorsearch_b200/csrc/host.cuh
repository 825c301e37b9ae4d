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

#include <atomic>
#include <map>
#include <memory>
#include <mutex>
#include <string>
#include <unordered_map>
#include <vector>

namespace svsb200 {

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

// A copy of `buf` with room for `want` elements whose first `used` elements are the old ones (no-op if it fits).
template <typename T> cudaError_t grow(DeviceBuffer<T>& buf, size_t used, size_t want) {
    if (want <= buf.count) return cudaSuccess;
    DeviceBuffer<T> bigger;
    cudaError_t e = bigger.ensure(want);
    if (e == cudaSuccess && used) e = cudaMemcpy(bigger.ptr, buf.ptr, used * sizeof(T), cudaMemcpyDeviceToDevice);
    if (e == cudaSuccess) buf = std::move(bigger);   // (the old block goes with `bigger`)
    return e;
}

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
    // filtered flat search, per call: each row's status (Valid = allowed), the allowed rows as a bitmap, their ids
    // compacted (count first), the bias with every other column empty, the gathered rows
    DeviceBuffer<uint32_t> flt_bits, flt_ids, flt_bias;
    DeviceBuffer<unsigned char> flt_status, flt_rows;
    DeviceBuffer<uint32_t> grow_unfinished;            // filtered and range search: queries whose lists must grow
    DeviceBuffer<uint32_t> range_counts;               // range search: results per query
    // host-buffer searches (run_host_search; the queries go in q_raw): the caller's bitmap and the outputs on their way
    // back.  No search body works in these, so a body's own use of the scratch never overwrites them.
    DeviceBuffer<uint32_t> stage_bitmap, stage_per_query;
    DeviceBuffer<uint64_t> stage_ids;
    DeviceBuffer<float> stage_dists;
    DeviceBuffer<uint32_t> dyn_ovf, dyn_qlist;        // dynamic search: overflowed queries, the list being re-run
    DeviceBuffer<uint32_t> point_rows;                 // svsb200_index_distances / _reconstruct: the rows named
    bool dyn_slot_ids = false;                         // dynamic search: write slots, not external ids (filtered / range)
    int (*cancel_fn)(void*) = nullptr;                 // the caller's cancellation predicate while a search runs
    void* cancel_arg = nullptr;
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
    DeviceBuffer<uint8_t> d_status;      // dynamic index: SlotStatus per slot
    DeviceBuffer<uint64_t> d_ext_ids;    // dynamic index: external id per slot
    // tensor-core flat search: the base vectors as warpgroup-MMA tiles + per-row bias, built on first use, one set per
    // operand kind (kept apart: one int8 / uint8 index can be searched with integer queries and with float32 queries)
    struct FlatBase {
        DeviceBuffer<unsigned char> tiles;
        DeviceBuffer<float> bias;            // 8-bit tiles: int32 |x|^2
        DeviceBuffer<float> norms;           // dynamic flat index, fp16 tiles: the norm of every slot's row
    };
    FlatBase flat_f16;                       // fp16 tiles
    DeviceBuffer<unsigned int> flat_xmax;    // ... and the largest norm of their rows
    bool flat_xmax_stale = false;            // dynamic flat index: the Valid slots changed since flat_xmax was taken
    // dynamic indexes: staging of a mutation (the added rows, their slots and ids, and the rows tiled 8 to a tile),
    // kept between calls so that an add or delete allocates -- and synchronises the device -- only when it outgrows them
    struct SlotStaging {
        DeviceBuffer<unsigned char> rows, tiles;
        DeviceBuffer<uint32_t> slots;
        DeviceBuffer<uint64_t> ids;
        DeviceBuffer<float> bias, norms;
    };
    SlotStaging staging;
    FlatBase flat_int;                       // int8 / uint8 tiles of the integer GEMM
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

// The rows of an index that keeps a slot table on its replica (the dynamic Vamana, dynamic flat and dynamic IVF
// indexes) are slots, which a mutation rewrites (after_searches).
inline bool rows_are_slots(const Replica* rep) { return rep->d_ext_ids.ptr != nullptr; }

// One call's hold on a scratch of a replica.  Checkout selects the replica's device first.
class ScratchLease {
  public:
    ScratchLease() = default;
    ScratchLease(const ScratchLease&) = delete;
    ScratchLease& operator=(const ScratchLease&) = delete;
    ScratchLease(ScratchLease&& o) noexcept : rep_(o.rep_), sc_(o.sc_), pooled_(o.pooled_) { o.sc_ = nullptr; }
    ~ScratchLease() {
        if (sc_ && pooled_) release(rep_, sc_);
    }
    // Blocking API: any idle scratch of the replica (a new one if all are busy -- one per concurrent caller), back in
    // the idle list when the lease ends.
    int checkout(Replica* rep) { return take(rep, true, nullptr); }
    // Enqueue-only API: the scratch bound to the caller's stream (NULL: one the replica keeps for that purpose).  Work
    // on one stream is ordered, so the scratch stays bound to it and the lease gives nothing back.
    int checkout(Replica* rep, void* stream) { return take(rep, false, static_cast<cudaStream_t>(stream)); }
    Scratch* get() const { return sc_; }
    Scratch* operator->() const { return sc_; }
    // Runs the search `body(scratch)`.  On an index whose rows are slots it then records the scratch's ev_done on its
    // stream, behind the body's last device write: after_searches waits for that event before a mutation rewrites the
    // rows or their external ids, so every search kind is covered without its body knowing.
    template <typename F> int run(F body) {
        Scratch* sc = sc_;
        if (int rc = body(sc)) return rc;
        if (rows_are_slots(rep_)) CUDA_TRY(cudaEventRecord(sc->ev_done, sc->stream));
        return 0;
    }

  private:
    int take(Replica* rep, bool pooled, cudaStream_t stream) {
        CUDA_TRY(cudaSetDevice(rep->device));
        std::string err;
        Scratch* sc = pooled ? acquire(rep, &err) : scratch_for_stream(rep, stream, &err);
        if (!sc) return fail(err);
        rep_ = rep;
        sc_ = sc;
        pooled_ = pooled;
        return 0;
    }
    static Scratch* acquire(Replica* rep, std::string* err) {
        std::lock_guard<std::mutex> lock(rep->mu);
        if (!rep->idle.empty()) {
            Scratch* sc = rep->idle.back();
            rep->idle.pop_back();
            return sc;
        }
        return new_scratch(rep, nullptr, err);
    }
    static void release(Replica* rep, Scratch* sc) {
        std::lock_guard<std::mutex> lock(rep->mu);
        rep->idle.push_back(sc);
    }
    static Scratch* scratch_for_stream(Replica* rep, cudaStream_t stream, std::string* err) {
        std::lock_guard<std::mutex> lock(rep->mu);
        auto it = rep->by_stream.find(stream);
        if (it != rep->by_stream.end()) return it->second;
        Scratch* sc = new_scratch(rep, stream, err);
        if (sc) rep->by_stream[stream] = sc;
        return sc;
    }
    Replica* rep_ = nullptr;
    Scratch* sc_ = nullptr;
    bool pooled_ = false;
};

// The device form of a search: `body(scratch)` on the scratch bound to the caller's stream, enqueued there.
template <typename F> int run_on_stream(Replica* rep, void* stream, F body) {
    ScratchLease lease;
    if (int rc = lease.checkout(rep, stream)) return rc;
    return lease.run(body);
}

// The buffers of a blocking search over host memory (run_host_search): the queries, the bitmap (NULL: none), k ids and
// distances per query (k = 0: none) and up to three per-query arrays of uint32 (NULL: not wanted).
struct HostBuffers {
    const void* queries = nullptr;
    const uint32_t* bitmap = nullptr;
    uint64_t* ids = nullptr;
    float* dists = nullptr;
    uint32_t* per_query[3] = {};
};
// ... and the same buffers in device memory, as run_host_search hands them to its body: the queries and the bitmap are
// copies the body may rewrite; a per-query array is NULL where the caller wants none.
struct StagedBuffers {
    const void* queries = nullptr;
    uint32_t* bitmap = nullptr;
    uint64_t* ids = nullptr;
    float* dists = nullptr;
    uint32_t* per_query[3] = {};
};

// The blocking form of a search over host buffers, on a scratch of the replica's pool: `query_bytes` of queries and
// `bitmap_words` of bitmap are copied in, `body(scratch, staged)` runs, the nq * k results and the per-query arrays are
// copied out, and the stream is synchronised.  Copies of zero bytes are skipped.
template <typename F>
int run_host_search(Replica* rep, const HostBuffers& host, size_t query_bytes, size_t bitmap_words, size_t nq, size_t k,
                    F body) {
    ScratchLease lease;
    if (int rc = lease.checkout(rep)) return rc;
    Scratch* sc = lease.get();
    const cudaStream_t s = sc->stream;
    const size_t results = nq * k;
    CUDA_TRY(sc->q_raw.ensure(std::max<size_t>(query_bytes, 1)));
    CUDA_TRY(sc->stage_ids.ensure(std::max<size_t>(results, 1)));
    CUDA_TRY(sc->stage_dists.ensure(std::max<size_t>(results, 1)));
    StagedBuffers dev{sc->q_raw.ptr, nullptr, sc->stage_ids.ptr, sc->stage_dists.ptr};
    if (query_bytes) CUDA_TRY(cudaMemcpyAsync(sc->q_raw.ptr, host.queries, query_bytes, cudaMemcpyHostToDevice, s));
    if (host.bitmap) {
        CUDA_TRY(sc->stage_bitmap.ensure(std::max<size_t>(bitmap_words, 1)));
        if (bitmap_words) CUDA_TRY(cudaMemcpyAsync(sc->stage_bitmap.ptr, host.bitmap, bitmap_words * 4, cudaMemcpyHostToDevice, s));
        dev.bitmap = sc->stage_bitmap.ptr;
    }
    for (int i = 0; i < 3; ++i) {
        if (!host.per_query[i]) continue;
        CUDA_TRY(sc->stage_per_query.ensure(3 * nq));
        dev.per_query[i] = sc->stage_per_query.ptr + i * nq;
    }
    if (int rc = lease.run([&](Scratch* scratch) { return body(scratch, dev); })) return rc;
    if (results) {
        CUDA_TRY(cudaMemcpyAsync(host.ids, dev.ids, results * 8, cudaMemcpyDeviceToHost, s));
        CUDA_TRY(cudaMemcpyAsync(host.dists, dev.dists, results * 4, cudaMemcpyDeviceToHost, s));
    }
    for (int i = 0; i < 3; ++i)
        if (host.per_query[i] && nq)
            CUDA_TRY(cudaMemcpyAsync(host.per_query[i], dev.per_query[i], nq * 4, cudaMemcpyDeviceToHost, s));
    CUDA_TRY(cudaStreamSynchronize(s));
    return 0;
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
    // dynamic index (svsb200_dynamic_*, MutableVamanaIndex): slot status and external ids live on the device
    // (Replica::d_status / d_ext_ids) and are mirrored here with the external -> slot translator (slots.h).
    bool dynamic = false;
    svsb200::SlotTable slots;         // also the dynamic flat and dynamic IVF indexes'
    long dyn_slack = -1;              // option "dynamic_slack"
    std::atomic<long> dyn_reruns{0};  // queries re-run with a larger buffer so far
    // dynamic flat index (svsb200_dynamic_flat_*, DynamicFlatIndex): the same slots, statuses Valid / Empty only, and
    // every flat search skips the slots that are not Valid and returns external ids.  `dynamic` stays false.
    bool slot_mask = false;
    // mutation parameters (alpha_, construction_window_size_, max_candidates_, prune_to_)
    float dyn_alpha = 0.f;
    size_t dyn_window = 0, dyn_max_candidates = 0, dyn_prune_to = 0;
};

// A flat index: the rows of an svsb200_index on one device, with no adjacency.  The exact scan walks the rows in blocks
// of deg_pad = round_up(gstride, 32) candidates and reads nothing else of the graph (search_kernel.cuh, EXH); the
// block is 32 rows, as for a Vamana index of degree <= 32.  (flat.cu; the IVF index holds its centroids in one.)
struct svsb200_flat {
    std::unique_ptr<svsb200_index> ix;
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
// The search's distance operator (Op) and query preparation (PrepMode) for `qdtype` queries on this index; fails for a
// query type its search refuses (search.cu).
int choose_op(const svsb200_index* ix, int qdtype, int* op, int* mode);

// Shared body of every graph-search entry point: everything on one device, enqueued on `stream`.  `exhaustive`
// scans every base row instead of walking the graph; with `row_status` (one byte per row, the filtered flat search's)
// it scans only the rows whose byte is SLOT_VALID, which replaces a dynamic flat index's own slot status.
int search_on_device(svsb200_index* ix, Replica* rep, Scratch* sc, const void* d_queries, int qdtype, size_t nq, size_t k,
                     size_t window, size_t capacity, void* d_out_ids, int id_bytes, float* d_out_dists, cudaStream_t stream,
                     bool exhaustive = false, const uint8_t* row_status = nullptr);

// ---- graph construction (build.cu), shared by svsb200_build_vamana and the dynamic index ----
// A float32 / float16 / int8 / uint8 graph (the dynamic index: float32 / float16) on the current device: n rows
// (row_stride apart), adjacency rows (gstride apart, neighbours first, kNoNeighbor padding) and the row lengths, with
// VamanaBuildParameters.
struct GraphBuild {
    int dtype = 0, metric = 0;
    size_t n = 0, dim = 0;
    uint32_t R = 0, gstride = 0, row_stride = 0;
    const void* vectors = nullptr;
    uint32_t* graph = nullptr;
    uint32_t* deg = nullptr;
    size_t window = 0, max_candidates = 0, prune_to = 0;
    float alpha = 1.f;                // forward pruning
    bool sq = false;                  // int8 / uint8 rows are SQ codes of `scale` and `bias` (svsb200_build_vamana_sq)
    float scale = 1.f, bias = 0.f;
    int sm_count = 0;
    cudaStream_t stream = nullptr;
};
// Fails ("<who>: ...") when the builder's search cannot run with these parameters on n rows.
int check_construct(const char* who, const GraphBuild& b);
// VamanaBuilder::construct(reverse_alpha, entry_point, nodes) (vamana_build.h:221-318): one pass over the nodes
// d_slots[0 .. count) (device list; NULL: nodes 0 .. count), in max(40, count / 4096) batches.  Blocking on b.stream.
int construct_graph(const char* who, const GraphBuild& b, float reverse_alpha, uint32_t entry_point, const uint32_t* d_slots,
                    size_t count);
// find_medioid (core/medioid.h:292-350) over the `count` rows whose status is Valid (d_status NULL: all n rows).
int medoid(const GraphBuild& b, const uint8_t* d_status, size_t count, uint32_t* out);
// b.deg[v] = length of adjacency row v, for every row (enqueued on b.stream).
int row_degrees(const GraphBuild& b);

// Slots -> external ids in place, `count` ids (padding ids stay all-ones; search.cu), enqueued on `stream`.
cudaError_t slots_to_external(uint64_t* d_ids, size_t count, const uint64_t* d_ext_ids, cudaStream_t stream);

// ---- mutations of the dynamic Vamana, dynamic flat and dynamic IVF indexes (dynamic.cu, dynamic_flat.cu,
// dynamic_ivf.cu): the device side of their slots (slots.cu; the host side is slots.h) ----
// rep->d_status / d_ext_ids hold the slots of `t`, with room for at least one slot (synchronous).
int upload_slots(Replica* rep, const SlotTable& t);
// The slot capacity an add to `slots` slots needs: 0 when rep->d_status already has room, else a geometric step (many
// small adds do not copy the per-slot arrays each time).
inline size_t slot_capacity(const Replica* rep, size_t slots) {
    const size_t have = rep->d_status.count;
    return slots <= have ? 0 : std::max(slots, 2 * have);
}
// rep->d_ext_ids, then rep->d_status, grown to `cap` slots, the first `used` kept; the new statuses are Empty.
// d_status's size is the capacity every later add checks, so an index grows its own per-slot arrays (rows, adjacency)
// to `cap` before calling this: a failed allocation then leaves the capacity as it was and the next add retries.
int grow_slots(Replica* rep, size_t used, size_t cap, cudaStream_t stream);
// The statuses and external ids after compaction: `ext.size()` Valid slots with external ids `ext`, Empty ones up to
// `cap`, in new buffers (the caller moves them into rep once the stream is drained), enqueued on `stream`.
int compacted_slots(const std::vector<uint64_t>& ext, size_t cap, DeviceBuffer<uint8_t>* status,
                    DeviceBuffer<uint64_t>* ext_ids, cudaStream_t stream);
// rep->d_status[d_slots[i]] = value and, with d_ids, rep->d_ext_ids[d_slots[i]] = d_ids[i], enqueued on `stream`.
cudaError_t mark_slots(const uint32_t* d_slots, const uint64_t* d_ids, size_t count, uint8_t value, Replica* rep,
                       cudaStream_t stream);
// Row dst_pos[i] of `dst` <- row src_pos[i] of `src` (an index array NULL: i; src NULL: no row moves), rows of
// row_stride bytes (a multiple of 16); with `entries`, entry dst_pos[i] <- vals[i] (vals NULL: all-ones).  Enqueued on
// `stream`.
cudaError_t move_rows(const void* src, const uint32_t* src_pos, void* dst, const uint32_t* dst_pos, const uint32_t* vals,
                      uint32_t* entries, size_t count, uint32_t row_stride, cudaStream_t stream);
// Runs a mutation `body(rep, stream)` on a scratch stream of the index's device, once every search of the index
// enqueued so far has finished: a device-buffer search returns with work still queued on the caller's stream (the
// mapping to external ids reads the slots' external ids, the scan reads the rows), and the mutation rewrites them.
// Every search of an index whose rows are slots runs through ScratchLease::run, which records its scratch's ev_done
// at its end -- except svsb200_search_cancellable on a dynamic Vamana index, which holds its leases itself: that search
// records ev_done behind each launch and waits for it (search_dynamic), and its kernel writes the external ids, so
// nothing of the index is read once it returns.
template <typename F> int after_searches(svsb200_index* ix, F body) {
    Replica* rep = ix->reps[0].get();
    CUDA_TRY(cudaSetDevice(rep->device));
    std::vector<cudaEvent_t> searches;
    {
        std::lock_guard<std::mutex> lock(rep->mu);
        for (const auto& sc : rep->all) searches.push_back(sc->ev_done);
    }
    for (cudaEvent_t ev : searches) CUDA_TRY(cudaEventSynchronize(ev));   // (never recorded: returns at once)
    ScratchLease lease;
    if (int rc = lease.checkout(rep)) return rc;
    return body(rep, lease->stream);
}

// ---- flat search (flat.cu), shared by the Flat handle and the dynamic flat index ----
// The device forms, enqueued on the caller's stream: `who` names the entry point in errors, `max_kc` is the deepest
// candidate list allowed.
int flat_search_device(const char* who, svsb200_index* ix, const void* d_queries, int qdtype, size_t nq, size_t k,
                       uint64_t* d_out_ids, float* d_out_dists, void* stream, uint32_t* fallback_queries, uint32_t max_kc);
// The filtered flat search (svsb200_flat_index_search_filtered): `bitmap` over the rows (a dynamic flat index: over
// the slots, Empty slots' bits ignored).
int flat_search_filtered_device(const char* who, svsb200_index* ix, const void* d_queries, int qdtype, size_t nq, size_t k,
                                const uint32_t* d_bitmap, uint64_t* d_out_ids, float* d_out_dists, void* stream,
                                size_t* out_allowed, uint32_t* fallback_queries);
// The blocking forms over host buffers: the same bodies on a scratch of the pool (run_host_search).
int flat_search_host(const char* who, svsb200_index* ix, const void* queries, int qdtype, size_t nq, size_t k,
                     uint64_t* out_ids, float* out_dists, uint32_t max_kc);
int flat_search_filtered_host(const char* who, svsb200_index* ix, const void* queries, int qdtype, size_t nq, size_t k,
                              const uint32_t* bitmap, uint64_t* out_ids, float* out_dists, size_t* out_allowed);
// Deepest list of the Flat handles' searches (k <= 121 on the GEMM).
uint32_t flat_max_kc_deep();
// Incremental upkeep of a dynamic flat index's GEMM operands, for every operand kind already built (nothing before the
// first search builds them), enqueued on `stream`.  Invariant afterwards: every Valid slot's blobs, bias and norm are
// what the full tiling writes for its row; every other row is a padding row (zero blobs, the empty bias).
//   flat_slots_grow:  the slots grow from old_n to new_n: whole 256-row tiles of padding rows behind the kept prefix;
//   flat_slots_place: rows i of the dense `d_rows` (ix->row_stride apart) are now Valid in slots d_slots[i];
//   flat_slots_clear: slots d_slots[i] are no longer Valid;
//   flat_slots_reset: the slots were renumbered (compaction): the tiles are dropped and rebuilt by the next search.
int flat_slots_grow(svsb200_index* ix, Replica* rep, size_t old_n, size_t new_n, cudaStream_t stream);
int flat_slots_place(svsb200_index* ix, Replica* rep, const void* d_rows, const uint32_t* d_slots, uint32_t count,
                     cudaStream_t stream);
int flat_slots_clear(svsb200_index* ix, Replica* rep, const uint32_t* d_slots, uint32_t count, cudaStream_t stream);
void flat_slots_reset(Replica* rep);

}  // namespace svsb200
