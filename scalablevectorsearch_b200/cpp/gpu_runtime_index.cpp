// gpu_runtime_index.cpp -- the FAISS-facing runtime ABI of the reference (SURVEY.md §8 f4), backed by libsvsb200.
//
// Implements `svs::runtime::v0::VamanaIndex` (bindings/cpp/include/svs/runtime/vamana_index.h:61-143) for the
// uncompressed storage kinds (FP32, FP16) and SQI8 on the GPU: `build` + `add` construct the graph with
// svsb200_build_vamana, `search` is the batched GPU search (optionally through an IDFilter evaluated on the device as a
// bitmap), `range_search` grows the result lists until they leave the radius.  SQI8 follows the reference's
// VamanaIndexImpl (vamana_index_impl.h:413-450): the first `add` compresses its float32 rows to int8 codes with one
// global scale and bias (svsb200_sq_compress; constant rows, or rows holding a NaN or an infinity, are a RUNTIME_ERROR)
// and builds the graph over the codes (svsb200_build_vamana_sq); the searches run the SQ search, `reconstruct_at`
// decompresses (scale * c + bias, the reference's DecompressionAccessor) and the host keeps the codes only.  It stands where the reference's
// libsvs_runtime implementation sits (bindings/cpp/src/vamana_index.cpp, vamana_index_impl.h:60-330): a program
// written against the runtime header links this object instead and runs on the H100.
//
// Compiles against the reference's runtime *headers* only (no svs core headers); the few out-of-line members of the
// header types that live in libsvs_runtime (Status message storage, the VamanaIndex destructor / static factories)
// are defined here.  save / load / LeanVec are the reference's CPU territory: NOT_IMPLEMENTED.
//
// It also implements `svs::runtime::v0::FlatIndex` (bindings/cpp/include/svs/runtime/flat_index.h) on the graph-free
// flat index of libsvsb200 (svsb200_flat_index_*), with the behaviour of the reference's FlatIndexImpl
// (bindings/cpp/src/flat_index_impl.h, flat_index.cpp): FP32 storage only, the first `add` creates the index and a
// second one is NOT_IMPLEMENTED, a search before it is NOT_INITIALIZED with labels -1 and distances +inf, k = 0 is
// INVALID_ARGUMENT.  Divergence: k > 1024 is INVALID_ARGUMENT (the GPU search returns at most 1024 neighbours).
//
// And `svs::runtime::v0::IVFIndex` (bindings/cpp/include/svs/runtime/ivf_index.h) on the IVF index of libsvsb200
// (svsb200_ivf_*) for FP32, FP16 and SQI8 storage: `build` clusters (svsb200_ivf_cluster, or
// svsb200_ivf_cluster_hierarchical when is_hierarchical is enabled) and assembles the index,
// `search` probes n_probes clusters (the build's default search parameters, overridden per call).  SQI8 follows the
// reference's init_impl: the float32 rows are clustered, then compressed to int8 (svsb200_sq_compress), then assembled
// with the clustering's assignments (svsb200_ivf_create_sq); data that cannot be compressed (constant, or holding a
// NaN or an infinity) is a RUNTIME_ERROR.  save / load, LeanVec and the other storage kinds are NOT_IMPLEMENTED;
// an unspecified is_hierarchical keeps the flat k-means, and the other unspecified build parameters take the Python
// IVFBuildParameters' defaults.  A non-null IDFilter becomes a bitmap over the ids (is_member(i) for every id) for
// svsb200_ivf_search_filtered, whose probe count grows per query until k allowed rows are in reach; filter_stop and
// filter_estimate_batch are honoured as described at filtered_search below.
//
// And `svs::runtime::v0::DynamicIVFIndex` (bindings/cpp/include/svs/runtime/dynamic_ivf_index.h) on the dynamic IVF
// index (svsb200_dynamic_ivf_*) for FP32, FP16 and SQI8 storage, with the behaviour of the reference's
// DynamicIVFIndexImpl (bindings/cpp/src/dynamic_ivf_index_impl.h): `build` with rows clusters (and for SQI8
// compresses) them as IVFIndex::build does and assembles the index; without rows there is no index until the first
// `add`, which clusters its own rows (and fixes the SQ scale and bias from them); a later SQI8 `add` passes its float32
// rows through, to be encoded with that scale and bias; before initialisation, `search`
// is NOT_INITIALIZED (labels -1, distances +inf), `remove` / `remove_selected` / `consolidate` / `compact` are
// NOT_INITIALIZED and `has_id` is false.  k = 0 is INVALID_ARGUMENT; save / load and LeanVec are NOT_IMPLEMENTED.  A
// non-null IDFilter becomes a bitmap over the slots (is_member(external id) for every Valid slot) for
// svsb200_dynamic_ivf_search_filtered, with IVFIndex's filter_stop and filter_estimate_batch.
//
// And `svs::runtime::v0::DynamicVamanaIndex` (bindings/cpp/include/svs/runtime/dynamic_vamana_index.h) on the dynamic
// Vamana index (svsb200_dynamic_*) for FP32, FP16 and SQI8 storage, with the behaviour of the reference's
// DynamicVamanaIndexImpl (bindings/cpp/src/dynamic_vamana_index_impl.h): the first `add` builds the index, `remove`
// consolidates and compacts once the soft deletions exceed half of the ids left, and `get_distance` / `reconstruct_at`
// read the rows on the device (svsb200_index_distances / _reconstruct), so no host copy is kept.  The GPU storage is not
// blocked: `blocksize_bytes` reports the block size the parameters ask for.  use_full_search_history = false is ignored
// (the GPU builder always keeps the full history).  save / load and LeanVec are NOT_IMPLEMENTED.
#include "svs/runtime/dynamic_ivf_index.h"
#include "svs/runtime/dynamic_vamana_index.h"
#include "svs/runtime/flat_index.h"
#include "svs/runtime/ivf_index.h"
#include "svs/runtime/vamana_index.h"

#include "svsb200.h"

#include <cmath>
#include <cstring>
#include <memory>
#include <new>
#include <random>
#include <vector>

namespace svs {
namespace runtime {
SVS_DECLARE_NAMESPACE_VERSION(0) {

// ---- out-of-line members of header types (bindings/cpp/src/api_defs.cpp:24-44) ----
void Status::store_message(const char* msg) noexcept {
    const size_t len = std::strlen(msg);
    message_storage_ = new (std::nothrow) char[len + 1];
    if (message_storage_) std::memcpy(message_storage_, msg, len + 1);
}
void Status::destroy_message() noexcept {
    delete[] message_storage_;
    message_storage_ = nullptr;
}

VamanaIndex::~VamanaIndex() = default;
FlatIndex::~FlatIndex() = default;
IVFIndex::~IVFIndex() = default;

namespace {

Status gpu_error() { return Status(ErrorCode::RUNTIME_ERROR, svsb200_last_error()); }

// The search window and buffer capacity of a Vamana search: the index's default search parameters (window 10 when
// unspecified), overridden by the call's, the window at least k and the capacity at least the window.
void window_of(const VamanaIndex::SearchParams& defaults, const VamanaIndex::SearchParams* params, size_t k, size_t& window,
               size_t& capacity) {
    window = is_specified(defaults.search_window_size) ? defaults.search_window_size : 10;
    capacity = is_specified(defaults.search_buffer_capacity) ? defaults.search_buffer_capacity : 0;
    if (params) {
        set_if_specified(window, params->search_window_size);
        set_if_specified(capacity, params->search_buffer_capacity);
    }
    window = window < k ? k : window;
    capacity = capacity < window ? window : capacity;
}

// float -> IEEE binary16, round to nearest even (FP16 storage)
uint16_t to_half(float f) {
    uint32_t x;
    std::memcpy(&x, &f, 4);
    const uint32_t sign = (x >> 16) & 0x8000u, ax = x & 0x7FFFFFFFu;
    if (ax >= 0x7F800000u) return uint16_t(sign | 0x7C00u | (ax > 0x7F800000u ? 0x200u : 0u));
    if (ax >= 0x477FF000u) return uint16_t(sign | 0x7C00u);   // rounds to >= 65520: inf
    if (ax < 0x38800000u) {                                    // below 2^-14: subnormal half
        const float v = std::fabs(f) * 16777216.0f;            // exact scaling by 2^24
        return uint16_t(sign | uint32_t(std::nearbyint(v)));
    }
    const uint32_t mant = ax & 0x7FFFFFu, exp = (ax >> 23) - 112;
    uint32_t h = (exp << 10) | (mant >> 13);
    const uint32_t rest = mant & 0x1FFFu;
    if (rest > 0x1000u || (rest == 0x1000u && (h & 1u))) ++h;
    return uint16_t(sign | h);
}

// IEEE binary16 -> float, exact (subnormals included)
float from_half(uint16_t h) {
    const uint32_t sign = uint32_t(h & 0x8000u) << 16, e = (h >> 10) & 0x1F, m = h & 0x3FFu;
    uint32_t x;
    if (e == 0) {
        if (m == 0) x = sign;
        else {
            int s = 0;
            uint32_t mm = m;
            while (!(mm & 0x400u)) {
                mm <<= 1;
                ++s;
            }
            x = sign | ((127 - 15 - s + 1) << 23) | ((mm & 0x3FFu) << 13);
        }
    } else if (e == 31) x = sign | 0x7F800000u | (m << 13);
    else x = sign | ((e - 15 + 127) << 23) | (m << 13);
    float f;
    std::memcpy(&f, &x, 4);
    return f;
}


class GpuVamanaIndex final : public VamanaIndex {
  public:
    GpuVamanaIndex(size_t dim, MetricType metric, StorageKind kind, const BuildParams& bp, const SearchParams& sp)
        : dim_(dim), metric_(metric), kind_(kind), bp_(bp), sp_(sp) {}
    ~GpuVamanaIndex() override { svsb200_index_destroy(index_); }

    // vamana_index_impl.h:92-107: the first `add` builds the (static) index, later ones are rejected
    Status add(size_t n, const float* x) noexcept override {
        if (index_) return Status(ErrorCode::INVALID_ARGUMENT, "Vamana index does not support adding points after initialization");
        if (n == 0 || !x) return Status(ErrorCode::INVALID_ARGUMENT, "no data");
        try {
            const int metric = metric_ == MetricType::L2 ? SVSB200_L2 : SVSB200_IP;
            const size_t R = is_specified(bp_.graph_max_degree) ? bp_.graph_max_degree : 32;
            const size_t window = is_specified(bp_.construction_window_size) ? bp_.construction_window_size : 200;
            const float alpha = is_specified(bp_.alpha) ? bp_.alpha : 0.f;
            const size_t pool = is_specified(bp_.max_candidate_pool_size) ? bp_.max_candidate_pool_size : 0;
            const size_t prune_to = is_specified(bp_.prune_to) ? bp_.prune_to : 0;
            std::vector<uint32_t> graph(n * (R + 1));
            uint32_t ep = 0;
            if (kind_ == StorageKind::SQI8) {   // int8 codes with one global scale and bias (vamana_index_impl.h:413-450)
                std::vector<int8_t> codes(n * dim_);
                float sq[2] = {0.f, 0.f};
                if (svsb200_sq_compress(x, n, dim_, SVSB200_I8, 0, codes.data(), &sq[0], &sq[1]) ||
                    svsb200_build_vamana_sq(codes.data(), SVSB200_I8, n, dim_, metric, sq[0], sq[1], alpha, R, window, pool,
                                            prune_to, 0, graph.data(), &ep) ||
                    svsb200_index_create(codes.data(), SVSB200_I8, n, dim_, 0, graph.data(), R + 1, ep, metric, SVSB200_SQ,
                                         sq, 0, &index_))
                    return gpu_error();
                codes_ = std::move(codes);
                scale_ = sq[0];
                bias_ = sq[1];
                n_ = n;
                graph_bytes_ = graph.size() * 4;
                return Status_Ok;
            }
            data_.assign(x, x + n * dim_);
            const void* rows = data_.data();
            int dtype = SVSB200_F32;
            if (kind_ == StorageKind::FP16) {   // stored as float16, like the reference's FP16 storage kind
                half_.resize(n * dim_);
                for (size_t i = 0; i < n * dim_; ++i) half_[i] = to_half(data_[i]);
                rows = half_.data();
                dtype = SVSB200_F16;
            }
            if (svsb200_build_vamana(rows, dtype, n, dim_, 0, metric, alpha, R, window, pool, prune_to, 0, graph.data(), &ep))
                return gpu_error();
            if (svsb200_index_create(rows, dtype, n, dim_, 0, graph.data(), R + 1, ep, metric, SVSB200_PLAIN, nullptr, 0, &index_))
                return gpu_error();
            n_ = n;
            graph_bytes_ = graph.size() * 4;
        } catch (const std::exception& e) {
            return Status(ErrorCode::RUNTIME_ERROR, e.what());
        }
        return Status_Ok;
    }

    Status reset() noexcept override {
        svsb200_index_destroy(index_);
        index_ = nullptr;
        data_.clear();
        half_.clear();
        codes_.clear();
        n_ = 0;
        return Status_Ok;
    }

    Status search(size_t n, const float* x, size_t k, float* distances, size_t* labels, const SearchParams* params,
                  IDFilter* filter) const noexcept override {
        if (!index_) return Status(ErrorCode::NOT_INITIALIZED, "Index not initialized");
        if (n == 0) return Status_Ok;
        if (k == 0) return Status(ErrorCode::INVALID_ARGUMENT, "k must be greater than 0");
        size_t window = 0, capacity = 0;
        window_of(sp_, params, k, window, capacity);
        static_assert(sizeof(size_t) == 8, "labels are 64-bit");
        if (!filter) {
            if (svsb200_search(index_, x, SVSB200_F32, n, k, window, capacity, 0, labels, 8, distances, nullptr)) return gpu_error();
            return Status_Ok;
        }
        try {   // IDFilter -> bitmap, evaluated on the device (vamana_index_impl.h:139-218 filters on the host)
            std::vector<uint32_t> bitmap((n_ + 31) / 32, 0u);
            for (size_t i = 0; i < n_; ++i)
                if (filter->is_member(i)) bitmap[i >> 5] |= 1u << (i & 31);
            if (svsb200_search_filtered(index_, x, SVSB200_F32, n, k, window, bitmap.data(),
                                        reinterpret_cast<uint64_t*>(labels), distances, nullptr))
                return gpu_error();
        } catch (const std::exception& e) {
            return Status(ErrorCode::RUNTIME_ERROR, e.what());
        }
        return Status_Ok;
    }

    Status range_search(size_t n, const float* x, float radius, const ResultsAllocator& results, const SearchParams* params,
                        IDFilter* filter) const noexcept override {
        if (!index_) return Status(ErrorCode::NOT_INITIALIZED, "Index not initialized");
        if (n == 0) return Status_Ok;
        size_t window = 0, capacity = 0;
        window_of(sp_, params, 10, window, capacity);
        try {
            std::vector<uint32_t> counts(n);
            uint64_t* ids = nullptr;
            float* dd = nullptr;
            if (svsb200_range_search(index_, x, SVSB200_F32, n, radius, window, counts.data(), &ids, &dd)) return gpu_error();
            std::unique_ptr<uint64_t, void (*)(void*)> ids_guard(ids, svsb200_free);
            std::unique_ptr<float, void (*)(void*)> dd_guard(dd, svsb200_free);
            std::vector<size_t> kept(n, 0);
            std::vector<size_t> offs(n + 1, 0);
            for (size_t q = 0; q < n; ++q) offs[q + 1] = offs[q] + counts[q];
            for (size_t q = 0; q < n; ++q)
                for (size_t j = offs[q]; j < offs[q + 1]; ++j)
                    if (!filter || filter->is_member(ids[j])) ++kept[q];
            SearchResultsStorage out = results.allocate(std::span<size_t>(kept.data(), kept.size()));
            size_t o = 0;
            for (size_t q = 0; q < n; ++q)
                for (size_t j = offs[q]; j < offs[q + 1]; ++j)
                    if (!filter || filter->is_member(ids[j])) {
                        out.labels[o] = ids[j];
                        out.distances[o] = dd[j];
                        ++o;
                    }
        } catch (const std::exception& e) {
            return Status(ErrorCode::RUNTIME_ERROR, e.what());
        }
        return Status_Ok;
    }

    Status get_distance(size_t id, const float* query, float* distance) const noexcept override {
        if (!index_) return Status(ErrorCode::NOT_INITIALIZED, "Index not initialized");
        if (id >= n_) return Status(ErrorCode::INVALID_ARGUMENT, "id out of range");
        // one stored vector against one query: the top-1 of a one-element filter is its exact distance
        std::vector<uint32_t> bitmap((n_ + 31) / 32, 0u);
        bitmap[id >> 5] = 1u << (id & 31);
        uint64_t label = 0;
        uint32_t found = 0;
        if (svsb200_search_filtered(index_, query, SVSB200_F32, 1, 1, n_ < 4096 ? n_ : 4096, bitmap.data(), &label, distance, &found))
            return gpu_error();
        if (!found && kind_ == StorageKind::SQI8) {   // not reached by the graph walk: the query-side compressed distance
            *distance = sq_distance(query, &codes_[id * dim_]);
        } else if (!found) {   // not reached by the graph walk: plain arithmetic on the host copy
            float acc = 0.f;
            for (size_t i = 0; i < dim_; ++i) {
                const float v = kind_ == StorageKind::FP16 ? from_half(half_[id * dim_ + i]) : data_[id * dim_ + i];
                acc += metric_ == MetricType::L2 ? (query[i] - v) * (query[i] - v) : query[i] * v;
            }
            *distance = acc;
        }
        return Status_Ok;
    }

    Status reconstruct_at(size_t n, const size_t* ids, float* output) noexcept override {
        for (size_t i = 0; i < n; ++i) {
            if (ids[i] >= n_) return Status(ErrorCode::INVALID_ARGUMENT, "id out of range");
            for (size_t d = 0; d < dim_; ++d)
                output[i * dim_ + d] = kind_ == StorageKind::SQI8   ? decompress(codes_[ids[i] * dim_ + d])
                                       : kind_ == StorageKind::FP16 ? from_half(half_[ids[i] * dim_ + d])
                                                                    : data_[ids[i] * dim_ + d];
        }
        return Status_Ok;
    }

    size_t get_memory_usage() const noexcept override { return index_ ? svsb200_index_device_bytes(index_) : 0; }
    Status get_memory_breakdown(MemoryBreakdown* out) const noexcept override {
        if (!out) return Status(ErrorCode::INVALID_ARGUMENT, "null output");
        out->graph_bytes = graph_bytes_;
        out->data_bytes = index_ ? svsb200_index_device_bytes(index_) - graph_bytes_ : 0;
        out->metadata_bytes = 0;
        return Status_Ok;
    }
    Status save(std::ostream&) const noexcept override {
        return Status(ErrorCode::NOT_IMPLEMENTED, "save stays on the reference's CPU index (index/vamana/index.h:825-854)");
    }

  private:
    // DecompressionAccessor (quantization/scalar/scalar.h:606-620): scale * c + bias, two roundings
    float decompress(int8_t c) const {
        const float scaled = scale_ * float(c);
        return scaled + bias_;
    }
    // The SQ search's distance of a float32 query to one row of codes (EuclideanCompressed / InnerProductCompressed,
    // quantization/scalar/scalar.h:58-153): L2 compresses the query and scales the integer L2 by scale^2; MIP is
    // scale * <q, c> + bias * sum(q).  The sums run in order (the device's MIP tree may round differently).
    float sq_distance(const float* q, const int8_t* c) const {
        if (metric_ == MetricType::L2) {
            int64_t l2 = 0;
            for (size_t i = 0; i < dim_; ++i) {
                float r = std::round((q[i] - bias_) / scale_);   // detail::compress
                r = r < -128.f ? -128.f : r > 127.f ? 127.f : r;
                const int64_t diff = int64_t(r) - int64_t(c[i]);
                l2 += diff * diff;
            }
            return (scale_ * scale_) * float(int32_t(l2));
        }
        float ip = 0.f, sum = 0.f;
        for (size_t i = 0; i < dim_; ++i) {
            ip += q[i] * float(c[i]);
            sum += q[i];
        }
        return scale_ * ip + bias_ * sum;
    }
    size_t dim_, n_ = 0, graph_bytes_ = 0;
    MetricType metric_;
    StorageKind kind_;
    BuildParams bp_;
    SearchParams sp_;
    std::vector<float> data_;
    std::vector<uint16_t> half_;
    std::vector<int8_t> codes_;   // SQI8: the codes, scale_ and bias_
    float scale_ = 1.f, bias_ = 0.f;
    svsb200_index* index_ = nullptr;
};

}  // namespace

Status VamanaIndex::check_storage_kind(StorageKind kind) noexcept {
    return kind == StorageKind::FP32 || kind == StorageKind::FP16 || kind == StorageKind::SQI8
               ? Status_Ok
               : Status(ErrorCode::NOT_IMPLEMENTED, "the GPU runtime holds FP32 / FP16 / SQI8 storage (LVQ and LeanVec: reference CPU library)");
}

Status VamanaIndex::build(VamanaIndex** index, size_t dim, MetricType metric, StorageKind storage_kind, const BuildParams& params,
                          const SearchParams& default_search_params) noexcept {
    if (!index) return Status(ErrorCode::INVALID_ARGUMENT, "null output");
    *index = nullptr;
    Status st = check_storage_kind(storage_kind);
    if (!st.ok()) return st;
    if (dim == 0) return Status(ErrorCode::INVALID_ARGUMENT, "dim must be positive");
    *index = new (std::nothrow) GpuVamanaIndex(dim, metric, storage_kind, params, default_search_params);
    return *index ? Status_Ok : Status(ErrorCode::RUNTIME_ERROR, "out of memory");
}

Status VamanaIndex::destroy(VamanaIndex* index) noexcept {
    delete index;
    return Status_Ok;
}

Status VamanaIndex::load(VamanaIndex** index, std::istream&, MetricType, StorageKind) noexcept {
    if (index) *index = nullptr;
    return Status(ErrorCode::NOT_IMPLEMENTED, "load stays on the reference's CPU library");
}
Status VamanaIndex::map_to_file(VamanaIndex** index, const char*, MetricType, StorageKind) noexcept {
    if (index) *index = nullptr;
    return Status(ErrorCode::NOT_IMPLEMENTED, "map_to_file stays on the reference's CPU library");
}
Status VamanaIndex::map_to_memory(VamanaIndex** index, void*, size_t, MetricType, StorageKind, size_t*) noexcept {
    if (index) *index = nullptr;
    return Status(ErrorCode::NOT_IMPLEMENTED, "map_to_memory stays on the reference's CPU library");
}

// ---- FlatIndex ----
namespace {

class GpuFlatIndex final : public FlatIndex {
  public:
    GpuFlatIndex(size_t dim, MetricType metric) : dim_(dim), metric_(metric) {}
    ~GpuFlatIndex() override { svsb200_flat_index_destroy(index_); }

    // flat_index_impl.h: the first `add` creates the index, later ones are rejected
    Status add(size_t n, const float* x) noexcept override {
        if (index_) return Status(ErrorCode::NOT_IMPLEMENTED, "Flat index does not support adding points after initialization");
        if (n == 0 || !x) return Status(ErrorCode::INVALID_ARGUMENT, "no data");
        const int metric = metric_ == MetricType::L2 ? SVSB200_L2 : SVSB200_IP;
        if (svsb200_flat_index_create(x, SVSB200_F32, n, dim_, 0, metric, 0, &index_)) return gpu_error();
        return Status_Ok;
    }

    Status search(size_t n, const float* x, size_t k, float* distances, size_t* labels) const noexcept override {
        if (!index_) {
            for (size_t i = 0; i < n * k; ++i) {
                distances[i] = INFINITY;
                labels[i] = static_cast<size_t>(-1);
            }
            return Status(ErrorCode::NOT_INITIALIZED, "Index not initialized");
        }
        if (k == 0) return Status(ErrorCode::INVALID_ARGUMENT, "k must be greater than 0");
        if (k > 1024) return Status(ErrorCode::INVALID_ARGUMENT, "k must be at most 1024 on the GPU");
        if (n == 0) return Status_Ok;
        static_assert(sizeof(size_t) == 8, "labels are 64-bit");
        if (svsb200_flat_index_search(index_, x, SVSB200_F32, n, k, reinterpret_cast<uint64_t*>(labels), distances))
            return gpu_error();
        return Status_Ok;
    }

    Status reset() noexcept override {
        svsb200_flat_index_destroy(index_);
        index_ = nullptr;
        return Status_Ok;
    }

    Status save(std::ostream&) const noexcept override {
        return Status(ErrorCode::NOT_IMPLEMENTED, "save stays on the reference's CPU index (index/flat/flat.h)");
    }

  private:
    size_t dim_;
    MetricType metric_;
    svsb200_flat* index_ = nullptr;
};

}  // namespace

Status FlatIndex::check_storage_kind(StorageKind kind) noexcept {
    return kind == StorageKind::FP32 ? Status_Ok
                                     : Status(ErrorCode::INVALID_ARGUMENT, "FlatIndex only supports FP32 storage kind");
}

Status FlatIndex::build(FlatIndex** index, size_t dim, MetricType metric) noexcept {
    if (!index) return Status(ErrorCode::INVALID_ARGUMENT, "null output");
    *index = nullptr;
    if (dim == 0) return Status(ErrorCode::INVALID_ARGUMENT, "dim must be positive");
    *index = new (std::nothrow) GpuFlatIndex(dim, metric);
    return *index ? Status_Ok : Status(ErrorCode::RUNTIME_ERROR, "out of memory");
}

Status FlatIndex::destroy(FlatIndex* index) noexcept {
    delete index;
    return Status_Ok;
}

Status FlatIndex::load(FlatIndex** index, std::istream&, MetricType) noexcept {
    if (index) *index = nullptr;
    return Status(ErrorCode::NOT_IMPLEMENTED, "load stays on the reference's CPU library");
}
Status FlatIndex::map_to_file(FlatIndex** index, const char*, MetricType) noexcept {
    if (index) *index = nullptr;
    return Status(ErrorCode::NOT_IMPLEMENTED, "map_to_file stays on the reference's CPU library");
}
Status FlatIndex::map_to_memory(FlatIndex** index, void*, size_t, MetricType, size_t* read_bytes) noexcept {
    if (index) *index = nullptr;
    if (read_bytes) *read_bytes = 0;
    return Status(ErrorCode::NOT_IMPLEMENTED, "map_to_memory stays on the reference's CPU library");
}

// ---- IVFIndex ----
namespace {

// Filtered IVF search.  As the reference's IVF runtime classes do (ivf_index_impl.h, dynamic_ivf_index_impl.h), two
// search parameters let a caller give up on a filter that lets too little through, so that it can fall back to an
// exact search: filter_stop (unspecified: 0, never give up) and filter_estimate_batch (unspecified: true).
//   * Estimate: with filter_estimate_batch, max(200, int(1 / filter_stop)) ids (at most the index's size) are drawn
//     uniformly from [0, size) with std::mt19937(42), at most four times as many draws, skipping ids the index does not
//     hold (dynamic index); when none of them or a fraction below filter_stop passes the filter, every row is padded.
//   * Per query: a query whose probed clusters hold allowed / rows < filter_stop (no allowed row included) gets a padded
//     row.  The reference divides by the candidates its iterator has yielded so far instead: a documented divergence.
// Padded rows are labels SIZE_MAX, distances +inf, and the status stays OK.
struct FilterStop {
    float stop = 0.0f;
    bool estimate = true;
};

template <typename SearchParams> FilterStop filter_stop_of(const SearchParams& sp, const SearchParams* params) {
    FilterStop fs;
    if (is_specified(sp.filter_stop)) fs.stop = sp.filter_stop;
    if (is_specified(sp.filter_estimate_batch)) fs.estimate = sp.filter_estimate_batch.is_enabled();
    if (params && is_specified(params->filter_stop)) fs.stop = params->filter_stop;
    if (params && is_specified(params->filter_estimate_batch)) fs.estimate = params->filter_estimate_batch.is_enabled();
    return fs;
}

// The estimate: true when the sampled ids say give up.  `held(id)` skips ids the index does not hold.
template <typename Held> bool sample_says_stop(const IDFilter& filter, size_t size, float stop, Held held) {
    if (!(stop > 0.0f) || size == 0) return false;
    const size_t want = std::min(std::max<size_t>(200, size_t(1.0f / stop)), size);
    std::mt19937 rng(42);
    std::uniform_int_distribution<size_t> draw(0, size - 1);
    size_t checked = 0, hits = 0;
    for (size_t tries = 0; checked < want && tries < 4 * want; ++tries) {
        const size_t id = draw(rng);
        if (!held(id)) continue;
        ++checked;
        if (filter.is_member(id)) ++hits;
    }
    return checked > 0 && (hits == 0 || float(hits) / float(checked) < stop);
}

void pad_rows(size_t from, size_t to, size_t k, float* distances, size_t* labels) {
    for (size_t i = from * k; i < to * k; ++i) {
        labels[i] = SIZE_MAX;
        distances[i] = INFINITY;
    }
}

// Runs `search(probes, allowed, rows)` (a filtered search writing labels and distances) and pads the rows of the
// queries below filter_stop.
template <typename Search>
Status filtered_search(size_t n, size_t k, float* distances, size_t* labels, float stop, Search search) {
    std::vector<uint32_t> probes(n), allowed(n), rows(n);
    if (search(probes.data(), allowed.data(), rows.data())) return gpu_error();
    if (stop > 0.0f)
        for (size_t q = 0; q < n; ++q)
            if (allowed[q] == 0 || float(allowed[q]) / float(rows[q]) < stop) pad_rows(q, q + 1, k, distances, labels);
    return Status_Ok;
}

class GpuIVFIndex final : public IVFIndex {
  public:
    GpuIVFIndex(svsb200_ivf* index, const SearchParams& sp, size_t threads, size_t intra)
        : index_(index), sp_(sp), threads_(threads), intra_(intra) {}
    ~GpuIVFIndex() override { svsb200_ivf_destroy(index_); }

    Status search(size_t n, const float* x, size_t k, float* distances, size_t* labels, const SearchParams* params,
                  IDFilter* filter) const noexcept override {
        if (k == 0) return Status(ErrorCode::INVALID_ARGUMENT, "k must be greater than 0");
        if (n == 0) return Status_Ok;
        size_t n_probes = is_specified(sp_.n_probes) ? sp_.n_probes : 1;
        float k_reorder = is_specified(sp_.k_reorder) ? sp_.k_reorder : 1.0f;
        if (params && is_specified(params->n_probes)) n_probes = params->n_probes;
        if (params && is_specified(params->k_reorder)) k_reorder = params->k_reorder;
        if (!(k_reorder >= 1.0f)) return Status(ErrorCode::INVALID_ARGUMENT, "k_reorder must be at least 1");
        static_assert(sizeof(size_t) == 8, "labels are 64-bit");
        if (filter) {
            const FilterStop fs = filter_stop_of(sp_, params);
            const size_t size = svsb200_ivf_size(index_);
            if (fs.estimate && sample_says_stop(*filter, size, fs.stop, [](size_t) { return true; })) {
                pad_rows(0, n, k, distances, labels);
                return Status_Ok;
            }
            try {
                std::vector<uint32_t> bitmap((size + 31) / 32, 0u);   // bit i: id i
                for (size_t i = 0; i < size; ++i)
                    if (filter->is_member(i)) bitmap[i >> 5] |= 1u << (i & 31);
                return filtered_search(n, k, distances, labels, fs.stop, [&](uint32_t* p, uint32_t* a, uint32_t* r) {
                    return svsb200_ivf_search_filtered(index_, x, SVSB200_F32, n, k, n_probes, bitmap.data(),
                                                       reinterpret_cast<uint64_t*>(labels), distances, p, a, r);
                });
            } catch (...) {
                return Status(ErrorCode::RUNTIME_ERROR, "out of memory");
            }
        }
        if (svsb200_ivf_search(index_, x, SVSB200_F32, n, k, n_probes, reinterpret_cast<uint64_t*>(labels), distances))
            return gpu_error();
        return Status_Ok;
    }
    Status save(std::ostream&) const noexcept override {
        return Status(ErrorCode::NOT_IMPLEMENTED, "save stays on the reference's CPU index");
    }
    Status set_num_threads(size_t n) noexcept override {
        threads_ = n;
        return Status_Ok;
    }
    Status get_num_threads(size_t* n) const noexcept override {
        if (n) *n = threads_;
        return Status_Ok;
    }
    Status set_intra_query_threads(size_t n) noexcept override {
        intra_ = n;
        return Status_Ok;
    }
    Status get_intra_query_threads(size_t* n) const noexcept override {
        if (n) *n = intra_;
        return Status_Ok;
    }

  private:
    svsb200_ivf* index_;
    SearchParams sp_;
    size_t threads_, intra_;
};

// Clusters n rows for IVFIndex / DynamicIVFIndex::build, unspecified parameters taking the Python defaults:
// svsb200_ivf_cluster_hierarchical when is_hierarchical is enabled (level-1 groups: hierarchical_level1_clusters, the
// square root of C when unspecified), else the flat svsb200_ivf_cluster.  Returns non-zero on a library error.
int cluster_rows(const IVFIndex::BuildParams& params, const void* rows, int dtype, size_t n, size_t dim, int metric, size_t C,
                 float* centroids, uint32_t* assignments) {
    const size_t minibatch = is_specified(params.minibatch_size) ? params.minibatch_size : 10000;
    const size_t iters = is_specified(params.num_iterations) ? params.num_iterations : 10;
    const float frac = is_specified(params.training_fraction) ? params.training_fraction : 0.1f;
    const size_t seed = is_specified(params.seed) ? params.seed : 0xC0FFEE;
    if (params.is_hierarchical.is_enabled()) {
        const size_t l1 = is_specified(params.hierarchical_level1_clusters) ? params.hierarchical_level1_clusters : 0;
        return svsb200_ivf_cluster_hierarchical(rows, dtype, n, dim, metric, C, l1, minibatch, iters, frac, seed, 0, centroids,
                                                assignments, nullptr);
    }
    return svsb200_ivf_cluster(rows, dtype, n, dim, metric, C, minibatch, iters, 0, frac, seed, 0, centroids, assignments);
}

}  // namespace

Status IVFIndex::check_storage_kind(StorageKind kind) noexcept {
    return kind == StorageKind::FP32 || kind == StorageKind::FP16 || kind == StorageKind::SQI8
               ? Status_Ok
               : Status(ErrorCode::NOT_IMPLEMENTED, "IVFIndex on the GPU supports FP32, FP16 and SQI8 storage only");
}

Status IVFIndex::build(IVFIndex** index, size_t dim, MetricType metric, StorageKind storage_kind, size_t n, const float* data,
                       const BuildParams& params, const SearchParams& default_search_params, size_t num_threads,
                       size_t intra_query_threads) noexcept {
    if (!index) return Status(ErrorCode::INVALID_ARGUMENT, "null output");
    *index = nullptr;
    if (Status st = check_storage_kind(storage_kind); !st.ok()) return st;
    if (dim == 0 || n == 0 || !data) return Status(ErrorCode::INVALID_ARGUMENT, "no data");
    try {
        const size_t C = is_specified(params.num_centroids) ? params.num_centroids : 1000;
        const int m = metric == MetricType::L2 ? SVSB200_L2 : SVSB200_IP;
        const void* rows = data;
        int dtype = SVSB200_F32;
        std::vector<uint16_t> half;
        if (storage_kind == StorageKind::FP16) {
            half.resize(n * dim);
            for (size_t i = 0; i < n * dim; ++i) half[i] = to_half(data[i]);
            rows = half.data();
            dtype = SVSB200_F16;
        }
        std::vector<float> centroids(C * dim);
        std::vector<uint32_t> assignments(n);
        if (cluster_rows(params, rows, dtype, n, dim, m, C, centroids.data(), assignments.data())) return gpu_error();
        svsb200_ivf* h = nullptr;
        if (storage_kind == StorageKind::SQI8) {   // compressed after clustering, as the reference's init_impl does
            std::vector<int8_t> codes(n * dim);
            float scale = 0.0f, bias = 0.0f;
            if (svsb200_sq_compress(data, n, dim, SVSB200_I8, 0, codes.data(), &scale, &bias) ||
                svsb200_ivf_create_sq(codes.data(), SVSB200_I8, n, dim, m, scale, bias, centroids.data(), C,
                                      assignments.data(), 0, &h))
                return gpu_error();
        } else if (svsb200_ivf_create(rows, dtype, n, dim, m, centroids.data(), C, assignments.data(), 0, &h)) {
            return gpu_error();
        }
        *index = new (std::nothrow) GpuIVFIndex(h, default_search_params, num_threads, intra_query_threads);
        if (!*index) {
            svsb200_ivf_destroy(h);
            return Status(ErrorCode::RUNTIME_ERROR, "out of memory");
        }
        return Status_Ok;
    } catch (...) {
        return Status(ErrorCode::RUNTIME_ERROR, "out of memory");
    }
}

Status IVFIndex::build(IVFIndex** index, size_t dim, MetricType metric, StorageKind storage_kind, size_t n, const float* data,
                       const BuildParams& params, size_t num_threads, size_t intra_query_threads) noexcept {
    return build(index, dim, metric, storage_kind, n, data, params, SearchParams{}, num_threads, intra_query_threads);
}

Status IVFIndex::destroy(IVFIndex* index) noexcept {
    delete index;
    return Status_Ok;
}

Status IVFIndex::load(IVFIndex** index, std::istream&, MetricType, StorageKind, size_t, size_t) noexcept {
    if (index) *index = nullptr;
    return Status(ErrorCode::NOT_IMPLEMENTED, "load stays on the reference's CPU library");
}

Status IVFIndexLeanVec::build(IVFIndex** index, size_t, MetricType, StorageKind, size_t, const float*, size_t,
                              const IVFIndex::BuildParams&, const IVFIndex::SearchParams&, size_t, size_t) noexcept {
    if (index) *index = nullptr;
    return Status(ErrorCode::NOT_IMPLEMENTED, "LeanVec storage is not available on the GPU");
}
Status IVFIndexLeanVec::build(IVFIndex** index, size_t, MetricType, StorageKind, size_t, const float*,
                              const LeanVecTrainingData*, const IVFIndex::BuildParams&, const IVFIndex::SearchParams&, size_t,
                              size_t) noexcept {
    if (index) *index = nullptr;
    return Status(ErrorCode::NOT_IMPLEMENTED, "LeanVec storage is not available on the GPU");
}

// ---- DynamicIVFIndex ----
namespace {

// Clusters n rows (cluster_rows) and assembles a dynamic index over them with the given labels.
Status cluster_and_assemble(size_t dim, MetricType metric, StorageKind kind, const IVFIndex::BuildParams& params, size_t n,
                            const float* data, const size_t* labels, svsb200_dynamic_ivf** out) {
    const size_t C = is_specified(params.num_centroids) ? params.num_centroids : 1000;
    const int m = metric == MetricType::L2 ? SVSB200_L2 : SVSB200_IP;
    const void* rows = data;
    int dtype = SVSB200_F32;
    std::vector<uint16_t> half;
    if (kind == StorageKind::FP16) {
        half.resize(n * dim);
        for (size_t i = 0; i < n * dim; ++i) half[i] = to_half(data[i]);
        rows = half.data();
        dtype = SVSB200_F16;
    }
    std::vector<float> centroids(C * dim);
    std::vector<uint32_t> assignments(n);
    if (cluster_rows(params, rows, dtype, n, dim, m, C, centroids.data(), assignments.data())) return gpu_error();
    static_assert(sizeof(size_t) == 8, "labels are 64-bit");
    const uint64_t* ids = reinterpret_cast<const uint64_t*>(labels);
    if (kind == StorageKind::SQI8) {   // compressed after clustering (dynamic_ivf_index_impl.h:391-425)
        std::vector<int8_t> codes(n * dim);
        float scale = 0.0f, bias = 0.0f;
        if (svsb200_sq_compress(data, n, dim, SVSB200_I8, 0, codes.data(), &scale, &bias) ||
            svsb200_dynamic_ivf_create_sq(codes.data(), SVSB200_I8, n, dim, m, scale, bias, centroids.data(), C,
                                          assignments.data(), ids, 0, out))
            return gpu_error();
        return Status_Ok;
    }
    if (svsb200_dynamic_ivf_create(rows, dtype, n, dim, m, centroids.data(), C, assignments.data(), ids, 0, out))
        return gpu_error();
    return Status_Ok;
}

Status not_initialized() { return Status(ErrorCode::NOT_INITIALIZED, "Index not initialized"); }

class GpuDynamicIVFIndex final : public DynamicIVFIndex {
  public:
    GpuDynamicIVFIndex(size_t dim, MetricType metric, StorageKind kind, const BuildParams& bp, const SearchParams& sp,
                       size_t threads, size_t intra)
        : dim_(dim), metric_(metric), kind_(kind), bp_(bp), sp_(sp), threads_(threads), intra_(intra) {}
    ~GpuDynamicIVFIndex() override {
        if (index_) svsb200_dynamic_ivf_destroy(index_);
    }
    Status init(size_t n, const float* data, const size_t* labels) noexcept {
        try {
            return cluster_and_assemble(dim_, metric_, kind_, bp_, n, data, labels, &index_);
        } catch (...) {
            return Status(ErrorCode::RUNTIME_ERROR, "out of memory");
        }
    }

    Status add(size_t n, const size_t* labels, const float* x, bool reuse_empty) noexcept override {
        if (n == 0) return Status_Ok;
        if (!labels || !x) return Status(ErrorCode::INVALID_ARGUMENT, "null input");
        if (!index_) return init(n, x, labels);   // the first add clusters its own rows (init_impl)
        try {
            const void* rows = x;
            int dtype = SVSB200_F32;
            std::vector<uint16_t> half;
            if (kind_ == StorageKind::FP16) {
                half.resize(n * dim_);
                for (size_t i = 0; i < n * dim_; ++i) half[i] = to_half(x[i]);
                rows = half.data();
                dtype = SVSB200_F16;
            }
            if (svsb200_dynamic_ivf_add(index_, rows, dtype, n, reinterpret_cast<const uint64_t*>(labels), reuse_empty ? 1 : 0,
                                        nullptr))
                return gpu_error();
            return Status_Ok;
        } catch (...) {
            return Status(ErrorCode::RUNTIME_ERROR, "out of memory");
        }
    }
    Status remove(size_t n, const size_t* labels) noexcept override {
        if (!index_) return not_initialized();
        if (svsb200_dynamic_ivf_delete(index_, reinterpret_cast<const uint64_t*>(labels), n)) return gpu_error();
        return Status_Ok;
    }
    Status remove_selected(size_t* num_removed, const IDFilter& selector) noexcept override {
        if (!index_) return not_initialized();
        try {
            size_t count = svsb200_dynamic_ivf_size(index_);
            std::vector<uint64_t> ids(count), gone;
            if (svsb200_dynamic_ivf_ids(index_, ids.data(), &count)) return gpu_error();
            for (size_t i = 0; i < count; ++i)
                if (selector(size_t(ids[i]))) gone.push_back(ids[i]);
            if (svsb200_dynamic_ivf_delete(index_, gone.data(), gone.size())) return gpu_error();
            if (num_removed) *num_removed = gone.size();
            return Status_Ok;
        } catch (...) {
            return Status(ErrorCode::RUNTIME_ERROR, "out of memory");
        }
    }
    Status has_id(bool* exists, size_t id) const noexcept override {
        if (!exists) return Status(ErrorCode::INVALID_ARGUMENT, "null output");
        *exists = false;
        if (!index_) return Status_Ok;
        int out = 0;
        if (svsb200_dynamic_ivf_has_id(index_, id, &out)) return gpu_error();
        *exists = out != 0;
        return Status_Ok;
    }
    Status consolidate() noexcept override { return index_ ? Status_Ok : not_initialized(); }
    Status compact(size_t) noexcept override {
        if (!index_) return not_initialized();
        if (svsb200_dynamic_ivf_compact(index_)) return gpu_error();
        return Status_Ok;
    }
    Status search(size_t n, const float* x, size_t k, float* distances, size_t* labels, const SearchParams* params,
                  IDFilter* filter) const noexcept override {
        if (!index_) {
            for (size_t i = 0; i < n * k; ++i) {
                labels[i] = size_t(-1);
                distances[i] = INFINITY;
            }
            return not_initialized();
        }
        if (k == 0) return Status(ErrorCode::INVALID_ARGUMENT, "k must be greater than 0");
        if (n == 0) return Status_Ok;
        size_t n_probes = is_specified(sp_.n_probes) ? sp_.n_probes : 1;
        float k_reorder = is_specified(sp_.k_reorder) ? sp_.k_reorder : 1.0f;
        if (params && is_specified(params->n_probes)) n_probes = params->n_probes;
        if (params && is_specified(params->k_reorder)) k_reorder = params->k_reorder;
        if (!(k_reorder >= 1.0f)) return Status(ErrorCode::INVALID_ARGUMENT, "k_reorder must be at least 1");
        if (filter) {
            const FilterStop fs = filter_stop_of(sp_, params);
            auto held = [this](size_t id) {
                int out = 0;
                return svsb200_dynamic_ivf_has_id(index_, id, &out) == 0 && out != 0;
            };
            if (fs.estimate && sample_says_stop(*filter, svsb200_dynamic_ivf_size(index_), fs.stop, held)) {
                pad_rows(0, n, k, distances, labels);
                return Status_Ok;
            }
            try {
                const size_t slots = svsb200_dynamic_ivf_num_slots(index_);
                std::vector<uint8_t> status(slots);
                std::vector<uint64_t> ext(slots);
                if (svsb200_dynamic_ivf_export(index_, status.data(), ext.data(), nullptr)) return gpu_error();
                std::vector<uint32_t> bitmap((slots + 31) / 32, 0u);   // bit s: slot s
                for (size_t s = 0; s < slots; ++s)
                    if (status[s] && filter->is_member(size_t(ext[s]))) bitmap[s >> 5] |= 1u << (s & 31);
                return filtered_search(n, k, distances, labels, fs.stop, [&](uint32_t* p, uint32_t* a, uint32_t* r) {
                    return svsb200_dynamic_ivf_search_filtered(index_, x, SVSB200_F32, n, k, n_probes, bitmap.data(),
                                                               reinterpret_cast<uint64_t*>(labels), distances, p, a, r);
                });
            } catch (...) {
                return Status(ErrorCode::RUNTIME_ERROR, "out of memory");
            }
        }
        if (svsb200_dynamic_ivf_search(index_, x, SVSB200_F32, n, k, n_probes, reinterpret_cast<uint64_t*>(labels),
                                       distances))
            return gpu_error();
        return Status_Ok;
    }
    Status save(std::ostream&) const noexcept override {
        return Status(ErrorCode::NOT_IMPLEMENTED, "save stays on the reference's CPU index");
    }
    Status set_num_threads(size_t n) noexcept override {
        threads_ = n;
        return Status_Ok;
    }
    Status get_num_threads(size_t* n) const noexcept override {
        if (n) *n = threads_;
        return Status_Ok;
    }
    Status set_intra_query_threads(size_t n) noexcept override {
        intra_ = n;
        return Status_Ok;
    }
    Status get_intra_query_threads(size_t* n) const noexcept override {
        if (n) *n = intra_;
        return Status_Ok;
    }

  private:
    svsb200_dynamic_ivf* index_ = nullptr;
    size_t dim_;
    MetricType metric_;
    StorageKind kind_;
    BuildParams bp_;
    SearchParams sp_;
    size_t threads_, intra_;
};

}  // namespace

Status DynamicIVFIndex::check_storage_kind(StorageKind kind) noexcept {
    return kind == StorageKind::FP32 || kind == StorageKind::FP16 || kind == StorageKind::SQI8
               ? Status_Ok
               : Status(ErrorCode::NOT_IMPLEMENTED, "DynamicIVFIndex on the GPU supports FP32, FP16 and SQI8 storage only");
}

Status DynamicIVFIndex::build(DynamicIVFIndex** index, size_t dim, MetricType metric, StorageKind storage_kind, size_t n,
                              const float* data, const size_t* labels, const IVFIndex::BuildParams& params,
                              const IVFIndex::SearchParams& default_search_params, size_t num_threads,
                              size_t intra_query_threads) noexcept {
    if (!index) return Status(ErrorCode::INVALID_ARGUMENT, "null output");
    *index = nullptr;
    if (Status st = check_storage_kind(storage_kind); !st.ok()) return st;
    if (dim == 0) return Status(ErrorCode::INVALID_ARGUMENT, "dim must be positive");
    auto* h = new (std::nothrow)
        GpuDynamicIVFIndex(dim, metric, storage_kind, params, default_search_params, num_threads, intra_query_threads);
    if (!h) return Status(ErrorCode::RUNTIME_ERROR, "out of memory");
    if (n > 0 && data && labels) {   // (no rows: the first add initialises the index)
        if (Status st = h->init(n, data, labels); !st.ok()) {
            delete h;
            return st;
        }
    }
    *index = h;
    return Status_Ok;
}

Status DynamicIVFIndex::destroy(DynamicIVFIndex* index) noexcept {
    delete index;
    return Status_Ok;
}

Status DynamicIVFIndex::load(DynamicIVFIndex** index, std::istream&, MetricType, StorageKind, size_t, size_t) noexcept {
    if (index) *index = nullptr;
    return Status(ErrorCode::NOT_IMPLEMENTED, "load stays on the reference's CPU library");
}

Status DynamicIVFIndexLeanVec::build(DynamicIVFIndex** index, size_t, MetricType, StorageKind, size_t, const float*,
                                     const size_t*, size_t, const IVFIndex::BuildParams&, const IVFIndex::SearchParams&,
                                     size_t, size_t) noexcept {
    if (index) *index = nullptr;
    return Status(ErrorCode::NOT_IMPLEMENTED, "LeanVec storage is not available on the GPU");
}
Status DynamicIVFIndexLeanVec::build(DynamicIVFIndex** index, size_t, MetricType, StorageKind, size_t, const float*,
                                     const size_t*, const LeanVecTrainingData*, const IVFIndex::BuildParams&,
                                     const IVFIndex::SearchParams&, size_t, size_t) noexcept {
    if (index) *index = nullptr;
    return Status(ErrorCode::NOT_IMPLEMENTED, "LeanVec storage is not available on the GPU");
}

// ---- DynamicVamanaIndex ----
namespace {

// The graph builder's parameters of a runtime BuildParams, unspecified ones as GpuVamanaIndex::add maps them: degree 32,
// window 200, and 0 (the library's default) for alpha, the candidate pool and prune_to.
struct GraphParams {
    size_t R, window, pool, prune_to;
    float alpha;
};
GraphParams graph_params(const VamanaIndex::BuildParams& bp) {
    return {is_specified(bp.graph_max_degree) ? bp.graph_max_degree : 32,
            is_specified(bp.construction_window_size) ? bp.construction_window_size : 200,
            is_specified(bp.max_candidate_pool_size) ? bp.max_candidate_pool_size : 0,
            is_specified(bp.prune_to) ? bp.prune_to : 0, is_specified(bp.alpha) ? bp.alpha : 0.f};
}

class GpuDynamicVamanaIndex final : public DynamicVamanaIndex {
  public:
    GpuDynamicVamanaIndex(size_t dim, MetricType metric, StorageKind kind, const BuildParams& bp, const SearchParams& sp,
                          const DynamicIndexParams& dp)
        : dim_(dim), metric_(metric), kind_(kind), bp_(bp), sp_(sp), dp_(dp) {}
    ~GpuDynamicVamanaIndex() override { svsb200_index_destroy(index_); }

    using DynamicVamanaIndex::add;   // (add(n, x) without labels: NOT_IMPLEMENTED, as the header defines it)

    // DynamicVamanaIndexImpl::add (dynamic_vamana_index_impl.h:95-102): the first add builds the index over its rows,
    // later ones are add_points with reuse_empty = false
    Status add(size_t n, const size_t* labels, const float* x) noexcept override {
        if (n == 0) return Status_Ok;
        if (!labels || !x) return Status(ErrorCode::INVALID_ARGUMENT, "null input");
        static_assert(sizeof(size_t) == 8, "labels are 64-bit");
        const uint64_t* ids = reinterpret_cast<const uint64_t*>(labels);
        try {
            if (!index_) return init(n, ids, x);
            const void* rows = x;
            int dtype = SVSB200_F32;   // (an SQI8 index encodes float32 rows with its fixed scale and bias)
            std::vector<uint16_t> half;
            if (kind_ == StorageKind::FP16) {
                half.resize(n * dim_);
                for (size_t i = 0; i < n * dim_; ++i) half[i] = to_half(x[i]);
                rows = half.data();
                dtype = SVSB200_F16;
            }
            if (svsb200_dynamic_add(index_, rows, dtype, n, ids, 0, nullptr)) return gpu_error();
            return Status_Ok;
        } catch (const std::exception& e) {
            return Status(ErrorCode::RUNTIME_ERROR, e.what());
        }
    }

    // DynamicVamanaIndexImpl::remove (:325-346): soft deletion, then consolidate and compact once the soft deletions
    // exceed half of the ids left, or none is left.  An index emptied this way is released: the next add builds anew.
    Status remove(size_t n, const size_t* labels) noexcept override {
        if (!index_) return not_initialized();
        if (n && !labels) return Status(ErrorCode::INVALID_ARGUMENT, "null input");
        if (svsb200_dynamic_delete(index_, reinterpret_cast<const uint64_t*>(labels), n)) return gpu_error();
        soft_deleted_ += n;
        size_t left = 0;
        if (svsb200_dynamic_ids(index_, nullptr, &left)) return gpu_error();
        if (left == 0) return reset();   // (nothing is left to consolidate towards)
        if (float(soft_deleted_) / float(left) > 0.5f) {
            if (svsb200_dynamic_consolidate(index_) || svsb200_dynamic_compact(index_)) return gpu_error();
            soft_deleted_ = 0;
        }
        return Status_Ok;
    }
    // remove_selected (:348-363): the Valid ids the selector accepts, in slot order, through remove
    Status remove_selected(size_t* num_removed, const IDFilter& selector) noexcept override {
        if (!index_) return not_initialized();
        try {
            size_t count = svsb200_index_size(index_);
            std::vector<uint64_t> ids(count);
            std::vector<size_t> gone;
            if (svsb200_dynamic_ids(index_, ids.data(), &count)) return gpu_error();
            for (size_t i = 0; i < count; ++i)
                if (selector(size_t(ids[i]))) gone.push_back(size_t(ids[i]));
            if (Status st = remove(gone.size(), gone.data()); !st.ok()) return st;
            if (num_removed) *num_removed = gone.size();
            return Status_Ok;
        } catch (const std::exception& e) {
            return Status(ErrorCode::RUNTIME_ERROR, e.what());
        }
    }

    Status reset() noexcept override {
        svsb200_index_destroy(index_);
        index_ = nullptr;
        soft_deleted_ = 0;
        return Status_Ok;
    }

    Status search(size_t n, const float* x, size_t k, float* distances, size_t* labels, const SearchParams* params,
                  IDFilter* filter) const noexcept override {
        if (!index_) {
            pad_rows(0, n, k, distances, labels);
            return not_initialized();
        }
        if (n == 0) return Status_Ok;
        if (k == 0) return Status(ErrorCode::INVALID_ARGUMENT, "k must be greater than 0");
        size_t window = 0, capacity = 0;
        window_of(sp_, params, k, window, capacity);
        if (!filter) {
            if (svsb200_search(index_, x, SVSB200_F32, n, k, window, capacity, 0, labels, 8, distances, nullptr))
                return gpu_error();
            return Status_Ok;
        }
        const FilterStop fs = filter_stop_of(sp_, params);
        size_t size = 0;
        if (svsb200_dynamic_ids(index_, nullptr, &size)) return gpu_error();
        auto held = [this](size_t id) {
            int out = 0;
            return svsb200_dynamic_has_id(index_, id, &out) == 0 && out != 0;
        };
        if (fs.estimate && sample_says_stop(*filter, size, fs.stop, held)) {
            pad_rows(0, n, k, distances, labels);
            return Status_Ok;
        }
        try {   // IDFilter -> bitmap over the slots: bit s when slot s is Valid and its external id a member
            const size_t slots = svsb200_index_size(index_);
            std::vector<uint8_t> status(slots);
            std::vector<uint64_t> ext(slots);
            if (svsb200_dynamic_export(index_, nullptr, status.data(), ext.data(), nullptr)) return gpu_error();
            std::vector<uint32_t> bitmap((slots + 31) / 32, 0u);
            for (size_t s = 0; s < slots; ++s)
                if (status[s] == 1 && filter->is_member(size_t(ext[s]))) bitmap[s >> 5] |= 1u << (s & 31);
            if (svsb200_search_filtered(index_, x, SVSB200_F32, n, k, window, bitmap.data(), reinterpret_cast<uint64_t*>(labels),
                                        distances, nullptr))
                return gpu_error();
        } catch (const std::exception& e) {
            return Status(ErrorCode::RUNTIME_ERROR, e.what());
        }
        return Status_Ok;
    }

    // range_search (:222-323): the search's results inside the radius, then the filter, as the static class applies it
    Status range_search(size_t n, const float* x, float radius, const ResultsAllocator& results, const SearchParams* params,
                        IDFilter* filter) const noexcept override {
        if (!index_) return not_initialized();
        if (radius <= 0) return Status(ErrorCode::INVALID_ARGUMENT, "radius must be greater than 0");
        if (n == 0) return Status_Ok;
        size_t window = 0, capacity = 0;
        window_of(sp_, params, 10, window, capacity);
        try {
            std::vector<uint32_t> counts(n);
            uint64_t* ids = nullptr;
            float* dd = nullptr;
            if (svsb200_range_search(index_, x, SVSB200_F32, n, radius, window, counts.data(), &ids, &dd)) return gpu_error();
            std::unique_ptr<uint64_t, void (*)(void*)> ids_guard(ids, svsb200_free);
            std::unique_ptr<float, void (*)(void*)> dd_guard(dd, svsb200_free);
            std::vector<size_t> kept(n, 0), offs(n + 1, 0);
            for (size_t q = 0; q < n; ++q) offs[q + 1] = offs[q] + counts[q];
            for (size_t q = 0; q < n; ++q)
                for (size_t j = offs[q]; j < offs[q + 1]; ++j)
                    if (!filter || filter->is_member(ids[j])) ++kept[q];
            SearchResultsStorage out = results.allocate(std::span<size_t>(kept.data(), kept.size()));
            size_t o = 0;
            for (size_t q = 0; q < n; ++q)
                for (size_t j = offs[q]; j < offs[q + 1]; ++j)
                    if (!filter || filter->is_member(ids[j])) {
                        out.labels[o] = ids[j];
                        out.distances[o] = dd[j];
                        ++o;
                    }
        } catch (const std::exception& e) {
            return Status(ErrorCode::RUNTIME_ERROR, e.what());
        }
        return Status_Ok;
    }

    // MutableVamanaIndex::get_distance / reconstruct_at on the device; an id the index does not hold is the reference's
    // ANNEXCEPTION, a RUNTIME_ERROR through runtime_error_wrapper
    Status get_distance(size_t id, const float* query, float* distance) const noexcept override {
        if (!index_) return not_initialized();
        const uint64_t ext = id;
        if (svsb200_index_distances(index_, query, SVSB200_F32, 1, &ext, distance)) return gpu_error();
        return Status_Ok;
    }
    Status reconstruct_at(size_t n, const size_t* ids, float* output) noexcept override {
        if (!index_) return not_initialized();
        if (svsb200_index_reconstruct(index_, reinterpret_cast<const uint64_t*>(ids), n, output)) return gpu_error();
        return Status_Ok;
    }

    size_t get_memory_usage() const noexcept override { return index_ ? svsb200_index_device_bytes(index_) : 0; }
    // The device bytes per slot: the row (16-byte aligned), the adjacency row (padded to whole 32-word groups) and its
    // 16-bit length, and the status byte and 64-bit external id.  The slots counted are the capacity the arrays hold.
    Status get_memory_breakdown(MemoryBreakdown* out) const noexcept override {
        if (!out) return Status(ErrorCode::INVALID_ARGUMENT, "memory breakdown output must not be null");
        *out = MemoryBreakdown{};
        if (!index_) return Status_Ok;
        const size_t total = svsb200_index_device_bytes(index_);
        const size_t elem = kind_ == StorageKind::FP32 ? 4 : kind_ == StorageKind::FP16 ? 2 : 1;
        const size_t row = (dim_ * elem + 15) / 16 * 16;
        const size_t R = svsb200_index_max_degree(index_);
        const size_t adjacency = (R + 31) / 32 * 32 * 4 + 2, meta = 1 + 8;
        const size_t cap = total / (row + adjacency + meta);
        out->data_bytes = cap * row;
        out->metadata_bytes = cap * meta;
        out->graph_bytes = total - out->data_bytes - out->metadata_bytes;
        return Status_Ok;
    }
    size_t blocksize_bytes() const noexcept override { return 1u << dp_.blocksize_exp; }

    Status save(std::ostream&) const noexcept override {
        return Status(ErrorCode::NOT_IMPLEMENTED, "save stays on the reference's CPU index (index/vamana/dynamic_index.h)");
    }

  private:
    static Status not_initialized() { return Status(ErrorCode::NOT_INITIALIZED, "Index not initialized"); }

    // The first add: the graph over its rows (svsb200_dynamic_build / _build_sq).  The builder needs two rows, so a
    // one-row index is assembled with an adjacency row of degree 0 and the build parameters as mutation parameters.
    Status init(size_t n, const uint64_t* ids, const float* x) {
        const GraphParams g = graph_params(bp_);
        const int metric = metric_ == MetricType::L2 ? SVSB200_L2 : SVSB200_IP;
        std::vector<uint32_t> graph(g.R + 1, 0u);   // (one row: degree 0)
        svsb200_index* h = nullptr;
        int rc = 0;
        if (kind_ == StorageKind::SQI8) {   // int8 codes with one global scale and bias, as the static class compresses
            std::vector<int8_t> codes(n * dim_);
            float sq[2] = {0.f, 0.f};
            if (svsb200_sq_compress(x, n, dim_, SVSB200_I8, 0, codes.data(), &sq[0], &sq[1])) return gpu_error();
            rc = n == 1 ? svsb200_dynamic_create_sq(codes.data(), SVSB200_I8, 1, dim_, sq[0], sq[1], graph.data(), g.R + 1, 0,
                                                    metric, ids, 0, &h)
                        : svsb200_dynamic_build_sq(codes.data(), SVSB200_I8, n, dim_, metric, sq[0], sq[1], g.alpha, g.R,
                                                   g.window, g.pool, g.prune_to, ids, 0, &h);
        } else {
            const void* rows = x;
            int dtype = SVSB200_F32;
            std::vector<uint16_t> half;
            if (kind_ == StorageKind::FP16) {
                half.resize(n * dim_);
                for (size_t i = 0; i < n * dim_; ++i) half[i] = to_half(x[i]);
                rows = half.data();
                dtype = SVSB200_F16;
            }
            rc = n == 1 ? svsb200_dynamic_create(rows, dtype, 1, dim_, graph.data(), g.R + 1, 0, metric, ids, 0, &h)
                        : svsb200_dynamic_build(rows, dtype, n, dim_, metric, g.alpha, g.R, g.window, g.pool, g.prune_to, ids,
                                                0, &h);
        }
        if (rc == 0 && n == 1) rc = svsb200_dynamic_set_build_parameters(h, g.alpha, g.window, g.pool, g.prune_to);
        if (rc) {
            const Status st = gpu_error();
            svsb200_index_destroy(h);
            return st;
        }
        index_ = h;
        soft_deleted_ = 0;
        return Status_Ok;
    }

    size_t dim_;
    MetricType metric_;
    StorageKind kind_;
    BuildParams bp_;
    SearchParams sp_;
    DynamicIndexParams dp_;
    svsb200_index* index_ = nullptr;
    size_t soft_deleted_ = 0;   // ntotal_soft_deleted
};

}  // namespace

Status DynamicVamanaIndex::check_storage_kind(StorageKind kind) noexcept {
    return kind == StorageKind::FP32 || kind == StorageKind::FP16 || kind == StorageKind::SQI8
               ? Status_Ok
               : Status(ErrorCode::NOT_IMPLEMENTED, "DynamicVamanaIndex on the GPU supports FP32, FP16 and SQI8 storage only");
}

// dynamic_vamana_index.cpp: the block size of the reference's blocked storage, 2^12 to 2^30 bytes
Status DynamicVamanaIndex::check_params(const VamanaIndex::DynamicIndexParams& dynamic_index_params) noexcept {
    if (dynamic_index_params.blocksize_exp > 30) return Status(ErrorCode::INVALID_ARGUMENT, "Blocksize is too large");
    if (dynamic_index_params.blocksize_exp < 12) return Status(ErrorCode::INVALID_ARGUMENT, "Blocksize is too small");
    return Status_Ok;
}

Status DynamicVamanaIndex::build(DynamicVamanaIndex** index, size_t dim, MetricType metric, StorageKind storage_kind,
                                 const VamanaIndex::BuildParams& params,
                                 const VamanaIndex::SearchParams& default_search_params) noexcept {
    return build(index, dim, metric, storage_kind, params, default_search_params, VamanaIndex::DynamicIndexParams{});
}

Status DynamicVamanaIndex::build(DynamicVamanaIndex** index, size_t dim, MetricType metric, StorageKind storage_kind,
                                 const VamanaIndex::BuildParams& params, const VamanaIndex::SearchParams& default_search_params,
                                 const VamanaIndex::DynamicIndexParams& dynamic_index_params) noexcept {
    if (!index) return Status(ErrorCode::INVALID_ARGUMENT, "null output");
    *index = nullptr;
    if (Status st = check_storage_kind(storage_kind); !st.ok()) return st;
    if (Status st = check_params(dynamic_index_params); !st.ok()) return st;
    if (dim == 0) return Status(ErrorCode::INVALID_ARGUMENT, "dim must be positive");
    *index = new (std::nothrow) GpuDynamicVamanaIndex(dim, metric, storage_kind, params, default_search_params,
                                                      dynamic_index_params);
    return *index ? Status_Ok : Status(ErrorCode::RUNTIME_ERROR, "out of memory");
}

Status DynamicVamanaIndex::destroy(DynamicVamanaIndex* index) noexcept {
    delete index;
    return Status_Ok;
}

Status DynamicVamanaIndex::load(DynamicVamanaIndex** index, std::istream&, MetricType, StorageKind) noexcept {
    if (index) *index = nullptr;
    return Status(ErrorCode::NOT_IMPLEMENTED, "load stays on the reference's CPU library");
}

Status DynamicVamanaIndexLeanVec::build(DynamicVamanaIndex** index, size_t, MetricType, StorageKind, size_t,
                                        const VamanaIndex::BuildParams&, const VamanaIndex::SearchParams&) noexcept {
    if (index) *index = nullptr;
    return Status(ErrorCode::NOT_IMPLEMENTED, "LeanVec storage is not available on the GPU");
}
Status DynamicVamanaIndexLeanVec::build(DynamicVamanaIndex** index, size_t, MetricType, StorageKind, size_t,
                                        const VamanaIndex::BuildParams&, const VamanaIndex::SearchParams&,
                                        const VamanaIndex::DynamicIndexParams&) noexcept {
    if (index) *index = nullptr;
    return Status(ErrorCode::NOT_IMPLEMENTED, "LeanVec storage is not available on the GPU");
}
Status DynamicVamanaIndexLeanVec::build(DynamicVamanaIndex** index, size_t, MetricType, StorageKind, const LeanVecTrainingData*,
                                        const VamanaIndex::BuildParams&, const VamanaIndex::SearchParams&) noexcept {
    if (index) *index = nullptr;
    return Status(ErrorCode::NOT_IMPLEMENTED, "LeanVec storage is not available on the GPU");
}
Status DynamicVamanaIndexLeanVec::build(DynamicVamanaIndex** index, size_t, MetricType, StorageKind, const LeanVecTrainingData*,
                                        const VamanaIndex::BuildParams&, const VamanaIndex::SearchParams&,
                                        const VamanaIndex::DynamicIndexParams&) noexcept {
    if (index) *index = nullptr;
    return Status(ErrorCode::NOT_IMPLEMENTED, "LeanVec storage is not available on the GPU");
}

}  // SVS_DECLARE_NAMESPACE_VERSION(0)
}  // namespace runtime
}  // namespace svs
