// gpu_runtime_index.cpp -- the FAISS-facing runtime ABI of the reference (SURVEY.md §8 f4), backed by libsvsb200.
//
// Implements `svs::runtime::v0::VamanaIndex` (bindings/cpp/include/svs/runtime/vamana_index.h:61-143) for the
// uncompressed storage kinds (FP32, FP16) on the GPU: `build` + `add` construct the graph with svsb200_build_vamana,
// `search` is the batched GPU search (optionally through an IDFilter evaluated on the device as a bitmap),
// `range_search` grows the result lists until they leave the radius.  It stands where the reference's
// libsvs_runtime implementation sits (bindings/cpp/src/vamana_index.cpp, vamana_index_impl.h:60-330): a program
// written against the runtime header links this object instead and runs on the H100.
//
// Compiles against the reference's runtime *headers* only (no svs core headers); the few out-of-line members of the
// header types that live in libsvs_runtime (Status message storage, the VamanaIndex destructor / static factories)
// are defined here.  save / load / LeanVec are the reference's CPU territory: NOT_IMPLEMENTED.
#include "svs/runtime/vamana_index.h"

#include "svsb200.h"

#include <cmath>
#include <cstring>
#include <memory>
#include <new>
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

namespace {

Status gpu_error() { return Status(ErrorCode::RUNTIME_ERROR, svsb200_last_error()); }

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
            data_.assign(x, x + n * dim_);
            const int metric = metric_ == MetricType::L2 ? SVSB200_L2 : SVSB200_IP;
            const size_t R = is_specified(bp_.graph_max_degree) ? bp_.graph_max_degree : 32;
            const size_t window = is_specified(bp_.construction_window_size) ? bp_.construction_window_size : 200;
            std::vector<uint32_t> graph(n * (R + 1));
            uint32_t ep = 0;
            const void* rows = data_.data();
            int dtype = SVSB200_F32;
            if (kind_ == StorageKind::FP16) {   // stored as float16, like the reference's FP16 storage kind
                half_.resize(n * dim_);
                for (size_t i = 0; i < n * dim_; ++i) half_[i] = to_half(data_[i]);
                rows = half_.data();
                dtype = SVSB200_F16;
            }
            if (svsb200_build_vamana(rows, dtype, n, dim_, 0, metric, is_specified(bp_.alpha) ? bp_.alpha : 0.f, R, window,
                                     is_specified(bp_.max_candidate_pool_size) ? bp_.max_candidate_pool_size : 0,
                                     is_specified(bp_.prune_to) ? bp_.prune_to : 0, 0, graph.data(), &ep))
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
        n_ = 0;
        return Status_Ok;
    }

    Status search(size_t n, const float* x, size_t k, float* distances, size_t* labels, const SearchParams* params,
                  IDFilter* filter) const noexcept override {
        if (!index_) return Status(ErrorCode::NOT_INITIALIZED, "Index not initialized");
        if (n == 0) return Status_Ok;
        if (k == 0) return Status(ErrorCode::INVALID_ARGUMENT, "k must be greater than 0");
        size_t window = 0, capacity = 0;
        window_of(params, k, window, capacity);
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
        window_of(params, 10, window, capacity);
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
        if (!found) {   // not reached by the graph walk: plain arithmetic on the host copy
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
                output[i * dim_ + d] = kind_ == StorageKind::FP16 ? from_half(half_[ids[i] * dim_ + d]) : data_[ids[i] * dim_ + d];
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
    void window_of(const SearchParams* params, size_t k, size_t& window, size_t& capacity) const {
        window = is_specified(sp_.search_window_size) ? sp_.search_window_size : 10;
        capacity = is_specified(sp_.search_buffer_capacity) ? sp_.search_buffer_capacity : 0;
        if (params) {
            set_if_specified(window, params->search_window_size);
            set_if_specified(capacity, params->search_buffer_capacity);
        }
        window = window < k ? k : window;
        capacity = capacity < window ? window : capacity;
    }
    static uint16_t to_half(float f) {   // round to nearest even, like lib/float16.h:54-79 (F16C)
        uint32_t x;
        std::memcpy(&x, &f, 4);
        const uint32_t sign = (x >> 16) & 0x8000u;
        int32_t e = int32_t((x >> 23) & 0xFF) - 127 + 15;
        uint32_t m = x & 0x7FFFFFu;
        if (((x >> 23) & 0xFF) == 0xFF) return uint16_t(sign | 0x7C00u | (m ? 0x200u : 0));
        if (e >= 31) return uint16_t(sign | 0x7C00u);
        if (e <= 0) {
            if (e < -10) return uint16_t(sign);
            m |= 0x800000u;
            const uint32_t shift = uint32_t(14 - e);
            uint32_t h = m >> shift;
            const uint32_t rem = m & ((1u << shift) - 1), half = 1u << (shift - 1);
            if (rem > half || (rem == half && (h & 1))) ++h;
            return uint16_t(sign | h);
        }
        uint32_t h = (uint32_t(e) << 10) | (m >> 13);
        const uint32_t rem = m & 0x1FFFu;
        if (rem > 0x1000u || (rem == 0x1000u && (h & 1))) ++h;
        return uint16_t(sign | h);
    }
    static float from_half(uint16_t h) {
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

    size_t dim_, n_ = 0, graph_bytes_ = 0;
    MetricType metric_;
    StorageKind kind_;
    BuildParams bp_;
    SearchParams sp_;
    std::vector<float> data_;
    std::vector<uint16_t> half_;
    svsb200_index* index_ = nullptr;
};

}  // namespace

Status VamanaIndex::check_storage_kind(StorageKind kind) noexcept {
    return kind == StorageKind::FP32 || kind == StorageKind::FP16
               ? Status_Ok
               : Status(ErrorCode::NOT_IMPLEMENTED, "the GPU runtime holds FP32 / FP16 storage (compressed kinds: reference CPU library)");
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

}  // SVS_DECLARE_NAMESPACE_VERSION(0)
}  // namespace runtime
}  // namespace svs
