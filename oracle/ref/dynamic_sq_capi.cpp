// oracle/_ref driver for the reference's MutableVamanaIndex over scalar-quantised codes -- TEST INFRASTRUCTURE ONLY
// (see oracle/README.md).
//
// A thin `extern "C"` façade over the *unmodified* reference headers (`-I/root/reference/include`, never copied),
// built by `make -C oracle -f dynamic_sq.mk dynamic_sq` into `_ref/libsvsref_dynamic_sq.so` and linked with the same
// `avx512.o` / `avx2.o` distance kernels as `libsvsref.so`.  The index holds SQDataset<int8_t / uint8_t> with a given
// scale and bias (what the runtime's DynamicVamanaIndex holds for StorageKind::SQI8):
//   index/vamana/dynamic_index.h:178-202   MutableVamanaIndex(graph, data, entry_point, distance, ids, threads)
//   index/vamana/dynamic_index.h:208-261   MutableVamanaIndex(parameters, data, ids, distance, threads)
//   index/vamana/dynamic_index.h:657-1013  add_points (float32 rows, encoded by SQDataset::set_datum), delete_entries,
//                                          compact, consolidate (the SQ build adaptor, extensions/vamana/scalar.h)
//   index/vamana/dynamic_index.h:525-571   search (the SQ search's compressed distance)
//
// Nothing in the product (libsvsb200.so / scalablevectorsearch_b200) links or loads this.

#include "svs/core/data.h"
#include "svs/core/distance.h"
#include "svs/core/graph.h"
#include "svs/extensions/vamana/scalar.h"
#include "svs/index/vamana/dynamic_index.h"
#include "svs/quantization/scalar/scalar.h"

#include <cstdint>
#include <cstring>
#include <span>
#include <string>
#include <vector>

namespace {

thread_local std::string g_error;

enum DType : int { I8 = 2, U8 = 3 };
enum Metric : int { L2 = 0, IP = 1, COS = 2 };
enum Slot : uint8_t { EMPTY = 0, VALID = 1, DELETED = 2 };

using Graph = svs::graphs::SimpleGraph<uint32_t, svs::lib::Allocator<uint32_t>>;
// A blocked allocator, as the runtime's dynamic indexes use (bindings/cpp/src/dynamic_vamana_index_impl.h): SQDataset
// resizes and compacts only over one (quantization/scalar/scalar.h:472-485).
template <typename T> using Alloc = svs::data::Blocked<svs::lib::Allocator<T>>;
template <typename T> using SQ = svs::quantization::scalar::SQDataset<T, svs::Dynamic, Alloc<T>>;

// `rows`: n x (max_degree + 1), element 0 the out-degree (core/graph/graph.h:103-114).
Graph make_graph(const uint32_t* rows, size_t n, size_t max_degree) {
    auto g = Graph(n, max_degree);
    for (size_t i = 0; i < n; ++i) {
        const uint32_t* r = rows + i * (max_degree + 1);
        g.replace_node(i, std::span<const uint32_t>(r + 1, r[0]));
    }
    return g;
}

template <typename T> SQ<T> sq_of(const void* src, size_t n, size_t dim, float scale, float bias) {
    auto d = svs::data::SimpleData<T, svs::Dynamic, Alloc<T>>(n, dim);
    const T* p = static_cast<const T*>(src);
    for (size_t i = 0; i < n; ++i) d.set_datum(i, std::span<const T>(p + i * dim, dim));
    return SQ<T>(std::move(d), scale, bias);
}

template <typename F> int guarded(F&& f) {
    try {
        f();
        return 0;
    } catch (const std::exception& e) {
        g_error = e.what();
        return 1;
    } catch (...) {
        g_error = "unknown exception";
        return 2;
    }
}

// The façade mirrors the slot status (the reference keeps it private), as ref/dynamic_capi.cpp does.
struct DynBase {
    virtual ~DynBase() = default;
    std::vector<uint8_t> status;
    virtual void set_params(float alpha, size_t window, size_t max_candidates, size_t prune_to) = 0;
    virtual void add(const float* data, size_t count, const uint64_t* ids, bool reuse, uint64_t* slots) = 0;
    virtual void remove(const uint64_t* ids, size_t count) = 0;
    virtual void consolidate() = 0;
    virtual void compact() = 0;
    virtual size_t slots() const = 0;
    virtual void export_state(uint32_t* graph, uint64_t* ext, uint32_t* ep, void* codes) = 0;
    virtual void search(const float* q, size_t nq, size_t k, size_t window, size_t capacity, uint64_t* ids, float* dists) = 0;
};

template <typename T, typename Dist> struct DynImpl : DynBase {
    using Index = svs::index::vamana::MutableVamanaIndex<Graph, SQ<T>, Dist>;
    Index index;

    DynImpl(Graph g, SQ<T> d, uint32_t ep, const std::vector<size_t>& ids, size_t threads)
        : index(std::move(g), std::move(d), ep, Dist{}, ids, threads) {
        status.assign(ids.size(), VALID);
    }
    DynImpl(const svs::index::vamana::VamanaBuildParameters& params, SQ<T> d, const std::vector<size_t>& ids, size_t threads)
        : index(params, std::move(d), ids, Dist{}, threads) {
        status.assign(ids.size(), VALID);
    }

    void set_params(float alpha, size_t window, size_t max_candidates, size_t prune_to) override {
        index.set_alpha(alpha);
        index.set_construction_window_size(window);
        index.set_max_candidates(max_candidates);
        index.set_prune_to(prune_to);
    }
    void add(const float* data, size_t count, const uint64_t* ids, bool reuse, uint64_t* slots) override {
        auto view = svs::data::ConstSimpleDataView<float>(data, count, index.dimensions());
        std::vector<size_t> ext(ids, ids + count);
        auto got = index.add_points(view, ext, reuse);
        for (size_t i = 0; i < got.size(); ++i) {
            slots[i] = got[i];
            if (got[i] >= status.size()) status.resize(got[i] + 1, EMPTY);
            status[got[i]] = VALID;
        }
    }
    void remove(const uint64_t* ids, size_t count) override {
        std::vector<size_t> ext(ids, ids + count);
        std::vector<size_t> internal;
        for (auto e : ext) {
            if (index.has_id(e)) internal.push_back(index.translate_external_id(e));
        }
        index.delete_entries(ext);
        for (auto i : internal) status[i] = DELETED;
    }
    void consolidate() override {
        index.consolidate();
        for (auto& s : status) {
            if (s == DELETED) s = EMPTY;
        }
    }
    void compact() override {
        index.compact();
        status.assign(index.size(), VALID);
    }
    size_t slots() const override { return status.size(); }
    void export_state(uint32_t* graph_out, uint64_t* ext, uint32_t* ep, void* codes) override {
        const size_t n = status.size();
        index.experimental_escape_hatch([&](const auto& graph, const auto& data, const auto&, auto) {
            const size_t R = graph.max_degree(), dim = data.dimensions();
            for (size_t i = 0; i < n; ++i) {
                auto nb = graph.get_node(i);
                uint32_t* row = graph_out + i * (R + 1);
                row[0] = static_cast<uint32_t>(nb.size());
                for (size_t j = 0; j < R; ++j) row[1 + j] = j < nb.size() ? nb[j] : 0;
                auto d = data.get_datum(i);
                std::memcpy(static_cast<T*>(codes) + i * dim, d.data(), dim * sizeof(T));
            }
        });
        for (size_t i = 0; i < n; ++i) ext[i] = status[i] == VALID ? index.translate_internal_id(i) : ~uint64_t(0);
        *ep = index.entry_point();
    }
    void search(const float* q, size_t nq, size_t k, size_t window, size_t capacity, uint64_t* ids, float* dists)
        override {
        auto view = svs::data::ConstSimpleDataView<float>(q, nq, index.dimensions());
        auto sp = index.get_search_parameters();
        sp.buffer_config({window, capacity});
        auto result = svs::QueryResultView<size_t>(
            svs::MatrixView<size_t>(svs::make_dims(nq, k), reinterpret_cast<size_t*>(ids)),
            svs::MatrixView<float>(svs::make_dims(nq, k), dists)
        );
        index.search(result, view, sp);
    }
};

template <typename T, typename... Args> DynBase* make_metric(int metric, Args&&... args) {
    switch (metric) {
        case L2: return new DynImpl<T, svs::distance::DistanceL2>(std::forward<Args>(args)...);
        case IP: return new DynImpl<T, svs::distance::DistanceIP>(std::forward<Args>(args)...);
        case COS: return new DynImpl<T, svs::distance::DistanceCosineSimilarity>(std::forward<Args>(args)...);
        default: throw ANNEXCEPTION("bad metric {}", metric);
    }
}

// f(SQ data) for the code type.
template <typename F> DynBase* with_codes(int dtype, const void* codes, size_t n, size_t dim, float scale, float bias, F&& f) {
    switch (dtype) {
        case I8: return f(sq_of<int8_t>(codes, n, dim, scale, bias));
        case U8: return f(sq_of<uint8_t>(codes, n, dim, scale, bias));
        default: throw ANNEXCEPTION("int8 / uint8 codes only, got dtype {}", dtype);
    }
}

}  // namespace

extern "C" {

const char* svsref_dynamic_sq_last_error() { return g_error.c_str(); }

/// MutableVamanaIndex(graph, SQ data, entry_point, distance, external_ids, threads) over int8 (dtype 2) / uint8 (3)
/// codes with the given scale and bias, then every mutation parameter set (the from-graph constructor leaves
/// max_candidates_ and prune_to_ uninitialised).
void* svsref_dynamic_sq_create(int dtype, const void* codes, size_t n, size_t dim, float scale, float bias,
                               const uint32_t* graph_rows, size_t max_degree, uint32_t entry_point, int metric,
                               const uint64_t* ids, float alpha, size_t window, size_t max_candidates, size_t prune_to,
                               size_t threads) {
    DynBase* out = nullptr;
    int rc = guarded([&] {
        std::vector<size_t> ext(ids, ids + n);
        out = with_codes(dtype, codes, n, dim, scale, bias, [&](auto data) {
            using T = typename decltype(data)::element_type;
            return make_metric<T>(metric, make_graph(graph_rows, n, max_degree), std::move(data), entry_point, ext, threads);
        });
        out->set_params(alpha, window, max_candidates, prune_to);
    });
    return rc == 0 ? out : nullptr;
}

/// MutableVamanaIndex(parameters, SQ data, external_ids, distance, threads): the reference's builder (two passes).
void* svsref_dynamic_sq_build(int dtype, const void* codes, size_t n, size_t dim, float scale, float bias, int metric,
                              float alpha, size_t max_degree, size_t window, size_t max_candidates, size_t prune_to,
                              const uint64_t* ids, size_t threads) {
    DynBase* out = nullptr;
    guarded([&] {
        auto params = svs::index::vamana::VamanaBuildParameters{alpha, max_degree, window, max_candidates, prune_to, true};
        std::vector<size_t> ext(ids, ids + n);
        out = with_codes(dtype, codes, n, dim, scale, bias, [&](auto data) {
            using T = typename decltype(data)::element_type;
            return make_metric<T>(metric, params, std::move(data), ext, threads);
        });
    });
    return out;
}

void svsref_dynamic_sq_destroy(void* h) { delete static_cast<DynBase*>(h); }

int svsref_dynamic_sq_set_params(void* h, float alpha, size_t window, size_t max_candidates, size_t prune_to) {
    return guarded([&] { static_cast<DynBase*>(h)->set_params(alpha, window, max_candidates, prune_to); });
}

/// add_points (dynamic_index.h:657-749) of float32 rows [count][dim], each encoded by SQDataset::set_datum; `slots`
/// receives the slots used.
int svsref_dynamic_sq_add(void* h, const float* data, size_t count, const uint64_t* ids, int reuse_empty, uint64_t* slots) {
    return guarded([&] { static_cast<DynBase*>(h)->add(data, count, ids, reuse_empty != 0, slots); });
}

int svsref_dynamic_sq_delete(void* h, const uint64_t* ids, size_t count) {
    return guarded([&] { static_cast<DynBase*>(h)->remove(ids, count); });
}

int svsref_dynamic_sq_consolidate(void* h) { return guarded([&] { static_cast<DynBase*>(h)->consolidate(); }); }

int svsref_dynamic_sq_compact(void* h) { return guarded([&] { static_cast<DynBase*>(h)->compact(); }); }

size_t svsref_dynamic_sq_slots(void* h) { return static_cast<DynBase*>(h)->slots(); }

/// Every slot: graph uint32[slots][R+1] degree first, status (0 Empty, 1 Valid, 2 Deleted), external id (2^64 - 1 for a
/// slot that is not Valid), entry point, and the codes [slots][dim] the dataset holds.
int svsref_dynamic_sq_export(void* h, uint32_t* graph, uint8_t* status, uint64_t* ext, uint32_t* ep, void* codes) {
    return guarded([&] {
        auto* d = static_cast<DynBase*>(h);
        d->export_state(graph, ext, ep, codes);
        std::memcpy(status, d->status.data(), d->status.size());
    });
}

/// MutableVamanaIndex::search with float32 queries; ids are external ids.
int svsref_dynamic_sq_search(void* h, const float* queries, size_t nq, size_t k, size_t window, size_t capacity,
                             uint64_t* ids, float* dists) {
    return guarded([&] { static_cast<DynBase*>(h)->search(queries, nq, k, window, capacity, ids, dists); });
}

}  // extern "C"
