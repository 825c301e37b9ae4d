// oracle/_ref driver for the reference's MutableVamanaIndex -- TEST INFRASTRUCTURE ONLY (see oracle/README.md).
//
// A thin `extern "C"` façade over the *unmodified* reference headers (`-I/root/reference/include`, never copied),
// built by `make -C oracle -f dynamic.mk` into `_ref/libsvsref_dynamic.so` next to `libsvsref.so` and linked
// with the same `avx512.o` / `avx2.o` distance kernels.  Tests drive the reference's dynamic index through it:
//   index/vamana/dynamic_index.h:178-202   MutableVamanaIndex(graph, data, entry_point, distance, ids, threads)
//   index/vamana/dynamic_index.h:208-261   MutableVamanaIndex(parameters, data, ids, distance, threads)
//   index/vamana/dynamic_index.h:316-371   set_alpha / set_construction_window_size / set_max_candidates / set_prune_to
//   index/vamana/dynamic_index.h:657-1013  add_points, delete_entries, compact, consolidate
//   index/vamana/dynamic_index.h:525-571   search
//
// Nothing in the product (libsvsb200.so / scalablevectorsearch_b200) links or loads this.

#include "svs/core/data.h"
#include "svs/core/distance.h"
#include "svs/core/graph.h"
#include "svs/index/vamana/dynamic_index.h"
#include "svs/lib/float16.h"

#include <cstdint>
#include <cstring>
#include <string>
#include <vector>

namespace {

thread_local std::string g_error;

enum DType : int { F32 = 0, F16 = 1 };
enum Metric : int { L2 = 0, IP = 1, COS = 2 };

using Graph = svs::graphs::SimpleGraph<uint32_t, svs::lib::Allocator<uint32_t>>;
template <typename T> using Data = svs::data::SimpleData<T, svs::Dynamic, svs::lib::Allocator<T>>;

// `rows`: n x (max_degree + 1), element 0 the out-degree (core/graph/graph.h:103-114).
Graph make_graph(const uint32_t* rows, size_t n, size_t max_degree) {
    auto g = Graph(n, max_degree);
    for (size_t i = 0; i < n; ++i) {
        const uint32_t* r = rows + i * (max_degree + 1);
        g.replace_node(i, std::span<const uint32_t>(r + 1, r[0]));
    }
    return g;
}

template <typename T> Data<T> make_data(const void* src, size_t n, size_t dim) {
    auto d = Data<T>(n, dim);
    const T* p = static_cast<const T*>(src);
    for (size_t i = 0; i < n; ++i) {
        d.set_datum(i, std::span<const T>(p + i * dim, dim));
    }
    return d;
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

// ---- MutableVamanaIndex ----
// The façade mirrors the slot status (the reference keeps it private): Valid / Deleted / Empty change exactly where
// add_points, delete_entries, consolidate and compact change them (dynamic_index.h:657-1013).
enum Slot : uint8_t { EMPTY = 0, VALID = 1, DELETED = 2 };

struct DynBase {
    virtual ~DynBase() = default;
    std::vector<uint8_t> status;
    virtual void set_params(float alpha, size_t window, size_t max_candidates, size_t prune_to) = 0;
    virtual void add(const void* data, size_t count, const uint64_t* ids, bool reuse, uint64_t* slots) = 0;
    virtual void remove(const uint64_t* ids, size_t count) = 0;
    virtual void consolidate() = 0;
    virtual void compact() = 0;
    virtual size_t slots() const = 0;
    virtual void export_state(uint32_t* graph, uint64_t* ext, uint32_t* ep) = 0;
    virtual void search(const float* q, size_t nq, size_t k, size_t window, size_t capacity, uint64_t* ids, float* dists) = 0;
};

template <typename T, typename Dist> struct DynImpl : DynBase {
    using Index = svs::index::vamana::MutableVamanaIndex<Graph, Data<T>, Dist>;
    Index index;

    DynImpl(Graph g, Data<T> d, uint32_t ep, const std::vector<size_t>& ids, size_t threads)
        : index(std::move(g), std::move(d), ep, Dist{}, ids, threads) {
        status.assign(ids.size(), VALID);
    }
    DynImpl(const svs::index::vamana::VamanaBuildParameters& params, Data<T> d, const std::vector<size_t>& ids, size_t threads)
        : index(params, std::move(d), ids, Dist{}, threads) {
        status.assign(ids.size(), VALID);
    }

    void set_params(float alpha, size_t window, size_t max_candidates, size_t prune_to) override {
        index.set_alpha(alpha);
        index.set_construction_window_size(window);
        index.set_max_candidates(max_candidates);
        index.set_prune_to(prune_to);
    }
    void add(const void* data, size_t count, const uint64_t* ids, bool reuse, uint64_t* slots) override {
        auto view = svs::data::ConstSimpleDataView<T>(static_cast<const T*>(data), count, index.dimensions());
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
    void export_state(uint32_t* graph_out, uint64_t* ext, uint32_t* ep) override {
        const auto& graph = index.view_graph();
        const size_t R = graph.max_degree();
        for (size_t i = 0; i < status.size(); ++i) {
            auto nb = graph.get_node(i);
            uint32_t* row = graph_out + i * (R + 1);
            row[0] = static_cast<uint32_t>(nb.size());
            for (size_t j = 0; j < R; ++j) {
                row[1 + j] = j < nb.size() ? nb[j] : 0;
            }
            ext[i] = status[i] == VALID ? index.translate_internal_id(i) : ~uint64_t(0);
        }
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

template <typename T, typename... Args> DynBase* make_dynamic(int metric, Args&&... args) {
    switch (metric) {
        case L2: return new DynImpl<T, svs::distance::DistanceL2>(std::forward<Args>(args)...);
        case IP: return new DynImpl<T, svs::distance::DistanceIP>(std::forward<Args>(args)...);
        case COS:
            return new DynImpl<T, svs::distance::DistanceCosineSimilarity>(std::forward<Args>(args)...);
        default: throw ANNEXCEPTION("bad metric {}", metric);
    }
}

} // namespace

extern "C" {

const char* svsref_dynamic_last_error() { return g_error.c_str(); }

/// MutableVamanaIndex(graph, data, entry_point, distance, external_ids, threads) (dynamic_index.h:178-202), then
/// set_alpha / set_construction_window_size / set_max_candidates / set_prune_to: the from-graph constructor leaves
/// max_candidates_ and prune_to_ uninitialised.
void* svsref_dynamic_create(
    int dtype,
    const void* data,
    size_t n,
    size_t dim,
    const uint32_t* graph_rows,
    size_t max_degree,
    uint32_t entry_point,
    int metric,
    const uint64_t* ids,
    float alpha,
    size_t window,
    size_t max_candidates,
    size_t prune_to,
    size_t threads
) {
    DynBase* out = nullptr;
    int rc = guarded([&] {
        auto g = make_graph(graph_rows, n, max_degree);
        std::vector<size_t> ext(ids, ids + n);
        switch (dtype) {
            case F32: out = make_dynamic<float>(metric, std::move(g), make_data<float>(data, n, dim), entry_point, ext, threads); break;
            case F16: out = make_dynamic<svs::Float16>(metric, std::move(g), make_data<svs::Float16>(data, n, dim), entry_point, ext, threads); break;
            default: throw ANNEXCEPTION("dynamic index: f32/f16 data, got {}", dtype);
        }
        out->set_params(alpha, window, max_candidates, prune_to);
    });
    return rc == 0 ? out : nullptr;
}

/// MutableVamanaIndex(parameters, data, external_ids, distance, threads) (dynamic_index.h:208-261).
void* svsref_dynamic_build(
    int dtype,
    const void* data,
    size_t n,
    size_t dim,
    int metric,
    float alpha,
    size_t max_degree,
    size_t window,
    size_t max_candidates,
    size_t prune_to,
    const uint64_t* ids,
    size_t threads
) {
    DynBase* out = nullptr;
    int rc = guarded([&] {
        auto params = svs::index::vamana::VamanaBuildParameters{
            alpha, max_degree, window, max_candidates, prune_to, true};
        std::vector<size_t> ext(ids, ids + n);
        switch (dtype) {
            case F32: out = make_dynamic<float>(metric, params, make_data<float>(data, n, dim), ext, threads); break;
            case F16: out = make_dynamic<svs::Float16>(metric, params, make_data<svs::Float16>(data, n, dim), ext, threads); break;
            default: throw ANNEXCEPTION("dynamic index: f32/f16 data, got {}", dtype);
        }
    });
    return rc == 0 ? out : nullptr;
}

void svsref_dynamic_destroy(void* h) { delete static_cast<DynBase*>(h); }

int svsref_dynamic_set_params(void* h, float alpha, size_t window, size_t max_candidates, size_t prune_to) {
    return guarded([&] { static_cast<DynBase*>(h)->set_params(alpha, window, max_candidates, prune_to); });
}

/// add_points (dynamic_index.h:657-749): rows of the index's element type; `slots` receives the slots used.
int svsref_dynamic_add(void* h, const void* data, size_t count, const uint64_t* ids, int reuse_empty, uint64_t* slots) {
    return guarded([&] { static_cast<DynBase*>(h)->add(data, count, ids, reuse_empty != 0, slots); });
}

int svsref_dynamic_delete(void* h, const uint64_t* ids, size_t count) {
    return guarded([&] { static_cast<DynBase*>(h)->remove(ids, count); });
}

int svsref_dynamic_consolidate(void* h) {
    return guarded([&] { static_cast<DynBase*>(h)->consolidate(); });
}

int svsref_dynamic_compact(void* h) {
    return guarded([&] { static_cast<DynBase*>(h)->compact(); });
}

size_t svsref_dynamic_slots(void* h) { return static_cast<DynBase*>(h)->slots(); }

/// Every slot: graph uint32[slots][R+1] degree first, status (0 Empty, 1 Valid, 2 Deleted), external id (2^64 - 1
/// for a slot that is not Valid), entry point.
int svsref_dynamic_export(void* h, uint32_t* graph, uint8_t* status, uint64_t* ext, uint32_t* ep) {
    return guarded([&] {
        auto* d = static_cast<DynBase*>(h);
        d->export_state(graph, ext, ep);
        std::memcpy(status, d->status.data(), d->status.size());
    });
}

/// MutableVamanaIndex::search with float32 queries; ids are external ids.
int svsref_dynamic_search(
    void* h, const float* queries, size_t nq, size_t k, size_t window, size_t capacity, uint64_t* ids, float* dists
) {
    return guarded([&] {
        static_cast<DynBase*>(h)->search(queries, nq, k, window, capacity, ids, dists);
    });
}

} // extern "C"
