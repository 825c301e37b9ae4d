// oracle/_ref driver for the reference's DynamicFlatIndex -- TEST INFRASTRUCTURE ONLY (see oracle/README.md).
//
// A thin `extern "C"` façade over the *unmodified* reference headers (`-I/root/reference/include`, never copied),
// built by `make -C oracle -f dynamic_flat.mk` into `_ref/libsvsref_dynamic_flat.so` next to `libsvsref.so` and linked
// with the same `avx512.o` / `avx2.o` distance kernels.  Tests drive the reference's dynamic flat index through it:
//   index/flat/dynamic_flat.h:94-113    DynamicFlatIndex(data, external_ids, distance, threadpool)
//   index/flat/dynamic_flat.h:214-276   add_points
//   index/flat/dynamic_flat.h:292-307   delete_entries
//   index/flat/dynamic_flat.h:335-367   compact
//   index/flat/dynamic_flat.h:513-573   search
// over SimpleData<T, Dynamic, Blocked<lib::Allocator<T>>> (the blocked layout add_points resizes) for float32,
// float16, int8 and uint8 rows and the three distances.
//
// Nothing in the product (libsvsb200.so / scalablevectorsearch_b200) links or loads this.

#include "svs/core/data.h"
#include "svs/core/distance.h"
#include "svs/index/flat/dynamic_flat.h"
#include "svs/lib/float16.h"

#include <cstdint>
#include <algorithm>
#include <string>
#include <type_traits>
#include <vector>

namespace {

thread_local std::string g_error;

enum DType : int { F32 = 0, F16 = 1, I8 = 2, U8 = 3 };
enum Metric : int { L2 = 0, IP = 1, COS = 2 };

template <typename T> using Data = svs::data::SimpleData<T, svs::Dynamic, svs::data::Blocked<svs::lib::Allocator<T>>>;

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

// Every slot's status is the reference's own `is_valid(i)` (dynamic_flat.h:311).  Only the number of slots is kept here
// (the reference keeps its data's size private): the largest slot add_points returned + 1, `size()` after compact.
enum Slot : uint8_t { EMPTY = 0, VALID = 1 };

struct FlatBase {
    virtual ~FlatBase() = default;
    size_t nslots = 0;
    virtual void add(const void* data, size_t count, const uint64_t* ids, bool reuse, uint64_t* slots) = 0;
    virtual void remove(const uint64_t* ids, size_t count) = 0;
    virtual void compact() = 0;
    virtual size_t size() const = 0;
    virtual void all_ids(uint64_t* out) const = 0;
    virtual void export_state(uint8_t* status, uint64_t* ext) const = 0;
    // queries: float32 for float rows, the rows' own type for int8 / uint8 rows
    virtual void search(const void* q, size_t nq, size_t k, uint64_t* ids, float* dists) = 0;
};

template <typename T, typename Dist> struct FlatImpl : FlatBase {
    using Index = svs::index::flat::DynamicFlatIndex<Data<T>, Dist>;
    using Q = std::conditional_t<std::is_integral_v<T>, T, float>;
    Index index;

    FlatImpl(Data<T> d, const std::vector<size_t>& ids, size_t threads) : index(std::move(d), ids, Dist{}, threads) {
        nslots = ids.size();
    }

    void add(const void* data, size_t count, const uint64_t* ids, bool reuse, uint64_t* slots) override {
        auto view = svs::data::ConstSimpleDataView<T>(static_cast<const T*>(data), count, index.dimensions());
        std::vector<size_t> ext(ids, ids + count);
        auto got = index.add_points(view, ext, reuse);
        for (size_t i = 0; i < got.size(); ++i) {
            slots[i] = got[i];
            nslots = std::max<size_t>(nslots, got[i] + 1);
        }
    }
    void remove(const uint64_t* ids, size_t count) override {
        std::vector<size_t> ext(ids, ids + count);
        index.delete_entries(ext);
    }
    void compact() override {
        index.compact();
        nslots = index.size();
    }
    size_t size() const override { return index.size(); }
    void all_ids(uint64_t* out) const override {
        auto ids = index.external_ids();
        for (size_t i = 0; i < ids.size(); ++i) out[i] = ids[i];
    }
    void export_state(uint8_t* status, uint64_t* ext) const override {
        for (size_t i = 0; i < nslots; ++i) {
            const bool valid = index.is_valid(i);
            status[i] = valid ? VALID : EMPTY;
            ext[i] = valid ? index.translate_internal_id(i) : ~uint64_t(0);
        }
    }
    void search(const void* q, size_t nq, size_t k, uint64_t* ids, float* dists) override {
        auto view = svs::data::ConstSimpleDataView<Q>(static_cast<const Q*>(q), nq, index.dimensions());
        auto result = svs::QueryResultView<size_t>(
            svs::MatrixView<size_t>(svs::make_dims(nq, k), reinterpret_cast<size_t*>(ids)),
            svs::MatrixView<float>(svs::make_dims(nq, k), dists)
        );
        index.search(result, view, index.get_search_parameters());
    }
};

template <typename T> Data<T> make_data(const void* src, size_t n, size_t dim) {
    auto d = Data<T>(n, dim);
    const T* p = static_cast<const T*>(src);
    for (size_t i = 0; i < n; ++i) {
        d.set_datum(i, std::span<const T>(p + i * dim, dim));
    }
    return d;
}

template <typename T> FlatBase* make_flat(int metric, const void* data, size_t n, size_t dim, const std::vector<size_t>& ids,
                                          size_t threads) {
    switch (metric) {
        case L2: return new FlatImpl<T, svs::distance::DistanceL2>(make_data<T>(data, n, dim), ids, threads);
        case IP: return new FlatImpl<T, svs::distance::DistanceIP>(make_data<T>(data, n, dim), ids, threads);
        case COS: return new FlatImpl<T, svs::distance::DistanceCosineSimilarity>(make_data<T>(data, n, dim), ids, threads);
        default: throw ANNEXCEPTION("bad metric {}", metric);
    }
}

} // namespace

extern "C" {

const char* svsref_dynamic_flat_last_error() { return g_error.c_str(); }

/// DynamicFlatIndex(data, external_ids, distance, threads) (dynamic_flat.h:94-113).
void* svsref_dynamic_flat_create(int dtype, const void* data, size_t n, size_t dim, int metric, const uint64_t* ids,
                                 size_t threads) {
    FlatBase* out = nullptr;
    int rc = guarded([&] {
        std::vector<size_t> ext(ids, ids + n);
        switch (dtype) {
            case F32: out = make_flat<float>(metric, data, n, dim, ext, threads); break;
            case F16: out = make_flat<svs::Float16>(metric, data, n, dim, ext, threads); break;
            case I8: out = make_flat<int8_t>(metric, data, n, dim, ext, threads); break;
            case U8: out = make_flat<uint8_t>(metric, data, n, dim, ext, threads); break;
            default: throw ANNEXCEPTION("dynamic flat index: bad dtype {}", dtype);
        }
    });
    return rc == 0 ? out : nullptr;
}

void svsref_dynamic_flat_destroy(void* h) { delete static_cast<FlatBase*>(h); }

/// add_points (dynamic_flat.h:214-276): rows of the index's element type; `slots` receives the slots used.
int svsref_dynamic_flat_add(void* h, const void* data, size_t count, const uint64_t* ids, int reuse_empty, uint64_t* slots) {
    return guarded([&] { static_cast<FlatBase*>(h)->add(data, count, ids, reuse_empty != 0, slots); });
}

int svsref_dynamic_flat_delete(void* h, const uint64_t* ids, size_t count) {
    return guarded([&] { static_cast<FlatBase*>(h)->remove(ids, count); });
}

int svsref_dynamic_flat_compact(void* h) {
    return guarded([&] { static_cast<FlatBase*>(h)->compact(); });
}

size_t svsref_dynamic_flat_slots(void* h) { return static_cast<FlatBase*>(h)->nslots; }
size_t svsref_dynamic_flat_size(void* h) { return static_cast<FlatBase*>(h)->size(); }

/// external_ids (dynamic_flat.h:192-197): the external ids of the Valid slots, in slot order.
int svsref_dynamic_flat_all_ids(void* h, uint64_t* out) {
    return guarded([&] { static_cast<FlatBase*>(h)->all_ids(out); });
}

/// Every slot: status (is_valid: 0 Empty, 1 Valid) and external id (2^64 - 1 for an Empty slot).
int svsref_dynamic_flat_export(void* h, uint8_t* status, uint64_t* ext) {
    return guarded([&] { static_cast<FlatBase*>(h)->export_state(status, ext); });
}

/// DynamicFlatIndex::search (dynamic_flat.h:513-573); ids are external ids.  Queries: float32 over float rows, the
/// rows' own type over int8 / uint8 rows.
int svsref_dynamic_flat_search(void* h, const void* queries, size_t nq, size_t k, uint64_t* ids, float* dists) {
    return guarded([&] { static_cast<FlatBase*>(h)->search(queries, nq, k, ids, dists); });
}

} // extern "C"
