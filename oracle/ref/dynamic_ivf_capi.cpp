// oracle/_ref driver for the reference's dynamic IVF index -- TEST INFRASTRUCTURE ONLY (see oracle/README.md).
//
// A thin `extern "C"` façade over the *unmodified* reference headers (`-I/root/reference/include`, never copied),
// built by `make -C oracle -f dynamic_ivf.mk` into `_ref/libsvsref_dynamic_ivf.so` and linked with the same `avx512.o`
// / `avx2.o` distance kernels as `libsvsref.so`.  It holds one DynamicIVFIndex (index/ivf/dynamic_ivf.h) per handle:
//   assemble_dynamic_from_clustering (:1127-1190), add_points (:475-504), delete_entries (:514-530), compact (:547-636),
//   external_ids (:456-461), search (:675-730; centroids ranked from cblas_sgemm, defined below as plain loops, as in
//   ref/ivf_capi.cpp).  float32 rows and queries; L2, inner product and cosine.
//
// Nothing in the product (libsvsb200.so / scalablevectorsearch_b200) links or loads this.

#include "svs/core/data.h"
#include "svs/core/distance.h"
#include "svs/index/ivf/dynamic_ivf.h"

#include <cstdint>
#include <cstring>
#include <memory>
#include <string>
#include <vector>

namespace {

thread_local std::string g_error;

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

// C = alpha A B^T + beta C (row-major, A m x k, B n x k): the only form the IVF code uses.
void gemm_abt(int m, int n, int k, float alpha, const float* a, int lda, const float* b, int ldb, float beta, float* c,
              int ldc) {
    for (int i = 0; i < m; ++i)
        for (int j = 0; j < n; ++j) {
            float s = 0.0f;
            for (int p = 0; p < k; ++p) s += a[size_t(i) * lda + p] * b[size_t(j) * ldb + p];
            float& out = c[size_t(i) * ldc + j];
            out = alpha * s + (beta == 0.0f ? 0.0f : beta * out);
        }
}

svs::data::SimpleData<float> rows_of(const float* x, size_t n, size_t dim) {
    auto rows = svs::data::SimpleData<float>(n, dim);
    for (size_t i = 0; i < n; ++i) rows.set_datum(i, std::span<const float>(x + i * dim, dim));
    return rows;
}

struct Handle {
    virtual ~Handle() = default;
    virtual void add(const float* x, size_t n, const uint64_t* ids, bool reuse, uint64_t* slots) = 0;
    virtual void remove(const uint64_t* ids, size_t n) = 0;
    virtual void compact() = 0;
    virtual std::vector<size_t> all_ids() const = 0;
    virtual void search(const float* q, size_t nq, size_t k, size_t n_probes, uint64_t* ids, float* dists) = 0;
    size_t dim = 0;
};

template <typename Index> struct Impl final : Handle {
    explicit Impl(Index&& ix) : index(std::move(ix)) {}
    void add(const float* x, size_t n, const uint64_t* ids, bool reuse, uint64_t* slots) override {
        auto rows = rows_of(x, n, dim);
        std::vector<size_t> ext(ids, ids + n);
        auto got = index.add_points(rows, ext, reuse);
        for (size_t i = 0; i < got.size(); ++i) slots[i] = got[i];
    }
    void remove(const uint64_t* ids, size_t n) override { index.delete_entries(std::vector<size_t>(ids, ids + n)); }
    void compact() override { index.compact(); }
    std::vector<size_t> all_ids() const override { return index.external_ids(); }
    void search(const float* q, size_t nq, size_t k, size_t n_probes, uint64_t* ids, float* dists) override {
        auto queries = svs::data::ConstSimpleDataView<float>(q, nq, dim);
        auto result = svs::QueryResultView<size_t>(
            svs::MatrixView<size_t>(svs::make_dims(nq, k), reinterpret_cast<size_t*>(ids)),
            svs::MatrixView<float>(svs::make_dims(nq, k), dists));
        index.search(result, queries, svs::index::ivf::IVFSearchParameters(n_probes, 1.0f));
    }
    Index index;
};

template <typename Dist> Handle* make(const float* data, size_t n, size_t dim, const float* centroids, size_t C,
                                      const uint32_t* assignments, const uint64_t* ids) {
    auto rows = rows_of(data, n, dim);
    auto cent = rows_of(centroids, C, dim);
    std::vector<std::vector<uint32_t>> clusters(C);
    for (size_t i = 0; i < n; ++i) clusters.at(assignments[i]).push_back(uint32_t(i));
    auto clustering = svs::index::ivf::Clustering<svs::data::SimpleData<float>, uint32_t>(std::move(cent), std::move(clusters));
    std::vector<size_t> ext(ids, ids + n);
    auto index = svs::index::ivf::assemble_dynamic_from_clustering(std::move(clustering), rows, std::span<const size_t>(ext),
                                                                   Dist(), size_t(1));
    auto* h = new Impl<decltype(index)>(std::move(index));
    h->dim = dim;
    return h;
}

} // namespace

extern "C" {

void cblas_sgemm(CBLAS_LAYOUT, CBLAS_TRANSPOSE, CBLAS_TRANSPOSE, int m, int n, int k, float alpha, const float* a, int lda,
                 const float* b, int ldb, float beta, float* c, int ldc) {
    gemm_abt(m, n, k, alpha, a, lda, b, ldb, beta, c, ldc);
}
void cblas_gemm_f16f16f32(CBLAS_LAYOUT, CBLAS_TRANSPOSE, CBLAS_TRANSPOSE, int, int, int, float, const uint16_t*, int,
                          const uint16_t*, int, float, float*, int) {
    throw std::runtime_error("float16 centroids are not used by this façade");
}
void cblas_gemm_bf16bf16f32(CBLAS_LAYOUT, CBLAS_TRANSPOSE, CBLAS_TRANSPOSE, int, int, int, float, const uint16_t*, int,
                            const uint16_t*, int, float, float*, int) {
    throw std::runtime_error("bfloat16 centroids are not used by this façade");
}

const char* svsref_dynivf_last_error() { return g_error.c_str(); }

/// assemble_dynamic_from_clustering: float32 rows [n][dim] with external ids [n], centroids [C][dim], assignments [n];
/// metric 0 L2, 1 inner product, 2 cosine.
int svsref_dynivf_create(const float* data, size_t n, size_t dim, int metric, const float* centroids, size_t C,
                         const uint32_t* assignments, const uint64_t* ids, void** out) {
    return guarded([&] {
        if (metric == 0) *out = make<svs::distance::DistanceL2>(data, n, dim, centroids, C, assignments, ids);
        else if (metric == 1) *out = make<svs::distance::DistanceIP>(data, n, dim, centroids, C, assignments, ids);
        else *out = make<svs::distance::DistanceCosineSimilarity>(data, n, dim, centroids, C, assignments, ids);
    });
}
void svsref_dynivf_destroy(void* h) { delete static_cast<Handle*>(h); }
int svsref_dynivf_add(void* h, const float* x, size_t n, const uint64_t* ids, int reuse_empty, uint64_t* slots_out) {
    return guarded([&] { static_cast<Handle*>(h)->add(x, n, ids, reuse_empty != 0, slots_out); });
}
int svsref_dynivf_delete(void* h, const uint64_t* ids, size_t n) {
    return guarded([&] { static_cast<Handle*>(h)->remove(ids, n); });
}
int svsref_dynivf_compact(void* h) {
    return guarded([&] { static_cast<Handle*>(h)->compact(); });
}
/// The external ids in slot order; *count: room on entry (out may be NULL), ids on return.
int svsref_dynivf_all_ids(void* h, uint64_t* out, size_t* count) {
    return guarded([&] {
        auto ids = static_cast<Handle*>(h)->all_ids();
        if (out) {
            if (*count < ids.size()) throw std::runtime_error("output too small");
            for (size_t i = 0; i < ids.size(); ++i) out[i] = ids[i];
        }
        *count = ids.size();
    });
}
int svsref_dynivf_search(void* h, const float* queries, size_t nq, size_t k, size_t n_probes, uint64_t* ids, float* dists) {
    return guarded([&] { static_cast<Handle*>(h)->search(queries, nq, k, n_probes, ids, dists); });
}

} // extern "C"
