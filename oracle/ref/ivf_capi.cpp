// oracle/_ref driver for the reference's IVF index -- TEST INFRASTRUCTURE ONLY (see oracle/README.md).
//
// A thin `extern "C"` façade over the *unmodified* reference headers (`-I/root/reference/include`, never copied),
// built by `make -C oracle -f ivf.mk` into `_ref/libsvsref_ivf.so` next to `libsvsref.so` and linked with the same
// `avx512.o` / `avx2.o` distance kernels.  Tests hand it a clustering (float32 centroids and one cluster per row) and
// search the reference's index with a given n_probes:
//   index/ivf/clustering.h:104-106   Clustering(centroids, clusters)
//   index/ivf/index.h:888-920        assemble_from_clustering
//   index/ivf/index.h:410-460        IVFIndex::search (centroids ranked from cblas_sgemm, common.h:641-684)
// The reference includes <mkl.h>; ref/shims/mkl.h declares the three CBLAS entry points it calls, defined below as
// plain loops.  float32 rows and queries; L2, inner product and cosine.
//
// Nothing in the product (libsvsb200.so / scalablevectorsearch_b200) links or loads this.

#include "svs/core/data.h"
#include "svs/core/distance.h"
#include "svs/index/ivf/index.h"

#include <cstdint>
#include <cstring>
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

float from_f16(uint16_t h) {
    const uint32_t sign = uint32_t(h & 0x8000u) << 16, exp = (h >> 10) & 0x1Fu, mant = h & 0x3FFu;
    float v;
    if (exp == 0) {
        v = float(mant) * 0x1p-24f;
    } else if (exp == 31) {
        v = mant ? __builtin_nanf("") : __builtin_inff();
    } else {
        v = std::ldexp(float(mant | 0x400u), int(exp) - 25);
    }
    uint32_t bits;
    std::memcpy(&bits, &v, 4);
    bits |= sign;
    std::memcpy(&v, &bits, 4);
    return v;
}
float from_bf16(uint16_t h) {
    const uint32_t bits = uint32_t(h) << 16;
    float v;
    std::memcpy(&v, &bits, 4);
    return v;
}

// C = alpha A B^T + beta C (row-major, A m x k, B n x k): the only form common.h uses.
template <typename T, typename Cvt>
void gemm_abt(int m, int n, int k, float alpha, const T* a, int lda, const T* b, int ldb, float beta, float* c, int ldc,
              Cvt cvt) {
    for (int i = 0; i < m; ++i)
        for (int j = 0; j < n; ++j) {
            float s = 0.0f;
            for (int p = 0; p < k; ++p) s += cvt(a[size_t(i) * lda + p]) * cvt(b[size_t(j) * ldb + p]);
            float& out = c[size_t(i) * ldc + j];
            out = alpha * s + (beta == 0.0f ? 0.0f : beta * out);
        }
}

template <typename Dist> void run(const float* data, size_t n, size_t dim, const float* centroids, size_t C,
                                  const uint32_t* assignments, const float* queries, size_t nq, size_t k, size_t n_probes,
                                  uint64_t* ids, float* dists) {
    auto rows = svs::data::SimpleData<float>(n, dim);
    for (size_t i = 0; i < n; ++i) rows.set_datum(i, std::span<const float>(data + i * dim, dim));
    auto cent = svs::data::SimpleData<float>(C, dim);
    for (size_t c = 0; c < C; ++c) cent.set_datum(c, std::span<const float>(centroids + c * dim, dim));
    std::vector<std::vector<uint32_t>> clusters(C);
    for (size_t i = 0; i < n; ++i) clusters.at(assignments[i]).push_back(uint32_t(i));
    auto clustering = svs::index::ivf::Clustering<svs::data::SimpleData<float>, uint32_t>(std::move(cent), std::move(clusters));
    auto index = svs::index::ivf::assemble_from_clustering(std::move(clustering), rows, Dist(), size_t(1));
    auto q = svs::data::ConstSimpleDataView<float>(queries, nq, dim);
    auto result = svs::QueryResultView<size_t>(svs::MatrixView<size_t>(svs::make_dims(nq, k), reinterpret_cast<size_t*>(ids)),
                                               svs::MatrixView<float>(svs::make_dims(nq, k), dists));
    index.search(result, q, svs::index::ivf::IVFSearchParameters(n_probes, 1.0f));
}

} // namespace

extern "C" {

void cblas_sgemm(CBLAS_LAYOUT, CBLAS_TRANSPOSE, CBLAS_TRANSPOSE, int m, int n, int k, float alpha, const float* a, int lda,
                 const float* b, int ldb, float beta, float* c, int ldc) {
    gemm_abt(m, n, k, alpha, a, lda, b, ldb, beta, c, ldc, [](float x) { return x; });
}
void cblas_gemm_f16f16f32(CBLAS_LAYOUT, CBLAS_TRANSPOSE, CBLAS_TRANSPOSE, int m, int n, int k, float alpha, const uint16_t* a,
                          int lda, const uint16_t* b, int ldb, float beta, float* c, int ldc) {
    gemm_abt(m, n, k, alpha, a, lda, b, ldb, beta, c, ldc, from_f16);
}
void cblas_gemm_bf16bf16f32(CBLAS_LAYOUT, CBLAS_TRANSPOSE, CBLAS_TRANSPOSE, int m, int n, int k, float alpha,
                            const uint16_t* a, int lda, const uint16_t* b, int ldb, float beta, float* c, int ldc) {
    gemm_abt(m, n, k, alpha, a, lda, b, ldb, beta, c, ldc, from_bf16);
}

const char* svsref_ivf_last_error() { return g_error.c_str(); }

/// assemble_from_clustering + search: float32 rows [n][dim], centroids [C][dim], assignments [n] (each < C), float32
/// queries [nq][dim]; metric 0 L2, 1 inner product, 2 cosine; ids uint64 [nq][k], distances float32 [nq][k].
int svsref_ivf_search(const float* data, size_t n, size_t dim, int metric, const float* centroids, size_t C,
                      const uint32_t* assignments, const float* queries, size_t nq, size_t k, size_t n_probes, uint64_t* ids,
                      float* dists) {
    return guarded([&] {
        if (metric == 0)
            run<svs::distance::DistanceL2>(data, n, dim, centroids, C, assignments, queries, nq, k, n_probes, ids, dists);
        else if (metric == 1)
            run<svs::distance::DistanceIP>(data, n, dim, centroids, C, assignments, queries, nq, k, n_probes, ids, dists);
        else
            run<svs::distance::DistanceCosineSimilarity>(data, n, dim, centroids, C, assignments, queries, nq, k, n_probes,
                                                         ids, dists);
    });
}

} // extern "C"
