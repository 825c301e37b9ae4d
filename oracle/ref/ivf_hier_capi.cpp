// oracle/_ref driver for the reference's hierarchical k-means -- TEST INFRASTRUCTURE ONLY (see oracle/README.md).
//
// A thin `extern "C"` façade over the *unmodified* reference headers (`-I/root/reference/include`, never copied),
// built by `make -C oracle -f ivf_hier.mk` into `_ref/libsvsref_ivf_hier.so` and linked with the same `avx512.o` /
// `avx2.o` distance kernels as `libsvsref.so`.  It runs
//   index/ivf/hierarchical_kmeans.h:68-358   hierarchical_kmeans_clustering<float>
// on float32 rows and returns the centroids and every row's cluster.  The reference draws from std::mt19937 and ranks
// centroids from cblas_sgemm, so its clustering is not the library's bit for bit; tests compare what an IVF index over
// each clustering recalls.  The reference includes <mkl.h>; ref/shims/mkl.h declares the three CBLAS entry points it
// calls, defined below as plain loops (as in ivf_capi.cpp).
//
// Nothing in the product (libsvsb200.so / scalablevectorsearch_b200) links or loads this.

#include "svs/core/data.h"
#include "svs/core/distance.h"
#include "svs/index/ivf/hierarchical_kmeans.h"

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

template <typename Dist> void run(const float* data, size_t n, size_t dim, const svs::index::ivf::IVFBuildParameters& bp,
                                  float* centroids, uint32_t* assignments) {
    auto rows = svs::data::SimpleData<float>(n, dim);
    for (size_t i = 0; i < n; ++i) rows.set_datum(i, std::span<const float>(data + i * dim, dim));
    auto distance = Dist();
    auto pool = svs::threads::SequentialThreadPool();
    auto [cent, clusters] = svs::index::ivf::hierarchical_kmeans_clustering<float>(bp, rows, distance, pool);
    for (size_t c = 0; c < cent.size(); ++c) {
        const auto row = cent.get_datum(c);
        std::copy(row.begin(), row.end(), centroids + c * dim);
    }
    for (size_t c = 0; c < clusters.size(); ++c)
        for (auto i : clusters[c]) assignments[i] = uint32_t(c);
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

const char* svsref_ivf_hier_last_error() { return g_error.c_str(); }

/// hierarchical_kmeans_clustering over float32 rows [n][dim]; metric 0 L2, 1 inner product, 2 cosine; centroids float32
/// [C][dim] (level-1 groups in order), assignments uint32 [n].
int svsref_ivf_cluster_hierarchical(const float* data, size_t n, size_t dim, int metric, size_t num_centroids,
                                    size_t level1_clusters, size_t minibatch_size, size_t num_iterations,
                                    float training_fraction, uint64_t seed, float* centroids, uint32_t* assignments) {
    return guarded([&] {
        const svs::index::ivf::IVFBuildParameters bp(num_centroids, minibatch_size, num_iterations, true, training_fraction,
                                                     level1_clusters, seed);
        if (metric == 0)
            run<svs::distance::DistanceL2>(data, n, dim, bp, centroids, assignments);
        else if (metric == 1)
            run<svs::distance::DistanceIP>(data, n, dim, bp, centroids, assignments);
        else
            run<svs::distance::DistanceCosineSimilarity>(data, n, dim, bp, centroids, assignments);
    });
}

} // extern "C"
