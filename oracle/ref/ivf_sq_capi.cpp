// oracle/_ref driver for the reference's IVF index over scalar-quantised rows -- TEST INFRASTRUCTURE ONLY (see
// oracle/README.md).
//
// A thin `extern "C"` façade over the *unmodified* reference headers (`-I/root/reference/include`, never copied),
// built by `make -C oracle -f ivf_sq.mk` into `_ref/libsvsref_ivf_sq.so` and linked with the same `avx512.o` / `avx2.o`
// distance kernels as `libsvsref.so`.  Tests hand it float32 rows, a clustering and queries; it compresses the rows
// with the reference's own SQDataset<int8_t / uint8_t>::compress and searches the reference's IVF index over them:
//   quantization/scalar/scalar.h:447-469   SQDataset::compress
//   extensions/ivf/scalar.h                the SQ leaf distances and dense clusters of IVF
//   index/ivf/index.h:888-920              assemble_from_clustering
//   index/ivf/index.h:410-460              IVFIndex::search (centroids ranked from cblas_sgemm)
// The reference includes <mkl.h>; ref/shims/mkl.h declares the CBLAS entry points, defined here as plain loops.
//
// Nothing in the product (libsvsb200.so / scalablevectorsearch_b200) links or loads this.

#include "svs/core/data.h"
#include "svs/core/distance.h"
#include "svs/extensions/ivf/scalar.h"
#include "svs/index/ivf/index.h"
#include "svs/quantization/scalar/scalar.h"

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

// C = alpha A B^T + beta C (row-major, A m x k, B n x k): the only form the IVF probe uses.
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

template <typename T, typename Dist>
void run(const float* data, size_t n, size_t dim, const float* centroids, size_t C, const uint32_t* assignments,
         const float* queries, size_t nq, size_t k, size_t n_probes, uint64_t* ids, float* dists, void* codes_out,
         float* scale_out, float* bias_out) {
    auto rows = svs::data::SimpleData<float>(n, dim);
    for (size_t i = 0; i < n; ++i) rows.set_datum(i, std::span<const float>(data + i * dim, dim));
    auto sq = svs::quantization::scalar::SQDataset<T>::compress(rows);
    *scale_out = sq.get_scale();
    *bias_out = sq.get_bias();
    for (size_t i = 0; i < n; ++i) {
        auto d = sq.get_datum(i);
        std::memcpy(static_cast<T*>(codes_out) + i * dim, d.data(), dim * sizeof(T));
    }
    auto cent = svs::data::SimpleData<float>(C, dim);
    for (size_t c = 0; c < C; ++c) cent.set_datum(c, std::span<const float>(centroids + c * dim, dim));
    std::vector<std::vector<uint32_t>> clusters(C);
    for (size_t i = 0; i < n; ++i) clusters.at(assignments[i]).push_back(uint32_t(i));
    auto clustering = svs::index::ivf::Clustering<svs::data::SimpleData<float>, uint32_t>(std::move(cent), std::move(clusters));
    auto index = svs::index::ivf::assemble_from_clustering(std::move(clustering), sq, Dist(), size_t(1));
    auto q = svs::data::ConstSimpleDataView<float>(queries, nq, dim);
    auto result = svs::QueryResultView<size_t>(svs::MatrixView<size_t>(svs::make_dims(nq, k), reinterpret_cast<size_t*>(ids)),
                                               svs::MatrixView<float>(svs::make_dims(nq, k), dists));
    index.search(result, q, svs::index::ivf::IVFSearchParameters(n_probes, 1.0f));
}

template <typename T>
void by_metric(int metric, const float* data, size_t n, size_t dim, const float* centroids, size_t C,
               const uint32_t* assignments, const float* queries, size_t nq, size_t k, size_t n_probes, uint64_t* ids,
               float* dists, void* codes_out, float* scale_out, float* bias_out) {
    if (metric == 0)
        run<T, svs::distance::DistanceL2>(data, n, dim, centroids, C, assignments, queries, nq, k, n_probes, ids, dists,
                                          codes_out, scale_out, bias_out);
    else if (metric == 1)
        run<T, svs::distance::DistanceIP>(data, n, dim, centroids, C, assignments, queries, nq, k, n_probes, ids, dists,
                                          codes_out, scale_out, bias_out);
    else
        run<T, svs::distance::DistanceCosineSimilarity>(data, n, dim, centroids, C, assignments, queries, nq, k, n_probes,
                                                        ids, dists, codes_out, scale_out, bias_out);
}

} // namespace

extern "C" {

void cblas_sgemm(CBLAS_LAYOUT, CBLAS_TRANSPOSE, CBLAS_TRANSPOSE, int m, int n, int k, float alpha, const float* a, int lda,
                 const float* b, int ldb, float beta, float* c, int ldc) {
    gemm_abt(m, n, k, alpha, a, lda, b, ldb, beta, c, ldc);
}
void cblas_gemm_f16f16f32(CBLAS_LAYOUT, CBLAS_TRANSPOSE, CBLAS_TRANSPOSE, int, int, int, float, const uint16_t*, int,
                          const uint16_t*, int, float, float*, int) {
    throw std::runtime_error("float16 GEMM is not used by the SQ façade");
}
void cblas_gemm_bf16bf16f32(CBLAS_LAYOUT, CBLAS_TRANSPOSE, CBLAS_TRANSPOSE, int, int, int, float, const uint16_t*, int,
                            const uint16_t*, int, float, float*, int) {
    throw std::runtime_error("bfloat16 GEMM is not used by the SQ façade");
}

const char* svsref_ivf_sq_last_error() { return g_error.c_str(); }

/// SQDataset<int8_t> (code_type 2) or <uint8_t> (3)::compress of float32 rows [n][dim], assemble_from_clustering with
/// centroids [C][dim] and assignments [n], search of float32 queries [nq][dim]; metric 0 L2, 1 inner product, 2
/// cosine.  Outputs: ids uint64 [nq][k], distances float32 [nq][k], the codes [n][dim], scale and bias.
int svsref_ivf_sq_search(const float* data, size_t n, size_t dim, int code_type, int metric, const float* centroids, size_t C,
                         const uint32_t* assignments, const float* queries, size_t nq, size_t k, size_t n_probes,
                         uint64_t* ids, float* dists, void* codes_out, float* scale_out, float* bias_out) {
    return guarded([&] {
        if (code_type == 2)
            by_metric<int8_t>(metric, data, n, dim, centroids, C, assignments, queries, nq, k, n_probes, ids, dists,
                              codes_out, scale_out, bias_out);
        else if (code_type == 3)
            by_metric<uint8_t>(metric, data, n, dim, centroids, C, assignments, queries, nq, k, n_probes, ids, dists,
                               codes_out, scale_out, bias_out);
        else
            throw std::runtime_error("code_type must be 2 (int8) or 3 (uint8)");
    });
}

} // extern "C"
