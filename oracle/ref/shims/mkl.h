// oracle/ref/shims/mkl.h -- TEST INFRASTRUCTURE ONLY (see oracle/README.md).
//
// A from-scratch stand-in for the three CBLAS entry points the reference's IVF code calls
// (include/svs/index/ivf/common.h) and the enums they take, so that the IVF façade (ref/ivf_capi.cpp) builds without
// a BLAS.  Declarations only; ref/ivf_capi.cpp defines them as plain row-major loops (float32 accumulation in k order).
#pragma once

#include <cstdint>

enum CBLAS_LAYOUT { CblasRowMajor = 101, CblasColMajor = 102 };
enum CBLAS_TRANSPOSE { CblasNoTrans = 111, CblasTrans = 112, CblasConjTrans = 113 };

extern "C" {
void cblas_sgemm(CBLAS_LAYOUT layout, CBLAS_TRANSPOSE ta, CBLAS_TRANSPOSE tb, int m, int n, int k, float alpha,
                 const float* a, int lda, const float* b, int ldb, float beta, float* c, int ldc);
void cblas_gemm_f16f16f32(CBLAS_LAYOUT layout, CBLAS_TRANSPOSE ta, CBLAS_TRANSPOSE tb, int m, int n, int k, float alpha,
                          const uint16_t* a, int lda, const uint16_t* b, int ldb, float beta, float* c, int ldc);
void cblas_gemm_bf16bf16f32(CBLAS_LAYOUT layout, CBLAS_TRANSPOSE ta, CBLAS_TRANSPOSE tb, int m, int n, int k, float alpha,
                            const uint16_t* a, int lda, const uint16_t* b, int ldb, float beta, float* c, int ldc);
}
