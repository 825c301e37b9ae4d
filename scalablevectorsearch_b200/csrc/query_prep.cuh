// query_prep.cuh -- the element and per-query rules of query preparation (distance::maybe_fix_argument), shared by the
// search's prepare_queries_kernel (search.cu), the graph builder's preparation of an SQ datum as its own query
// (build_kernels.cuh, stage_sq_datum) and the hierarchical k-means's rows prepared as queries (ivf_kernel.cuh,
// ivf_group_assign_kernel).
#pragma once

#include "common.cuh"

namespace svsb200 {

// Float16 -> float the way non-SIMD reference code does it (lib/float16.h:45-52):
// subnormals flush to signed zero.
__device__ __forceinline__ float f16_scalar(uint16_t x) {
    if ((x & 0x7C00u) == 0) return __uint_as_float(uint32_t(x & 0x8000u) << 16);
    return __half2float(__ushort_as_half(x));
}

// Element i of a query as the SIMD kernels load it, and as the scalar code (norms, compression) reads it.
template <int QT> __device__ __forceinline__ float q_simd(const void* q, uint32_t i) {
    if constexpr (QT == SVSB200_F32) return static_cast<const float*>(q)[i];
    if constexpr (QT == SVSB200_F16) return __half2float(__ushort_as_half(static_cast<const uint16_t*>(q)[i]));
    if constexpr (QT == SVSB200_I8) return float(static_cast<const int8_t*>(q)[i]);
    return float(static_cast<const uint8_t*>(q)[i]);
}
template <int QT> __device__ __forceinline__ float q_scalar(const void* q, uint32_t i) {
    if constexpr (QT == SVSB200_F16) return f16_scalar(static_cast<const uint16_t*>(q)[i]);
    return q_simd<QT>(q, i);
}

// detail::compress (quantization/scalar/scalar.h:38-42): clamp(round((x - bias) / scale)) as an int8 / uint8 code byte.
__device__ __forceinline__ uint8_t sq_compress_code(float x, int code_type, float scale, float bias) {
    const float lo = code_type == SVSB200_I8 ? -128.f : 0.f, hi = code_type == SVSB200_I8 ? 127.f : 255.f;
    float r = roundf(__fdiv_rn(__fsub_rn(x, bias), scale));
    r = fminf(fmaxf(r, lo), hi);
    return code_type == SVSB200_I8 ? uint8_t(int8_t(int(r))) : uint8_t(int(r));
}

// detail::decompress (quantization/scalar/scalar.h:44-46): scale * c + bias, not contracted.
__device__ __forceinline__ float sq_decompress(int c, float scale, float bias) {
    return __fadd_rn(__fmul_rn(scale, float(c)), bias);
}

// InnerProductCompressed::fix_argument's offset (scalar.h:123-131): bias * std::reduce over the fp32 query
// (libstdc++: four at a time, then the tail).
__device__ __forceinline__ float sq_ip_offset(const float* f, uint32_t dim, float bias) {
    float acc = 0.f;
    uint32_t i = 0;
    for (; i + 4 <= dim; i += 4) {
        float v1 = __fadd_rn(f[i], f[i + 1]);
        float v2 = __fadd_rn(f[i + 2], f[i + 3]);
        acc = __fadd_rn(acc, __fadd_rn(v1, v2));
    }
    for (; i < dim; ++i) acc = __fadd_rn(acc, f[i]);
    return __fmul_rn(bias, acc);
}

// distance::norm (distance_core.h:45-66): sequential fp32 `accum += v * v`, sqrt; square(i) is the i-th v * v.
template <typename Square> __device__ __forceinline__ float sequential_norm(uint32_t dim, Square square) {
    float acc = 0.f;
    for (uint32_t i = 0; i < dim; ++i) acc = __fadd_rn(acc, square(i));
    return __fsqrt_rn(acc);
}

}  // namespace svsb200
