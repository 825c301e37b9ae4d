// build_f32.cu -- graph-builder kernel instantiations for f32 base vectors.
#include "build_kernels.cuh"

namespace svsb200 {

template <> cudaError_t launch_build_search<SVSB200_F32>(int op, const SearchParams& p, const LaunchConfig& cfg) {
    switch (op) {
        case OP_L2F: return launch_fast_dims<SVSB200_F32, OP_L2F, true>(p, cfg);
        case OP_IPF: return launch_fast_dims<SVSB200_F32, OP_IPF, true>(p, cfg);
        case OP_COSF: return launch_fast_dims<SVSB200_F32, OP_COSF, true>(p, cfg);
        default: return cudaErrorInvalidValue;
    }
}
template <> cudaError_t launch_build_prune_op<SVSB200_F32>(int op, const SearchParams& p, const BuildParams& bp, int grid,
                                                           cudaStream_t stream) {
    switch (op) {
        case OP_L2F: return launch_build_prune<SVSB200_F32, OP_L2F>(p, bp, grid, stream);
        case OP_IPF: return launch_build_prune<SVSB200_F32, OP_IPF>(p, bp, grid, stream);
        case OP_COSF: return launch_build_prune<SVSB200_F32, OP_COSF>(p, bp, grid, stream);
        default: return cudaErrorInvalidValue;
    }
}

template <> cudaError_t launch_consolidate_pool_op<SVSB200_F32>(int op, const SearchParams& p, const BuildParams& bp, int grid,
                                                                cudaStream_t stream) {
    switch (op) {
        case OP_L2F: return launch_consolidate_pool<SVSB200_F32, OP_L2F>(p, bp, grid, stream);
        case OP_IPF: return launch_consolidate_pool<SVSB200_F32, OP_IPF>(p, bp, grid, stream);
        case OP_COSF: return launch_consolidate_pool<SVSB200_F32, OP_COSF>(p, bp, grid, stream);
        default: return cudaErrorInvalidValue;
    }
}

}  // namespace svsb200
