// build_u8.cu -- graph-builder kernel instantiations for uint8 base vectors: exact integer distances (OP_*I).
#include "build_kernels.cuh"

namespace svsb200 {

template <> cudaError_t launch_build_search<SVSB200_U8>(int op, const SearchParams& p, const LaunchConfig& cfg) {
    switch (op) {
        case OP_L2I: return launch_fast_dims<SVSB200_U8, OP_L2I, true>(p, cfg);
        case OP_IPI: return launch_fast_dims<SVSB200_U8, OP_IPI, true>(p, cfg);
        case OP_COSI: return launch_fast_dims<SVSB200_U8, OP_COSI, true>(p, cfg);
        default: return cudaErrorInvalidValue;
    }
}
template <> cudaError_t launch_build_prune_op<SVSB200_U8>(int op, const SearchParams& p, const BuildParams& bp, int grid,
                                                          cudaStream_t stream) {
    switch (op) {
        case OP_L2I: return launch_build_prune<SVSB200_U8, OP_L2I>(p, bp, grid, stream);
        case OP_IPI: return launch_build_prune<SVSB200_U8, OP_IPI>(p, bp, grid, stream);
        case OP_COSI: return launch_build_prune<SVSB200_U8, OP_COSI>(p, bp, grid, stream);
        default: return cudaErrorInvalidValue;
    }
}

}  // namespace svsb200
