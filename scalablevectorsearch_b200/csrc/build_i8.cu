// build_i8.cu -- graph-builder kernel instantiations for int8 base vectors: exact integer distances (OP_*I).
#include "build_kernels.cuh"

namespace svsb200 {

template cudaError_t launch_build_search<SVSB200_I8>(int, const SearchParams&, const LaunchConfig&);
template cudaError_t launch_build_prune_op<SVSB200_I8>(int, const SearchParams&, const BuildParams&, int, cudaStream_t);

}  // namespace svsb200
