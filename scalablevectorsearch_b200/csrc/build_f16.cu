// build_f16.cu -- graph-builder kernel instantiations for f16 base vectors.
#include "build_kernels.cuh"

namespace svsb200 {

template cudaError_t launch_build_search<SVSB200_F16>(int, const SearchParams&, const LaunchConfig&);
template cudaError_t launch_build_prune_op<SVSB200_F16>(int, const SearchParams&, const BuildParams&, int, cudaStream_t);
template cudaError_t launch_consolidate_pool_op<SVSB200_F16>(int, const SearchParams&, const BuildParams&, int, cudaStream_t);

}  // namespace svsb200
