// build_sq_i8.cu -- graph-builder kernel instantiations for SQ int8 codes: the SQ search's operators (BuildSqOps), and
// consolidation's candidate pools of a dynamic index over such codes.
#include "build_kernels.cuh"

namespace svsb200 {

template cudaError_t launch_build_search_sq<SVSB200_I8>(int, const SearchParams&, const LaunchConfig&);
template cudaError_t launch_build_prune_sq<SVSB200_I8>(int, const SearchParams&, const BuildParams&, int, cudaStream_t);
template cudaError_t launch_build_batch_sq<SVSB200_I8>(int, const SearchParams&, uint32_t, uint32_t, const uint32_t*, float*,
                                                        uint8_t*, float*, cudaStream_t);
template cudaError_t launch_consolidate_pool_sq<SVSB200_I8>(int, const SearchParams&, const BuildParams&, int, cudaStream_t);

}  // namespace svsb200
