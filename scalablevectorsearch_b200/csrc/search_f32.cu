// search_f32.cu -- search-kernel instantiations for f32 base vectors.
#include "search_kernel.cuh"

namespace svsb200 {

template cudaError_t launch_search<SVSB200_F32>(int, const SearchParams&, const LaunchConfig&, int);
template cudaError_t launch_search_exhaustive<SVSB200_F32>(int, const SearchParams&, const LaunchConfig&);

}  // namespace svsb200
