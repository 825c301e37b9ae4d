// fast_dynamic.cu -- lean search-kernel instantiations in MutableBuffer mode (search_fast.cuh, MUT = true): the
// search of a dynamic index over f32 / f16 rows.
#include "search_fast.cuh"

namespace svsb200 {

template cudaError_t launch_search_dynamic<SVSB200_F32>(int, const SearchParams&, const LaunchConfig&);
template cudaError_t launch_search_dynamic<SVSB200_F16>(int, const SearchParams&, const LaunchConfig&);

}  // namespace svsb200
