// fast_dynamic_sq.cu -- lean search-kernel instantiations in MutableBuffer mode (search_fast.cuh, MUT = true) over SQ
// int8 / uint8 codes: the search of a dynamic index with SQ storage, with the SQ search's operators (DynamicSqOps).
#include "search_fast.cuh"

namespace svsb200 {

template cudaError_t launch_search_dynamic_sq<SVSB200_I8>(int, const SearchParams&, const LaunchConfig&);
template cudaError_t launch_search_dynamic_sq<SVSB200_U8>(int, const SearchParams&, const LaunchConfig&);

}  // namespace svsb200
