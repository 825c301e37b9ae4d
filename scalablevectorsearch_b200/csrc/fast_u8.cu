// fast_u8.cu -- lean search-kernel instantiations (search_fast.cuh) for u8 rows.
#include "search_fast.cuh"

namespace svsb200 {

template cudaError_t launch_search_fast<SVSB200_U8>(int, const SearchParams&, const LaunchConfig&);

}  // namespace svsb200
