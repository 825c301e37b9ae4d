// fast_f16.cu -- lean search-kernel instantiations (search_fast.cuh) for f16 rows.
#include "search_fast.cuh"

namespace svsb200 {

template cudaError_t launch_search_fast<SVSB200_F16>(int, const SearchParams&, const LaunchConfig&);

}  // namespace svsb200
