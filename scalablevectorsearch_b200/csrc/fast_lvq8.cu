// fast_lvq8.cu -- lean search-kernel instantiations (search_fast.cuh) for lvq8 rows.
#include "search_fast.cuh"

namespace svsb200 {

template cudaError_t launch_search_fast<ROW_LVQ8>(int, const SearchParams&, const LaunchConfig&);

}  // namespace svsb200
