// search_lvq8.cu -- search-kernel instantiations for LVQ-8 rows (fused decompress + distance).
#include "search_kernel.cuh"

namespace svsb200 {

template cudaError_t launch_search<ROW_LVQ8>(int, const SearchParams&, const LaunchConfig&, int);
template cudaError_t launch_search_exhaustive<ROW_LVQ8>(int, const SearchParams&, const LaunchConfig&);

}  // namespace svsb200
