// fast_dynamic.cu -- lean search-kernel instantiations in MutableBuffer mode (search_fast.cuh, MUT = true): the
// search of a dynamic index over f32 / f16 rows.
#include "search_fast.cuh"

namespace svsb200 {

template <int ROWT> static cudaError_t launch_dynamic_rows(int op, const SearchParams& p, const LaunchConfig& cfg) {
    switch (op) {
        case OP_L2F: return launch_fast_dims_mut<ROWT, OP_L2F>(p, cfg);
        case OP_IPF: return launch_fast_dims_mut<ROWT, OP_IPF>(p, cfg);
        case OP_COSF: return launch_fast_dims_mut<ROWT, OP_COSF>(p, cfg);
        default: return cudaErrorInvalidValue;
    }
}

cudaError_t launch_search_dynamic(int rowt, int op, const SearchParams& p, const LaunchConfig& cfg) {
    if (rowt == SVSB200_F32) return launch_dynamic_rows<SVSB200_F32>(op, p, cfg);
    if (rowt == SVSB200_F16) return launch_dynamic_rows<SVSB200_F16>(op, p, cfg);
    return cudaErrorInvalidValue;
}

}  // namespace svsb200
