// fast_f32.cu -- lean search-kernel instantiations (search_fast.cuh) for f32 rows.
#include "search_fast.cuh"

namespace svsb200 {

template cudaError_t launch_search_fast<SVSB200_F32>(int, const SearchParams&, const LaunchConfig&);

}  // namespace svsb200

#ifdef SVSB200_PHASE_CLOCKS
// diagnostic build only: cycles per hop phase {next+adjacency, filter, distances, merge, hops} summed over the f32 launches
extern "C" int svsb200_debug_phase_clocks(unsigned long long* out, int reset) {
    if (cudaMemcpyFromSymbol(out, svsb200::g_phase_clocks, 8 * sizeof(unsigned long long)) != cudaSuccess) return -1;
    if (reset) {
        unsigned long long zero[8] = {};
        if (cudaMemcpyToSymbol(svsb200::g_phase_clocks, zero, sizeof(zero)) != cudaSuccess) return -1;
    }
    return 0;
}
#endif
