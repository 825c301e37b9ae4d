// common.cuh -- shared definitions for libsvsb200 (sm_90a only).
#pragma once

#include <cuda_runtime.h>
#include <cuda_fp16.h>

#include <cstddef>
#include <cstdint>
#include <cstdio>
#include <string>
#include <type_traits>

#include "../../include/svsb200.h"
#include "slots.h"   // SlotStatus

namespace svsb200 {

constexpr uint32_t kNoNeighbor = 0xFFFFFFFFu;   // padding of adjacency rows in HBM
constexpr uint32_t kVisitedBit = 0x80000000u;   // SearchNeighbor::visited packed into the id
constexpr uint32_t kIdMask = 0x7FFFFFFFu;

// Internal row kinds of the search kernel: the four ABI element types plus LVQ-8 rows
// (uint8 codes followed by the per-vector {delta, lower} as two float16; DESIGN.md §10).
constexpr int ROW_LVQ8 = 4;

// Distance operator of the search kernel.
//   *F: the reference's fp32 expression tree (generic_simd_op, simd_utils.h:204-252)
//   *I: exact int32 arithmetic for (int8,int8)/(uint8,uint8) (L2VNNIOp/IPVNNIOp)
enum Op : int { OP_L2F = 0, OP_IPF = 1, OP_COSF = 2, OP_L2I = 3, OP_IPI = 4, OP_COSI = 5 };

// Everything the search kernel needs; passed by value (__grid_constant__).
struct SearchParams {
    // index
    const void* vectors;       // HBM, row-major, `row_stride` bytes apart (multiple of 16)
    const uint32_t* graph;     // HBM, uint32[n][gstride], neighbours then kNoNeighbor padding
    const uint16_t* ref_degree; // HBM, out-degree as the reference stores it (repeats included); counters only
    uint32_t n;
    uint32_t dim;
    uint32_t row_stride;
    uint32_t lvq_const_offset;  // LVQ-8: byte offset of {delta, lower} (2 x f16) inside a row
    uint32_t gstride;
    uint32_t entry_point;
    const uint32_t* entry_points;   // more than one entry point (index/vamana/index.h:304-312 holds a vector): device array
    uint32_t n_entry;               // 0 or 1: `entry_point` alone
    // distance post-processing
    int greater;               // comparator std::greater (IP / cosine): keys are negated
    int sq;                    // rows are scalar-quantised codes
    int lvq;                   // rows are LVQ-8 (mean-removed, per-vector delta/lower)
    int no_split;              // tuning: keep wide rows on the narrow (G threads per row) mapping
    float scale, bias, scale_sq;
    // prepared queries (output of prepare_queries)
    const float* qf;           // [nq][qstride] fp32 operands of the float tree
    const uint8_t* qcodes;     // [nq][qstride] int8/uint8 operands of the integer kernels
    const float* qaux;         // [nq][2]: {a_norm | offset, float(sum x*x)}
    uint32_t qstride;          // elements; multiple of 16
    uint32_t nq;
    // search buffer configuration
    uint32_t k, window, capacity;
    uint32_t cap_pad;          // capacity+1 rounded up to 32
    uint32_t deg_pad;          // gstride rounded up to 32
    uint32_t filter_slots;     // per-query exact visited filter (power of two, 0 = off)
    uint32_t filter_shift;     // tag = id >> filter_shift: log2(sets) = log2(filter_slots / 2) in tag16 mode,
                               // log2(filter_slots) (unused: full ids are stored) otherwise
    uint32_t filter_tag16;     // 1: two 16-bit tags per 32-bit set (exact while (n-1) >> filter_shift < 0xFFFF)
    // outputs
    void* out_ids;
    int id_bytes;
    uint64_t id_offset;        // added to every valid 64-bit output id (this index is a shard of a larger one)
    float* out_dists;
    // bookkeeping
    unsigned int* work_counter;  // dynamic query scheduler
    uint32_t* hops;              // optional per-query counters
    uint32_t* evals;
    uint32_t* fetched;           // rows actually read from HBM (after the visited filter)
    const int* cancel;           // optional device flag: non-zero stops the batch (polled per query and per hop)
    uint32_t exh_split;          // exhaustive scan: base rows are cut into this many ranges, one work item per (query, range)
    // graph builder only (HIST kernels): per query, every expanded node {key bits, id}
    uint2* hist;
    uint32_t* hist_count;
    uint32_t hist_cap;
    // dynamic index only (MUT kernels, the reference's MutableBuffer search): per-slot status, external ids, buffer room
    const uint8_t* status;       // [n] SlotMetadata: a Deleted slot is walked through but never returned
    const uint64_t* ext_ids;     // [n] external id of every slot (what the copy-out writes; NULL: the slot itself)
    uint32_t buf_cap;            // entries the buffer may hold: capacity + slack for Deleted entries
    uint32_t* ovf;               // [1 + nq] count, then the queries whose buffer ran out of slack (not written)
    const uint32_t* qlist;       // optional: run only these queries (a re-run of overflowed ones)
};

constexpr uint32_t kInvalidBit = 0x40000000u;   // MUT kernels: PredicatedSearchNeighbor::valid() == false, packed into the id

struct LaunchConfig {
    int grid;
    int warps_per_cta;
    size_t smem_bytes;
    cudaStream_t stream;
};

// Per-warp shared-memory footprint of the search kernel (bytes), mirrored on the host.
__host__ __device__ inline size_t warp_smem_bytes(uint32_t qstride, uint32_t cap_pad, uint32_t deg_pad,
                                                  uint32_t filter_bytes) {
    // query (fp32 or bytes, reserve fp32) + buffer keys/ids + candidate keys/ids +
    // survivor keys/pos/ids/final-pos + visited filter
    // + two staged adjacency rows
    return size_t(qstride) * 4 + size_t(cap_pad) * 8 + size_t(deg_pad) * 8 + size_t(deg_pad) * 16 +
           size_t(filter_bytes) + size_t(deg_pad) * 8;
}

// Per-CTA (= per-warp = per-query) shared memory of the fast kernel, mirrored on the host.
__host__ __device__ inline size_t fast_smem_bytes(uint32_t qstride, uint32_t cap_pad, uint32_t deg_pad,
                                                  uint32_t filter_bytes) {
    // filter | query | buffer {key,id} | candidate keys | candidate ids
    return size_t((filter_bytes + 15u) & ~15u) + size_t(qstride) * 4 + size_t(cap_pad) * 8 + size_t(deg_pad) * 8;
}

constexpr int kFastMaxGW = 4;   // adjacency rows up to 128 neighbours (4 x 32) are register-staged

constexpr size_t kSmemOptInMax = 227 * 1024;   // dynamic shared memory a block may opt in to on sm_90

// ---- Which (row type, distance operator) pairs every kernel family has ----------------------------------------------
//   family                                        rows      F32, F16       I8, U8            LVQ8
//   generic search, exhaustive scan, lean search  SearchRows  L2F IPF COSF   all six           L2F IPF
//   builder search (HIST), builder prune          DataRows    L2F IPF COSF   L2I IPI COSI      -
//   the same over SQ codes (build_sq_<type>.cu)   BuildSqRows -              L2I IPF COSF      -
//   consolidate pool, dynamic search (MUT)        DynamicRows L2F IPF COSF   -                 -
//   the same over SQ codes (fast_dynamic_sq.cu)   DynamicSqRows -            L2I IPF COSF      -
//   flat rescore                                  DataRows    L2F IPF        L2F IPF L2I IPI   -
//   IVF leaf scan (ivf_kernel.cuh)                IvfRows     L2F IPF COSF   -                 -
//   IVF leaf scan over SQ codes                   IvfSqRows   -              IPF COSF (+ the
//                                                                            tensor-core L2 leaf)
// int8 / uint8 rows take float and integer queries in a search; the builder's datum is its own query.  Over SQ codes
// the builder's datum is decompressed and prepared as the SQ search's fp32 query, so it takes the SQ search's operators;
// so does the dynamic index over SQ codes, in its search and in consolidation's candidate pools.
template <int... V> struct IntList {};
template <int ROWT> constexpr bool kIntRow = ROWT == SVSB200_I8 || ROWT == SVSB200_U8;
using FloatOps = IntList<OP_L2F, OP_IPF, OP_COSF>;
using IntOps = IntList<OP_L2I, OP_IPI, OP_COSI>;

using SearchRows = IntList<SVSB200_F32, SVSB200_F16, SVSB200_I8, SVSB200_U8, ROW_LVQ8>;
using DataRows = IntList<SVSB200_F32, SVSB200_F16, SVSB200_I8, SVSB200_U8>;   // the four element types of the ABI
using DynamicRows = IntList<SVSB200_F32, SVSB200_F16>;
template <int ROWT>
using SearchOps = std::conditional_t<ROWT == ROW_LVQ8, IntList<OP_L2F, OP_IPF>,
                                     std::conditional_t<kIntRow<ROWT>, IntList<OP_L2F, OP_IPF, OP_COSF, OP_L2I, OP_IPI, OP_COSI>,
                                                        FloatOps>>;
template <int ROWT> using BuildOps = std::conditional_t<kIntRow<ROWT>, IntOps, FloatOps>;
using BuildSqRows = IntList<SVSB200_I8, SVSB200_U8>;
using BuildSqOps = IntList<OP_L2I, OP_IPF, OP_COSF>;
using DynamicOps = FloatOps;
using DynamicSqRows = IntList<SVSB200_I8, SVSB200_U8>;
using DynamicSqOps = BuildSqOps;
using IvfRows = IntList<SVSB200_F32, SVSB200_F16>;
using IvfOps = FloatOps;
using IvfSqRows = IntList<SVSB200_I8, SVSB200_U8>;
using IvfSqOps = IntList<OP_IPF, OP_COSF>;
template <int ROWT>
using RescoreOps = std::conditional_t<kIntRow<ROWT>, IntList<OP_L2F, OP_IPF, OP_L2I, OP_IPI>, IntList<OP_L2F, OP_IPF>>;

// f(std::integral_constant<int, V>{}) for the V of the list equal to `v`; cudaErrorInvalidValue when the list lacks it.
template <int... V, typename F> cudaError_t dispatch(IntList<V...>, int v, F&& f) {
    cudaError_t err = cudaErrorInvalidValue;
    (void)((v == V && (err = f(std::integral_constant<int, V>{}), true)) || ...);
    return err;
}

// The compile-time shape of a distance pass for rows of `dim` elements: f(DS, KS), DS the static dimension (0: any) and
// KS the factor by which a float row's accumulators are split over more threads.  Static dimensions get fully unrolled
// loads (all of a row's loads in flight at once), like the reference's static-N vs Dynamic kernels
// (distance_core.h:31-42); rows of 256 and more split (float_rows_split) when `split` allows it.  The integer distance
// code has one shape for every dimension.  The families differ in two ways only: DIM128 (no static 128 for the builder's
// kernels) and `split` (the searches take it from SearchParams::no_split, the builder and consolidation always split).
template <int OP, bool DIM128, typename F> cudaError_t with_shape(uint32_t dim, bool split, F&& f) {
    using One = std::integral_constant<int, 1>;
    if constexpr (OP < OP_L2I) {
        if (dim == 96) return f(std::integral_constant<int, 96>{}, One{});
        if constexpr (DIM128) {
            if (dim == 128) return f(std::integral_constant<int, 128>{}, One{});
        }
        if (dim >= 256 && split) return f(std::integral_constant<int, 0>{}, std::integral_constant<int, 4>{});
    }
    return f(std::integral_constant<int, 0>{}, One{});
}

void count_launch();

// kernel<<<grid, cfg.warps_per_cta * 32, cfg.smem_bytes, cfg.stream>>>(args...), counted, returning the launch error.
// cfg.grid > 0 is the grid; cfg.grid < 0 asks for a persistent one, -cfg.grid SMs x the CTAs of `kernel` resident per
// SM.  Either way at most `max_ctas` CTAs.  With `opt_in` the kernel first opts in to cfg.smem_bytes of shared memory.
template <typename K, typename... Args>
cudaError_t launch_kernel(K kernel, const LaunchConfig& cfg, size_t max_ctas, bool opt_in, const Args&... args) {
    const int block = cfg.warps_per_cta * 32;
    if (opt_in) {
        cudaError_t err = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, int(cfg.smem_bytes));
        if (err != cudaSuccess) return err;
    }
    int grid = cfg.grid;
    if (grid < 0) {
        int resident = 0;
        cudaError_t err = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&resident, kernel, block, cfg.smem_bytes);
        if (err != cudaSuccess) return err;
        grid = -grid * (resident > 0 ? resident : 1);
    }
    if (size_t(grid) > max_ctas) grid = int(max_ctas);
    kernel<<<grid, block, cfg.smem_bytes, cfg.stream>>>(args...);
    count_launch();
    return cudaGetLastError();
}

// The search launchers, one per (family, row type), dispatching on the operator.  Defined in search_kernel.cuh and
// search_fast.cuh, instantiated in search_<type>.cu / fast_<type>.cu / fast_dynamic.cu.
template <int ROWT> cudaError_t launch_search(int op, const SearchParams& p, const LaunchConfig& cfg, int rows_in_flight);
// Exhaustive scan with the same distance code (ground truth / flat search).
template <int ROWT> cudaError_t launch_search_exhaustive(int op, const SearchParams& p, const LaunchConfig& cfg);
// The lean one-warp-per-CTA form of the same search.
template <int ROWT> cudaError_t launch_search_fast(int op, const SearchParams& p, const LaunchConfig& cfg);
// The lean kernel in its MutableBuffer mode (dynamic indexes, DynamicRows).
template <int ROWT> cudaError_t launch_search_dynamic(int op, const SearchParams& p, const LaunchConfig& cfg);
// The same over SQ codes (DynamicSqRows, DynamicSqOps).
template <int ROWT> cudaError_t launch_search_dynamic_sq(int op, const SearchParams& p, const LaunchConfig& cfg);

}  // namespace svsb200
