/* svsb200.h -- C ABI of libsvsb200.so: the H100-native Vamana batched-search hot path.
 *
 * This is the drop-in boundary for the reference's Vamana search (SURVEY.md §8b).  Each
 * entry point names the reference interface it replaces (file:line relative to
 * /root/reference).  Plain pointers and sizes only -- no C++/torch types -- so it binds
 * from C++ (scalablevectorsearch_b200/cpp/gpu_vamana_index.h), Python ctypes
 * (scalablevectorsearch_b200/_lib.py) or anything else with a C FFI.
 *
 * Conventions
 *   * every function returns 0 on success, non-zero on failure; svsb200_last_error()
 *     gives the message for the calling thread (the C++ adapter rethrows it as
 *     svs::ANNException, matching include/svs/lib/exception.h);
 *   * there is no CPU fallback: if no sm_90-class device is usable, create/search fail;
 *   * "host" pointers may be pageable or pinned; "device" pointers must live on the
 *     index's device;
 *   * ids are the reference's internal uint32 ids (core/graph/graph.h:388) widened to
 *     `id_bytes` (4 or 8; the orchestrator boundary uses size_t, orchestrators/manager.h:79).
 */
#ifndef SVSB200_H
#define SVSB200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define SVSB200_VERSION 201

/* Element types: svs::DataType float32 / float16 / int8 / uint8 (lib/datatype.h). */
enum { SVSB200_F32 = 0, SVSB200_F16 = 1, SVSB200_I8 = 2, SVSB200_U8 = 3 };
/* svs::DistanceType (core/distance.h:41-60): L2, MIP, Cosine. */
enum { SVSB200_L2 = 0, SVSB200_IP = 1, SVSB200_COSINE = 2 };
/* Storage of the base vectors:
 *   PLAIN  svs::data::SimpleData<T>                       (core/data/simple.h:259-618)
 *   SQ     svs::quantization::scalar::SQDataset<int8|uint8> (quantization/scalar/scalar.h:363-551);
 *          aux = {scale, bias}
 *   LVQ8   one-level 8-bit locally-adaptive quantisation (closed-source in the reference,
 *          own specification: DESIGN.md §LVQ-8); aux = per-dataset mean[dim] */
enum { SVSB200_PLAIN = 0, SVSB200_SQ = 1, SVSB200_LVQ8 = 2 };

typedef struct svsb200_index svsb200_index;

const char* svsb200_last_error(void);
int svsb200_version(void);
/* Number of usable CUDA devices (0 if none); fills `sm` with the compute capability*10
 * of `device` when non-NULL. */
int svsb200_device_count(void);
int svsb200_device_sm(int device, int* sm);

/* Replaces: VamanaIndex(graph, data, entry_point, distance, threadpool)
 *           (include/svs/index/vamana/index.h:364-378) / auto_assemble (:1022-1077).
 * Copies the host arrays into HBM (the caller keeps ownership of its memory):
 *   vectors     n rows of `dim` elements of `dtype`, `row_stride_bytes` apart (0 = dense);
 *               for SQ the rows are the int8/uint8 codes, for LVQ8 see svsb200_lvq8_*.
 *   graph_rows  the reference's in-memory adjacency: uint32[n][graph_row_len], element 0 =
 *               out-degree, then the neighbours (include/svs/core/graph/graph.h:103-114);
 *               graph_row_len = max_degree + 1.
 *   entry_point the medoid / configured entry point (index.h:312,373).
 */
int svsb200_index_create(
    const void* vectors, int dtype, size_t n, size_t dim, size_t row_stride_bytes,
    const uint32_t* graph_rows, size_t graph_row_len, uint32_t entry_point, int metric,
    int storage, const float* aux, int device, svsb200_index** out);

/* The same index replicated on several GPUs of this process (SURVEY.md 8e mode A, the multi-device form of
 * the reference's `num_threads`): replica 0 is uploaded from the host arrays, the others are copied device to
 * device.  svsb200_search on such an index splits every batch with threads::balance
 * (lib/threads/types.h:311-329), one contiguous slice per device, and the slices' results land in disjoint
 * rows of the caller's arrays -- no collective. */
int svsb200_index_create_multi(
    const void* vectors, int dtype, size_t n, size_t dim, size_t row_stride_bytes,
    const uint32_t* graph_rows, size_t graph_row_len, uint32_t entry_point, int metric,
    int storage, const float* aux, const int* devices, size_t ndevices, svsb200_index** out);

/* Replaces: index::vamana::auto_assemble(config_path, GraphLoader, VectorDataLoader, distance, threads)
 * (include/svs/index/vamana/index.h:1022-1050) for uncompressed data: the VamanaIndexParameters TOML
 * (`svs_config.toml` inside `config_path`, or the file itself; index.h:53-178) is parsed here (entry point, saved
 * search parameters -> svsb200_get_option "config_search_window_size" / "config_search_buffer_capacity"), and
 * the native v1 `.svs` containers (core/io/native.h:315-345; `graph_0.svs` / `data_0.svs` inside a directory) or
 * `[fibh]vecs` files (core/io/vecs.h:137-273) are streamed through pinned staging buffers straight into HBM --
 * no host copy of the dataset is made.  `expected_dims` != 0 is VectorDataLoader's `dims` check. */
int svsb200_index_assemble(
    const char* config_path, const char* graph_path, const char* data_path, int dtype, size_t expected_dims,
    int metric, const int* devices, size_t ndevices, svsb200_index** out);
/* The TOML subset reader behind it (tables, dotted table names, integers, floats, booleans, strings): copies the
 * raw text of `table.key` into `out`. */
int svsb200_toml_get(const char* path, const char* dotted_key, char* out, size_t capacity);

/* Several entry points: VamanaIndex keeps a vector of them (include/svs/index/vamana/index.h:304-312) and
 * EntryPointInitializer pushes every one before the walk starts (index/vamana/greedy_search.h:62-94).  1..32 distinct
 * ids; the first replaces the entry point given at creation. */
int svsb200_set_entry_points(svsb200_index* index, const uint32_t* entry_points, size_t count);

int svsb200_index_destroy(svsb200_index* index);

/* Introspection used by the host-side mirror (size()/dimensions()/get_graph_max_degree,
 * orchestrators/vamana.h:127-275). */
size_t svsb200_index_size(const svsb200_index* index);
size_t svsb200_index_dimensions(const svsb200_index* index);
size_t svsb200_index_max_degree(const svsb200_index* index);
size_t svsb200_index_device_bytes(const svsb200_index* index);
int svsb200_index_device(const svsb200_index* index);         /* first replica's device */
size_t svsb200_index_num_devices(const svsb200_index* index);

/* Replaces: VamanaIndex::search(QueryResultView<I>, queries, VamanaSearchParameters, cancel)
 *           (include/svs/index/vamana/index.h:564-611) for a whole batch.
 *   queries      nq x dim, dense row-major, element type `qdtype` (HOST memory);
 *   window / capacity = SearchBufferConfig (index/vamana/search_buffer.h:39-96); as in
 *               index.h:590-592, a capacity < k resets both to k;
 *   use_visited_set = VamanaSearchParameters::search_buffer_visited_set_
 *               (search_params.h:42); performance-only, results identical;
 *   out_ids      nq x k ids of `id_bytes` each; out_dists nq x k float (HOST memory).
 * Rows with fewer than k reachable candidates are padded with id = all-ones and
 * dist = +/-inf (the reference leaves stale buffer contents there, extensions.h:588-590).
 * Blocking: returns after the results are in the host buffers.  The H2D copy, the search
 * kernel and the D2H copy run on `stream` (a cudaStream_t; NULL selects the index's own
 * non-blocking stream -- pass cudaStreamLegacy / cudaStreamPerThread to name a default stream). */
int svsb200_search(
    svsb200_index* index, const void* queries, int qdtype, size_t nq, size_t k, size_t window,
    size_t capacity, int use_visited_set, void* out_ids, int id_bytes, float* out_dists,
    void* stream);

/* svsb200_search with the reference's cancellation predicate (`const lib::DefaultPredicate& cancel`,
 * index/vamana/index.h:568): while the batch runs, the calling thread polls `cancel(cancel_arg)`; once it
 * returns non-zero a device flag is raised that every search warp polls per query and per expanded node
 * (extensions.h:579, greedy_search.h:155) and the call returns as soon as the kernels have drained.  As in
 * the reference, the result rows of a cancelled call are unspecified. */
int svsb200_search_cancellable(
    svsb200_index* index, const void* queries, int qdtype, size_t nq, size_t k, size_t window,
    size_t capacity, int use_visited_set, void* out_ids, int id_bytes, float* out_dists,
    void* stream, int (*cancel)(void*), void* cancel_arg);

/* Threading: concurrent svsb200_search* calls on one index from several host threads are allowed (as the
 * reference allows concurrent searches with external scratch, index/vamana/index.h:455-470,512-526): every
 * call checks out its own stream + scratch buffers (svsb200_get_option "streams" reports how many exist). */

/* Same search with every buffer already resident in HBM on the index's device and no
 * synchronisation: enqueues on `stream` and returns (bench.py's device-resident `value`,
 * multi-GPU pipelines that feed NCCL directly).  The index keeps one set of scratch buffers
 * (prepared queries, work counter) per caller stream -- the analogue of the reference's
 * per-thread scratch space (index/vamana/index.h:455-470) -- so different streams may search
 * concurrently; single-device indexes only. */
int svsb200_search_device(
    svsb200_index* index, const void* d_queries, int qdtype, size_t nq, size_t k, size_t window,
    size_t capacity, int use_visited_set, void* d_out_ids, int id_bytes, float* d_out_dists,
    void* stream);

/* Work counters of the most recent search on this index, per query (device arrays are
 * copied to the host buffers; either may be NULL): expanded nodes and distance
 * evaluations -- the quantities a reference GreedySearchTracker reports
 * (index/vamana/greedy_search.h:38-42,165).  Used for the algorithmic-bytes roofline.
 * Counting is off by default; enable it before the search. */
int svsb200_set_counting(svsb200_index* index, int enabled);
int svsb200_get_counters(svsb200_index* index, size_t nq, uint32_t* hops, uint32_t* evals);
/* Rows of base vectors the kernel actually read per query (entry point included): equal to
 * `evals` with the visited filter off, smaller with it on.  This -- not the reference-
 * equivalent `evals` -- is what the HBM roofline of the kernel is computed from. */
int svsb200_get_fetched(svsb200_index* index, size_t nq, uint32_t* fetched);
/* Duration in milliseconds of the search kernel of the last svsb200_search* call on this
 * index (CUDA events on the launching stream; synchronises on the stop event).  A host-buffer
 * batch that was cut into pieces ("host_chunks") reports its last piece, from that piece's
 * enqueue to its end -- i.e. including the time it waited for SMs behind the earlier pieces. */
int svsb200_last_kernel_ms(svsb200_index* index, float* ms);
/* Number of kernels this library launched so far in this process. */
uint64_t svsb200_launch_count(void);

/* Tuning knobs (performance only; results never change):
 *   "warps_per_cta", "ctas_per_sm", "rows_in_flight" (0 restores the default);
 *   "visited_filter_slots": size of the per-query exact visited filter, the GPU form of
 *   VamanaSearchParameters::search_buffer_visited_set_ (-1 default, 0 off, else 2^n >= 8);
 *   "host_chunks": pieces a host-buffer batch is cut into per device so that the copies of one piece run under
 *   the kernel of another (0 = automatic: up to 4 for large batches; one piece when a cancel predicate or a
 *   caller stream is given). */
int svsb200_set_option(svsb200_index* index, const char* name, long value);
/* Reads a knob back; also "last_kernel": which kernel the most recent search ran on (1 = the lean
 * one-warp-per-CTA kernel, 0 = the generic kernel that covers every other configuration), and
 * "generic_kernel" (set to 1 to force the generic kernel; results are identical). */
int svsb200_get_option(svsb200_index* index, const char* name, long* value);

/* The filtered and range searches of the reference's runtime ABI (svs::runtime::v0::VamanaIndex::search with an
 * IDFilter, ::range_search; bindings/cpp/include/svs/runtime/vamana_index.h:75-92, implemented in
 * bindings/cpp/src/vamana_index_impl.h:139-300 with a batch iterator that keeps asking for further candidates).
 * Here the membership test runs on the device: the caller hands the filter over as a bitmap of n bits
 * (bit i = id i may be returned), every query searches with a result list that grows (x4) until k members were
 * found or the search is exhausted, and the first k members in result order are returned -- distances are the graph
 * search's.  Short rows are padded with id = all-ones, distance = +inf (the reference's `Unspecify`).
 *   svsb200_range_search returns, per query, the results closer than `radius` (further than, for MIP):
 *   counts[nq] and two malloc'ed arrays holding the concatenated ids / distances (release with svsb200_free). */
int svsb200_search_filtered(
    svsb200_index* index, const void* queries, int qdtype, size_t nq, size_t k, size_t window,
    const uint32_t* id_bitmap, uint64_t* out_ids, float* out_dists, uint32_t* out_found);
int svsb200_range_search(
    svsb200_index* index, const void* queries, int qdtype, size_t nq, float radius, size_t window,
    uint32_t* out_counts, uint64_t** out_ids, float** out_dists);
void svsb200_free(void* p);

/* Mode B of SURVEY.md §8e inside one process: `shards[s]` are single-device indexes over disjoint,
 * contiguous id ranges of one dataset, each with its own graph and entry point and its id range's first id
 * set with svsb200_set_id_offset.  Every query is searched on every shard; the per-shard top-k rows are
 * gathered on shard 0's device -- written there directly by the shards' search kernels over NVLink when
 * peer access exists, by peer copies otherwise -- and merged G*k -> k with the reference's TotalOrder
 * (distance, then id; lib/neighbor.h:143-155).  Host buffers in, host buffers out; blocking. */
int svsb200_set_id_offset(svsb200_index* index, uint64_t offset);
int svsb200_search_sharded(
    svsb200_index* const* shards, size_t nshards, const void* queries, int qdtype, size_t nq, size_t k,
    size_t window, size_t capacity, uint64_t* out_ids, float* out_dists);

/* Mode B of SURVEY.md §8e -- merge per-shard top-k lists (after an NCCL all-gather) into a
 * global top-k with the reference's TotalOrder (distance, then id; lib/neighbor.h:143-155).
 *   d_ids   [nshards][nq][k] uint64 global ids, d_dists same shape; outputs [nq][k].
 * metric selects the comparator (L2: smaller is better; IP/cosine: larger is better). */
int svsb200_merge_topk_device(
    const uint64_t* d_ids, const float* d_dists, size_t nshards, size_t nq, size_t k, int metric,
    uint64_t* d_out_ids, float* d_out_dists, int device, void* stream);

/* LVQ-8 (one-level, 8-bit locally-adaptive vector quantisation).  The reference's LVQ lives in a
 * closed-source library (examples/cpp/shared/example_vamana_with_compression_lvq.cpp:38,
 * `LVQDataset<8>::compress(data, threadpool, padding)`); this is an own specification
 * (DESIGN.md §10) and parity with Intel's binary is unpinned.
 *   row layout  : dim uint8 codes, padded to 4 bytes, then {delta, lower} as two IEEE float16,
 *                 row stride = svsb200_lvq8_row_stride(dim) (a multiple of 32 bytes);
 *   compress    : encodes n float32 vectors against `mean[dim]` on the GPU into `out_rows`
 *                 (host buffers); pass the same `mean` as `aux` to svsb200_index_create with
 *                 storage = SVSB200_LVQ8, dtype = SVSB200_U8, row_stride_bytes = the stride. */
size_t svsb200_lvq8_row_stride(size_t dim);
int svsb200_lvq8_compress(const float* data, size_t n, size_t dim, const float* mean, void* out_rows,
                          int device);

/* GPU graph construction.  Replaces: index::vamana::auto_build / VamanaIndex(VamanaBuildParameters, ...)
 * (include/svs/index/vamana/index.h:404-440,968-994) and VamanaBuilder::construct
 * (index/vamana/vamana_build.h:221-599): medoid entry point (core/medioid.h:292-330), two passes over
 * batches of max(40, n/4096) rounds, greedy search with full search history + alpha-robust pruning
 * (prune.h: Progressive strategy for L2, Iterative for MIP and cosine), reverse edges with overflow re-pruning to
 * `prune_to`.  Arguments are VamanaBuildParameters (index/vamana/build_params.h): 0 selects the reference's
 * default (alpha 1.2 / 0.95, max_candidate_pool_size = 3 * window_size, prune_to = max_degree - 4).
 *   vectors     n x dim float32 / float16 rows in HOST memory (row_stride_bytes apart, 0 = dense);
 *   graph_rows_out  uint32[n][graph_max_degree + 1], the reference's in-memory layout (degree first), HOST;
 * The reference's result depends on thread timing, so parity is its own bar: recall equivalence of the
 * built index (tests/integration/vamana/index_build.cpp:96,139-140). */
int svsb200_build_vamana(
    const void* vectors, int dtype, size_t n, size_t dim, size_t row_stride_bytes, int metric,
    float alpha, size_t graph_max_degree, size_t window_size, size_t max_candidate_pool_size,
    size_t prune_to, int device, uint32_t* graph_rows_out, uint32_t* entry_point_out);

/* How svsb200_flat_search* will split a problem of `nq` queries over `n` base vectors on a device with `sm_count`
 * SMs (introspection, host arithmetic only; nothing in the reference corresponds): `ctas` thread blocks are
 * launched; the 128-query tiles are taken `share` at a time and the (row group, 256-row base tile) pairs form one
 * row-major sequence cut into ctas / share equal segments, each walked by `share` blocks together;
 * `lists_per_query` candidate lists of 33 entries reach the rescoring step.  `segment_begin` (optional,
 * ctas / share + 1 entries) receives the first pair of every segment and the total. */
int svsb200_flat_plan(size_t nq, size_t n, int sm_count, uint32_t* ctas, uint32_t* share, uint32_t* lists_per_query,
                      uint64_t* segment_begin);

/* Exact exhaustive (flat) search on the tensor cores.  Replaces: svs::Flat / FlatIndex::search
 * (include/svs/index/flat/flat.h:159,421-465): top-k of every query against all `n` base vectors inside `index`.
 * A query-tile x base-tile fp16 GEMM (wgmma, operands staged by bulk copies) selects candidates, the
 * candidates are re-scored with the graph search's own bit-exact distance code, and an error bound on the fp16
 * products proves per query that no other vector can belong to the top k; queries that fail the proof are
 * re-run by the exact scan.  The result therefore always equals svsb200_exhaustive_device bit for bit (ids and
 * distances; ties by id).  float32/float16 data and queries, L2 and MIP, k <= 25; other shapes take the scan.
 * `fallback_queries` (optional) receives how many queries needed the scan. */
int svsb200_flat_search_device(
    svsb200_index* index, const void* d_queries, int qdtype, size_t nq, size_t k,
    uint64_t* d_out_ids, float* d_out_dists, void* stream, uint32_t* fallback_queries);
/* The same with HOST buffers (blocking). */
int svsb200_flat_search(
    svsb200_index* index, const void* queries, int qdtype, size_t nq, size_t k,
    uint64_t* out_ids, float* out_dists);

/* Exhaustive search used by the harness for ground truth (replaces svs::Flat /
 * index/flat/flat.h:159 for recall measurement only): top-k of every query against all
 * `n` base vectors already on the device inside `index`. Distances use the same exact
 * expression tree as the graph search, ties broken by id. */
int svsb200_exhaustive_device(
    svsb200_index* index, const void* d_queries, int qdtype, size_t nq, size_t k,
    uint64_t* d_out_ids, float* d_out_dists, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* SVSB200_H */
