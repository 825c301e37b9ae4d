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
 * search's.  Short rows are padded with id = all-ones, distance = +inf for every metric (the reference's
 * `Unspecify`; the plain search pads MIP / cosine rows with -inf instead).
 *   The whole batch shares one list length: it starts at max(k, window), is at most n, and stops growing at 16384 or
 *   once no query is short of k members with its search not exhausted; every query's row is taken from the last list.
 *   svsb200_range_search returns, per query, the results closer than `radius` (further than, for MIP / cosine; the
 *   comparison is strict, so a NaN radius returns nothing): counts[nq] and two malloc'ed arrays holding the
 *   concatenated ids / distances (release with svsb200_free).  Its list starts at max(window, 16) and grows the same
 *   way while some query's whole list is inside the radius.
 *   On a shard (svsb200_set_id_offset) the bitmap is over the shard's own rows, bit i = row i, and both calls return
 *   ids with the offset added, as the plain search does. */
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
 *                 storage = SVSB200_LVQ8, dtype = SVSB200_U8, row_stride_bytes = the stride.
 *                 It fails, naming the first offending row and writing nothing, when a residual x_i - mean_i is
 *                 not finite (a NaN or infinite input) or a row's delta or lower bound is not finite in float16
 *                 (a residual range of 255 x 65520 or more, or a lower bound at or below -65520): such a row
 *                 would decode to NaN or -inf.  A subnormal or zero float16 delta is finite and accepted; every
 *                 element then still decodes within 0.5 delta16 + |lower - lower16| + 255 |delta - delta16| of
 *                 its residual, plus fp32 rounding (DESIGN.md §12). */
size_t svsb200_lvq8_row_stride(size_t dim);
int svsb200_lvq8_compress(const float* data, size_t n, size_t dim, const float* mean, void* out_rows,
                          int device);

/* GPU graph construction.  Replaces: index::vamana::auto_build / VamanaIndex(VamanaBuildParameters, ...)
 * (include/svs/index/vamana/index.h:404-440,968-994) and VamanaBuilder::construct
 * (index/vamana/vamana_build.h:221-599): medoid entry point (core/medioid.h:292-330), two passes over
 * batches of max(40, n/4096) rounds, greedy search with full search history + alpha-robust pruning
 * (prune.h: Progressive strategy for L2, Iterative for MIP and cosine), reverse edges with overflow re-pruning to
 * `prune_to`.  Arguments are VamanaBuildParameters (index/vamana/build_params.h): 0 selects the reference's
 * default (alpha 1.2 / 0.95, max_candidate_pool_size = 3 * window_size clamped to 512, prune_to = max_degree - 4).
 * The candidate pool holds 512 entries, so max_candidate_pool_size > 512 is refused.  A construction search that
 * expands more than 4096 nodes fails the build rather than prune from an incomplete history.
 *   vectors     n x dim float32 / float16 / int8 / uint8 rows in HOST memory (row_stride_bytes apart, 0 = dense).
 *               int8 / uint8 rows are built with exact int x int distances throughout, as the reference builds
 *               SimpleData<int8_t / uint8_t> (the datum is its own query); the cosine norm is distance::norm's
 *               sequential fp32 sum;
 *   graph_rows_out  uint32[n][graph_max_degree + 1], the reference's in-memory layout (degree first), HOST;
 * The reference's result depends on thread timing in rounds of several nodes.  Where every round holds one node
 * (n <= 40) the rows equal the reference's; larger builds are held to recall equivalence, the reference's own bar
 * (tests/integration/vamana/index_build.cpp:96,139-140). */
int svsb200_build_vamana(
    const void* vectors, int dtype, size_t n, size_t dim, size_t row_stride_bytes, int metric,
    float alpha, size_t graph_max_degree, size_t window_size, size_t max_candidate_pool_size,
    size_t prune_to, int device, uint32_t* graph_rows_out, uint32_t* entry_point_out);

/* GPU graph construction over scalar-quantised codes.  Replaces: auto_build over SQDataset<int8_t / uint8_t>
 * (the reference's VamanaBuildAdaptor for SQ data, extensions/vamana/scalar.h:47-95).  Every datum is its own query
 * through DecompressionAdaptor (quantization/scalar/scalar.h:547-600): its codes are decompressed to fp32 as
 * scale * c + bias and prepared as the SQ search prepares an fp32 query, so the build's distances are the SQ
 * search's: L2 compresses the decompressed row again (the round trip may move codes) and scales the integer L2 of the
 * two code rows by scale^2; MIP is scale * <v, c> + bias * sum(v); cosine decompresses both sides.  The entry point is
 * the medoid of the codes as integers (find_medioid over get_datum).  The result is searched with
 * svsb200_index_create(..., SVSB200_SQ, {scale, bias}).
 *   codes       n x dim int8 / uint8 codes (`code_type` SVSB200_I8 / SVSB200_U8), dense, HOST (svsb200_sq_compress
 *               writes them);
 *   scale, bias the SQ parameters: the scale finite and positive, the bias finite;
 * everything else, the output layout, the defaults, the refusals and the parity bar are svsb200_build_vamana's. */
int svsb200_build_vamana_sq(
    const void* codes, int code_type, size_t n, size_t dim, int metric, float scale, float bias,
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
 * distances; ties by id).  GEMM shapes, all with L2 or MIP, plain storage, k <= 25 and n >= 512:
 *   - float32/float16 data with float32/float16 queries, and int8/uint8 data with float32 queries: the fp16 GEMM;
 *   - (int8, int8) and (uint8, uint8) up to dim 32768: an exact int8/uint8 GEMM (wgmma s32.s8.s8 / s32.u8.u8) whose
 *     candidate lists are exact in (distance, id) order, so no query needs the scan while distances stay below 2^24.
 * Other shapes (cosine, SQ, LVQ-8, integer rows wider than 32768, float rows wider than about 55000, ...) take
 * the scan.
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

/* Stored rows of a graph index.  Replaces: VamanaIndex::get_distance / MutableVamanaIndex::get_distance and
 * reconstruct_at (index/vamana/index.h:915-933, dynamic_index.h:1152-1190, 1306-1322).  An id is what the handle's
 * searches return: on a dynamic index the external id of a Valid slot (a Deleted or absent id is refused), otherwise a
 * row id plus any svsb200_set_id_offset.  Every id is checked before any device work; a refused call names the first
 * offending id and writes nothing.  All buffers are dense HOST memory; count = 0 succeeds and does nothing.  Plain and
 * SQ rows (LVQ-8 is refused); a replicated index reads its first replica.  Blocking.
 *   svsb200_index_distances: out[i] = the distance the index's search computes between query i (queries[count][dim]
 *     of `qdtype`, any type svsb200_search takes on this handle) and the row named ids[i], bit for bit: the same query
 *     preparation and the same expression tree, one warp per pair.
 *   svsb200_index_reconstruct: out[count][dim] float32: plain rows widened (float16 as the reference's Float16
 *     converts: subnormals become signed zero), SQ codes decompressed as scale * c + bias with two roundings
 *     (DecompressionAccessor, quantization/scalar/scalar.h:606-620). */
int svsb200_index_distances(svsb200_index* index, const void* queries, int qdtype, size_t count, const uint64_t* ids,
                            float* out);
int svsb200_index_reconstruct(svsb200_index* index, const uint64_t* ids, size_t count, float* out);

/* The svsb200_flat_search* split for a given k (host arithmetic only, like svsb200_flat_plan): for k <= 25 exactly what
 * svsb200_flat_plan returns, with `list_entries` = 33; for 26 <= k <= 121 and nq > 256 the deep lists of a flat index
 * (svsb200_flat_index_search*): `list_entries` = 129, one list per query and piece, lists_per_query x 129 <= 1024.
 * For 26 <= k <= 121 and nq <= 256 that search runs the exact scan: every output is 0 (segment_begin is untouched).
 * Fails for k = 0 and k > 121 (those searches do not use the GEMM). */
int svsb200_flat_plan_k(size_t nq, size_t n, size_t k, int sm_count, uint32_t* ctas, uint32_t* share,
                        uint32_t* lists_per_query, uint32_t* list_entries, uint64_t* segment_begin);

/* Flat index: rows only, no graph.  Replaces: svs::Flat (include/svs/index/flat/flat.h:159) and the runtime's
 * FlatIndex (bindings/cpp/include/svs/runtime/flat_index.h).  A distinct handle type, so that no graph call can be
 * made on it. */
typedef struct svsb200_flat svsb200_flat;

/* Uploads n x dim float32 / float16 / int8 / uint8 rows from HOST memory (row_stride_bytes apart, 0 = dense) to
 * `device` for `metric` (L2, IP or cosine).  Nothing for a graph is allocated. */
int svsb200_flat_index_create(const void* vectors, int dtype, size_t n, size_t dim, size_t row_stride_bytes, int metric,
                              int device, svsb200_flat** out);
/* Frees the handle and its device memory (NULL is ignored). */
int svsb200_flat_index_destroy(svsb200_flat* index);
/* Number of rows, their dimension, and the device memory the rows hold (the GEMM's operand tiles, built on the first
 * search, are not counted); 0 for NULL. */
size_t svsb200_flat_index_size(const svsb200_flat* index);
size_t svsb200_flat_index_dimensions(const svsb200_flat* index);
size_t svsb200_flat_index_device_bytes(const svsb200_flat* index);

/* FlatIndex::search / svs::Flat::search (index/flat/flat.h:421-465): the exact top k (1 <= k <= 1024) of every query
 * over all rows, ids as uint64, ties by id; the result equals svsb200_exhaustive_device over the same rows bit for bit.
 * Routing: k <= 25 runs the GEMM of svsb200_flat_search; 26 <= k <= 121 with nq > 256 the same GEMM with deep
 * candidate lists (129 entries per query and base range; one 128-query tile keeps at most 7 SMs busy with them, and
 * batches of one or two tiles run faster on the scan); larger k, cosine, n < 512 and the shapes svsb200_flat_search
 * leaves to the scan run the exact scan.  Queries: float32 / float16 over float rows, float32 or the rows' own type over int8 /
 * uint8 rows.  If k > n the rows are padded with all-ones ids and +-inf distances, as the scan pads them.
 * `fallback_queries` (optional) receives how many queries ran on the scan.  The device form is enqueued on `stream`
 * apart from one synchronisation (the fallback count). */
int svsb200_flat_index_search_device(svsb200_flat* index, const void* d_queries, int qdtype, size_t nq, size_t k,
                                     uint64_t* d_out_ids, float* d_out_dists, void* stream, uint32_t* fallback_queries);
/* The same with HOST buffers (blocking). */
int svsb200_flat_index_search(svsb200_flat* index, const void* queries, int qdtype, size_t nq, size_t k, uint64_t* out_ids,
                              float* out_dists);

/* Filtered exact search: FlatIndex::search with a predicate over the data index (index/flat/flat.h:421-465).
 * `id_bitmap` ((n + 31) / 32 words; NULL is refused): bit i % 32 of word i / 32 set means row i may be returned; bits
 * past n are ignored.  Each query gets the exact top k (1 <= k <= 1024) over the A allowed rows: the scan's bit-exact
 * distances, ordered by (distance, id), min(k, A) real entries, the rest padded with all-ones ids and +inf for EVERY
 * metric.  The result equals svsb200_flat_index_search over a Flat built from the allowed rows in ascending id order,
 * its ids mapped back, bit for bit (only the padding's distance differs: +inf).  Query and row types, metrics and
 * limits are svsb200_flat_index_search's.  `out_allowed` (optional) receives A.
 * Routes (svsb200_flat_filter_plan): the dense route runs svsb200_flat_index_search's routing with the disallowed
 * rows masked (the GEMM never offers them to a list, the scans skip them); the sparse route gathers the allowed rows
 * and runs the exact scan over them alone.  All per-call state lives in the caller stream's scratch, so searches of
 * one index with different bitmaps may run concurrently on different streams.  `fallback_queries` (optional) receives
 * how many queries ran on a scan.  The device form (queries, bitmap and outputs in device memory) is enqueued on
 * `stream` apart from one synchronisation for A and, on the dense route, the fallback count's. */
int svsb200_flat_index_search_filtered_device(svsb200_flat* index, const void* d_queries, int qdtype, size_t nq, size_t k,
                                              const uint32_t* d_id_bitmap, uint64_t* d_out_ids, float* d_out_dists,
                                              void* stream, size_t* out_allowed, uint32_t* fallback_queries);
/* The same with HOST buffers (blocking). */
int svsb200_flat_index_search_filtered(svsb200_flat* index, const void* queries, int qdtype, size_t nq, size_t k,
                                       const uint32_t* id_bitmap, uint64_t* out_ids, float* out_dists, size_t* out_allowed);
/* The route of a filtered flat search with `allowed` of `n` rows allowed (host arithmetic only): SPARSE when
 * allowed * 64 <= n (so always when allowed = 0), DENSE otherwise.  Fails for allowed > n. */
enum { SVSB200_FLAT_ROUTE_DENSE = 0, SVSB200_FLAT_ROUTE_SPARSE = 1 };
int svsb200_flat_filter_plan(size_t n, size_t allowed, int* route);

/* Dynamic index.  Replaces: MutableVamanaIndex(graph, data, entry_point, distance, external_ids, threadpool)
 * (include/svs/index/vamana/dynamic_index.h:178-202) for float32 / float16 plain storage (SQ codes:
 * svsb200_dynamic_create_sq) on one device, adjacency rows
 * of at most 128 neighbours, L2 / MIP / cosine.  Arguments as svsb200_index_create (dense rows), plus one distinct
 * external id per row; every slot starts Valid.  The result is an ordinary index handle:
 *   * svsb200_search / _cancellable / _device run MutableVamanaIndex::search (dynamic_index.h:482-571): the walk goes
 *     through Deleted slots (ValidBuilder, :93-108) but the MutableBuffer (dynamic_search_buffer.h) never counts or
 *     returns them; ids are the EXTERNAL ids (id_bytes must be 8).  Short rows are padded with all-ones / +-inf.
 *     These calls block until the kernels are done (a query whose list outgrows the buffer's room for Deleted entries
 *     is re-run with more room; the "dynamic_slack" option sets the initial room, "dynamic_reruns" counts re-runs);
 *     a cancellation predicate is polled while they run;
 *   * svsb200_search_filtered takes a bitmap over the slots, clears the slots that are not Valid from it and returns
 *     external ids; svsb200_range_search returns external ids;
 *   * flat, exhaustive and sharded searches, set_entry_points and set_id_offset fail on it.
 * External id 2^64 - 1 is reserved (it marks padding).
 * Mutations must not run concurrently with searches of the same index. */
int svsb200_dynamic_create(
    const void* vectors, int dtype, size_t n, size_t dim, const uint32_t* graph_rows, size_t graph_row_len,
    uint32_t entry_point, int metric, const uint64_t* external_ids, int device, svsb200_index** out);
/* delete_entries (dynamic_index.h:773-788): soft deletion.  Fails without changing anything unless every id is
 * present (and listed once); afterwards the slots are Deleted and the ids unknown. */
int svsb200_dynamic_delete(svsb200_index* index, const uint64_t* ids, size_t count);
/* all_ids / has_id: the external ids of the Valid slots, in slot order.  *count is the room of out_ids on entry
 * (out_ids may be NULL to ask for the count) and the number of ids on return. */
int svsb200_dynamic_ids(const svsb200_index* index, uint64_t* out_ids, size_t* count);
int svsb200_dynamic_has_id(const svsb200_index* index, uint64_t id, int* out);
/* The index's state for inspection: graph uint32[n][max_degree + 1] (degree first), status uint8[n]
 * (0 Empty, 1 Valid, 2 Deleted), external ids uint64[n] and the entry point; n = svsb200_index_size (slots).
 * Any output may be NULL. */
int svsb200_dynamic_export(const svsb200_index* index, uint32_t* graph_rows_out, uint8_t* status_out,
                           uint64_t* ext_ids_out, uint32_t* entry_point_out);

/* Mutation parameters: alpha_, construction_window_size_, max_candidates_ and prune_to_ of MutableVamanaIndex
 * (dynamic_index.h:316-371), used by svsb200_dynamic_add and svsb200_dynamic_consolidate.  0 selects the default:
 * alpha 1.2 (L2) / 0.95 (MIP, cosine), window 2 * max_degree, max_candidates 3 * window clamped to 512, prune_to
 * max_degree - 4 (max_degree when below 16).  The GPU builder's candidate pool holds 512 entries, so max_candidates
 * above 512 is an error, as are an alpha on the wrong side of 1, prune_to > max_degree and a window that leaves the
 * pool no room.  An index starts with the defaults (svsb200_dynamic_build: with its build parameters).  The search
 * history is always kept in full (use_full_search_history = true). */
int svsb200_dynamic_set_build_parameters(svsb200_index* index, float alpha, size_t window_size, size_t max_candidates,
                                         size_t prune_to);
/* Any output may be NULL. */
int svsb200_dynamic_get_build_parameters(const svsb200_index* index, float* alpha, size_t* window_size,
                                         size_t* max_candidates, size_t* prune_to);
/* add_points (dynamic_index.h:657-749): `count` rows of the index's dtype (dense, HOST) with one new external id
 * each.  Slots are chosen as the reference chooses them: Empty slots from first_empty (from slot 0 when reuse_empty
 * is non-zero), then new slots past the end; first_empty becomes max(first_empty, last slot + 1).  The rows are
 * linked in by one pass of the graph builder over the slots (VamanaBuilder::construct with alpha), whose search walks
 * Deleted slots too; the slots become Valid afterwards.  Everything (dtype, repeated, present or reserved ids) is
 * checked before anything changes.  `slots_out` (optional, `count` entries) receives the slots used.  The device
 * arrays grow geometrically; svsb200_index_size then reports the new number of slots. */
int svsb200_dynamic_add(svsb200_index* index, const void* vectors, int dtype, size_t count, const uint64_t* ids,
                        int reuse_empty, uint64_t* slots_out);
/* consolidate (dynamic_index.h:976-1013, consolidate.h): a Deleted entry point is replaced by the medoid of the Valid
 * rows (fails, changing nothing, when none is left); every Valid node with a neighbour that is not Valid gets its
 * row rebuilt from its Valid neighbours and the rows of the others, truncated to max_candidates and pruned to
 * prune_to with alpha; then every Deleted slot becomes Empty.  Ties among exactly equal distances are broken by id
 * (the reference leaves their order unspecified). */
int svsb200_dynamic_consolidate(svsb200_index* index);
/* compact (dynamic_index.h:817-916): the Valid slots move, in ascending order, to [0, size): rows, adjacency rows
 * (ids remapped), status, external ids and entry point; the allocations shrink to fit.  Fails without changing
 * anything while a Deleted slot is present (consolidate first). */
int svsb200_dynamic_compact(svsb200_index* index);
/* MutableVamanaIndex(parameters, data, external_ids, distance) (dynamic_index.h:208-261): svsb200_build_vamana's
 * two passes, then svsb200_dynamic_create; the build parameters (defaults as for svsb200_dynamic_set_build_parameters)
 * become the mutation parameters. */
int svsb200_dynamic_build(const void* vectors, int dtype, size_t n, size_t dim, int metric, float alpha,
                          size_t graph_max_degree, size_t window_size, size_t max_candidates, size_t prune_to,
                          const uint64_t* external_ids, int device, svsb200_index** out);
/* Dynamic index over scalar-quantised codes.  Replaces: MutableVamanaIndex over SQDataset<int8_t / uint8_t> (the
 * runtime's DynamicVamanaIndex with StorageKind::SQI8 and its uint8 twin): n x dim int8 / uint8 codes (`code_type`,
 * HOST, dense; svsb200_sq_compress writes them) with the `scale` (finite, positive) and `bias` (finite) they were
 * compressed with, which stay fixed for the life of the index.  Arguments otherwise as svsb200_dynamic_create (one
 * distinct external id per row, every slot Valid, n = 0 refused), and the result is an index handle with storage
 * SVSB200_SQ on which every svsb200_dynamic_* call and search works as on a float index, with these differences:
 *   * searches take float32 / float16 queries and measure with the SQ search's distances (svsb200_build_vamana_sq);
 *   * svsb200_dynamic_add takes float32 rows only (float16 and integer rows, and rows holding a NaN or an infinity, are
 *     refused before anything changes) and encodes them on the device as SQDataset::set_datum does (quantization/
 *     scalar/scalar.h:417-429): clamp(roundf((x - bias) / scale), MIN, MAX), so values outside the compressed range
 *     clamp; the codes are then linked in with the SQ builder's distances;
 *   * svsb200_dynamic_consolidate measures candidates with the build adaptor's general distance over SQ data
 *     (consolidate.h:241-244): the node decompressed and prepared as an SQ query, the SQ search's operators; a
 *     Deleted entry point is replaced by the medoid of the Valid codes as integers;
 *   * the rows take dim bytes of device memory (rounded up to 16) instead of 4 x dim or 2 x dim. */
int svsb200_dynamic_create_sq(const void* codes, int code_type, size_t n, size_t dim, float scale, float bias,
                              const uint32_t* graph_rows, size_t graph_row_len, uint32_t entry_point, int metric,
                              const uint64_t* external_ids, int device, svsb200_index** out);
/* MutableVamanaIndex(parameters, SQ data, external_ids, distance): svsb200_build_vamana_sq, then
 * svsb200_dynamic_create_sq; the build parameters become the mutation parameters, as in svsb200_dynamic_build.  The
 * code type, scale, bias and ids are checked before the build runs. */
int svsb200_dynamic_build_sq(const void* codes, int code_type, size_t n, size_t dim, int metric, float scale, float bias,
                             float alpha, size_t graph_max_degree, size_t window_size, size_t max_candidates,
                             size_t prune_to, const uint64_t* external_ids, int device, svsb200_index** out);

/* Dynamic flat index.  Replaces: DynamicFlatIndex (include/svs/index/flat/dynamic_flat.h:65) with svs::DynamicFlat
 * (orchestrators/dynamic_flat.h): an exact index over a mutable set of float32 / float16 / int8 / uint8 rows on one
 * device, L2 / MIP / cosine, addressed by external ids.  A distinct handle type: neither the graph calls nor the
 * svsb200_flat_index_* calls accept it.  Every slot is Valid or Empty; deleting a slot empties it at once (there is no
 * Deleted state and nothing to consolidate).  External id 2^64 - 1 is reserved (it marks padding).  Searches may run
 * concurrently with each other; mutations must not run concurrently with searches of the same index.  A mutation
 * (add, delete, compact) first waits for every search of the index enqueued so far, including the work that
 * svsb200_dynamic_flat_search_device leaves queued on the caller's stream, so it may follow such a call without a
 * synchronisation; a search enqueued while a mutation runs is the caller's error. */
typedef struct svsb200_dynamic_flat svsb200_dynamic_flat;

/* DynamicFlatIndex(data, external_ids, distance, threadpool) (dynamic_flat.h:94-113): n x dim dense rows from HOST
 * memory, one distinct external id each; every slot starts Valid.  n = 0 makes an empty index to be filled by
 * svsb200_dynamic_flat_add. */
int svsb200_dynamic_flat_create(const void* vectors, int dtype, size_t n, size_t dim, int metric, const uint64_t* external_ids,
                                int device, svsb200_dynamic_flat** out);
/* Frees the handle and its device memory (NULL is ignored). */
int svsb200_dynamic_flat_destroy(svsb200_dynamic_flat* index);
/* size() (dynamic_flat.h:146-150): Valid rows; the number of slots; dimensions() (:153); the device memory held by the
 * rows, statuses and external ids of the allocated slots (the GEMM's operand tiles are not counted).  0 for NULL. */
size_t svsb200_dynamic_flat_size(const svsb200_dynamic_flat* index);
size_t svsb200_dynamic_flat_num_slots(const svsb200_dynamic_flat* index);
size_t svsb200_dynamic_flat_dimensions(const svsb200_dynamic_flat* index);
size_t svsb200_dynamic_flat_device_bytes(const svsb200_dynamic_flat* index);
/* add_points (dynamic_flat.h:214-276): `count` rows of the index's dtype (dense, HOST) with one new external id each.
 * Empty slots are taken in ascending order from first_empty (from slot 0 when reuse_empty is non-zero), then new slots
 * past the end; first_empty becomes max(first_empty, last slot + 1).  Everything (dtype, repeated, present or reserved
 * ids) is checked before anything changes.  `slots_out` (optional, `count` entries) receives the slots used.  The
 * device arrays grow geometrically. */
int svsb200_dynamic_flat_add(svsb200_dynamic_flat* index, const void* vectors, int dtype, size_t count, const uint64_t* ids,
                             int reuse_empty, uint64_t* slots_out);
/* delete_entries (dynamic_flat.h:292-307): the slots become Empty and first_empty = min(first_empty, slot).  Fails
 * without changing anything unless every id is present and listed once. */
int svsb200_dynamic_flat_delete(svsb200_dynamic_flat* index, const uint64_t* ids, size_t count);
/* compact (dynamic_flat.h:335-367): the Valid slots move, in ascending order, to [0, size); first_empty = size; the
 * allocations shrink to fit.  (The reference's batch size only tunes its copy; there is none here.)  consolidate
 * (:376-378) is a no-op and has no function here. */
int svsb200_dynamic_flat_compact(svsb200_dynamic_flat* index);
/* external_ids / has_id (dynamic_flat.h:174,182-197): the external ids of the Valid slots, in slot order.  *count is
 * the room of out_ids on entry (out_ids may be NULL to ask for the count) and the number of ids on return. */
int svsb200_dynamic_flat_ids(const svsb200_dynamic_flat* index, uint64_t* out_ids, size_t* count);
int svsb200_dynamic_flat_has_id(const svsb200_dynamic_flat* index, uint64_t id, int* out);
/* The slot state for inspection: status uint8[slots] (0 Empty, 1 Valid) and external ids uint64[slots] (2^64 - 1 for
 * an Empty slot); slots = svsb200_dynamic_flat_num_slots.  Either output may be NULL. */
int svsb200_dynamic_flat_export(const svsb200_dynamic_flat* index, uint8_t* status_out, uint64_t* ext_ids_out);
/* search (dynamic_flat.h:513-573): the exact top k (1 <= k <= 1024) of every query over the Valid slots, as EXTERNAL
 * ids, with the routing, query types, distances and fallback count of svsb200_flat_index_search_device; ties are
 * broken by slot (the reference leaves their order unspecified).  The result equals svsb200_flat_index_search over the
 * Valid rows in slot order, its ids mapped to the external ids, bit for bit.  Rows are padded with all-ones ids and
 * +-inf distances when fewer than k slots are Valid.  The device form is enqueued on `stream` apart from the
 * fallback count's synchronisation (and, on the first search after a mutation, the maximum norm over the Valid rows). */
int svsb200_dynamic_flat_search_device(svsb200_dynamic_flat* index, const void* d_queries, int qdtype, size_t nq, size_t k,
                                       uint64_t* d_out_ids, float* d_out_dists, void* stream, uint32_t* fallback_queries);
/* The same with HOST buffers (blocking). */
int svsb200_dynamic_flat_search(svsb200_dynamic_flat* index, const void* queries, int qdtype, size_t nq, size_t k,
                                uint64_t* out_ids, float* out_dists);
/* search with a predicate over the data index (dynamic_flat.h:513-573, 653-661): svsb200_flat_index_search_filtered's
 * contract with the bitmap over SLOTS ((num_slots + 31) / 32 words; Empty slots' bits are ignored), EXTERNAL ids and
 * ties by slot.  The result equals svsb200_flat_index_search over the rows of the slots that are both Valid and
 * allowed, in slot order, its ids mapped to the external ids.  `out_allowed` receives the number of such slots.  As
 * every search here, the device form records the scratch's event, so a mutation waits for it. */
int svsb200_dynamic_flat_search_filtered_device(svsb200_dynamic_flat* index, const void* d_queries, int qdtype, size_t nq,
                                                size_t k, const uint32_t* d_slot_bitmap, uint64_t* d_out_ids,
                                                float* d_out_dists, void* stream, size_t* out_allowed,
                                                uint32_t* fallback_queries);
/* The same with HOST buffers (blocking). */
int svsb200_dynamic_flat_search_filtered(svsb200_dynamic_flat* index, const void* queries, int qdtype, size_t nq, size_t k,
                                         const uint32_t* slot_bitmap, uint64_t* out_ids, float* out_dists,
                                         size_t* out_allowed);

/* IVF index.  Replaces: IVFIndex (include/svs/index/ivf/index.h) with svs::IVF and svs::Clustering
 * (index/ivf/kmeans.h, common.h): float32 / float16 rows on one device, L2 / MIP / cosine, grouped into C clusters
 * around float32 centroids.  A search probes, per query, the n_probes centroids nearest under the metric (the flat
 * search's exact distances over the centroids, ties to the lower centroid; the reference ranks them from an sgemm whose
 * rounding is the BLAS's) and returns the exact top k (1 <= k <= 1024) over the union of the probed clusters' rows:
 * the search path's bit-exact distances, ordered by distance, then original row id, padded with all-ones ids and
 * +-inf distances when the probed clusters hold fewer than k rows.  With n_probes = C the result equals
 * svsb200_exhaustive_device over the same rows bit for bit.  Integer and LVQ rows are refused; SQ codes are assembled by
 * svsb200_ivf_create_sq. */
typedef struct svsb200_ivf svsb200_ivf;

/* The random sequence of svsb200_ivf_cluster: the first `count` outputs of splitmix64 seeded with `seed` (state +=
 * 0x9E3779B97F4A7C15, then the two xor-shift-multiply rounds).  An own sequence, documented so that a model can
 * reproduce the clustering bit for bit. */
int svsb200_ivf_random(uint64_t seed, size_t count, uint64_t* out);
/* Clustering.build / kmeans_clustering (ivf/kmeans.h:40-131, common.h:446-634) over n x dim dense rows in HOST memory,
 * the flat (non-hierarchical) k-means, deterministic: is_hierarchical must be 0 (hierarchical k-means is refused).
 *   1. m = min(n, max(min(2 C, n), ceil(float(n) * training_fraction))) training rows, refused when m < C: the first m
 *      of a Fisher-Yates shuffle of [0, n) (draw i swaps position i with i + r % (n - i)), taken in ascending order;
 *   2. centroid c = training row p[c], p the first C of the same shuffle of [0, m) (continuing the sequence);
 *   3. num_iterations rounds of: assign every training row to its exact nearest centroid (the flat search, k = 1, in
 *      batches of minibatch_size rows, which changes no result); add every member, in ascending row order, in float32
 *      onto its old centroid and multiply a centroid with members by float(1.0 / (count + 1)); split every empty
 *      cluster i in ascending order as the reference does (j cycles from 0 over the populated clusters until a draw
 *      r = (x >> 40) 2^-24 < float(count_j) / float(m); i copies j; even coordinates of i and odd ones of j times
 *      1 + 2^-10, the others times 1 - 2^-10, rounded from double; count_i = count_j / 2, count_j -= count_i); for MIP
 *      and cosine, normalise every centroid (x * (1 / sqrt(sequential float32 sum of squares)), zero rows untouched),
 *      as also done once after step 2;
 *   4. assign all n rows to their exact nearest final centroid.
 * out_centroids: float32 [C][dim]; out_assignments: uint32 [n]. */
int svsb200_ivf_cluster(const void* vectors, int dtype, size_t n, size_t dim, int metric, size_t num_centroids,
                        size_t minibatch_size, size_t num_iterations, int is_hierarchical, float training_fraction,
                        uint64_t seed, int device, float* out_centroids, uint32_t* out_assignments);
/* hierarchical_kmeans_clustering (ivf/hierarchical_kmeans.h:68-358), the reference's default IVF clustering, over the
 * rows svsb200_ivf_cluster takes (float32 / float16, L2 / MIP / cosine, the same checks), deterministic:
 *   1. the m training rows of svsb200_ivf_cluster's step 1 (m from C, refused when m < C);
 *   2. L1 = level1_clusters, or size_t(sqrt(double(C))) when it is 0; refused when L1 > C;
 *   3. svsb200_ivf_cluster's steps 2-3 with L1 centroids on the sample (split draws take m as denominator);
 *   4. every training row to its exact nearest level-1 centroid: t_g rows in group g;
 *   5. c_g = size_t(double(t_g) / m * C) level-2 centroids per group, then until they sum to C: j = r % L1 for the next
 *      draw r, c_j += 1 unless t_j = 0 or c_j = t_j (then the draw is discarded), so that c_g <= t_g always;
 *   6. every row to its exact nearest level-1 centroid among the groups with c_g > 0 (ties to the lower index);
 *   7. per group g with c_g > 0, all groups in lockstep: its training rows in ascending order; centroid j = its row
 *      p[j], p the first c_g of a shuffle of [0, t_g); num_iterations rounds of step 3 among its own rows and centroids
 *      (assignment to the nearest of its own centroids, the same update, splits with t_g as denominator, MIP / cosine
 *      normalised); finally each row of group g goes to the nearest of g's final centroids.
 * The random sequence is svsb200_ivf_random's: the main stream (seeded with `seed`) draws the sample shuffle, the
 * level-1 shuffle, the level-1 splits, the draws of step 5, then one value per level-1 group in ascending order (groups
 * with c_g = 0 included), which seeds that group's own stream for its shuffle and then its splits.  Distances are exact
 * (the search path's), ties to the lower centroid.
 * out_centroids: float32 [C][dim], group by group (group g's from cluster_start_g = sum of c_h over h < g);
 * out_assignments: uint32 [n], cluster_start_g + the row's centroid within its group g (not necessarily the globally
 * nearest centroid); out_level2_counts (optional, NULL allowed): uint32 [L1], c_g. */
int svsb200_ivf_cluster_hierarchical(const void* vectors, int dtype, size_t n, size_t dim, int metric, size_t num_centroids,
                                     size_t level1_clusters, size_t minibatch_size, size_t num_iterations,
                                     float training_fraction, uint64_t seed, int device, float* out_centroids,
                                     uint32_t* out_assignments, uint32_t* out_level2_counts);
/* IVFIndex::assemble_from_clustering: n x dim rows (HOST) grouped by `assignments` (uint32 [n], each < C; NULL:
 * every row goes to its exact nearest centroid, computed on the device) around C float32 centroids [C][dim]. */
int svsb200_ivf_create(const void* vectors, int dtype, size_t n, size_t dim, int metric, const float* centroids,
                       size_t num_centroids, const uint32_t* assignments, int device, svsb200_ivf** out);
/* Scalar quantisation, SQDataset<int8_t / uint8_t>::compress (quantization/scalar/scalar.h:447-469), on the device:
 * n x dim float32 rows (HOST) become codes (int8 / uint8, `code_type`, HOST, n x dim) with one global scale and bias:
 * scale = (max - min) / (MAX - MIN), bias = min - MIN * scale (each operation rounded on its own), code =
 * clamp(roundf((x - bias) / scale), MIN, MAX), [MIN, MAX] = [-128, 127] or [0, 255].  Data holding a NaN or an infinity,
 * and constant data (max == min), are refused: the reference's result is undefined there. */
int svsb200_sq_compress(const float* data, size_t n, size_t dim, int code_type, int device, void* out_codes, float* out_scale,
                        float* out_bias);
/* assemble_from_clustering over SQ codes (IVFIndex with StorageKind::SQI8 and its uint8 twin): n x dim int8 / uint8
 * codes (HOST) with the `scale` (finite, positive) and `bias` (finite) they were compressed with, C float32 centroids,
 * and REQUIRED assignments (uint32 [n], each < C): without float rows nothing can be ranked against the centroids.
 * The handle is an ordinary svsb200_ivf.  The probe is unchanged (float32 / float16 queries against the float32
 * centroids); the result is the exact top k over the probed clusters with the SQ search path's bit-exact distances
 * (EuclideanCompressed, InnerProductCompressed, CosineSimilarityCompressed), ordered by (distance, id).  With
 * n_probes = C it equals svsb200_exhaustive_device on an SQ svsb200_index over the same codes.  L2 runs on the integer
 * tensor cores (int32 sums, which wrap past dim * 255^2 >= 2^31 exactly as the search path's do); MIP and cosine run
 * the float trees. */
int svsb200_ivf_create_sq(const void* codes, int code_type, size_t n, size_t dim, int metric, float scale, float bias,
                          const float* centroids, size_t num_centroids, const uint32_t* assignments, int device,
                          svsb200_ivf** out);
/* Frees the handle and its device memory (NULL is ignored). */
int svsb200_ivf_destroy(svsb200_ivf* index);
/* Rows, dimensions, clusters, device memory held (rows, ids, centroids); 0 for NULL. */
size_t svsb200_ivf_size(const svsb200_ivf* index);
size_t svsb200_ivf_dimensions(const svsb200_ivf* index);
size_t svsb200_ivf_num_clusters(const svsb200_ivf* index);
size_t svsb200_ivf_device_bytes(const svsb200_ivf* index);
/* Rows per cluster (uint32 [C]) and the centroids (float32 [C][dim]), HOST buffers. */
int svsb200_ivf_cluster_sizes(const svsb200_ivf* index, uint32_t* out);
int svsb200_ivf_centroids(const svsb200_ivf* index, float* out);
/* search: float32 / float16 queries (DEVICE buffers), 1 <= k <= 1024, 1 <= n_probes <= min(C, 1024); ids uint64
 * [nq][k], distances float32 [nq][k].  Enqueued on `stream` apart from the synchronisations of the centroid search. */
int svsb200_ivf_search_device(svsb200_ivf* index, const void* d_queries, int qdtype, size_t nq, size_t k, size_t n_probes,
                              uint64_t* d_out_ids, float* d_out_dists, void* stream);
/* The same with HOST buffers (blocking). */
int svsb200_ivf_search(svsb200_ivf* index, const void* queries, int qdtype, size_t nq, size_t k, size_t n_probes,
                       uint64_t* out_ids, float* out_dists);
/* Filtered search (svs::runtime::v0::IVFIndex::search with an IDFilter): the plain search restricted to the ALLOWED rows,
 * with the probe count growing per query until k allowed rows are in reach.
 *   Bitmap: bit i (word i / 32, bit i % 32) set = original id i may be returned; (n + 31) / 32 words.  NULL is refused.
 *   Growth: the probe order is the plain search's (the flat search over the centroids, ties to the lower centroid).
 *   P_0 = n_probes, P_{j+1} = min(4 P_j, P_max), P_max = min(C, 1024).  Query q uses the first P_j whose nearest P_j
 *   clusters hold at least k allowed rows, or P_max when none does.  The choice is per query: a query's row does not
 *   depend on the other queries of the batch.
 *   Result: the exact top k over the allowed rows of the query's probed clusters, with the scan's bit-exact distances,
 *   ordered by distance, then original id.  Short rows are padded with all-ones ids and +inf distances for EVERY metric
 *   (as svsb200_search_filtered; the plain search pads MIP / cosine with -inf).
 *   Per-query outputs, uint32 [nq] each, each may be NULL: out_probes the P used, out_allowed the allowed rows in those
 *   clusters, out_rows all rows in those clusters; min(k, out_allowed) entries of the row are not padding.
 *   Limits and refusals are the plain search's (1 <= k <= 1024, 1 <= n_probes <= P_max, float32 / float16 queries,
 *   every row type and storage kind). */
int svsb200_ivf_search_filtered(svsb200_ivf* index, const void* queries, int qdtype, size_t nq, size_t k, size_t n_probes,
                                const uint32_t* id_bitmap, uint64_t* out_ids, float* out_dists, uint32_t* out_probes,
                                uint32_t* out_allowed, uint32_t* out_rows);
/* The same with the queries, bitmap and every output in DEVICE memory, enqueued on `stream` apart from the
 * synchronisations of the centroid searches and of each growth decision (which reads the allowed counts back). */
int svsb200_ivf_search_filtered_device(svsb200_ivf* index, const void* d_queries, int qdtype, size_t nq, size_t k,
                                       size_t n_probes, const uint32_t* d_id_bitmap, uint64_t* d_out_ids, float* d_out_dists,
                                       uint32_t* d_out_probes, uint32_t* d_out_allowed, uint32_t* d_out_rows, void* stream);

/* The shape svsb200_ivf_search* and svsb200_dynamic_ivf_search* run (introspection, host arithmetic only, like
 * svsb200_flat_plan; the search calls this same arithmetic) for an index of `dim`-element rows of `dtype`: float32 /
 * float16 with `storage` SVSB200_PLAIN, or int8 / uint8 codes with SVSB200_SQ; `dynamic` nonzero for the dynamic index
 * and the filtered searches (the leaf's DYN form).
 *   tile_rows:        rows per shared-memory ring slot: 32, halved while two slots would pass 96 KB;
 *   queries_per_item: Q, the queries a work item scores together (at most 64);
 *   ctas_per_sm:      2 where Q >= 1 fits half of the 227 KB - 1 KB a CTA may use, else 1;
 *   query_chunk:      queries per pass, min(nq, max(1, min(8192, 256 MiB / (12 n_probes k))));
 *   leaf:             0 = the float-tree scan (float rows; SQ MIP / cosine), 1 = the SQ L2 tensor-core scan;
 *   static_dim:       96 or 128 where the float tree runs at that static dimension, else 0 (and 0 for leaf 1);
 *   rows_per_pass:    rows per group and pass of the float tree (1 or 2; 0 for leaf 1);
 *   smem_bytes:       dynamic shared memory of one CTA.
 * Fails, with the search's own message, where no Q >= 1 fits one CTA per SM. */
int svsb200_ivf_plan(size_t dim, int dtype, int storage, int metric, size_t k, size_t n_probes, size_t nq, int dynamic,
                     uint32_t* tile_rows, uint32_t* queries_per_item, uint32_t* ctas_per_sm, uint32_t* query_chunk,
                     uint32_t* leaf, uint32_t* static_dim, uint32_t* rows_per_pass, uint64_t* smem_bytes);
/* The grouped assignment of svsb200_ivf_cluster_hierarchical for `dim`-element rows (host arithmetic only): `tile`
 * rows per work item (64, halved while two tiles of prepared rows would pass 96 KB), the group's centroids staged
 * `chunk` at a time, `smem_bytes` of dynamic shared memory per CTA.  Fails, with the clustering's own message, where
 * that passes 227 KB - 1 KB. */
int svsb200_ivf_group_plan(size_t dim, uint32_t* tile, uint32_t* chunk, uint64_t* smem_bytes);

/* Dynamic IVF index.  Replaces: DynamicIVFIndex (include/svs/index/ivf/dynamic_ivf.h) with svs::DynamicIVF: the IVF
 * index over a mutable set of float32 / float16 rows (or SQ codes, svsb200_dynamic_ivf_create_sq) on one device, L2 /
 * MIP / cosine, addressed by external ids.  A distinct handle type.  Every slot (internal id) is Valid or Empty; a
 * delete empties it at once and leaves a tombstone in its cluster, which no search returns.  The centroids never move
 * after assembly: an added row joins its nearest centroid, ranked as a probe ranks centroids (the flat search at k = 1,
 * ties to the lower centroid).  External id 2^64 - 1 is reserved (it marks padding).  Searches may run concurrently
 * with each other; a mutation (add, delete, compact) first waits for every search of the index enqueued so far,
 * including the work that svsb200_dynamic_ivf_search_device leaves queued on the caller's stream, so it may follow such
 * a call without a synchronisation; a search enqueued while a mutation runs is the caller's error. */
typedef struct svsb200_dynamic_ivf svsb200_dynamic_ivf;

/* assemble_from_clustering: n x dim rows (HOST) with one distinct external id each, grouped by `assignments` (uint32
 * [n], each < C; NULL: every row goes to its nearest centroid) around C float32 centroids [C][dim].  Row i takes slot
 * i.  n = 0 makes an empty index to be filled by svsb200_dynamic_ivf_add. */
int svsb200_dynamic_ivf_create(const void* vectors, int dtype, size_t n, size_t dim, int metric, const float* centroids,
                               size_t num_centroids, const uint32_t* assignments, const uint64_t* external_ids, int device,
                               svsb200_dynamic_ivf** out);
/* assemble_from_clustering over SQ codes (DynamicIVFIndex with StorageKind::SQI8 and its uint8 twin): n x dim int8 /
 * uint8 codes (HOST) with the `scale` (finite, positive) and `bias` (finite) they were compressed with, C float32
 * centroids, one distinct external id per row, and assignments (uint32 [n], each < C), REQUIRED when n > 0: without
 * float rows nothing can be ranked against the centroids.  Row i takes slot i.  n = 0 makes an empty SQ index whose
 * scale and bias are fixed from the start.  Slots, mutations and refusals are the float index's, except that
 * svsb200_dynamic_ivf_add takes float32 rows only (float16 and integer rows, and rows holding a NaN or an infinity, are
 * refused before anything changes): each joins its nearest centroid, ranked from its float32 values as in a float
 * index, and is encoded with the index's scale and bias as SQDataset::set_datum does (quantization/scalar/scalar.h:
 * 417-429): clamp(roundf((x - bias) / scale), MIN, MAX), each operation rounded on its own, so that values outside
 * the compressed range clamp.  A search returns the exact top k over the Valid rows of the probed clusters with the SQ
 * search path's bit-exact distances (as svsb200_ivf_create_sq), ordered by (distance, slot); with n_probes = C it
 * equals svsb200_exhaustive_device on an SQ svsb200_index over the Valid slots' codes in slot order. */
int svsb200_dynamic_ivf_create_sq(const void* codes, int code_type, size_t n, size_t dim, int metric, float scale, float bias,
                                  const float* centroids, size_t num_centroids, const uint32_t* assignments,
                                  const uint64_t* external_ids, int device, svsb200_dynamic_ivf** out);
/* Frees the handle and its device memory (NULL is ignored). */
int svsb200_dynamic_ivf_destroy(svsb200_dynamic_ivf* index);
/* Valid rows, slots (Valid or Empty), dimensions, clusters, and the device memory held (rows pool with its dead
 * regions until a compaction, entries, statuses, external ids, centroids); 0 for NULL. */
size_t svsb200_dynamic_ivf_size(const svsb200_dynamic_ivf* index);
size_t svsb200_dynamic_ivf_num_slots(const svsb200_dynamic_ivf* index);
size_t svsb200_dynamic_ivf_dimensions(const svsb200_dynamic_ivf* index);
size_t svsb200_dynamic_ivf_num_clusters(const svsb200_dynamic_ivf* index);
size_t svsb200_dynamic_ivf_device_bytes(const svsb200_dynamic_ivf* index);
/* Valid rows per cluster (uint32 [C]) and the centroids (float32 [C][dim]), HOST buffers. */
int svsb200_dynamic_ivf_cluster_sizes(const svsb200_dynamic_ivf* index, uint32_t* out);
int svsb200_dynamic_ivf_centroids(const svsb200_dynamic_ivf* index, float* out);
/* add_points (dynamic_ivf.h:474-527): `count` rows of the index's dtype (float32 for an SQ index; dense, HOST) with one
 * new external id each.
 * Without reuse_empty every row takes a new slot past the end; with it, Empty slots are taken in ascending order from
 * slot 0 first.  Each row is appended to its nearest centroid's cluster, in input order.  Everything (dtype, repeated,
 * present or reserved ids, 2^31-1 slots) is checked before anything changes.  `slots_out` (optional, `count` entries)
 * receives the slots used. */
int svsb200_dynamic_ivf_add(svsb200_dynamic_ivf* index, const void* vectors, int dtype, size_t count, const uint64_t* ids,
                            int reuse_empty, uint64_t* slots_out);
/* delete_entries (dynamic_ivf.h:547-636): the slots become Empty and their stored rows tombstones.  Fails without
 * changing anything unless every id is present and listed once. */
int svsb200_dynamic_ivf_delete(svsb200_dynamic_ivf* index, const uint64_t* ids, size_t count);
/* compact (dynamic_ivf.h:932-961): the Valid slots are renumbered 0 .. size-1 in slot order, the tombstones dropped;
 * every cluster keeps the order of its rows and is laid out tightly again.  consolidate is a no-op and has no function
 * here. */
int svsb200_dynamic_ivf_compact(svsb200_dynamic_ivf* index);
/* The external ids of the Valid slots, in slot order (*count: room on entry, out_ids may be NULL; ids on return), and
 * has_id. */
int svsb200_dynamic_ivf_ids(const svsb200_dynamic_ivf* index, uint64_t* out_ids, size_t* count);
int svsb200_dynamic_ivf_has_id(const svsb200_dynamic_ivf* index, uint64_t id, int* out);
/* The slot state for inspection, per slot: status uint8 (0 Empty, 1 Valid), external id uint64 (2^64 - 1 when Empty)
 * and cluster uint32 (2^32 - 1 when Empty); slots = svsb200_dynamic_ivf_num_slots.  Any output may be NULL. */
int svsb200_dynamic_ivf_export(const svsb200_dynamic_ivf* index, uint8_t* status_out, uint64_t* ext_ids_out,
                               uint32_t* cluster_out);
/* search: the exact top k (1 <= k <= 1024) over the Valid rows of the n_probes (1 <= n_probes <= min(C, 1024)) probed
 * clusters, as EXTERNAL ids: the scan's bit-exact distances, ordered by distance, then slot, padded with all-ones ids
 * and +-inf distances.  With n_probes = C the result is the exact scan over the Valid rows in slot order, its ids mapped
 * through the slots.  Queries float32 / float16 in DEVICE buffers, enqueued on `stream` apart from the synchronisations
 * of the centroid search. */
int svsb200_dynamic_ivf_search_device(svsb200_dynamic_ivf* index, const void* d_queries, int qdtype, size_t nq, size_t k,
                                      size_t n_probes, uint64_t* d_out_ids, float* d_out_dists, void* stream);
/* The same with HOST buffers (blocking). */
int svsb200_dynamic_ivf_search(svsb200_dynamic_ivf* index, const void* queries, int qdtype, size_t nq, size_t k,
                               size_t n_probes, uint64_t* out_ids, float* out_dists);
/* Filtered search: svsb200_ivf_search_filtered over the Valid rows, with the bitmap over SLOTS ((num_slots + 31) / 32
 * words, bit s = slot s may be returned; the bits of Empty slots are ignored), as svsb200_search_filtered does for the
 * dynamic Vamana index.  Results are ordered by distance, then slot, and returned as EXTERNAL ids; out_rows counts the
 * Valid rows of the probed clusters.  Like every search, a mutation waits for it, the device form included. */
int svsb200_dynamic_ivf_search_filtered(svsb200_dynamic_ivf* index, const void* queries, int qdtype, size_t nq, size_t k,
                                        size_t n_probes, const uint32_t* slot_bitmap, uint64_t* out_ids, float* out_dists,
                                        uint32_t* out_probes, uint32_t* out_allowed, uint32_t* out_rows);
int svsb200_dynamic_ivf_search_filtered_device(svsb200_dynamic_ivf* index, const void* d_queries, int qdtype, size_t nq,
                                               size_t k, size_t n_probes, const uint32_t* d_slot_bitmap, uint64_t* d_out_ids,
                                               float* d_out_dists, uint32_t* d_out_probes, uint32_t* d_out_allowed,
                                               uint32_t* d_out_rows, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* SVSB200_H */
