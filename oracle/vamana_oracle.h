/* oracle/vamana_oracle.h -- CPU restatement of the reference Vamana batched-search path.
 *
 * TEST INFRASTRUCTURE ONLY.  Nothing under scalablevectorsearch_b200/ or include/ may
 * include, link or load this; it exists so tests/, __graft_entry__.smoke() and bench.py's
 * cpu_baseline leg can check the CUDA path.  Pinned against the compiled reference
 * (oracle/_ref/libsvsref.so) and the reference's golden recalls by tests/test_oracle_*.py.
 */
#ifndef VAMANA_ORACLE_H
#define VAMANA_ORACLE_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

enum { ORACLE_F32 = 0, ORACLE_F16 = 1, ORACLE_I8 = 2, ORACLE_U8 = 3 };
enum { ORACLE_L2 = 0, ORACLE_IP = 1, ORACLE_COS = 2 };

const char* oracle_last_error(void);

/* distance::compute(f, query, row) for every row, after one maybe_fix_argument(query). */
int oracle_distance_rows(int metric, int qtype, int dtype, const void* query, const void* rows,
                         size_t nrows, size_t dim, float* out);
/* The same over compressed rows, through the code the SQ and LVQ-8 index searches use:
 * SQ int8 / uint8 codes (dense, dim bytes each) with their scale and bias, and LVQ-8 rows
 * (svsb200_lvq8_row_stride apart) with the dataset mean.  Queries are float32 or float16. */
int oracle_sq_distance_rows(int metric, int qtype, int code_type, float scale, float bias, const void* query,
                            const void* codes, size_t nrows, size_t dim, float* out);
int oracle_lvq8_distance_rows(int metric, int qtype, const void* query, const void* rows, size_t nrows, size_t dim,
                              const float* mean, float* out);

/* graph_rows: uint32[n][max_degree+1], out-degree in element 0 (reference in-memory layout). */
void* oracle_index_create(int dtype, const void* data, size_t n, size_t dim,
                          const uint32_t* graph_rows, size_t max_degree, uint32_t entry_point,
                          int metric, size_t threads);
/* data is f32; codes/scale/bias are produced with the reference's SQDataset::compress rule. */
void* oracle_sq_index_create(int code_type, const float* data, size_t n, size_t dim,
                             const uint32_t* graph_rows, size_t max_degree, uint32_t entry_point,
                             int metric, size_t threads, float* scale_out, float* bias_out,
                             void* codes_out);
/* LVQ-8 (own specification; the reference's LVQ is closed source, parity unpinned). */
size_t oracle_lvq8_row_stride(size_t dim);
/* Fails, naming the first offending row, on a non-finite residual or float16 constant. */
int oracle_lvq8_compress(const float* data, size_t n, size_t dim, const float* mean, void* out_rows);
void* oracle_lvq8_index_create(const void* rows, size_t n, size_t dim, const float* mean,
                               const uint32_t* graph_rows, size_t max_degree, uint32_t entry_point, int metric);
/* Several (distinct) entry points, as VamanaIndex::entry_point_ allows (index/vamana/index.h:304-312). */
int oracle_index_set_entry_points(void* index, const uint32_t* entry_points, size_t count);
void oracle_index_destroy(void* index);
int oracle_index_search(void* index, int qtype, const void* queries, size_t nq, size_t k,
                        size_t window, size_t capacity, int visited_set, uint64_t* ids,
                        float* dists);
int oracle_index_counts(void* index, int qtype, const void* queries, size_t nq, size_t window,
                        size_t capacity, uint64_t* hops, uint64_t* evals);

#ifdef __cplusplus
}
#endif
#endif
