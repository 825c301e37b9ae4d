/* oracle/vamana_oracle.c -- plain-C restatement of the reference Vamana batched-search path.
 *
 * TEST INFRASTRUCTURE ONLY (see vamana_oracle.h).  Every function cites the reference
 * file:line (relative to /root/reference/include/svs) whose behaviour it restates.  The
 * restatement is pinned bit-for-bit against the compiled reference (oracle/_ref) by
 * tests/test_oracle_golden.py (live _ref comparison) and against the reference's 17 golden recalls by
 * tests/test_oracle_golden.py.
 *
 * Floating-point contract (SURVEY.md Appendix B): the reference's AVX-512 kernels are a
 * fixed expression tree -- 16 lanes, 4 accumulators over 64-element blocks, fused
 * multiply-add, (s0+s1)+(s2+s3), 16-wide tail blocks into s0, masked remainder, then the
 * 8/4/2/1 butterfly of _mm512_reduce_add_ps.  Compile with -ffp-contract=off so the only
 * fused operations are the explicit fmaf() calls.
 */
#include "vamana_oracle.h"

#include <math.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

static _Thread_local char g_error[256];
const char* oracle_last_error(void) { return g_error; }
#define FAIL(...)                                          \
    do {                                                   \
        snprintf(g_error, sizeof(g_error), __VA_ARGS__);   \
        return 1;                                          \
    } while (0)

/* ------------------------------------------------------------------------------------
 * Element conversion.
 * ---------------------------------------------------------------------------------- */

/* Exact IEEE binary16 -> binary32 including subnormals: what the SIMD loads do
 * (`_mm512_cvtph_ps`, core/distance/simd_utils.h:270-276). */
static float f16_to_f32_exact(uint16_t h) {
    uint32_t s = ((uint32_t)h & 0x8000u) << 16, e = (h >> 10) & 31u, m = h & 1023u, r;
    if (e == 0) {
        if (m == 0) {
            r = s;
        } else {
            int sh = 0;
            while (!(m & 1024u)) {
                m <<= 1;
                ++sh;
            }
            m &= 1023u;
            r = s | ((uint32_t)(113 - sh) << 23) | (m << 13);
        }
    } else if (e == 31) {
        r = s | 0x7F800000u | (m << 13);
    } else {
        r = s | ((e + 112u) << 23) | (m << 13);
    }
    float f;
    memcpy(&f, &r, 4);
    return f;
}

/* The reference's *scalar* Float16 -> float (lib/float16.h:45-52): flushes subnormals
 * to signed zero.  Used wherever the reference touches Float16 outside a SIMD kernel
 * (query norm, SQ query preparation). */
static float f16_to_f32_scalar(uint16_t x) {
    uint32_t e = (x & 0x7C00u) >> 10, m = ((uint32_t)x & 0x03FFu) << 13;
    uint32_t r = ((uint32_t)x & 0x8000u) << 16 | (uint32_t)(e != 0) * ((e + 112u) << 23 | m);
    float f;
    memcpy(&f, &r, 4);
    return f;
}

static size_t elem_size(int t) { return t == ORACLE_F32 ? 4 : t == ORACLE_F16 ? 2 : 1; }

/* SIMD-load conversion to float (simd_utils.h:262-301): all exact. */
static void load_as_float(int t, const void* src, size_t n, float* dst) {
    switch (t) {
        case ORACLE_F32: memcpy(dst, src, n * 4); break;
        case ORACLE_F16:
            for (size_t i = 0; i < n; ++i) dst[i] = f16_to_f32_exact(((const uint16_t*)src)[i]);
            break;
        case ORACLE_I8:
            for (size_t i = 0; i < n; ++i) dst[i] = (float)((const int8_t*)src)[i];
            break;
        default:
            for (size_t i = 0; i < n; ++i) dst[i] = (float)((const uint8_t*)src)[i];
    }
}

/* Scalar element -> float as `static_cast<float>(T)` does it in non-SIMD code. */
static float scalar_as_float(int t, const void* src, size_t i) {
    switch (t) {
        case ORACLE_F32: return ((const float*)src)[i];
        case ORACLE_F16: return f16_to_f32_scalar(((const uint16_t*)src)[i]);
        case ORACLE_I8: return (float)((const int8_t*)src)[i];
        default: return (float)((const uint8_t*)src)[i];
    }
}

/* ------------------------------------------------------------------------------------
 * The distance expression tree: generic_simd_op (core/distance/simd_utils.h:204-252)
 * instantiated with L2FloatOp<16> (euclidean.h:240-259), IPFloatOp<16>
 * (inner_product.h:199-216) or CosineFloatOp<16> (cosine.h:224-256).
 * ---------------------------------------------------------------------------------- */

/* _mm512_reduce_add_ps as GCC 13 expands it: lanes (l+8)+(l), (l+4)+(l), then
 * (t[0]+t[2]) + (t[1]+t[3]). */
static float reduce16(const float* v) {
    float t8[8], t4[4];
    for (int l = 0; l < 8; ++l) t8[l] = v[l + 8] + v[l];
    for (int l = 0; l < 4; ++l) t4[l] = t8[l + 4] + t8[l];
    float u0 = t4[0] + t4[2], u1 = t4[1] + t4[3];
    return u0 + u1;
}

/* op: 0 = L2, 1 = IP, 2 = cosine (also fills *norm_out with sum b*b). */
static float float_tree(int op, const float* a, const float* b, size_t n, float* norm_out) {
    float s[4][16], t[4][16];
    memset(s, 0, sizeof(s));
    memset(t, 0, sizeof(t));
#define STEP(k, base, lanes)                                                 \
    for (size_t l = 0; l < (lanes); ++l) {                                   \
        float x = a[(base) + l], y = b[(base) + l];                          \
        if (op == 0) {                                                       \
            float c = x - y;                                                 \
            s[k][l] = fmaf(c, c, s[k][l]);                                   \
        } else {                                                             \
            s[k][l] = fmaf(x, y, s[k][l]);                                   \
            if (op == 2) t[k][l] = fmaf(y, y, t[k][l]);                      \
        }                                                                    \
    }
    size_t i = 0;
    if (i + 64 <= n) {
        for (; i + 64 <= n; i += 64) {
            STEP(0, i, 16) STEP(1, i + 16, 16) STEP(2, i + 32, 16) STEP(3, i + 48, 16)
        }
        for (int l = 0; l < 16; ++l) {
            s[0][l] = (s[0][l] + s[1][l]) + (s[2][l] + s[3][l]);
            t[0][l] = (t[0][l] + t[1][l]) + (t[2][l] + t[3][l]);
        }
    }
    for (; i + 16 <= n; i += 16) {
        STEP(0, i, 16)
    }
    if (i < n) {
        STEP(0, i, n - i) /* masked: untouched lanes keep their value */
    }
#undef STEP
    if (norm_out) *norm_out = reduce16(t[0]);
    return reduce16(s[0]);
}

/* Exact integer kernels for (i8,i8) and (u8,u8): L2VNNIOp / IPVNNIOp
 * (euclidean.h:265-313, inner_product.h:222-267) and the VNNI cosine loop
 * (cosine.h:262-326).  int32 accumulation is exact for dim < 33 025. */
static void int_sums(int t, const void* a, const void* b, size_t n, int32_t* l2, int32_t* ip,
                     int32_t* bb) {
    int32_t sl2 = 0, sip = 0, sbb = 0;
    for (size_t i = 0; i < n; ++i) {
        int32_t x = t == ORACLE_I8 ? ((const int8_t*)a)[i] : ((const uint8_t*)a)[i];
        int32_t y = t == ORACLE_I8 ? ((const int8_t*)b)[i] : ((const uint8_t*)b)[i];
        sl2 += (x - y) * (x - y);
        sip += x * y;
        sbb += y * y;
    }
    *l2 = sl2;
    *ip = sip;
    *bb = sbb;
}

/* distance::norm (core/distance/distance_core.h:45-66): sequential `accum += i * i` in
 * fp32 (separate multiply and add), then sqrt.  Integer element types multiply as int. */
static float query_norm(int qtype, const void* q, size_t n) {
    float acc = 0.0f;
    for (size_t i = 0; i < n; ++i) {
        float sq;
        if (qtype == ORACLE_I8 || qtype == ORACLE_U8) {
            int v = qtype == ORACLE_I8 ? ((const int8_t*)q)[i] : ((const uint8_t*)q)[i];
            sq = (float)(v * v);
        } else {
            float v = scalar_as_float(qtype, q, i);
            sq = v * v;
        }
        acc += sq;
    }
    return sqrtf(acc);
}

static int pair_supported(int qtype, int dtype) {
    /* The (query,row) pairs with SIMD specialisations (euclidean.h:293-358 etc.). */
    if (qtype == ORACLE_F32) return 1;
    if (qtype == ORACLE_F16) return dtype == ORACLE_F32 || dtype == ORACLE_F16;
    return qtype == dtype;
}

/* ------------------------------------------------------------------------------------
 * A "fixed" query: the state maybe_fix_argument leaves behind (concepts/distance.h:90-130).
 * ---------------------------------------------------------------------------------- */
typedef struct {
    int metric, qtype, dtype, sq; /* sq: rows are scalar-quantised codes */
    size_t dim;
    float scale, bias;
    const void* q_raw; /* original query */
    float* q_f32;      /* SIMD-converted query (float tree) */
    void* q_codes;     /* SQ/L2: query compressed to the code type */
    float a_norm;      /* cosine */
    float offset;      /* SQ/IP: bias * sum(q) */
    float* row_f32;    /* scratch for the converted / decompressed row */
    int lvq;           /* rows are LVQ-8 (own spec, see oracle_lvq8_compress) */
    const float* mean; /* LVQ-8 dataset mean */
    size_t lvq_const_offset;
} FixedQuery;

static int fixed_query_init(FixedQuery* f, int metric, int qtype, int dtype, int sq, size_t dim,
                            float scale, float bias) {
    memset(f, 0, sizeof(*f));
    f->metric = metric;
    f->qtype = qtype;
    f->dtype = dtype;
    f->sq = sq;
    f->dim = dim;
    f->scale = scale;
    f->bias = bias;
    f->q_f32 = (float*)malloc(dim * sizeof(float) + 16);
    f->row_f32 = (float*)malloc(dim * sizeof(float) + 16);
    f->q_codes = malloc(dim + 16);
    return !(f->q_f32 && f->row_f32 && f->q_codes);
}
static void fixed_query_free(FixedQuery* f) {
    free(f->q_f32);
    free(f->row_f32);
    free(f->q_codes);
}

static void fix_argument(FixedQuery* f, const void* query) {
    size_t n = f->dim;
    f->q_raw = query;
    if (f->lvq) {
        /* LVQ-8 (own specification): L2 removes the dataset mean from the query once;
         * IP keeps the query and adds <q, mean> (sequential fma) to every result. */
        load_as_float(f->qtype, query, n, f->q_f32);
        if (f->metric == ORACLE_L2) {
            for (size_t i = 0; i < n; ++i) f->q_f32[i] = f->q_f32[i] - f->mean[i];
        } else {
            float acc = 0.0f;
            for (size_t i = 0; i < n; ++i) acc = fmaf(f->q_f32[i], f->mean[i], acc);
            f->offset = acc;
        }
        return;
    }
    if (!f->sq) {
        load_as_float(f->qtype, query, n, f->q_f32);
        /* DistanceCosineSimilarity::fix_argument (cosine.h:117-119). */
        if (f->metric == ORACLE_COS) f->a_norm = query_norm(f->qtype, query, n);
        return;
    }
    if (f->metric == ORACLE_L2) {
        /* EuclideanCompressed::fix_argument (quantization/scalar/scalar.h:75-82) with
         * detail::compress (:38-42): clamp(round((v - bias) / scale), MIN, MAX). */
        float lo = f->dtype == ORACLE_I8 ? -128.0f : 0.0f, hi = f->dtype == ORACLE_I8 ? 127.0f : 255.0f;
        for (size_t i = 0; i < n; ++i) {
            float v = scalar_as_float(f->qtype, query, i);
            float r = roundf((v - f->bias) / f->scale);
            r = r < lo ? lo : (r > hi ? hi : r);
            if (f->dtype == ORACLE_I8)
                ((int8_t*)f->q_codes)[i] = (int8_t)r;
            else
                ((uint8_t*)f->q_codes)[i] = (uint8_t)r;
        }
    } else {
        /* InnerProductCompressed / CosineSimilarityCompressed::fix_argument
         * (scalar.h:123-131,168-171): query copied to fp32 element by element. */
        for (size_t i = 0; i < n; ++i) f->q_f32[i] = scalar_as_float(f->qtype, query, i);
        if (f->metric == ORACLE_IP) {
            /* std::reduce(begin, end, 0.0F, plus) -- libstdc++ 13 <numeric> evaluates
             * random-access ranges four at a time: init += (x0+x1)+(x2+x3), then a
             * sequential tail. */
            float acc = 0.0f;
            size_t i = 0;
            for (; i + 4 <= n; i += 4) {
                float v1 = f->q_f32[i] + f->q_f32[i + 1];
                float v2 = f->q_f32[i + 2] + f->q_f32[i + 3];
                float v3 = v1 + v2;
                acc = acc + v3;
            }
            for (; i < n; ++i) acc = acc + f->q_f32[i];
            f->offset = f->bias * acc;
        } else {
            f->a_norm = query_norm(f->qtype, query, n);
        }
    }
}

static float compute_distance(FixedQuery* f, const void* row) {
    size_t n = f->dim;
    if (f->lvq) {
        /* decode y_i = fma(delta, code_i, lower), then the reference's float tree */
        _Float16 consts[2];
        memcpy(consts, (const char*)row + f->lvq_const_offset, 4);
        float delta = (float)consts[0], lower = (float)consts[1];
        for (size_t i = 0; i < n; ++i) f->row_f32[i] = fmaf(delta, (float)((const uint8_t*)row)[i], lower);
        if (f->metric == ORACLE_L2) return float_tree(0, f->q_f32, f->row_f32, n, NULL);
        return float_tree(1, f->q_f32, f->row_f32, n, NULL) + f->offset;
    }
    if (f->sq) {
        if (f->metric == ORACLE_L2) {
            /* EuclideanCompressed::compute (scalar.h:88-94): scale^2 * L2_int(qc, row). */
            int32_t l2, ip, bb;
            int_sums(f->dtype, f->q_codes, row, n, &l2, &ip, &bb);
            return (f->scale * f->scale) * (float)l2;
        }
        if (f->metric == ORACLE_IP) {
            /* InnerProductCompressed::compute (scalar.h:135-142): scale * IP(q_f32,row) + offset. */
            load_as_float(f->dtype, row, n, f->row_f32);
            float ip = float_tree(1, f->q_f32, f->row_f32, n, NULL);
            float prod = f->scale * ip;
            return prod + f->offset;
        }
        /* CosineSimilarityCompressed::compute (scalar.h:177-185): decompress (scale*v+bias,
         * :44-46) then the f32 x f32 cosine. */
        for (size_t i = 0; i < n; ++i) {
            float v = f->dtype == ORACLE_I8 ? (float)((const int8_t*)row)[i] : (float)((const uint8_t*)row)[i];
            float p = f->scale * v;
            f->row_f32[i] = p + f->bias;
        }
        float nb, sum = float_tree(2, f->q_f32, f->row_f32, n, &nb);
        return sum / (sqrtf(nb) * f->a_norm);
    }
    if ((f->qtype == ORACLE_I8 || f->qtype == ORACLE_U8) && f->qtype == f->dtype) {
        int32_t l2, ip, bb;
        int_sums(f->dtype, f->q_raw, row, n, &l2, &ip, &bb);
        if (f->metric == ORACLE_L2) return (float)l2;
        if (f->metric == ORACLE_IP) return (float)ip;
        /* cosine.h:292-296: float(sum) / (a_norm * sqrt(float(bnorm))). */
        float b_norm = sqrtf((float)bb);
        return (float)ip / (f->a_norm * b_norm);
    }
    load_as_float(f->dtype, row, n, f->row_f32);
    if (f->metric == ORACLE_L2) return float_tree(0, f->q_f32, f->row_f32, n, NULL);
    if (f->metric == ORACLE_IP) return float_tree(1, f->q_f32, f->row_f32, n, NULL);
    float nb, sum = float_tree(2, f->q_f32, f->row_f32, n, &nb);
    /* cosine.h:334-335: sum / (sqrt(norm) * a_norm). */
    return sum / (sqrtf(nb) * f->a_norm);
}

int oracle_distance_rows(int metric, int qtype, int dtype, const void* query, const void* rows,
                         size_t nrows, size_t dim, float* out) {
    if (!pair_supported(qtype, dtype)) FAIL("unsupported (query,data) pair %d %d", qtype, dtype);
    FixedQuery f;
    if (fixed_query_init(&f, metric, qtype, dtype, 0, dim, 0, 0)) FAIL("out of memory");
    fix_argument(&f, query);
    for (size_t i = 0; i < nrows; ++i)
        out[i] = compute_distance(&f, (const char*)rows + i * dim * elem_size(dtype));
    fixed_query_free(&f);
    return 0;
}

int oracle_sq_distance_rows(int metric, int qtype, int code_type, float scale, float bias, const void* query,
                            const void* codes, size_t nrows, size_t dim, float* out) {
    if (qtype != ORACLE_F32 && qtype != ORACLE_F16) FAIL("SQ: float32 / float16 queries only, got %d", qtype);
    if (code_type != ORACLE_I8 && code_type != ORACLE_U8) FAIL("bad SQ code type %d", code_type);
    FixedQuery f;
    if (fixed_query_init(&f, metric, qtype, code_type, 1, dim, scale, bias)) FAIL("out of memory");
    fix_argument(&f, query);
    for (size_t i = 0; i < nrows; ++i) out[i] = compute_distance(&f, (const char*)codes + i * dim);
    fixed_query_free(&f);
    return 0;
}

int oracle_lvq8_distance_rows(int metric, int qtype, const void* query, const void* rows, size_t nrows, size_t dim,
                              const float* mean, float* out) {
    if (qtype != ORACLE_F32 && qtype != ORACLE_F16) FAIL("LVQ-8: float32 / float16 queries only, got %d", qtype);
    if (metric == ORACLE_COS) FAIL("LVQ-8: cosine is not supported");
    FixedQuery f;
    if (fixed_query_init(&f, metric, qtype, ORACLE_U8, 0, dim, 0, 0)) FAIL("out of memory");
    f.lvq = 1;
    f.mean = mean;
    f.lvq_const_offset = (dim + 3) / 4 * 4;
    fix_argument(&f, query);
    size_t stride = oracle_lvq8_row_stride(dim);
    for (size_t i = 0; i < nrows; ++i) out[i] = compute_distance(&f, (const char*)rows + i * stride);
    fixed_query_free(&f);
    return 0;
}

/* ------------------------------------------------------------------------------------
 * SearchBuffer (index/vamana/search_buffer.h:104-497).
 * ---------------------------------------------------------------------------------- */
typedef struct {
    uint32_t id;
    float dist;
    int visited;
} Entry; /* SearchNeighbor<uint32_t> (lib/neighbor.h:199-217) */

typedef struct {
    Entry* e; /* capacity + 1 slots (search_buffer.h:142) */
    size_t size, best_unvisited, window, capacity;
    int greater;       /* comparator: std::less for L2, std::greater for IP/cosine */
    uint16_t* visited; /* VisitedFilter<uint32_t,16> (filter.h:49-130) or NULL */
} Buffer;

static int cmp(const Buffer* b, float x, float y) { return b->greater ? x > y : x < y; }

static void buffer_clear(Buffer* b) { /* :229-235 */
    b->size = 0;
    b->best_unvisited = 0;
    if (b->visited) memset(b->visited, 0xFF, 65536 * sizeof(uint16_t));
}
static int buffer_done(const Buffer* b) { /* :280 */
    size_t upper = b->size < b->window ? b->size : b->window;
    return b->best_unvisited == upper;
}
static Entry buffer_next(Buffer* b) { /* :294-304 */
    Entry* node = &b->e[b->best_unvisited];
    node->visited = 1;
    size_t upper = b->size < b->window ? b->size : b->window;
    while (++b->best_unvisited != upper && b->e[b->best_unvisited].visited) {}
    return *node;
}
static void buffer_push_back(Buffer* b, Entry n) { /* :311-316 */
    if (b->size != b->capacity) b->e[b->size++] = n;
}
static int emplace_visited(Buffer* b, uint32_t id) { /* :462-464 + filter.h:111-117 */
    if (!b->visited) return 0;
    uint16_t* v = &b->visited[id & 0xFFFFu];
    int hit = (uint16_t)(id >> 16) == *v;
    *v = (uint16_t)(id >> 16);
    return hit;
}
/* Returns what the reference's insert returns: the insertion index, size() when the
 * candidate is skipped, size()+1 when it is a duplicate id. */
static size_t buffer_insert(Buffer* b, Entry n) { /* :353-403 */
    int full = b->size == b->capacity;
    if (full && (b->capacity == 0 || cmp(b, b->e[b->size - 1].dist, n.dist))) return b->size; /* can_skip */
    /* lower_bound with !cmp(d, other): first slot whose entry is strictly worse than d. */
    size_t lo = 0, hi = b->size;
    while (lo < hi) {
        size_t mid = lo + (hi - lo) / 2;
        if (!cmp(b, n.dist, b->e[mid].dist))
            lo = mid + 1;
        else
            hi = mid;
    }
    size_t pos = lo;
    for (size_t back = pos; back > 0;) { /* duplicate-id scan over the equal-distance run */
        --back;
        if (cmp(b, b->e[back].dist, n.dist)) break;
        if (b->e[back].id == n.id) return b->size + 1;
    }
    memmove(&b->e[pos + 1], &b->e[pos], (b->size - pos) * sizeof(Entry)); /* copy_backward */
    b->e[pos] = n;
    b->size = b->size + 1 < b->capacity ? b->size + 1 : b->capacity;
    if (pos < b->best_unvisited) b->best_unvisited = pos;
    return pos;
}
/* ------------------------------------------------------------------------------------
 * Index + greedy search.
 * ---------------------------------------------------------------------------------- */
typedef struct {
    int dtype, metric, sq;
    size_t n, dim, max_degree;
    void* data;      /* owned copy, row-major */
    uint32_t* graph; /* owned copy, n x (max_degree + 1) */
    uint32_t entry_point;
    uint32_t entry_points[32]; /* index/vamana/index.h:304-312 holds a vector of entry points */
    uint32_t n_entry;
    float scale, bias;
    int lvq;
    size_t row_stride, lvq_const_offset; /* row_stride 0 = dense */
    float* mean;
} Index;

/* greedy_search (index/vamana/greedy_search.h:124-203) with EntryPointInitializer (:62-94). */
static void greedy_search(const Index* ix, FixedQuery* f, const void* query, Buffer* buf,
                          uint64_t* hops, uint64_t* evals) {
    size_t row_bytes = ix->row_stride ? ix->row_stride : ix->dim * elem_size(ix->dtype);
    fix_argument(f, query); /* :140 */
    buffer_clear(buf);      /* :79 */
    {
        /* EntryPointInitializer (:62-94): push_back every entry point, then buffer.sort().  With one entry point
         * there is nothing to order; with several (distinct ones) the sort is restated as a stable insertion sort
         * by the comparator -- std::sort leaves the order of exactly tied distances unspecified. */
        uint32_t ne = ix->n_entry > 1 ? ix->n_entry : 1;
        for (uint32_t i = 0; i < ne; ++i) {
            uint32_t id = ix->n_entry > 1 ? ix->entry_points[i] : ix->entry_point;
            Entry e = {id, compute_distance(f, (const char*)ix->data + (size_t)id * row_bytes), 0};
            buffer_push_back(buf, e);
            if (evals) ++*evals;
        }
        for (size_t i = 1; i < buf->size; ++i) {
            Entry x = buf->e[i];
            size_t j = i;
            while (j > 0 && cmp(buf, x.dist, buf->e[j - 1].dist)) {
                buf->e[j] = buf->e[j - 1];
                --j;
            }
            buf->e[j] = x;
        }
    }
    while (!buffer_done(buf)) { /* :153 */
        Entry node = buffer_next(buf);
        const uint32_t* row = ix->graph + (size_t)node.id * (ix->max_degree + 1);
        uint32_t deg = row[0]; /* core/graph/graph.h:103-114 */
        if (hops) ++*hops;
        if (evals) *evals += deg; /* tracker.visited(node, neighbors.size()) (:165) */
        for (uint32_t j = 0; j < deg; ++j) { /* adjacency order (:190) */
            uint32_t id = row[1 + j];
            if (emplace_visited(buf, id)) continue; /* :191 */
            Entry e = {id, compute_distance(f, (const char*)ix->data + (size_t)id * row_bytes), 0};
            buffer_insert(buf, e); /* :199-200 */
        }
    }
}

static Index* index_new(int dtype, const void* data, size_t n, size_t dim, const uint32_t* graph,
                        size_t max_degree, uint32_t entry_point, int metric) {
    Index* ix = (Index*)calloc(1, sizeof(Index));
    if (!ix) return NULL;
    ix->dtype = dtype;
    ix->metric = metric;
    ix->n = n;
    ix->dim = dim;
    ix->max_degree = max_degree;
    ix->entry_point = entry_point;
    size_t db = n * dim * elem_size(dtype), gb = n * (max_degree + 1) * sizeof(uint32_t);
    ix->data = malloc(db ? db : 1);
    ix->graph = (uint32_t*)malloc(gb ? gb : 1);
    if (!ix->data || !ix->graph) return NULL;
    if (data) memcpy(ix->data, data, db);
    memcpy(ix->graph, graph, gb);
    return ix;
}

void* oracle_index_create(int dtype, const void* data, size_t n, size_t dim,
                          const uint32_t* graph_rows, size_t max_degree, uint32_t entry_point,
                          int metric, size_t threads) {
    (void)threads;
    Index* ix = index_new(dtype, data, n, dim, graph_rows, max_degree, entry_point, metric);
    if (!ix) snprintf(g_error, sizeof(g_error), "out of memory");
    return ix;
}

void* oracle_sq_index_create(int code_type, const float* data, size_t n, size_t dim,
                             const uint32_t* graph_rows, size_t max_degree, uint32_t entry_point,
                             int metric, size_t threads, float* scale_out, float* bias_out,
                             void* codes_out) {
    (void)threads;
    if (code_type != ORACLE_I8 && code_type != ORACLE_U8) {
        snprintf(g_error, sizeof(g_error), "bad SQ code type %d", code_type);
        return NULL;
    }
    Index* ix = index_new(code_type, NULL, n, dim, graph_rows, max_degree, entry_point, metric);
    if (!ix) {
        snprintf(g_error, sizeof(g_error), "out of memory");
        return NULL;
    }
    /* SQDataset::compress (quantization/scalar/scalar.h:447-469). */
    float mn = 3.402823466e+38f, mx = -3.402823466e+38f;
    for (size_t i = 0; i < n * dim; ++i) {
        mn = data[i] < mn ? data[i] : mn;
        mx = data[i] > mx ? data[i] : mx;
    }
    float MIN = code_type == ORACLE_I8 ? -128.0f : 0.0f, MAX = code_type == ORACLE_I8 ? 127.0f : 255.0f;
    float scale = (mx - mn) / (MAX - MIN);
    float t = MIN * scale;
    float bias = mn - t;
    for (size_t i = 0; i < n * dim; ++i) {
        float r = roundf((data[i] - bias) / scale);
        r = r < MIN ? MIN : (r > MAX ? MAX : r);
        if (code_type == ORACLE_I8)
            ((int8_t*)ix->data)[i] = (int8_t)r;
        else
            ((uint8_t*)ix->data)[i] = (uint8_t)r;
    }
    ix->sq = 1;
    ix->scale = scale;
    ix->bias = bias;
    *scale_out = scale;
    *bias_out = bias;
    if (codes_out) memcpy(codes_out, ix->data, n * dim);
    return ix;
}

/* ------------------------------------------------------------------------------------
 * LVQ-8, own specification (the reference's LVQ is closed source: parity UNPINNED).
 *   r_i = x_i - mean_i; lower = min r; upper = max r; delta = (upper - lower) / 255
 *   {delta, lower} stored as IEEE float16 (RNE); codes against the stored constants:
 *   c_i = clamp(rint((r_i - lower16) / delta16), 0, 255), 0 when delta16 == 0.
 *   Row = dim codes, padded to 4 bytes, then delta16, lower16; stride multiple of 32.
 * A row with a residual that is not finite, or whose delta16 or lower16 is not finite (the range
 * reaches 255 x 65520 or lower reaches -65520), is refused: it would decode to NaN or -inf.  A
 * subnormal or zero delta16 is kept.  Nothing is written when a row is refused.
 * ---------------------------------------------------------------------------------- */
size_t oracle_lvq8_row_stride(size_t dim) { return ((((dim + 3) / 4 * 4) + 4) + 31) / 32 * 32; }

int oracle_lvq8_compress(const float* data, size_t n, size_t dim, const float* mean, void* out_rows) {
    size_t stride = oracle_lvq8_row_stride(dim), off = (dim + 3) / 4 * 4;
    for (size_t r = 0; r < n; ++r) {
        const float* x = data + r * dim;
        float lo = INFINITY, hi = -INFINITY;
        for (size_t i = 0; i < dim; ++i) {
            float v = x[i] - mean[i];
            if (!isfinite(v)) FAIL("LVQ-8: row %zu holds an element that is not finite after removing the mean", r);
            lo = v < lo ? v : lo;
            hi = v > hi ? v : hi;
        }
        _Float16 consts[2] = {(_Float16)((hi - lo) / 255.0f), (_Float16)lo};
        if (!isfinite((float)consts[0]) || !isfinite((float)consts[1]))
            FAIL("LVQ-8: row %zu has a delta or lower bound that float16 cannot hold", r);
    }
    for (size_t r = 0; r < n; ++r) {
        const float* x = data + r * dim;
        uint8_t* out = (uint8_t*)out_rows + r * stride;
        memset(out, 0, stride);
        float lo = INFINITY, hi = -INFINITY;
        for (size_t i = 0; i < dim; ++i) {
            float v = x[i] - mean[i];
            lo = v < lo ? v : lo;
            hi = v > hi ? v : hi;
        }
        float range = hi - lo;
        _Float16 consts[2] = {(_Float16)(range / 255.0f), (_Float16)lo};
        float d = (float)consts[0], l = (float)consts[1];
        for (size_t i = 0; i < dim && d > 0.0f; ++i) {
            float v = x[i] - mean[i];
            float q = rintf((v - l) / d);
            q = q < 0.0f ? 0.0f : (q > 255.0f ? 255.0f : q);
            out[i] = (uint8_t)(int)q;
        }
        memcpy(out + off, consts, 4);
    }
    return 0;
}

void* oracle_lvq8_index_create(const void* rows, size_t n, size_t dim, const float* mean,
                               const uint32_t* graph_rows, size_t max_degree, uint32_t entry_point, int metric) {
    if (metric == ORACLE_COS) {
        snprintf(g_error, sizeof(g_error), "LVQ-8: cosine is not supported");
        return NULL;
    }
    Index* ix = index_new(ORACLE_U8, NULL, 0, dim, graph_rows, max_degree, entry_point, metric);
    if (!ix) return NULL;
    /* index_new sized the graph for 0 nodes: redo with the real count */
    free(ix->graph);
    free(ix->data);
    ix->n = n;
    ix->row_stride = oracle_lvq8_row_stride(dim);
    ix->lvq_const_offset = (dim + 3) / 4 * 4;
    ix->lvq = 1;
    ix->data = malloc(n * ix->row_stride);
    ix->graph = (uint32_t*)malloc(n * (max_degree + 1) * sizeof(uint32_t));
    ix->mean = (float*)malloc(dim * sizeof(float));
    if (!ix->data || !ix->graph || !ix->mean) return NULL;
    memcpy(ix->data, rows, n * ix->row_stride);
    memcpy(ix->graph, graph_rows, n * (max_degree + 1) * sizeof(uint32_t));
    memcpy(ix->mean, mean, dim * sizeof(float));
    return ix;
}

/* index/vamana/index.h:304-312: the index holds a vector of entry points; all of them start a search. */
int oracle_index_set_entry_points(void* h, const uint32_t* entry_points, size_t count) {
    Index* ix = (Index*)h;
    if (!ix || !entry_points || count == 0 || count > 32) {
        snprintf(g_error, sizeof(g_error), "between 1 and 32 entry points");
        return -1;
    }
    for (size_t i = 0; i < count; ++i) {
        if (entry_points[i] >= ix->n) {
            snprintf(g_error, sizeof(g_error), "entry point out of range");
            return -1;
        }
        for (size_t j = 0; j < i; ++j)
            if (entry_points[j] == entry_points[i]) {
                snprintf(g_error, sizeof(g_error), "entry points must be distinct");
                return -1;
            }
    }
    memcpy(ix->entry_points, entry_points, count * sizeof(uint32_t));
    ix->n_entry = (uint32_t)count;
    ix->entry_point = entry_points[0];
    return 0;
}

void oracle_index_destroy(void* h) {
    Index* ix = (Index*)h;
    if (!ix) return;
    free(ix->mean);
    free(ix->data);
    free(ix->graph);
    free(ix);
}

static int run_batch(Index* ix, int qtype, const void* queries, size_t nq, size_t k, size_t window,
                     size_t capacity, int visited_set, uint64_t* ids, float* dists, uint64_t* hops,
                     uint64_t* evals) {
    if ((ix->sq || ix->lvq) ? !(qtype == ORACLE_F32 || qtype == ORACLE_F16) : !pair_supported(qtype, ix->dtype))
        FAIL("unsupported (query,data) pair %d %d", qtype, ix->dtype);
    if (window > capacity) FAIL("search window %zu exceeds capacity %zu", window, capacity);
    /* VamanaIndex::search (index/vamana/index.h:590-592): a buffer smaller than k is
     * re-created with window = capacity = k. */
    if (capacity < k) window = capacity = k;
    Buffer buf;
    memset(&buf, 0, sizeof(buf));
    buf.window = window;
    buf.capacity = capacity;
    buf.greater = ix->metric != ORACLE_L2; /* distance::comparator */
    buf.e = (Entry*)calloc(capacity + 1, sizeof(Entry));
    if (visited_set) buf.visited = (uint16_t*)malloc(65536 * sizeof(uint16_t));
    FixedQuery f;
    if (!buf.e || fixed_query_init(&f, ix->metric, qtype, ix->dtype, ix->sq, ix->dim, ix->scale, ix->bias))
        FAIL("out of memory");
    f.lvq = ix->lvq;
    f.mean = ix->mean;
    f.lvq_const_offset = ix->lvq_const_offset;
    size_t qbytes = ix->dim * elem_size(qtype);
    for (size_t q = 0; q < nq; ++q) {
        uint64_t h = 0, e = 0;
        greedy_search(ix, &f, (const char*)queries + q * qbytes, &buf, &h, &e);
        if (hops) hops[q] = h;
        if (evals) evals[q] = e;
        /* extensions.h:588-590 copies buffer[j] for j < k regardless of size; slots past
         * `size` hold stale entries from earlier queries there.  The oracle reports them the way
         * the C ABI documents (include/svsb200.h): id = all-ones, dist = +inf (L2) / -inf (IP, cosine). */
        for (size_t j = 0; ids && j < k; ++j) {
            int valid = j < buf.size;
            ids[q * k + j] = valid ? buf.e[j].id : ~0ull;
            dists[q * k + j] = valid ? buf.e[j].dist : (buf.greater ? -INFINITY : INFINITY);
        }
    }
    fixed_query_free(&f);
    free(buf.e);
    free(buf.visited);
    return 0;
}

/* ------------------------------------------------------------------------------------
 * Test-only access to the SearchBuffer restatement, so tests/ can replay the reference's own
 * known-answer insert sequence (tests/svs/index/vamana/search_buffer.cpp:382-519) and fuzz it
 * against an independent model (same file, :74-244).
 * ---------------------------------------------------------------------------------- */
void* oracle_buffer_new(size_t window, size_t capacity, int greater) {
    Buffer* b = (Buffer*)calloc(1, sizeof(Buffer));
    if (!b) return NULL;
    b->window = window;
    b->capacity = capacity;
    b->greater = greater;
    b->e = (Entry*)calloc(capacity + 1, sizeof(Entry));
    return b;
}
void oracle_buffer_free(void* h) {
    Buffer* b = (Buffer*)h;
    if (!b) return;
    free(b->e);
    free(b);
}
void oracle_buffer_clear(void* h) { buffer_clear((Buffer*)h); }
void oracle_buffer_push_back(void* h, uint32_t id, float dist) {
    Entry e = {id, dist, 0};
    buffer_push_back((Buffer*)h, e);
}
size_t oracle_buffer_insert(void* h, uint32_t id, float dist) {
    Entry e = {id, dist, 0};
    return buffer_insert((Buffer*)h, e);
}
size_t oracle_buffer_size(void* h) { return ((Buffer*)h)->size; }
size_t oracle_buffer_best_unvisited(void* h) { return ((Buffer*)h)->best_unvisited; }
int oracle_buffer_done(void* h) { return buffer_done((Buffer*)h); }
uint32_t oracle_buffer_next(void* h) { return buffer_next((Buffer*)h).id; }
void oracle_buffer_set_visited(void* h, size_t i) { ((Buffer*)h)->e[i].visited = 1; }
void oracle_buffer_get(void* h, size_t i, uint32_t* id, float* dist, int* visited) {
    Entry e = ((Buffer*)h)->e[i];
    *id = e.id;
    *dist = e.dist;
    *visited = e.visited;
}
void oracle_buffer_sort(void* h) { /* buffer.sort(): std::sort by the comparator (:408) */
    Buffer* b = (Buffer*)h;
    for (size_t i = 1; i < b->size; ++i) {   /* insertion sort: small, and stable is fine */
        Entry x = b->e[i];
        size_t j = i;
        while (j > 0 && cmp(b, x.dist, b->e[j - 1].dist)) {
            b->e[j] = b->e[j - 1];
            --j;
        }
        b->e[j] = x;
    }
}

int oracle_index_search(void* h, int qtype, const void* queries, size_t nq, size_t k, size_t window,
                        size_t capacity, int visited_set, uint64_t* ids, float* dists) {
    return run_batch((Index*)h, qtype, queries, nq, k, window, capacity, visited_set, ids, dists, NULL,
                     NULL);
}

int oracle_index_counts(void* h, int qtype, const void* queries, size_t nq, size_t window,
                        size_t capacity, uint64_t* hops, uint64_t* evals) {
    return run_batch((Index*)h, qtype, queries, nq, 0, window, capacity, 0, NULL, NULL, hops, evals);
}
