// search.cu -- graph search of the C ABI (include/svsb200.h): query preparation (the device-side maybe_fix_argument),
// kernel choice and launch, the blocking / enqueue-only / cancellable / sharded / filtered / range / exhaustive entry
// points, result gather, and the counters and kernel time of the last search.
#include "host.cuh"
#include "query_prep.cuh"

#include <algorithm>
#include <chrono>
#include <cmath>
#include <thread>
#include <type_traits>

namespace svsb200 {

// ---------------------------------------------------------------------------------------
// Query preparation == distance::maybe_fix_argument for the whole batch
// (concepts/distance.h:90-130), one warp per query.
// ---------------------------------------------------------------------------------------

template <int QT>
__global__ void prepare_queries_kernel(const void* __restrict__ queries, uint32_t nq, uint32_t dim, uint32_t qstride,
                                       int mode, int metric, int code_type, float scale, float bias,
                                       const float* __restrict__ mean, float* __restrict__ qf,
                                       uint8_t* __restrict__ qcodes, float* __restrict__ qaux) {
    const uint32_t q = blockIdx.x * (blockDim.x / 32) + threadIdx.x / 32;
    const int lane = threadIdx.x & 31;
    if (q >= nq) return;
    constexpr size_t QES = QT == SVSB200_F32 ? 4 : QT == SVSB200_F16 ? 2 : 1;
    const void* src = static_cast<const char*>(queries) + size_t(q) * dim * QES;
    float* f = qf + size_t(q) * qstride;
    uint8_t* c = qcodes + size_t(q) * qstride;

    for (uint32_t i = lane; i < qstride; i += 32) {
        float fv = 0.f;
        uint8_t cv = 0;
        if (i < dim) {
            if (mode == PREP_FLOAT || mode == PREP_LVQ_IP) {
                fv = q_simd<QT>(src, i);
            } else if (mode == PREP_LVQ_L2) {
                fv = __fsub_rn(q_simd<QT>(src, i), mean[i]);
            } else if (mode == PREP_INT) {
                if constexpr (QT == SVSB200_I8 || QT == SVSB200_U8) cv = static_cast<const uint8_t*>(src)[i];
            } else if (mode == PREP_SQ_L2) {
                cv = sq_compress_code(q_scalar<QT>(src, i), code_type, scale, bias);
            } else {
                fv = q_scalar<QT>(src, i);
            }
        }
        f[i] = fv;
        c[i] = cv;
    }
    __syncwarp();
    if (lane != 0) return;

    float aux0 = 0.f, aux1 = 0.f;
    if (mode == PREP_INT || mode == PREP_SQ_L2) {
        int xx = 0;
        const bool is_signed = (mode == PREP_INT) ? (QT == SVSB200_I8) : (code_type == SVSB200_I8);
        for (uint32_t i = 0; i < dim; ++i) {
            int v = is_signed ? int(int8_t(c[i])) : int(c[i]);
            xx += v * v;
        }
        aux1 = __int_as_float(xx);
    }
    const bool need_norm = (metric == SVSB200_COSINE) && (mode == PREP_FLOAT || mode == PREP_INT || mode == PREP_SQ_COS);
    if (need_norm) {
        aux0 = sequential_norm(dim, [&](uint32_t i) {
            if constexpr (QT == SVSB200_I8 || QT == SVSB200_U8) {
                int v = QT == SVSB200_I8 ? int(static_cast<const int8_t*>(src)[i]) : int(static_cast<const uint8_t*>(src)[i]);
                return float(v * v);
            } else {
                float v = q_scalar<QT>(src, i);
                return __fmul_rn(v, v);
            }
        });
    } else if (mode == PREP_LVQ_IP) {
        float acc = 0.f;
        for (uint32_t i = 0; i < dim; ++i) acc = __fmaf_rn(f[i], mean[i], acc);
        aux0 = acc;
    } else if (mode == PREP_SQ_IP) {
        aux0 = sq_ip_offset(f, dim, bias);
    }
    qaux[2 * size_t(q)] = aux0;
    qaux[2 * size_t(q) + 1] = aux1;
}

// ---------------------------------------------------------------------------------------
// Cross-shard top-k merge with TotalOrder (lib/neighbor.h:143-155): distance, then id.
// ---------------------------------------------------------------------------------------
// One warp per query selects the k smallest (key, id) pairs among all nshards * k candidates by repeated
// "smallest entry greater than the previous output" -- a full TotalOrder sort of the candidates' prefix, so
// the result does not depend on how ties are ordered inside a shard's list (they come out of the search
// buffer in insertion order, not id order).  Padding entries (id = all-ones) are ignored.
__device__ __forceinline__ uint32_t total_order_key(float d, int greater) {
    float k = greater ? -d : d;
    k = __fadd_rn(k, 0.0f);                       // -0 == +0 under operator<
    const uint32_t u = __float_as_uint(k);
    return (u & 0x80000000u) ? ~u : (u | 0x80000000u);   // monotone float -> uint
}
__global__ void merge_topk_kernel(const uint64_t* __restrict__ ids, const float* __restrict__ dists, uint32_t nshards,
                                  uint32_t nq, uint32_t k, int greater, uint64_t* __restrict__ out_ids,
                                  float* __restrict__ out_dists) {
    const uint32_t q = blockIdx.x * (blockDim.x / 32) + threadIdx.x / 32;
    const int lane = threadIdx.x & 31;
    if (q >= nq) return;
    constexpr unsigned FULL = 0xFFFFFFFFu;
    const uint32_t n = nshards * k;
    // (key, id) of the previous output; "nothing yet" sorts before everything
    bool have_last = false;
    uint32_t last_key = 0;
    uint64_t last_id = 0;
    for (uint32_t j = 0; j < k; ++j) {
        uint32_t best_key = 0xFFFFFFFFu;
        uint64_t best_id = ~uint64_t(0);
        float best_d = 0.f;
        bool found = false;
        for (uint32_t c = lane; c < n; c += 32) {
            const uint32_t sh = c / k, jj = c - sh * k;
            const size_t o = (size_t(sh) * nq + q) * k + jj;
            const uint64_t id = ids[o];
            if (id == ~uint64_t(0)) continue;
            const float d = dists[o];
            const uint32_t key = total_order_key(d, greater);
            if (have_last && (key < last_key || (key == last_key && id <= last_id))) continue;
            if (!found || key < best_key || (key == best_key && id < best_id)) {
                best_key = key;
                best_id = id;
                best_d = d;
                found = true;
            }
        }
        // warp argmin over (found, key, id)
        for (int off = 16; off; off >>= 1) {
            const uint32_t okey = __shfl_xor_sync(FULL, best_key, off);
            const uint64_t oid = __shfl_xor_sync(FULL, best_id, off);
            const float od = __shfl_xor_sync(FULL, best_d, off);
            const bool ofound = __shfl_xor_sync(FULL, int(found), off) != 0;
            if (ofound && (!found || okey < best_key || (okey == best_key && oid < best_id))) {
                best_key = okey;
                best_id = oid;
                best_d = od;
                found = true;
            }
        }
        if (lane == 0) {
            const size_t o = size_t(q) * k + j;
            out_ids[o] = found ? best_id : ~uint64_t(0);
            out_dists[o] = found ? best_d : (greater ? -INFINITY : INFINITY);
        }
        if (!found) {
            for (uint32_t r = j + 1 + lane; r < k; r += 32) {   // nothing left: pad the tail
                out_ids[size_t(q) * k + r] = ~uint64_t(0);
                out_dists[size_t(q) * k + r] = greater ? -INFINITY : INFINITY;
            }
            return;
        }
        have_last = true;
        last_key = best_key;
        last_id = best_id;
    }
}

// Filtered search (bindings/cpp/src/vamana_index_impl.h:139-218): out of a query's `kk` search results (sorted), keep
// the first k whose id is a member of the filter bitmap; `found[q]` = how many there were.  The bitmap is over the
// index's own rows: on a shard the listed ids carry `id_offset`, which is taken off for the membership test only.
__global__ void filter_topk_kernel(const uint64_t* __restrict__ ids, const float* __restrict__ dists, uint32_t nq, uint32_t kk,
                                   uint32_t k, const uint32_t* __restrict__ bitmap, uint64_t id_offset,
                                   uint64_t* __restrict__ out_ids, float* __restrict__ out_dists, uint32_t* __restrict__ found,
                                   uint32_t* __restrict__ unfinished) {
    const uint32_t q = blockIdx.x * (blockDim.x / 32) + threadIdx.x / 32;
    const uint32_t lane = threadIdx.x & 31;
    if (q >= nq) return;
    uint32_t cnt = 0;
    bool exhausted = false;   // the search returned fewer than kk valid entries: nothing more to find
    for (uint32_t j0 = 0; j0 < kk && cnt < k; j0 += 32) {
        const uint32_t j = j0 + lane;
        const uint64_t id = j < kk ? ids[size_t(q) * kk + j] : ~uint64_t(0);
        const bool valid = id != ~uint64_t(0);
        const uint64_t row = id - id_offset;
        const bool pass = valid && ((bitmap[row >> 5] >> (row & 31)) & 1u);
        const unsigned m = __ballot_sync(0xFFFFFFFFu, pass);
        const uint32_t o = cnt + __popc(m & ((1u << lane) - 1u));
        if (pass && o < k) {
            out_ids[size_t(q) * k + o] = id;
            out_dists[size_t(q) * k + o] = dists[size_t(q) * kk + j];
        }
        cnt += __popc(m);
        if (__any_sync(0xFFFFFFFFu, j < kk && !valid)) exhausted = true;
    }
    cnt = min(cnt, k);
    if (lane == 0) {
        found[q] = cnt;
        if (cnt < k && !exhausted) atomicAdd(unfinished, 1u);
    }
}

// Range search (vamana_index_impl.h:227-300): number of a query's sorted results inside the radius; a query whose
// last result is still inside needs a longer list.
__global__ void range_count_kernel(const float* __restrict__ dists, const uint64_t* __restrict__ ids, uint32_t nq, uint32_t kk,
                                   float radius, int greater, uint32_t* __restrict__ counts, uint32_t* __restrict__ unfinished) {
    const uint32_t q = blockIdx.x * blockDim.x + threadIdx.x;
    if (q >= nq) return;
    uint32_t c = 0;
    bool exhausted = false;
    for (; c < kk; ++c) {
        if (ids[size_t(q) * kk + c] == ~uint64_t(0)) {
            exhausted = true;
            break;
        }
        const float d = dists[size_t(q) * kk + c];
        if (greater ? !(d > radius) : !(d < radius)) break;
    }
    counts[q] = c;
    if (c == kk && !exhausted) atomicAdd(unfinished, 1u);
}

// Dynamic index, filtered search: members whose slot is not Valid are cleared from the bitmap (one thread per word).
__global__ void keep_valid_kernel(uint32_t* __restrict__ bitmap, const uint8_t* __restrict__ status, size_t n) {
    const size_t w = size_t(blockIdx.x) * blockDim.x + threadIdx.x;
    if (w * 32 >= n) return;
    uint32_t keep = 0;
    for (uint32_t b = 0; b < 32 && w * 32 + b < n; ++b) keep |= (status[w * 32 + b] == SLOT_VALID ? 1u : 0u) << b;
    bitmap[w] &= keep;
}

// Dynamic index: slots -> external ids in place (padding ids stay all-ones).
__global__ void slots_to_external_kernel(uint64_t* __restrict__ ids, size_t count, const uint64_t* __restrict__ ext_ids) {
    const size_t i = size_t(blockIdx.x) * blockDim.x + threadIdx.x;
    if (i < count && ids[i] != ~uint64_t(0)) ids[i] = ext_ids[ids[i]];
}

cudaError_t slots_to_external(uint64_t* d_ids, size_t count, const uint64_t* d_ext_ids, cudaStream_t stream) {
    if (count == 0) return cudaSuccess;
    slots_to_external_kernel<<<unsigned((count + 255) / 256), 256, 0, stream>>>(d_ids, count, d_ext_ids);
    count_launch();
    return cudaGetLastError();
}

// ---------------------------------------------------------------------------------------
// Host side
// ---------------------------------------------------------------------------------------

int prepare_queries(const svsb200_index* ix, const Replica* rep, Scratch* sc, const void* d_queries, int qdtype, size_t nq,
                    int mode, cudaStream_t stream) {
    const uint32_t qstride = query_stride(ix->dim);
    CUDA_TRY(sc->q_f32.ensure(nq * qstride));
    CUDA_TRY(sc->q_codes.ensure(nq * qstride));
    CUDA_TRY(sc->q_aux.ensure(nq * 2));
    const int warps = 8;
    const LaunchConfig cfg{int((nq + warps - 1) / warps), warps, 0, stream};
    CUDA_TRY(dispatch(DataRows{}, qdtype, [&](auto qt) {
        return launch_kernel(prepare_queries_kernel<decltype(qt)::value>, cfg, cfg.grid, false, d_queries, uint32_t(nq),
                             uint32_t(ix->dim), qstride, mode, ix->metric, ix->dtype, ix->scale, ix->bias, rep->d_mean.ptr,
                             sc->q_f32.ptr, sc->q_codes.ptr, sc->q_aux.ptr);
    }));
    return 0;
}

// threads::balance (lib/threads/types.h:311-329): contiguous ranges whose sizes differ by at most one.
static void balance(size_t n, size_t parts, size_t i, size_t* lo, size_t* hi) {
    const size_t base = n / parts, rem = n % parts;
    *lo = i * base + (i < rem ? i : rem);
    *hi = *lo + base + (i < rem ? 1 : 0);
}

// Which (query, data) pairs exist, mirroring the SIMD specialisations (euclidean.h:293-358) and the SQ CPOs
// (extensions/vamana/scalar.h:32-43): the distance operator and the query preparation for them.
int choose_op(const svsb200_index* ix, int qdtype, int* op, int* mode) {
    const int metric = ix->metric;
    if (ix->storage == SVSB200_LVQ8) {
        if (qdtype != SVSB200_F32 && qdtype != SVSB200_F16) return fail("LVQ-8 datasets take float32/float16 queries");
        if (metric == SVSB200_COSINE) return fail("LVQ-8: cosine is not supported (L2 and MIP are)");
        *op = metric == SVSB200_L2 ? OP_L2F : OP_IPF;
        *mode = metric == SVSB200_L2 ? PREP_LVQ_L2 : PREP_LVQ_IP;
    } else if (ix->storage == SVSB200_SQ) {
        if (qdtype != SVSB200_F32 && qdtype != SVSB200_F16) return fail("SQ datasets take float32/float16 queries");
        *op = metric == SVSB200_L2 ? OP_L2I : metric == SVSB200_IP ? OP_IPF : OP_COSF;
        *mode = metric == SVSB200_L2 ? PREP_SQ_L2 : metric == SVSB200_IP ? PREP_SQ_IP : PREP_SQ_COS;
    } else if (qdtype == SVSB200_I8 || qdtype == SVSB200_U8) {
        if (qdtype != ix->dtype) return fail("int8/uint8 queries need a dataset of the same type");
        *op = metric == SVSB200_L2 ? OP_L2I : metric == SVSB200_IP ? OP_IPI : OP_COSI;
        *mode = PREP_INT;
    } else {
        if (qdtype == SVSB200_F16 && ix->dtype != SVSB200_F32 && ix->dtype != SVSB200_F16)
            return fail("float16 queries need a float32/float16 dataset");
        *op = metric == SVSB200_L2 ? OP_L2F : metric == SVSB200_IP ? OP_IPF : OP_COSF;
        *mode = PREP_FLOAT;
    }
    return 0;
}

// The kernel parameters of a search over this replica with the generic kernel's visited filter; the lean kernel's
// filter and buffer padding are set by choose_launch.
static SearchParams search_params(const svsb200_index* ix, const Replica* rep, const Scratch* sc, size_t nq, size_t k,
                                  size_t window, size_t capacity, void* d_out_ids, int id_bytes, float* d_out_dists,
                                  bool exhaustive) {
    const bool counting = ix->counting != 0;
    SearchParams p{};
    p.vectors = rep->d_vectors.ptr;
    p.graph = rep->d_graph.ptr;
    p.ref_degree = rep->d_ref_degree.ptr;
    p.n = uint32_t(ix->n);
    p.dim = uint32_t(ix->dim);
    p.row_stride = ix->row_stride;
    p.gstride = ix->gstride;
    p.entry_point = ix->entry_point;
    p.entry_points = rep->d_entry.ptr;
    // push_back drops entry points once the buffer is full (search_buffer.h:311-316): only the first `capacity` count
    p.n_entry = rep->d_entry.ptr ? uint32_t(std::min<size_t>(ix->n_entry, capacity)) : 1;
    p.greater = ix->metric != SVSB200_L2;
    p.sq = ix->storage == SVSB200_SQ;
    p.lvq = ix->storage == SVSB200_LVQ8;
    p.no_split = int(ix->no_split);
    p.lvq_const_offset = ix->lvq_const_offset;
    p.scale = ix->scale;
    p.bias = ix->bias;
    p.scale_sq = ix->scale * ix->scale;   // EuclideanCompressed ctor (scalar.h:68-72)
    p.qf = sc->q_f32.ptr;
    p.qcodes = sc->q_codes.ptr;
    p.qaux = sc->q_aux.ptr;
    p.qstride = query_stride(ix->dim);
    p.nq = uint32_t(nq);
    p.k = uint32_t(k);
    p.window = uint32_t(window);
    p.capacity = uint32_t(capacity);
    p.cap_pad = uint32_t(round_up(capacity + 1, 32));
    p.deg_pad = uint32_t(round_up(ix->gstride, 32));
    p.out_ids = d_out_ids;
    p.id_bytes = id_bytes;
    p.id_offset = id_bytes == 8 ? ix->id_offset : 0;
    p.out_dists = d_out_dists;
    p.work_counter = sc->d_counter.ptr;
    p.cancel = sc->poll_cancel ? sc->d_cancel.ptr : nullptr;   // (no predicate: no per-hop poll in the kernel)
    p.hops = counting ? sc->hops.ptr : nullptr;
    p.evals = counting ? sc->evals.ptr : nullptr;
    p.fetched = counting ? sc->fetched.ptr : nullptr;
    p.filter_slots = exhaustive ? 0u : (ix->filter_slots < 0 ? 4096u : uint32_t(ix->filter_slots));
    // generic kernel: 16-bit tags (two per 32-bit set, 2-way LRU) are exact as long as every id >> log2(sets) fits
    // below the 0xFFFF "empty" mark; larger indexes fall back to direct-mapped 32-bit entries.
    p.filter_shift = 0;
    while ((2u << p.filter_shift) < p.filter_slots) ++p.filter_shift;   // log2(sets) with sets = slots / 2
    p.filter_tag16 = p.filter_slots >= 2 && ((uint64_t(ix->n - 1) >> p.filter_shift) < 0xFFFFull) && ix->filter_tag16 != 0;
    if (!p.filter_tag16) {
        p.filter_shift = 0;
        while ((1u << p.filter_shift) < p.filter_slots) ++p.filter_shift;
    }
    return p;
}

// Picks the kernel (lean or generic) and its launch configuration; for the lean kernel it also sets the buffer padding
// and visited filter in `p`.
static int choose_launch(const svsb200_index* ix, const Replica* rep, SearchParams* p, bool exhaustive, cudaStream_t stream,
                         LaunchConfig* cfg, bool* use_fast) {
    // The lean kernel (search_fast.cuh) covers the common shape: 16-bit-tag filter on, adjacency rows of up to
    // 128 neighbours; anything else (and the exhaustive scan) runs on the generic kernel.  Its filter: default 256
    // sets (4 KB), more when n needs it for exactness.
    const uint32_t fast_cap_pad = uint32_t(round_up(p->capacity, 32));
    const LeanFilter lean = lean_filter(ix->n, ix->filter_slots < 0 ? 2048u : uint32_t(ix->filter_slots));
    const size_t fast_bytes = fast_smem_bytes(p->qstride, fast_cap_pad, p->deg_pad, lean.slots * 2u);
    *use_fast = !exhaustive && !ix->generic_kernel && lean.slots >= 64 && ix->filter_tag16 &&
                p->deg_pad <= 32u * kFastMaxGW && p->gstride % 32u == 0 && fast_bytes <= kSmemOptInMax;
    cfg->stream = stream;
    if (*use_fast) {
        p->cap_pad = fast_cap_pad;
        p->filter_slots = lean.slots;
        p->filter_shift = lean.shift;
        p->filter_tag16 = 1;
        cfg->warps_per_cta = 1;
        cfg->smem_bytes = fast_bytes;
        cfg->grid = ix->ctas_per_sm ? rep->sm_count * int(ix->ctas_per_sm) : -rep->sm_count;
        return 0;
    }
    const size_t per_warp = warp_smem_bytes(p->qstride, p->cap_pad, p->deg_pad, p->filter_slots * (p->filter_tag16 ? 2u : 4u));
    int warps = ix->warps_per_cta ? int(ix->warps_per_cta) : 4;
    while (warps > 1 && per_warp * warps > kSmemOptInMax) warps >>= 1;
    if (per_warp * warps > kSmemOptInMax) return fail("search buffer capacity too large for shared memory");
    cfg->warps_per_cta = warps;
    cfg->smem_bytes = per_warp * warps;
    // grid: persistent CTAs; the launcher clamps to what is resident.  ctas_per_sm == 0
    // means "as many as fit" (computed by the launcher through the occupancy API).
    cfg->grid = rep->sm_count * (ix->ctas_per_sm ? int(ix->ctas_per_sm) : 0);
    if (cfg->grid == 0 || exhaustive) cfg->grid = -rep->sm_count;   // negative: launcher multiplies by occupancy
    return 0;
}

// Waits for the event `ev` of a dynamic search's launch.  With a cancellation predicate in the scratch it polls it
// meanwhile and, once it returns non-zero, raises the device flag the kernel polls per query and per hop, waits for the
// kernel to drain and lowers the flag again.  *cancelled tells whether that happened.
static int wait_dynamic(Scratch* sc, cudaEvent_t ev, bool* cancelled) {
    *cancelled = false;
    if (!sc->cancel_fn) {
        CUDA_TRY(cudaEventSynchronize(ev));
        return 0;
    }
    for (;;) {
        const cudaError_t q = cudaEventQuery(ev);
        if (q == cudaSuccess) break;
        if (q != cudaErrorNotReady) return fail(std::string("cudaEventQuery: ") + cudaGetErrorString(q));
        if (!*cancelled && sc->cancel_fn(sc->cancel_arg)) {
            *cancelled = true;
            CUDA_TRY(cudaMemsetAsync(sc->d_cancel.ptr, 1, sizeof(int), sc->ctl));
        }
        std::this_thread::sleep_for(std::chrono::microseconds(20));
    }
    if (*cancelled) {
        CUDA_TRY(cudaMemsetAsync(sc->d_cancel.ptr, 0, sizeof(int), sc->ctl));
        CUDA_TRY(cudaStreamSynchronize(sc->ctl));
    }
    return 0;
}

// Search of a dynamic index (MutableVamanaIndex::search, dynamic_index.h:482-571) on the lean kernel's MUT form.  The
// buffer holds `capacity + slack` entries; queries whose list outgrows it are listed by the kernel and re-run here with
// four times the room until none is left, so the answer never depends on the slack.  Blocking on `stream`; a
// cancellation predicate in the scratch is polled while the kernels run (the rows of a cancelled search are unspecified,
// as in the reference).  The ids written are external ids, or slots when the scratch asks for them (dyn_slot_ids).
static int search_dynamic(svsb200_index* ix, Replica* rep, Scratch* sc, SearchParams p, LaunchConfig cfg, int op, bool use_fast,
                          cudaStream_t stream) {
    const int rowt = ix->dtype;
    const bool sq = ix->storage == SVSB200_SQ;
    if (sq ? rowt != SVSB200_I8 && rowt != SVSB200_U8
           : ix->storage != SVSB200_PLAIN || (rowt != SVSB200_F32 && rowt != SVSB200_F16))
        return fail("dynamic index: float32 / float16 plain storage or int8 / uint8 SQ codes only");
    // (over SQ codes, L2 runs the integer operator on the compressed query: choose_op's OP_L2I)
    if (!use_fast || (sq ? op != OP_L2I && op != OP_IPF && op != OP_COSF : op > OP_COSF))
        return fail("dynamic index: the search needs the lean kernel (visited filter on, generic_kernel off, float queries)");
    const size_t fixed = fast_smem_bytes(p.qstride, 0, p.deg_pad, p.filter_slots * 2u);
    const size_t max_cap = std::min<size_t>((kSmemOptInMax - fixed) / 8 / 32 * 32, size_t(1) << 24);
    const size_t C = p.capacity;
    size_t slack = ix->dyn_slack >= 0 ? size_t(ix->dyn_slack) : 3 * C + 32;
    // a list never holds more than n distinct slots, so n entries of room can never overflow
    size_t bcap = std::min(std::max(C + slack, C), std::max<size_t>(ix->n, C));
    if (C > max_cap) return fail("search buffer capacity too large for shared memory");
    bcap = std::min(bcap, max_cap);
    p.status = rep->d_status.ptr;
    p.ext_ids = sc->dyn_slot_ids ? nullptr : rep->d_ext_ids.ptr;
    CUDA_TRY(sc->dyn_ovf.ensure(1 + size_t(p.nq)));
    CUDA_TRY(sc->dyn_qlist.ensure(size_t(p.nq)));
    p.ovf = sc->dyn_ovf.ptr;
    p.qlist = nullptr;
    CUDA_TRY(cudaEventRecord(sc->ev_start, stream));
    for (;;) {
        p.buf_cap = uint32_t(bcap);
        p.cap_pad = uint32_t(round_up(bcap, 32));
        cfg.smem_bytes = fast_smem_bytes(p.qstride, p.cap_pad, p.deg_pad, p.filter_slots * 2u);
        CUDA_TRY(cudaMemsetAsync(sc->d_counter.ptr, 0, sizeof(unsigned int), stream));
        CUDA_TRY(cudaMemsetAsync(p.ovf, 0, sizeof(uint32_t), stream));
        CUDA_TRY(sq ? dispatch(DynamicSqRows{}, rowt, [&](auto t) { return launch_search_dynamic_sq<decltype(t)::value>(op, p, cfg); })
                    : dispatch(DynamicRows{}, rowt, [&](auto t) { return launch_search_dynamic<decltype(t)::value>(op, p, cfg); }));
        CUDA_TRY(cudaEventRecord(sc->ev_done, stream));
        bool cancelled = false;
        if (int rc = wait_dynamic(sc, sc->ev_done, &cancelled)) return rc;
        if (cancelled) break;
        uint32_t over = 0;
        CUDA_TRY(cudaMemcpyAsync(&over, p.ovf, sizeof(uint32_t), cudaMemcpyDeviceToHost, stream));
        CUDA_TRY(cudaStreamSynchronize(stream));
        if (over == 0) break;
        if (bcap >= std::max<size_t>(ix->n, C) || bcap >= max_cap)
            return fail("dynamic index: the search buffer cannot hold the Deleted entries of this query in shared memory");
        ix->dyn_reruns += long(over);
        CUDA_TRY(cudaMemcpyAsync(sc->dyn_qlist.ptr, p.ovf + 1, size_t(over) * sizeof(uint32_t), cudaMemcpyDeviceToDevice,
                                 stream));
        p.qlist = sc->dyn_qlist.ptr;
        p.nq = over;
        bcap = std::min(std::min(4 * bcap + 32, std::max<size_t>(ix->n, C)), max_cap);
    }
    CUDA_TRY(cudaEventRecord(sc->ev_stop, stream));
    sc->timed = true;
    {
        std::lock_guard<std::mutex> lock(ix->mu);
        ix->last = sc;
    }
    return 0;
}

int search_on_device(svsb200_index* ix, Replica* rep, Scratch* sc, const void* d_queries, int qdtype, size_t nq, size_t k,
                     size_t window, size_t capacity, void* d_out_ids, int id_bytes, float* d_out_dists, cudaStream_t stream,
                     bool exhaustive, const uint8_t* row_status) {
    if (id_bytes != 4 && id_bytes != 8) return fail("id_bytes must be 4 or 8");
    if (qdtype < SVSB200_F32 || qdtype > SVSB200_U8) return fail("bad query dtype");
    if (ix->dynamic && id_bytes != 8) return fail("a dynamic index returns 64-bit external ids: id_bytes must be 8");
    if (ix->dynamic && exhaustive) return fail("exhaustive search is not available on a dynamic index");
    if (window > capacity) {
        // SearchBufferConfig::check_invariants (search_buffer.h:87-96)
        return fail("Improper configuration for search buffer! search window size cannot exceed capacity");
    }
    if (capacity < k) window = capacity = k;   // index/vamana/index.h:590-592
    if (capacity == 0) return fail("search buffer capacity is zero");
    if (nq == 0) return 0;
    if (nq >= (size_t(1) << 31)) return fail("too many queries in one batch");
    int op = 0, mode = 0;
    if (int rc = choose_op(ix, qdtype, &op, &mode)) return rc;

    if (ix->counting) {
        CUDA_TRY(sc->hops.ensure(nq));
        CUDA_TRY(sc->evals.ensure(nq));
        CUDA_TRY(sc->fetched.ensure(nq));
        sc->counted_nq = nq;
    }
    if (int rc = prepare_queries(ix, rep, sc, d_queries, qdtype, nq, mode, stream)) return rc;
    CUDA_TRY(cudaMemsetAsync(sc->d_counter.ptr, 0, sizeof(unsigned int), stream));
    // (sc->d_cancel is zero here: only wait_kernels raises it, and lowers it again once the kernels have finished)

    SearchParams p = search_params(ix, rep, sc, nq, k, window, capacity, d_out_ids, id_bytes, d_out_dists, exhaustive);
    if (exhaustive && ix->slot_mask) p.status = rep->d_status.ptr;   // dynamic flat index: the Valid slots only
    if (exhaustive && row_status) p.status = row_status;             // filtered flat search: the allowed rows only
    LaunchConfig cfg{};
    bool use_fast = false;
    if (int rc = choose_launch(ix, rep, &p, exhaustive, stream, &cfg, &use_fast)) return rc;
    sc->last_kernel = use_fast ? 1 : 0;
    if (ix->dynamic) return search_dynamic(ix, rep, sc, p, cfg, op, use_fast, stream);
    const int nrows = ix->rows_in_flight ? int(ix->rows_in_flight) : 2;
    uint32_t split = 1;
    if (exhaustive) {
        // few queries: cut the base rows into ranges so that (query, range) work items fill the GPU; the per-range
        // top-k lists are merged with TotalOrder (== the scan's own order: key, then id)
        const size_t want_items = size_t(rep->sm_count) * 32;
        split = uint32_t(std::min<size_t>(64, std::max<size_t>(1, want_items / nq)));
        while (split > 1 && ix->n / split < 4 * k + 64) --split;
        if (split > 1) {
            CUDA_TRY(sc->exh_ids.ensure(size_t(split) * nq * k));
            CUDA_TRY(sc->exh_dists.ensure(size_t(split) * nq * k));
            p.out_ids = sc->exh_ids.ptr;
            p.out_dists = sc->exh_dists.ptr;
            p.exh_split = split;
        }
    }

    CUDA_TRY(cudaEventRecord(sc->ev_start, stream));
    const int rowt = ix->storage == SVSB200_LVQ8 ? ROW_LVQ8 : ix->dtype;
    CUDA_TRY(dispatch(SearchRows{}, rowt, [&](auto row) {
        constexpr int ROWT = decltype(row)::value;
        if (exhaustive) return launch_search_exhaustive<ROWT>(op, p, cfg);
        if (use_fast) return launch_search_fast<ROWT>(op, p, cfg);
        return launch_search<ROWT>(op, p, cfg, nrows);
    }));
    if (split > 1) {
        const unsigned warps = 4;
        merge_topk_kernel<<<unsigned((nq + warps - 1) / warps), warps * 32, 0, stream>>>(
            sc->exh_ids.ptr, sc->exh_dists.ptr, split, uint32_t(nq), uint32_t(k), ix->metric != SVSB200_L2,
            static_cast<uint64_t*>(d_out_ids), d_out_dists);
        count_launch();
        CUDA_TRY(cudaGetLastError());
    }
    CUDA_TRY(cudaEventRecord(sc->ev_stop, stream));
    sc->timed = true;
    {
        std::lock_guard<std::mutex> lock(ix->mu);
        ix->last = sc;
    }
    return 0;
}

// Waits for the search kernels of `scs` (their ev_stop events); with a cancel callback it polls the callback
// meanwhile and raises the device flags the kernels poll per query and per hop (greedy_search.h:155,
// extensions.h:579).
static int wait_kernels(const std::vector<Scratch*>& scs, int (*cancel)(void*), void* cancel_arg) {
    if (!cancel) return 0;   // nothing to poll for: the stream order of the copies behind the kernels is enough
    bool raised = false;
    int rc = 0;
    for (;;) {
        bool busy = false;
        for (Scratch* sc : scs) {
            if (!sc->timed) continue;
            cudaSetDevice(sc->device);
            cudaError_t q = cudaEventQuery(sc->ev_stop);
            if (q == cudaErrorNotReady) busy = true;
            else if (q != cudaSuccess) rc = fail(std::string("cudaEventQuery: ") + cudaGetErrorString(q));
        }
        if (!busy || rc) break;
        if (!raised && cancel(cancel_arg)) {
            raised = true;
            for (Scratch* sc : scs) {
                cudaSetDevice(sc->device);
                cudaError_t e = cudaMemsetAsync(sc->d_cancel.ptr, 1, sizeof(int), sc->ctl);
                if (e != cudaSuccess) rc = fail(std::string("cudaMemsetAsync: ") + cudaGetErrorString(e));
            }
        }
        std::this_thread::sleep_for(std::chrono::microseconds(20));
    }
    if (raised) {   // the kernels are done (or failed): lower the flags for the next search of these scratch sets
        for (Scratch* sc : scs) {
            cudaSetDevice(sc->device);
            cudaStreamSynchronize(sc->stream);
            cudaMemsetAsync(sc->d_cancel.ptr, 0, sizeof(int), sc->ctl);
            cudaStreamSynchronize(sc->ctl);
        }
    }
    return rc;
}
static int wait_all(const std::vector<Scratch*>& scs) {
    for (Scratch* sc : scs) {
        cudaSetDevice(sc->device);
        CUDA_TRY(cudaStreamSynchronize(sc->stream));
    }
    return 0;
}

// Filtered and range search: runs the batch `d_queries` with result lists of `kk` entries per query
// (window = capacity = max(window, kk)) into the scratch's own id / distance blocks, and lets `check(kk, d_unfinished)`
// launch the kernel that counts in *d_unfinished the queries that need a longer list.  Lists grow (x4) until no query
// is unfinished, a list holds the whole index or 16384 entries, like the reference's batch iterator asks for further
// batches (vamana_index_impl.h:183-205).  Returns the final list length in *kk.
template <typename Check>
static int grow_until_done(svsb200_index* ix, Replica* rep, Scratch* sc, const void* d_queries, int qdtype, size_t nq,
                           size_t window, size_t* kk, Check check) {
    CUDA_TRY(sc->grow_unfinished.ensure(1));
    uint32_t* d_unfinished = sc->grow_unfinished.ptr;
    for (;;) {
        *kk = std::min(*kk, ix->n);
        CUDA_TRY(sc->ids.ensure(nq * *kk * 8));
        CUDA_TRY(sc->dists.ensure(nq * *kk));
        const size_t w = std::max(window, *kk);
        if (int rc = search_on_device(ix, rep, sc, d_queries, qdtype, nq, *kk, w, w, sc->ids.ptr, 8, sc->dists.ptr, sc->stream))
            return rc;
        CUDA_TRY(cudaMemsetAsync(d_unfinished, 0, 4, sc->stream));
        check(*kk, d_unfinished);
        count_launch();
        CUDA_TRY(cudaGetLastError());
        uint32_t unfinished = 0;
        CUDA_TRY(cudaMemcpyAsync(&unfinished, d_unfinished, 4, cudaMemcpyDeviceToHost, sc->stream));
        CUDA_TRY(cudaStreamSynchronize(sc->stream));
        if (unfinished == 0 || *kk >= ix->n || *kk >= 16384) return 0;
        *kk *= 4;
    }
}

// Filtered search body on device buffers: `d_bitmap` (rewritten on a dynamic index), the k results per query and the
// number found per query, enqueued on sc->stream apart from the growth decisions, which synchronise it.
static int search_filtered(svsb200_index* ix, Replica* rep, Scratch* sc, const void* d_queries, int qdtype, size_t nq, size_t k,
                           size_t window, uint32_t* d_bitmap, uint64_t* d_oi, float* d_od, uint32_t* d_found) {
    const size_t words = (ix->n + 31) / 32;
    CUDA_TRY(cudaMemsetAsync(d_oi, 0xFF, nq * k * 8, sc->stream));
    if (ix->dynamic) {
        // the bitmap is over slots: only Valid slots may be returned; the search lists slots, translated at the end
        keep_valid_kernel<<<unsigned((words + 255) / 256), 256, 0, sc->stream>>>(d_bitmap, rep->d_status.ptr, ix->n);
        count_launch();
        CUDA_TRY(cudaGetLastError());
        sc->dyn_slot_ids = true;
    }
    // lists grow until every query has k members or its search is exhausted
    size_t kk = std::max(k, window);
    int rc = grow_until_done(ix, rep, sc, d_queries, qdtype, nq, window, &kk, [&](size_t len, uint32_t* d_unfinished) {
        filter_topk_kernel<<<unsigned((nq + 3) / 4), 128, 0, sc->stream>>>(
            reinterpret_cast<const uint64_t*>(sc->ids.ptr), sc->dists.ptr, uint32_t(nq), uint32_t(len), uint32_t(k),
            d_bitmap, ix->id_offset, d_oi, d_od, d_found, d_unfinished);
    });
    sc->dyn_slot_ids = false;
    if (rc) return rc;
    if (ix->dynamic) {
        slots_to_external_kernel<<<unsigned((nq * k + 255) / 256), 256, 0, sc->stream>>>(d_oi, nq * k, rep->d_ext_ids.ptr);
        count_launch();
        CUDA_TRY(cudaGetLastError());
    }
    return 0;
}

// Range search body, on the batch `d_queries` in the scratch checked out by the caller; blocks.
static int range_search(svsb200_index* ix, Replica* rep, Scratch* sc, const void* d_queries, int qdtype, size_t nq,
                        float radius, size_t window, uint32_t* out_counts, uint64_t** out_ids, float** out_dists) {
    CUDA_TRY(sc->range_counts.ensure(nq));
    uint32_t* d_counts = sc->range_counts.ptr;
    size_t kk = std::max<size_t>(window, 16);
    int rc = grow_until_done(ix, rep, sc, d_queries, qdtype, nq, window, &kk, [&](size_t len, uint32_t* d_unfinished) {
        range_count_kernel<<<unsigned((nq + 127) / 128), 128, 0, sc->stream>>>(
            sc->dists.ptr, reinterpret_cast<const uint64_t*>(sc->ids.ptr), uint32_t(nq), uint32_t(len), radius,
            ix->metric != SVSB200_L2, d_counts, d_unfinished);
    });
    if (rc) return rc;   // (on a dynamic index the list holds no Deleted slot and its ids are already external)
    CUDA_TRY(cudaMemcpyAsync(out_counts, d_counts, nq * 4, cudaMemcpyDeviceToHost, sc->stream));
    std::vector<uint64_t> ids(nq * kk);
    std::vector<float> dd(nq * kk);
    CUDA_TRY(cudaMemcpyAsync(ids.data(), sc->ids.ptr, nq * kk * 8, cudaMemcpyDeviceToHost, sc->stream));
    CUDA_TRY(cudaMemcpyAsync(dd.data(), sc->dists.ptr, nq * kk * 4, cudaMemcpyDeviceToHost, sc->stream));
    CUDA_TRY(cudaStreamSynchronize(sc->stream));
    size_t total = 0;
    for (size_t q = 0; q < nq; ++q) total += out_counts[q];
    uint64_t* oi = static_cast<uint64_t*>(malloc(std::max<size_t>(total, 1) * 8));
    float* od = static_cast<float*>(malloc(std::max<size_t>(total, 1) * 4));
    if (!oi || !od) {
        free(oi);
        free(od);
        return fail("svsb200_range_search: out of host memory");
    }
    size_t o = 0;
    for (size_t q = 0; q < nq; ++q)
        for (size_t j = 0; j < out_counts[q]; ++j, ++o) {
            oi[o] = ids[q * kk + j];
            od[o] = dd[q * kk + j];
        }
    *out_ids = oi;
    *out_dists = od;
    return 0;
}

// Sharded search body, on one scratch set per shard checked out by the caller: every query on every shard, merged on
// shard 0's device.
static int search_sharded(svsb200_index* const* shards, const std::vector<Scratch*>& scs, const void* queries, int qdtype,
                          size_t nq, size_t k, size_t window, size_t capacity, uint64_t* out_ids, float* out_dists) {
    const size_t nshards = scs.size();
    const size_t qbytes = nq * shards[0]->dim * esize(qdtype);
    const size_t cnt = nq * k;
    // the merging device is shard 0's; its scratch holds the [nshards][nq][k] gather block
    Replica* rep0 = shards[0]->reps[0].get();
    Scratch* sc0 = scs[0];
    CUDA_TRY(cudaSetDevice(rep0->device));
    CUDA_TRY(sc0->gather_ids.ensure(nshards * cnt));
    CUDA_TRY(sc0->gather_dists.ensure(nshards * cnt));
    CUDA_TRY(sc0->merged_ids.ensure(cnt));
    CUDA_TRY(sc0->merged_dists.ensure(cnt));
    for (size_t s = 0; s < nshards; ++s) {
        Replica* rep = shards[s]->reps[0].get();
        Scratch* sc = scs[s];
        CUDA_TRY(cudaSetDevice(rep->device));
        CUDA_TRY(sc->q_raw.ensure(qbytes));
        CUDA_TRY(cudaMemcpyAsync(sc->q_raw.ptr, queries, qbytes, cudaMemcpyHostToDevice, sc->stream));
        // With peer access the shard's kernel writes its rows straight into the merging device's block over
        // NVLink (the gather is fused into the search kernel's copy-out); otherwise it writes locally and the
        // block is moved by a peer copy.
        bool direct = rep->device == rep0->device;
        if (!direct) {
            int can = 0;
            if (cudaDeviceCanAccessPeer(&can, rep->device, rep0->device) == cudaSuccess && can) {
                cudaError_t pe = cudaDeviceEnablePeerAccess(rep0->device, 0);
                direct = pe == cudaSuccess || pe == cudaErrorPeerAccessAlreadyEnabled;
                cudaGetLastError();
            }
        }
        uint64_t* ids_dst = sc0->gather_ids.ptr + s * cnt;
        float* d_dst = sc0->gather_dists.ptr + s * cnt;
        if (!direct) {
            CUDA_TRY(sc->ids.ensure(cnt * 8));
            CUDA_TRY(sc->dists.ensure(cnt));
        }
        int rc = search_on_device(shards[s], rep, sc, sc->q_raw.ptr, qdtype, nq, k, window, capacity,
                                  direct ? static_cast<void*>(ids_dst) : static_cast<void*>(sc->ids.ptr), 8,
                                  direct ? d_dst : sc->dists.ptr, sc->stream);
        if (rc) return rc;
        CUDA_TRY(cudaEventRecord(sc->ev_done, sc->stream));
        if (s != 0) {
            CUDA_TRY(cudaSetDevice(rep0->device));
            CUDA_TRY(cudaStreamWaitEvent(sc0->stream, sc->ev_done, 0));
            if (!direct) {
                CUDA_TRY(cudaMemcpyPeerAsync(ids_dst, rep0->device, sc->ids.ptr, rep->device, cnt * 8, sc0->stream));
                CUDA_TRY(cudaMemcpyPeerAsync(d_dst, rep0->device, sc->dists.ptr, rep->device, cnt * 4, sc0->stream));
            }
        }
    }
    CUDA_TRY(cudaSetDevice(rep0->device));
    const unsigned warps = 4;
    merge_topk_kernel<<<unsigned((nq + warps - 1) / warps), warps * 32, 0, sc0->stream>>>(
        sc0->gather_ids.ptr, sc0->gather_dists.ptr, uint32_t(nshards), uint32_t(nq), uint32_t(k),
        shards[0]->metric != SVSB200_L2, sc0->merged_ids.ptr, sc0->merged_dists.ptr);
    count_launch();
    CUDA_TRY(cudaGetLastError());
    CUDA_TRY(cudaMemcpyAsync(out_ids, sc0->merged_ids.ptr, cnt * 8, cudaMemcpyDeviceToHost, sc0->stream));
    CUDA_TRY(cudaMemcpyAsync(out_dists, sc0->merged_dists.ptr, cnt * 4, cudaMemcpyDeviceToHost, sc0->stream));
    return 0;
}

static Scratch* last_scratch(svsb200_index* ix) {
    std::lock_guard<std::mutex> lock(ix->mu);
    return ix->last;
}

}  // namespace svsb200

using namespace svsb200;

// =========================================================================================
// C ABI
// =========================================================================================
extern "C" {

int svsb200_search_device(svsb200_index* ix, const void* d_queries, int qdtype, size_t nq, size_t k, size_t window,
                          size_t capacity, int use_visited_set, void* d_out_ids, int id_bytes, float* d_out_dists,
                          void* stream_) {
    (void)use_visited_set;   // performance-only in the reference (search_buffer.h:420); results identical
    if (!ix) return fail("svsb200_search_device: NULL index");
    if (nq && (!d_queries || !d_out_ids || !d_out_dists)) return fail("svsb200_search_device: NULL buffer");
    if (ix->reps.size() != 1) return fail("svsb200_search_device: the index must live on exactly one device");
    Replica* rep = ix->reps[0].get();
    return run_on_stream(rep, stream_, [&](Scratch* sc) {
        return search_on_device(ix, rep, sc, d_queries, qdtype, nq, k, window, capacity, d_out_ids, id_bytes, d_out_dists,
                                sc->stream);
    });
}

int svsb200_search_cancellable(svsb200_index* ix, const void* queries, int qdtype, size_t nq, size_t k, size_t window,
                               size_t capacity, int use_visited_set, void* out_ids, int id_bytes, float* out_dists,
                               void* stream_, int (*cancel)(void*), void* cancel_arg) {
    (void)use_visited_set;
    if (!ix) return fail("svsb200_search: NULL index");
    if (nq == 0) return 0;
    if (!queries || !out_ids || !out_dists) return fail("svsb200_search: NULL buffer");
    if (qdtype < SVSB200_F32 || qdtype > SVSB200_U8) return fail("bad query dtype");
    if (id_bytes != 4 && id_bytes != 8) return fail("id_bytes must be 4 or 8");
    const size_t R = ix->reps.size();
    if (stream_ && R != 1) return fail("svsb200_search: a caller stream needs a single-device index");
    if (cancel && cancel(cancel_arg)) return 0;   // index.h:575 checks before any work
    const size_t qrow = ix->dim * esize(qdtype);
    struct Piece {
        ScratchLease lease;
        size_t lo, m;   // the piece's queries: [lo, lo + m)
    };
    std::vector<Piece> pieces;
    int rc = 0;
    // Every device's share is cut into C pieces, each on its own stream: the host-to-device copy of piece i+1 and the
    // device-to-host copy of piece i-1 run under the kernel of piece i (the kernels of consecutive pieces overlap
    // too -- the next one's CTAs start as the previous one's retire).  C = 1 on a caller's stream (enqueue order is
    // the caller's) and for small shares.
    size_t C = 1;
    if (!stream_ && !ix->counting && !cancel) {   // (the diagnostic counters describe one launch; a predicate: one piece)
        const size_t share = (nq + R - 1) / R;
        // (measured on C2: 1 piece 6.5 M QPS end to end, 4 pieces 7.1 M, 8 pieces 6.8-6.9 M -- the enqueue calls of a piece
        // cost the host about as much as 1 000 queries cost the GPU)
        C = ix->host_chunks > 0 ? size_t(ix->host_chunks) : (share >= 4096 ? 4 : share >= 1024 ? 2 : 1);
        C = std::min(C, share);
    }
    for (size_t part = 0; part < R * C && rc == 0; ++part) {
        const size_t r = part / C;
        size_t lo, hi;
        balance(nq, R * C, part, &lo, &hi);
        if (hi == lo) continue;
        Replica* rep = ix->reps[r].get();
        ScratchLease lease;
        rc = stream_ ? lease.checkout(rep, stream_) : lease.checkout(rep);
        if (rc) break;
        Scratch* sc = lease.get();
        const size_t m = hi - lo;
        pieces.push_back({std::move(lease), lo, m});
        sc->timed = false;
        sc->poll_cancel = cancel != nullptr;
        sc->cancel_fn = ix->dynamic ? cancel : nullptr;   // a dynamic search waits for its kernels itself
        sc->cancel_arg = cancel_arg;
        auto step = [&]() -> int {
            CUDA_TRY(sc->q_raw.ensure(m * qrow));
            CUDA_TRY(sc->ids.ensure(m * k * size_t(id_bytes)));
            CUDA_TRY(sc->dists.ensure(m * k));
            CUDA_TRY(cudaMemcpyAsync(sc->q_raw.ptr, static_cast<const char*>(queries) + lo * qrow, m * qrow,
                                     cudaMemcpyHostToDevice, sc->stream));
            return search_on_device(ix, rep, sc, sc->q_raw.ptr, qdtype, m, k, window, capacity, sc->ids.ptr, id_bytes,
                                    sc->dists.ptr, sc->stream);
        };
        rc = step();
    }
    std::string first_error = svsb200_last_error();
    std::vector<Scratch*> used;
    for (const Piece& piece : pieces) used.push_back(piece.lease.get());
    // the kernels of every replica are in flight: poll the predicate until they finish (a copy into pageable host
    // memory would block this thread, so the device-to-host copies are only enqueued afterwards)
    int rc_wait = wait_kernels(used, cancel, cancel_arg);
    for (size_t i = 0; i < pieces.size() && rc == 0 && rc_wait == 0; ++i) {
        Scratch* sc = used[i];
        if (!sc->timed) continue;
        const Piece& piece = pieces[i];
        auto copy_out = [&]() -> int {
            CUDA_TRY(cudaSetDevice(sc->device));
            CUDA_TRY(cudaMemcpyAsync(static_cast<char*>(out_ids) + piece.lo * k * size_t(id_bytes), sc->ids.ptr,
                                     piece.m * k * size_t(id_bytes), cudaMemcpyDeviceToHost, sc->stream));
            CUDA_TRY(cudaMemcpyAsync(out_dists + piece.lo * k, sc->dists.ptr, piece.m * k * sizeof(float),
                                     cudaMemcpyDeviceToHost, sc->stream));
            return 0;
        };
        rc = copy_out();
        if (rc) first_error = svsb200_last_error();
    }
    if (rc_wait == 0) rc_wait = wait_all(used);
    for (Scratch* sc : used) {   // (before the leases give the pooled scratch sets back)
        sc->poll_cancel = false;
        sc->cancel_fn = nullptr;
    }
    if (rc) return fail(first_error);
    return rc_wait;
}

int svsb200_search(svsb200_index* ix, const void* queries, int qdtype, size_t nq, size_t k, size_t window,
                   size_t capacity, int use_visited_set, void* out_ids, int id_bytes, float* out_dists, void* stream_) {
    return svsb200_search_cancellable(ix, queries, qdtype, nq, k, window, capacity, use_visited_set, out_ids, id_bytes,
                                      out_dists, stream_, nullptr, nullptr);
}

int svsb200_search_filtered(svsb200_index* ix, const void* queries, int qdtype, size_t nq, size_t k, size_t window,
                            const uint32_t* id_bitmap, uint64_t* out_ids, float* out_dists, uint32_t* out_found) {
    if (!ix) return fail("svsb200_search_filtered: NULL index");
    if (nq == 0) return 0;
    if (!queries || !id_bitmap || !out_ids || !out_dists) return fail("svsb200_search_filtered: NULL buffer");
    if (k == 0) return fail("k must be greater than 0");
    if (qdtype < SVSB200_F32 || qdtype > SVSB200_U8) return fail("bad query dtype");
    Replica* rep = ix->reps[0].get();
    std::vector<uint32_t> found(nq);
    if (int rc = run_host_search(rep, {queries, id_bitmap, out_ids, out_dists, {found.data()}}, nq * ix->dim * esize(qdtype),
                                 (ix->n + 31) / 32, nq, k, [&](Scratch* sc, const StagedBuffers& d) {
                                     return search_filtered(ix, rep, sc, d.queries, qdtype, nq, k, window, d.bitmap, d.ids,
                                                            d.dists, d.per_query[0]);
                                 }))
        return rc;
    for (size_t q = 0; q < nq; ++q) {   // pad like the reference: unspecified id (all-ones), +inf distance
        for (size_t j = found[q]; j < k; ++j) {
            out_ids[q * k + j] = ~uint64_t(0);
            out_dists[q * k + j] = INFINITY;
        }
        if (out_found) out_found[q] = found[q];
    }
    return 0;
}

int svsb200_range_search(svsb200_index* ix, const void* queries, int qdtype, size_t nq, float radius, size_t window,
                         uint32_t* out_counts, uint64_t** out_ids, float** out_dists) {
    if (!ix) return fail("svsb200_range_search: NULL index");
    if (nq == 0) return 0;
    if (!queries || !out_counts || !out_ids || !out_dists) return fail("svsb200_range_search: NULL buffer");
    if (qdtype < SVSB200_F32 || qdtype > SVSB200_U8) return fail("bad query dtype");
    *out_ids = nullptr;
    *out_dists = nullptr;
    Replica* rep = ix->reps[0].get();
    return run_host_search(rep, {queries}, nq * ix->dim * esize(qdtype), 0, nq, 0, [&](Scratch* sc, const StagedBuffers& d) {
        return range_search(ix, rep, sc, d.queries, qdtype, nq, radius, window, out_counts, out_ids, out_dists);
    });
}

void svsb200_free(void* p) { free(p); }

int svsb200_search_sharded(svsb200_index* const* shards, size_t nshards, const void* queries, int qdtype, size_t nq,
                           size_t k, size_t window, size_t capacity, uint64_t* out_ids, float* out_dists) {
    if (!shards || nshards == 0) return fail("svsb200_search_sharded: no shards");
    if (nshards > 1024) return fail("svsb200_search_sharded: at most 1024 shards");
    if (nq == 0) return 0;
    if (!queries || !out_ids || !out_dists) return fail("svsb200_search_sharded: NULL buffer");
    if (qdtype < SVSB200_F32 || qdtype > SVSB200_U8) return fail("bad query dtype");
    for (size_t s = 0; s < nshards; ++s) {
        if (!shards[s] || shards[s]->reps.size() != 1) return fail("svsb200_search_sharded: every shard is a single-device index");
        if (shards[s]->dynamic) return fail("svsb200_search_sharded: a dynamic index cannot be a shard");
        if (shards[s]->dim != shards[0]->dim || shards[s]->metric != shards[0]->metric)
            return fail("svsb200_search_sharded: shards disagree on dimension or metric");
    }
    std::vector<ScratchLease> leases(nshards);
    std::vector<Scratch*> scs;
    for (size_t s = 0; s < nshards; ++s) {
        if (int rc = leases[s].checkout(shards[s]->reps[0].get())) return rc;
        scs.push_back(leases[s].get());
    }
    int rc = search_sharded(shards, scs, queries, qdtype, nq, k, window, capacity, out_ids, out_dists);
    const std::string first_error = svsb200_last_error();
    int rc_wait = wait_all(scs);
    if (rc) return fail(first_error);
    return rc_wait;
}

int svsb200_get_fetched(svsb200_index* ix, size_t nq, uint32_t* fetched) {
    if (!ix || !fetched) return fail("svsb200_get_fetched: NULL argument");
    Scratch* sc = last_scratch(ix);
    if (!ix->counting || !sc || sc->counted_nq < nq) return fail("svsb200_get_fetched: counting was not enabled for that many queries");
    CUDA_TRY(cudaSetDevice(sc->device));
    CUDA_TRY(cudaDeviceSynchronize());
    CUDA_TRY(cudaMemcpy(fetched, sc->fetched.ptr, nq * sizeof(uint32_t), cudaMemcpyDeviceToHost));
    return 0;
}

int svsb200_get_counters(svsb200_index* ix, size_t nq, uint32_t* hops, uint32_t* evals) {
    if (!ix) return fail("svsb200_get_counters: NULL index");
    Scratch* sc = last_scratch(ix);
    if (!ix->counting || !sc || sc->counted_nq < nq) return fail("svsb200_get_counters: counting was not enabled for that many queries");
    CUDA_TRY(cudaSetDevice(sc->device));
    CUDA_TRY(cudaDeviceSynchronize());
    if (hops) CUDA_TRY(cudaMemcpy(hops, sc->hops.ptr, nq * sizeof(uint32_t), cudaMemcpyDeviceToHost));
    if (evals) CUDA_TRY(cudaMemcpy(evals, sc->evals.ptr, nq * sizeof(uint32_t), cudaMemcpyDeviceToHost));
    return 0;
}

int svsb200_last_kernel_ms(svsb200_index* ix, float* ms) {
    if (!ix || !ms) return fail("svsb200_last_kernel_ms: NULL argument");
    Scratch* sc = last_scratch(ix);
    if (!sc || !sc->timed) return fail("svsb200_last_kernel_ms: no search has run yet");
    CUDA_TRY(cudaSetDevice(sc->device));
    CUDA_TRY(cudaEventSynchronize(sc->ev_stop));
    CUDA_TRY(cudaEventElapsedTime(ms, sc->ev_start, sc->ev_stop));
    return 0;
}

int svsb200_merge_topk_device(const uint64_t* d_ids, const float* d_dists, size_t nshards, size_t nq, size_t k, int metric,
                              uint64_t* d_out_ids, float* d_out_dists, int device, void* stream) {
    if (nshards == 0 || nshards > 1024) return fail("svsb200_merge_topk_device: 1..1024 shards supported");
    if (nq == 0 || k == 0) return 0;
    CUDA_TRY(cudaSetDevice(device));
    const unsigned warps = 4;
    merge_topk_kernel<<<unsigned((nq + warps - 1) / warps), warps * 32, 0, static_cast<cudaStream_t>(stream)>>>(
        d_ids, d_dists, uint32_t(nshards), uint32_t(nq), uint32_t(k), metric != SVSB200_L2, d_out_ids, d_out_dists);
    count_launch();
    CUDA_TRY(cudaGetLastError());
    return 0;
}

int svsb200_exhaustive_device(svsb200_index* ix, const void* d_queries, int qdtype, size_t nq, size_t k, uint64_t* d_out_ids,
                              float* d_out_dists, void* stream_) {
    if (!ix) return fail("svsb200_exhaustive_device: NULL index");
    if (nq && (!d_queries || !d_out_ids || !d_out_dists)) return fail("svsb200_exhaustive_device: NULL buffer");
    if (k == 0 || k > 1024) return fail("svsb200_exhaustive_device: k must be in [1, 1024]");
    if (ix->reps.size() != 1) return fail("svsb200_exhaustive_device: the index must live on exactly one device");
    Replica* rep = ix->reps[0].get();
    return run_on_stream(rep, stream_, [&](Scratch* sc) {
        return search_on_device(ix, rep, sc, d_queries, qdtype, nq, k, k, k, d_out_ids, 8, d_out_dists, sc->stream, true);
    });
}

}  // extern "C"
