// dynamic_ivf.cu -- the dynamic IVF index of the C ABI (svsb200_dynamic_ivf_*): DynamicIVFIndex
// (index/ivf/dynamic_ivf.h), the IVF index over a mutable set of rows addressed by external ids (DESIGN.md §16).
//
// Layout: one pool of rows (the replica's d_vectors) with one uint32 entry per pooled row (svsb200_ivf::d_row_ids):
// the slot stored there, all-ones for a tombstone or padding.  Cluster c owns the region [start, start + cap) of the
// pool, cap a multiple of 32 and start on a 32-row boundary; its first `count` entries are stored rows (tombstones
// included) and the rest of the region is zero rows with all-ones entries, as the ring of ivf_scan_kernel needs.  An
// add that overflows a cluster moves the cluster to the pool's tail with a doubled capacity; the pool itself grows by
// doubling; compaction lays every cluster out tightly again.  Slots, their statuses, external ids and the external ->
// slot translator follow slots.h's rules, as the dynamic flat index's do; the host also keeps the pool's entries and
// every Valid slot's (cluster, index in the cluster).
//
// Searches are the IVF index's (ivf.cu) with the scan's DYN form: tombstones are not candidates, and the lists are
// ordered by (distance, slot) before the slots become external ids.
//
// SQ storage (svsb200_dynamic_ivf_create_sq): the pool holds int8 / uint8 codes under one scale and bias fixed at
// assembly.  An add takes float32 rows, ranks them against the centroids as a float index does, and encodes them on the
// device (sq_encode) before they are placed; delete and compact move codes as they move float rows.
#include "ivf.cuh"

#include <algorithm>
#include <cmath>

struct svsb200_dynamic_ivf {
    svsb200_ivf iv;                         // the rows pool, its entries, the clusters and the centroids
    std::vector<uint32_t> start, count, cap, live;   // per cluster: region, stored entries, capacity, Valid rows
    std::vector<uint32_t> entries;          // host copy of the entries of the used pool
    std::vector<uint32_t> slot_cluster, slot_index;  // per slot: where its entry is (all-ones for an Empty slot)
    size_t pool_used = 0;                   // pool rows handed out to cluster regions
    // staging of a mutation, kept between calls
    svsb200::DeviceBuffer<unsigned char> dense, rows, codes;   // (codes: an SQ index's added rows, encoded)
    svsb200::DeviceBuffer<uint32_t> assign, src_pos, dst_pos;   // (the entries' values go in Replica::staging.slots)
};

namespace svsb200 {

constexpr uint32_t IVF_NONE = 0xFFFFFFFFu;
constexpr size_t IVF_MIN_POOL = 32;   // rows: an index without rows still has one ring tile of pool

template <typename T> static cudaError_t upload(DeviceBuffer<T>& buf, const std::vector<T>& v, cudaStream_t stream) {
    cudaError_t e = buf.ensure(std::max<size_t>(v.size(), 1));
    if (e == cudaSuccess && !v.empty())
        e = cudaMemcpyAsync(buf.ptr, v.data(), v.size() * sizeof(T), cudaMemcpyHostToDevice, stream);
    return e;
}

static void update_device_bytes(svsb200_dynamic_ivf* h) {
    svsb200_index* ix = h->iv.ix.get();
    const Replica* rep = ix->reps[0].get();
    ix->device_bytes = rep->d_vectors.count + h->iv.d_row_ids.count * 4 + h->iv.C * 8 +
                       rep->d_status.count * (1 + sizeof(uint64_t)) + h->iv.cent->ix->device_bytes;
}

// A fresh pool of `rows` rows: zero rows, all-ones entries.
static int new_pool(DeviceBuffer<unsigned char>& pool, DeviceBuffer<uint32_t>& entries, size_t rows, uint32_t row_stride,
                    cudaStream_t stream) {
    CUDA_TRY(pool.ensure(rows * row_stride));
    CUDA_TRY(entries.ensure(rows));
    CUDA_TRY(cudaMemsetAsync(pool.ptr, 0, rows * row_stride, stream));
    CUDA_TRY(cudaMemsetAsync(entries.ptr, 0xFF, rows * 4, stream));
    return 0;
}

// Room for `used` pool rows, growing the pool by doubling; rows past h->pool_used stay zero with all-ones entries.
static int reserve_pool(svsb200_dynamic_ivf* h, Replica* rep, size_t used, cudaStream_t stream) {
    const size_t have = h->iv.d_row_ids.count, stride = h->iv.ix->row_stride;
    if (used <= have) return 0;
    const size_t want = std::max(used, 2 * have);
    DeviceBuffer<unsigned char> pool;
    DeviceBuffer<uint32_t> entries;
    if (int rc = new_pool(pool, entries, want, uint32_t(stride), stream)) return rc;
    CUDA_TRY(cudaMemcpyAsync(pool.ptr, rep->d_vectors.ptr, h->pool_used * stride, cudaMemcpyDeviceToDevice, stream));
    CUDA_TRY(cudaMemcpyAsync(entries.ptr, h->iv.d_row_ids.ptr, h->pool_used * 4, cudaMemcpyDeviceToDevice, stream));
    CUDA_TRY(cudaStreamSynchronize(stream));
    rep->d_vectors = std::move(pool);   // (the old blocks are freed with the locals)
    h->iv.d_row_ids = std::move(entries);
    return 0;
}

static svsb200_ivf* ivf_of(svsb200_dynamic_ivf* h) { return h ? &h->iv : nullptr; }

}  // namespace svsb200

using namespace svsb200;

// assemble_from_clustering over checked rows (SQ codes when `storage` is SVSB200_SQ): the static layout, clusters in
// order, each from a 32-row boundary, its rows in ascending slot.
static int dynamic_ivf_assemble(const char* who, const void* vectors, int dtype, int storage, float scale, float bias,
                                size_t n, size_t dim, int metric, const float* centroids, size_t num_centroids,
                                const uint32_t* assignments, const uint64_t* external_ids, int device,
                                svsb200_dynamic_ivf** out) {
    const std::string w(who);
    if (metric < SVSB200_L2 || metric > SVSB200_COSINE) return fail(w + ": bad metric");
    if (dim == 0) return fail(w + ": dim must be positive");
    if (n >= (size_t(1) << 31)) return fail(w + ": more than 2^31-1 slots");
    const size_t C = num_centroids;
    if (!centroids) return fail(w + ": NULL centroids");
    if (C == 0 || C >= (size_t(1) << 31)) return fail(w + ": num_centroids must be in [1, 2^31)");
    if (assignments)
        for (size_t i = 0; i < n; ++i)
            if (assignments[i] >= C)
                return fail(w + ": assignment " + std::to_string(i) + " is not a cluster");
    SlotTable slot_table;
    if (int rc = slot_table.assign(who, external_ids, n)) return rc;
    cudaDeviceProp prop;
    if (int rc = check_device(who, device, &prop)) return rc;
    CUDA_TRY(cudaSetDevice(device));
    auto h = std::make_unique<svsb200_dynamic_ivf>();
    svsb200_ivf& iv = h->iv;
    iv.C = C;
    iv.centroids.assign(centroids, centroids + C * dim);
    if (int rc = ivf_centroid_index(centroids, C, dim, metric, device, &iv.cent)) return rc;
    iv.ix = std::make_unique<svsb200_index>();
    svsb200_index* ix = iv.ix.get();
    ix->dtype = dtype;
    ix->metric = metric;
    ix->storage = storage;
    ix->scale = scale;
    ix->bias = bias;
    ix->dim = dim;
    ix->row_stride = data_row_stride(storage, dtype, dim);
    ix->gstride = 32;
    ix->slots = std::move(slot_table);
    ix->reps.push_back(std::make_unique<Replica>());
    Replica* rep = ix->reps.back().get();
    rep->device = device;
    rep->sm_count = prop.multiProcessorCount;
    const size_t row_bytes = dim * esize(dtype);
    OwnStream own;
    CUDA_TRY(cudaStreamCreateWithFlags(&own.s, cudaStreamNonBlocking));
    std::vector<uint32_t> assign(n);
    if (assignments) {
        std::copy(assignments, assignments + n, assign.begin());
    } else if (n) {
        CUDA_TRY(h->dense.ensure(n * row_bytes));
        CUDA_TRY(h->assign.ensure(n));
        CUDA_TRY(cudaMemcpy(h->dense.ptr, vectors, n * row_bytes, cudaMemcpyHostToDevice));
        if (int rc = ivf_assign(iv.cent.get(), reinterpret_cast<const char*>(h->dense.ptr), dtype, n, row_bytes, 65536,
                                h->assign.ptr, own.s))
            return rc;
        CUDA_TRY(cudaMemcpy(assign.data(), h->assign.ptr, n * 4, cudaMemcpyDeviceToHost));
    }
    // the static layout: clusters in order, each from a 32-row boundary, its rows in ascending slot
    h->count.assign(C, 0);
    for (uint32_t a : assign) ++h->count[a];
    h->start.assign(C, 0);
    h->cap.assign(C, 0);
    size_t used = 0;
    for (size_t c = 0; c < C; ++c) {
        h->start[c] = uint32_t(used);
        h->cap[c] = uint32_t(round_up(h->count[c], 32));
        used += h->cap[c];
    }
    if (used >= (size_t(1) << 32)) return fail(w + ": too many rows");
    h->live = h->count;
    h->pool_used = used;
    const size_t pool = std::max(used, IVF_MIN_POOL);
    h->entries.assign(used, IVF_NONE);
    h->slot_cluster.assign(n, 0);
    h->slot_index.assign(n, 0);
    std::vector<char> rows(pool * size_t(ix->row_stride), 0);
    std::vector<uint32_t> fill(C, 0);
    const char* src = static_cast<const char*>(vectors);
    for (size_t i = 0; i < n; ++i) {
        const uint32_t c = assign[i], r = h->start[c] + fill[c];
        h->slot_cluster[i] = c;
        h->slot_index[i] = fill[c]++;
        h->entries[r] = uint32_t(i);
        std::copy(src + i * row_bytes, src + (i + 1) * row_bytes, rows.data() + size_t(r) * ix->row_stride);
    }
    std::vector<uint32_t> entries(pool, IVF_NONE);
    std::copy(h->entries.begin(), h->entries.end(), entries.begin());
    CUDA_TRY(rep->d_vectors.ensure(rows.size()));
    CUDA_TRY(cudaMemcpy(rep->d_vectors.ptr, rows.data(), rows.size(), cudaMemcpyHostToDevice));
    CUDA_TRY(iv.d_row_ids.ensure(pool));
    CUDA_TRY(cudaMemcpy(iv.d_row_ids.ptr, entries.data(), pool * 4, cudaMemcpyHostToDevice));
    CUDA_TRY(iv.d_start.ensure(C));
    CUDA_TRY(cudaMemcpy(iv.d_start.ptr, h->start.data(), C * 4, cudaMemcpyHostToDevice));
    CUDA_TRY(iv.d_count.ensure(C));
    CUDA_TRY(cudaMemcpy(iv.d_count.ptr, h->count.data(), C * 4, cudaMemcpyHostToDevice));
    if (int rc = upload_slots(rep, ix->slots)) return rc;
    update_device_bytes(h.get());
    *out = h.release();
    return 0;
}

extern "C" {

int svsb200_dynamic_ivf_create(const void* vectors, int dtype, size_t n, size_t dim, int metric, const float* centroids,
                               size_t num_centroids, const uint32_t* assignments, const uint64_t* external_ids, int device,
                               svsb200_dynamic_ivf** out) {
    if (!out) return fail("svsb200_dynamic_ivf_create: NULL output");
    *out = nullptr;
    if (n && (!vectors || !external_ids)) return fail("svsb200_dynamic_ivf_create: NULL input");
    if (dtype != SVSB200_F32 && dtype != SVSB200_F16)
        return fail("svsb200_dynamic_ivf_create: rows must be float32 or float16 (integer, SQ and LVQ rows are not supported)");
    return dynamic_ivf_assemble("svsb200_dynamic_ivf_create", vectors, dtype, SVSB200_PLAIN, 0.0f, 0.0f, n, dim, metric,
                                centroids, num_centroids, assignments, external_ids, device, out);
}

int svsb200_dynamic_ivf_create_sq(const void* codes, int code_type, size_t n, size_t dim, int metric, float scale, float bias,
                                  const float* centroids, size_t num_centroids, const uint32_t* assignments,
                                  const uint64_t* external_ids, int device, svsb200_dynamic_ivf** out) {
    const char* who = "svsb200_dynamic_ivf_create_sq";
    if (!out) return fail("svsb200_dynamic_ivf_create_sq: NULL output");
    *out = nullptr;
    if (n && (!codes || !external_ids)) return fail("svsb200_dynamic_ivf_create_sq: NULL input");
    if (code_type != SVSB200_I8 && code_type != SVSB200_U8)
        return fail("svsb200_dynamic_ivf_create_sq: SQ codes must be int8 or uint8");
    if (int rc = sq_check_params(who, scale, bias)) return rc;
    if (n && !assignments)
        return fail("svsb200_dynamic_ivf_create_sq: SQ rows need assignments (there is no float row to rank)");
    return dynamic_ivf_assemble(who, codes, code_type, SVSB200_SQ, scale, bias, n, dim, metric, centroids, num_centroids,
                                assignments, external_ids, device, out);
}

int svsb200_dynamic_ivf_destroy(svsb200_dynamic_ivf* index) {
    if (index) cudaSetDevice(index->iv.ix->reps[0]->device);
    delete index;
    return 0;
}

size_t svsb200_dynamic_ivf_size(const svsb200_dynamic_ivf* index) { return index ? index->iv.ix->slots.size() : 0; }
size_t svsb200_dynamic_ivf_num_slots(const svsb200_dynamic_ivf* index) { return index ? index->iv.ix->slots.num_slots() : 0; }
size_t svsb200_dynamic_ivf_dimensions(const svsb200_dynamic_ivf* index) { return index ? index->iv.ix->dim : 0; }
size_t svsb200_dynamic_ivf_num_clusters(const svsb200_dynamic_ivf* index) { return index ? index->iv.C : 0; }
size_t svsb200_dynamic_ivf_device_bytes(const svsb200_dynamic_ivf* index) { return index ? index->iv.ix->device_bytes : 0; }

int svsb200_dynamic_ivf_cluster_sizes(const svsb200_dynamic_ivf* index, uint32_t* out) {
    if (!index || !out) return fail("svsb200_dynamic_ivf_cluster_sizes: NULL argument");
    std::copy(index->live.begin(), index->live.end(), out);
    return 0;
}

int svsb200_dynamic_ivf_centroids(const svsb200_dynamic_ivf* index, float* out) {
    if (!index || !out) return fail("svsb200_dynamic_ivf_centroids: NULL argument");
    std::copy(index->iv.centroids.begin(), index->iv.centroids.end(), out);
    return 0;
}

int svsb200_dynamic_ivf_add(svsb200_dynamic_ivf* index, const void* vectors, int dtype, size_t count, const uint64_t* ids,
                            int reuse_empty, uint64_t* slots_out) {
    const char* who = "svsb200_dynamic_ivf_add";
    if (!index) return fail("svsb200_dynamic_ivf_add: NULL index");
    if (count == 0) return 0;
    if (!vectors || !ids) return fail("svsb200_dynamic_ivf_add: NULL argument");
    svsb200_dynamic_ivf* h = index;
    svsb200_index* ix = h->iv.ix.get();
    // an SQ index takes float32 rows and encodes them with its fixed scale and bias (SQDataset::set_datum)
    const bool sq = ix->storage == SVSB200_SQ;
    if (sq) {
        if (dtype != SVSB200_F32) return fail("svsb200_dynamic_ivf_add: an SQ index takes float32 points");
        const float* x = static_cast<const float*>(vectors);
        for (size_t i = 0; i < count * ix->dim; ++i)
            if (!std::isfinite(x[i])) return fail("svsb200_dynamic_ivf_add: the points hold a NaN or an infinity");
    } else if (dtype != ix->dtype) {
        return fail("svsb200_dynamic_ivf_add: the points' dtype differs from the index's");
    }
    if (int rc = ix->slots.check_new(who, ids, count)) return rc;
    // slots (add_points, dynamic_ivf.h:474-527): Empty ones from slot 0 with reuse_empty, then appended
    std::vector<uint32_t> slots;
    const size_t old_n = ix->slots.num_slots();
    const size_t new_n = ix->slots.choose(count, reuse_empty ? 0 : old_n, &slots);
    if (new_n >= (size_t(1) << 31)) return fail("svsb200_dynamic_ivf_add: more than 2^31-1 slots");
    const size_t C = h->iv.C, stride = ix->row_stride, in_bytes = ix->dim * esize(dtype), row_bytes = ix->dim * esize(ix->dtype);
    // the new layout, made inside the mutation and taken over once every device step has succeeded
    std::vector<uint32_t> assign(count), index_in(count), start = h->start, cnt = h->count, cap = h->cap;
    std::vector<uint32_t> reloc_src, reloc_dst, reloc_val;
    size_t used = h->pool_used;
    int rc = after_searches(ix, [&](Replica* rep, cudaStream_t stream) -> int {
        // Nothing a search reads changes before the last step: the new entries lie past the clusters' old counts or in
        // regions the old starts do not reach, until the new starts and counts are uploaded.
        if (const size_t cap = slot_capacity(rep, new_n))
            if (int rc2 = grow_slots(rep, old_n, cap, stream)) return rc2;
        // 1. the nearest centroid of every row, as a probe ranks them
        CUDA_TRY(h->dense.ensure(count * in_bytes));
        CUDA_TRY(h->assign.ensure(count));
        CUDA_TRY(cudaMemcpyAsync(h->dense.ptr, vectors, count * in_bytes, cudaMemcpyHostToDevice, stream));
        if (int rc2 = ivf_assign(h->iv.cent.get(), reinterpret_cast<const char*>(h->dense.ptr), dtype, count, in_bytes,
                                 65536, h->assign.ptr, stream))
            return rc2;
        CUDA_TRY(cudaMemcpy(assign.data(), h->assign.ptr, count * 4, cudaMemcpyDeviceToHost));
        // 2. positions: appended in input order within each cluster (insert_into_clusters, dynamic_ivf.h:966-985)
        for (size_t i = 0; i < count; ++i) index_in[i] = cnt[assign[i]]++;
        // 3. clusters that overflow move to the pool's tail with room to grow
        for (size_t c = 0; c < C; ++c) {
            if (cnt[c] <= cap[c]) continue;
            const uint32_t ncap = uint32_t(round_up(std::max<size_t>(2 * size_t(cap[c]), cnt[c]), 32));
            for (uint32_t j = 0; j < h->count[c]; ++j) {
                reloc_src.push_back(start[c] + j);
                reloc_dst.push_back(uint32_t(used + j));
                reloc_val.push_back(h->entries[start[c] + j]);
            }
            start[c] = uint32_t(used);
            cap[c] = ncap;
            used += ncap;
        }
        if (used >= (size_t(1) << 32)) return fail("svsb200_dynamic_ivf_add: the rows pool would pass 2^32 rows");
        if (int rc2 = reserve_pool(h, rep, used, stream)) return rc2;
        Replica::SlotStaging& st = rep->staging;
        if (!reloc_src.empty()) {
            CUDA_TRY(upload(h->src_pos, reloc_src, stream));
            CUDA_TRY(upload(h->dst_pos, reloc_dst, stream));
            CUDA_TRY(upload(st.slots, reloc_val, stream));
            CUDA_TRY(move_rows(rep->d_vectors.ptr, h->src_pos.ptr, rep->d_vectors.ptr, h->dst_pos.ptr, st.slots.ptr,
                               h->iv.d_row_ids.ptr, reloc_src.size(), uint32_t(stride), stream));
            CUDA_TRY(cudaStreamSynchronize(stream));   // (before the staging buffers are refilled)
        }
        // 4. the rows (SQ: their codes) and their slots into place
        const void* src = h->dense.ptr;
        const void* from = vectors;   // the dense rows as stored, `row_bytes` apart
        cudaMemcpyKind kind = cudaMemcpyHostToDevice;
        if (sq) {
            const size_t values = count * ix->dim;
            const unsigned grid = unsigned(std::min<size_t>((values + 255) / 256, size_t(rep->sm_count) * 8));
            CUDA_TRY(h->codes.ensure(values));
            CUDA_TRY(sq_encode(reinterpret_cast<const float*>(h->dense.ptr), values, ix->dtype, ix->scale, ix->bias,
                               h->codes.ptr, grid, stream));
            src = from = h->codes.ptr;
            kind = cudaMemcpyDeviceToDevice;
        }
        if (row_bytes != stride) {   // (the row padding stays zero)
            CUDA_TRY(h->rows.ensure(count * stride));
            CUDA_TRY(cudaMemsetAsync(h->rows.ptr, 0, count * stride, stream));
            CUDA_TRY(cudaMemcpy2DAsync(h->rows.ptr, stride, from, row_bytes, row_bytes, count, kind, stream));
            src = h->rows.ptr;
        }
        std::vector<uint32_t> dst(count);
        for (size_t i = 0; i < count; ++i) dst[i] = start[assign[i]] + index_in[i];
        CUDA_TRY(upload(h->dst_pos, dst, stream));
        CUDA_TRY(upload(st.slots, slots, stream));
        CUDA_TRY(move_rows(src, nullptr, rep->d_vectors.ptr, h->dst_pos.ptr, st.slots.ptr, h->iv.d_row_ids.ptr, count,
                           uint32_t(stride), stream));
        // 5. the slots become Valid, then the clusters' new layout takes effect
        CUDA_TRY(st.ids.ensure(count));
        CUDA_TRY(cudaMemcpyAsync(st.ids.ptr, ids, count * 8, cudaMemcpyHostToDevice, stream));
        CUDA_TRY(mark_slots(st.slots.ptr, st.ids.ptr, count, SLOT_VALID, rep, stream));
        CUDA_TRY(cudaMemcpyAsync(h->iv.d_start.ptr, start.data(), C * 4, cudaMemcpyHostToDevice, stream));
        CUDA_TRY(cudaMemcpyAsync(h->iv.d_count.ptr, cnt.data(), C * 4, cudaMemcpyHostToDevice, stream));
        CUDA_TRY(cudaStreamSynchronize(stream));
        return 0;
    });
    if (rc) return rc;
    h->entries.resize(used, IVF_NONE);
    for (size_t r = 0; r < reloc_src.size(); ++r) h->entries[reloc_dst[r]] = reloc_val[r];
    h->start = std::move(start);
    h->count = std::move(cnt);
    h->cap = std::move(cap);
    h->pool_used = used;
    h->slot_cluster.resize(new_n, IVF_NONE);
    h->slot_index.resize(new_n, IVF_NONE);
    for (size_t i = 0; i < count; ++i) {
        const uint32_t s = slots[i], c = assign[i];
        h->entries[h->start[c] + index_in[i]] = s;
        h->slot_cluster[s] = c;
        h->slot_index[s] = index_in[i];
        ++h->live[c];
    }
    ix->slots.commit_add(slots, ids, slots_out);
    update_device_bytes(h);
    return 0;
}

int svsb200_dynamic_ivf_delete(svsb200_dynamic_ivf* index, const uint64_t* ids, size_t count) {
    if (!index) return fail("svsb200_dynamic_ivf_delete: NULL index");
    if (count && !ids) return fail("svsb200_dynamic_ivf_delete: NULL ids");
    svsb200_dynamic_ivf* h = index;
    svsb200_index* ix = h->iv.ix.get();
    // nothing changes unless every id is present, once (dynamic_ivf.h:547-636)
    std::vector<uint32_t> slots, pos;
    if (int rc = ix->slots.find("svsb200_dynamic_ivf_delete", ids, count, &slots)) return rc;
    if (count == 0) return 0;
    pos.reserve(count);
    for (uint32_t s : slots) pos.push_back(h->start[h->slot_cluster[s]] + h->slot_index[s]);
    int rc = after_searches(ix, [&](Replica* rep, cudaStream_t stream) -> int {
        // the entries become tombstones, then the slots Empty
        CUDA_TRY(upload(h->dst_pos, pos, stream));
        CUDA_TRY(upload(rep->staging.slots, slots, stream));
        CUDA_TRY(move_rows(nullptr, nullptr, nullptr, h->dst_pos.ptr, nullptr, h->iv.d_row_ids.ptr, count,
                           uint32_t(ix->row_stride), stream));
        CUDA_TRY(mark_slots(rep->staging.slots.ptr, nullptr, count, SLOT_EMPTY, rep, stream));
        CUDA_TRY(cudaStreamSynchronize(stream));
        return 0;
    });
    if (rc) return rc;
    for (size_t i = 0; i < count; ++i) {
        const uint32_t s = slots[i];
        h->entries[pos[i]] = IVF_NONE;
        --h->live[h->slot_cluster[s]];
        h->slot_cluster[s] = IVF_NONE;
        h->slot_index[s] = IVF_NONE;
    }
    ix->slots.commit_delete(slots, ids, SLOT_EMPTY);
    return 0;
}

int svsb200_dynamic_ivf_compact(svsb200_dynamic_ivf* index) {
    if (!index) return fail("svsb200_dynamic_ivf_compact: NULL index");
    svsb200_dynamic_ivf* h = index;
    svsb200_index* ix = h->iv.ix.get();
    const size_t C = h->iv.C, stride = ix->row_stride;
    // compact (dynamic_ivf.h:932-961): the Valid slots renumbered 0 .. m-1 in slot order; every cluster keeps the
    // stored order of its live entries, laid out tightly from a 32-row boundary
    std::vector<uint64_t> ext;
    const std::vector<uint32_t> new_to_old = ix->slots.valid_slots(&ext);
    const size_t m = new_to_old.size();
    std::vector<uint32_t> renum(ix->slots.num_slots(), IVF_NONE);
    for (size_t i = 0; i < m; ++i) renum[new_to_old[i]] = uint32_t(i);
    std::vector<uint32_t> start(C), cap(C), src, dst, val, slot_cluster(m), slot_index(m);
    size_t used = 0;
    for (size_t c = 0; c < C; ++c) {
        start[c] = uint32_t(used);
        cap[c] = uint32_t(round_up(h->live[c], 32));
        uint32_t j = 0;
        for (uint32_t e = 0; e < h->count[c]; ++e) {
            const uint32_t s = h->entries[h->start[c] + e];
            if (s == IVF_NONE) continue;
            src.push_back(h->start[c] + e);
            dst.push_back(uint32_t(used + j));
            val.push_back(renum[s]);
            slot_cluster[renum[s]] = uint32_t(c);
            slot_index[renum[s]] = j++;
        }
        used += cap[c];
    }
    const size_t pool = std::max(used, IVF_MIN_POOL), slots = std::max<size_t>(m, 1);
    int rc = after_searches(ix, [&](Replica* rep, cudaStream_t stream) -> int {
        DeviceBuffer<unsigned char> vectors;
        DeviceBuffer<uint32_t> entries;
        DeviceBuffer<uint8_t> status;
        DeviceBuffer<uint64_t> ext_ids;
        if (int rc2 = new_pool(vectors, entries, pool, uint32_t(stride), stream)) return rc2;
        if (int rc2 = compacted_slots(ext, slots, &status, &ext_ids, stream)) return rc2;
        CUDA_TRY(upload(h->src_pos, src, stream));
        CUDA_TRY(upload(h->dst_pos, dst, stream));
        CUDA_TRY(upload(rep->staging.slots, val, stream));
        CUDA_TRY(move_rows(rep->d_vectors.ptr, h->src_pos.ptr, vectors.ptr, h->dst_pos.ptr, rep->staging.slots.ptr,
                           entries.ptr, m, uint32_t(stride), stream));
        CUDA_TRY(cudaMemcpyAsync(h->iv.d_start.ptr, start.data(), C * 4, cudaMemcpyHostToDevice, stream));
        CUDA_TRY(cudaMemcpyAsync(h->iv.d_count.ptr, h->live.data(), C * 4, cudaMemcpyHostToDevice, stream));
        CUDA_TRY(cudaStreamSynchronize(stream));
        rep->d_vectors = std::move(vectors);   // (the old blocks are freed with the locals)
        h->iv.d_row_ids = std::move(entries);
        rep->d_status = std::move(status);
        rep->d_ext_ids = std::move(ext_ids);
        return 0;
    });
    if (rc) return rc;
    h->entries.assign(used, IVF_NONE);
    for (size_t i = 0; i < m; ++i) h->entries[dst[i]] = val[i];
    h->start = std::move(start);
    h->cap = std::move(cap);
    h->count = h->live;
    h->pool_used = used;
    h->slot_cluster = std::move(slot_cluster);
    h->slot_index = std::move(slot_index);
    ix->slots.commit_compact(std::move(ext));
    update_device_bytes(h);
    return 0;
}

int svsb200_dynamic_ivf_ids(const svsb200_dynamic_ivf* index, uint64_t* out_ids, size_t* count) {
    if (!index) return fail("svsb200_dynamic_ivf_ids: NULL index");
    return index->iv.ix->slots.ids("svsb200_dynamic_ivf_ids", out_ids, count);
}

int svsb200_dynamic_ivf_has_id(const svsb200_dynamic_ivf* index, uint64_t id, int* out) {
    if (!index) return fail("svsb200_dynamic_ivf_has_id: NULL index");
    return index->iv.ix->slots.has_id("svsb200_dynamic_ivf_has_id", id, out);
}

int svsb200_dynamic_ivf_export(const svsb200_dynamic_ivf* index, uint8_t* status_out, uint64_t* ext_ids_out,
                               uint32_t* cluster_out) {
    if (!index) return fail("svsb200_dynamic_ivf_export: NULL index");
    index->iv.ix->slots.export_to(status_out, ext_ids_out);
    if (cluster_out) std::copy(index->slot_cluster.begin(), index->slot_cluster.end(), cluster_out);
    return 0;
}

int svsb200_dynamic_ivf_search_device(svsb200_dynamic_ivf* index, const void* d_queries, int qdtype, size_t nq, size_t k,
                                      size_t n_probes, uint64_t* d_out_ids, float* d_out_dists, void* stream_) {
    if (int rc = ivf_check_search("svsb200_dynamic_ivf_search_device", ivf_of(index), qdtype, k, n_probes)) return rc;
    if (nq == 0) return 0;
    if (!d_queries || !d_out_ids || !d_out_dists) return fail("svsb200_dynamic_ivf_search_device: NULL buffer");
    Replica* rep = index->iv.ix->reps[0].get();
    return run_on_stream(rep, stream_, [&](Scratch* sc) {
        return ivf_search_on_device(&index->iv, sc, d_queries, qdtype, nq, k, n_probes, d_out_ids, d_out_dists,
                                    rep->d_ext_ids.ptr);
    });
}

int svsb200_dynamic_ivf_search(svsb200_dynamic_ivf* index, const void* queries, int qdtype, size_t nq, size_t k,
                               size_t n_probes, uint64_t* out_ids, float* out_dists) {
    if (int rc = ivf_check_search("svsb200_dynamic_ivf_search", ivf_of(index), qdtype, k, n_probes)) return rc;
    if (nq == 0) return 0;
    if (!queries || !out_ids || !out_dists) return fail("svsb200_dynamic_ivf_search: NULL buffer");
    Replica* rep = index->iv.ix->reps[0].get();
    return run_host_search(rep, {queries, nullptr, out_ids, out_dists}, nq * index->iv.ix->dim * esize(qdtype), 0, nq, k,
                           [&](Scratch* sc, const StagedBuffers& d) {
                               return ivf_search_on_device(&index->iv, sc, d.queries, qdtype, nq, k, n_probes, d.ids, d.dists,
                                                           rep->d_ext_ids.ptr);
                           });
}

int svsb200_dynamic_ivf_search_filtered_device(svsb200_dynamic_ivf* index, const void* d_queries, int qdtype, size_t nq,
                                               size_t k, size_t n_probes, const uint32_t* d_slot_bitmap, uint64_t* d_out_ids,
                                               float* d_out_dists, uint32_t* d_out_probes, uint32_t* d_out_allowed,
                                               uint32_t* d_out_rows, void* stream_) {
    const char* who = "svsb200_dynamic_ivf_search_filtered_device";
    if (int rc = ivf_check_search(who, ivf_of(index), qdtype, k, n_probes)) return rc;
    if (!d_slot_bitmap) return fail("svsb200_dynamic_ivf_search_filtered_device: NULL bitmap");
    if (nq == 0) return 0;
    if (!d_queries || !d_out_ids || !d_out_dists) return fail("svsb200_dynamic_ivf_search_filtered_device: NULL buffer");
    Replica* rep = index->iv.ix->reps[0].get();
    return run_on_stream(rep, stream_, [&](Scratch* sc) {
        return ivf_search_filtered_on_device(&index->iv, sc, d_queries, qdtype, nq, k, n_probes, d_slot_bitmap, d_out_ids,
                                             d_out_dists, d_out_probes, d_out_allowed, d_out_rows, rep->d_ext_ids.ptr);
    });
}

int svsb200_dynamic_ivf_search_filtered(svsb200_dynamic_ivf* index, const void* queries, int qdtype, size_t nq, size_t k,
                                        size_t n_probes, const uint32_t* slot_bitmap, uint64_t* out_ids, float* out_dists,
                                        uint32_t* out_probes, uint32_t* out_allowed, uint32_t* out_rows) {
    if (int rc = ivf_check_search("svsb200_dynamic_ivf_search_filtered", ivf_of(index), qdtype, k, n_probes)) return rc;
    if (!slot_bitmap) return fail("svsb200_dynamic_ivf_search_filtered: NULL bitmap");
    if (nq == 0) return 0;
    if (!queries || !out_ids || !out_dists) return fail("svsb200_dynamic_ivf_search_filtered: NULL buffer");
    Replica* rep = index->iv.ix->reps[0].get();
    return run_host_search(rep, {queries, slot_bitmap, out_ids, out_dists, {out_probes, out_allowed, out_rows}},
                           nq * index->iv.ix->dim * esize(qdtype), (index->iv.ix->slots.num_slots() + 31) / 32, nq, k,
                           [&](Scratch* sc, const StagedBuffers& d) {
                               return ivf_search_filtered_on_device(&index->iv, sc, d.queries, qdtype, nq, k, n_probes, d.bitmap,
                                                                    d.ids, d.dists, d.per_query[0], d.per_query[1],
                                                                    d.per_query[2], rep->d_ext_ids.ptr);
                           });
}

}  // extern "C"
