// dynamic_flat.cu -- the dynamic flat index of the C ABI: DynamicFlatIndex (index/flat/dynamic_flat.h), an exact index
// over a mutable set of rows addressed by external ids.  A slot is Valid or Empty (there is no Deleted state and nothing
// to consolidate); status and external ids live in HBM (Replica::d_status / d_ext_ids) with the external -> slot
// translator on the host, as for the dynamic Vamana index.  Searches take the Flat handle's path (flat.cu): the
// tensor-core GEMM over tiles that every mutation keeps exact (a slot that is not Valid is a padding row, which the
// GEMM never offers to a list), then the rescoring and its certificate unchanged, and the exact scan over the Valid
// slots alone for the queries and shapes the GEMM leaves to it.  Ids are mapped to external ids on every route.
#include "host.cuh"

#include <algorithm>
#include <unordered_set>

struct svsb200_dynamic_flat {
    std::unique_ptr<svsb200_index> ix;
};

namespace svsb200 {

// status[slots[i]] = value and, with `ids`, ext_ids[slots[i]] = ids[i]
__global__ void mark_slots_kernel(const uint32_t* __restrict__ slots, const uint64_t* __restrict__ ids, uint32_t count,
                                  uint8_t value, uint8_t* __restrict__ status, uint64_t* __restrict__ ext_ids) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= count) return;
    status[slots[i]] = value;
    if (ids) ext_ids[slots[i]] = ids[i];
}

// Row dst_idx[i] of `dst` <- row src_idx[i] of `src` (an index array NULL: i), rows of `words` 16-byte words; one warp
// per row.
__global__ void move_rows_kernel(const uint4* __restrict__ src, const uint32_t* __restrict__ src_idx, uint4* __restrict__ dst,
                                 const uint32_t* __restrict__ dst_idx, uint32_t count, uint32_t words) {
    const uint32_t i = blockIdx.x * (blockDim.x / 32) + threadIdx.x / 32;
    const uint32_t lane = threadIdx.x & 31;
    if (i >= count) return;
    const size_t s = src_idx ? src_idx[i] : i, d = dst_idx ? dst_idx[i] : i;
    for (uint32_t j = lane; j < words; j += 32) dst[d * words + j] = src[s * words + j];
}

static cudaError_t move_rows(const void* src, const uint32_t* src_idx, void* dst, const uint32_t* dst_idx, size_t count,
                             uint32_t row_stride, cudaStream_t stream) {
    if (count == 0) return cudaSuccess;
    move_rows_kernel<<<unsigned((count + 7) / 8), 256, 0, stream>>>(static_cast<const uint4*>(src), src_idx,
                                                                    static_cast<uint4*>(dst), dst_idx, uint32_t(count),
                                                                    row_stride / 16);
    count_launch();
    return cudaGetLastError();
}

cudaError_t mark_slots(const uint32_t* d_slots, const uint64_t* d_ids, size_t count, uint8_t value, Replica* rep,
                       cudaStream_t stream) {
    if (count == 0) return cudaSuccess;
    mark_slots_kernel<<<unsigned((count + 255) / 256), 256, 0, stream>>>(d_slots, d_ids, uint32_t(count), value,
                                                                          rep->d_status.ptr, rep->d_ext_ids.ptr);
    count_launch();
    return cudaGetLastError();
}

// Bytes of device memory the rows, statuses and external ids of `slots` slots hold (the GEMM's tiles not counted).
static size_t slot_bytes(const svsb200_index* ix, size_t slots) {
    return slots * (size_t(ix->row_stride) + 1 + sizeof(uint64_t));
}

static svsb200_index* index_of(svsb200_dynamic_flat* h) { return h ? h->ix.get() : nullptr; }
static const svsb200_index* index_of(const svsb200_dynamic_flat* h) { return h ? h->ix.get() : nullptr; }

}  // namespace svsb200

using namespace svsb200;

extern "C" {

int svsb200_dynamic_flat_create(const void* vectors, int dtype, size_t n, size_t dim, int metric, const uint64_t* external_ids,
                                int device, svsb200_dynamic_flat** out) {
    const char* who = "svsb200_dynamic_flat_create";
    if (!out) return fail("svsb200_dynamic_flat_create: NULL output");
    *out = nullptr;
    if (n && (!vectors || !external_ids)) return fail("svsb200_dynamic_flat_create: NULL input");
    if (dtype < SVSB200_F32 || dtype > SVSB200_U8) return fail("svsb200_dynamic_flat_create: bad dtype");
    if (metric < SVSB200_L2 || metric > SVSB200_COSINE) return fail("svsb200_dynamic_flat_create: bad metric");
    if (dim == 0) return fail("svsb200_dynamic_flat_create: dim must be positive");
    if (n >= (size_t(1) << 31)) return fail("svsb200_dynamic_flat_create: more than 2^31-1 slots");
    // IDTranslator::insert (core/translation.h:105-127)
    std::unordered_map<uint64_t, uint32_t> translator;
    translator.reserve(n);
    for (size_t i = 0; i < n; ++i)
        if (external_ids[i] == ~uint64_t(0))   // (marks the padding of short result rows)
            return fail("svsb200_dynamic_flat_create: external id 2^64 - 1 is reserved");
        else if (!translator.emplace(external_ids[i], uint32_t(i)).second)
            return fail("svsb200_dynamic_flat_create: External IDs contain repeat elements!");
    cudaDeviceProp prop;
    if (int rc = check_device(who, device, &prop)) return rc;
    auto h = std::make_unique<svsb200_dynamic_flat>();
    h->ix = std::make_unique<svsb200_index>();
    svsb200_index* ix = h->ix.get();
    ix->dtype = dtype;
    ix->metric = metric;
    ix->storage = SVSB200_PLAIN;
    ix->n = n;
    ix->dim = dim;
    ix->row_stride = data_row_stride(SVSB200_PLAIN, dtype, dim);
    ix->gstride = 32;   // the scan's block of rows, as for the Flat handle; there is no adjacency
    ix->slot_mask = true;
    ix->status.assign(n, SLOT_VALID);
    ix->ext_ids.assign(external_ids, external_ids + n);
    ix->translator = std::move(translator);
    ix->first_empty = n;
    ix->reps.push_back(std::make_unique<Replica>());
    Replica* rep = ix->reps.back().get();
    rep->device = device;
    rep->sm_count = prop.multiProcessorCount;
    CUDA_TRY(cudaSetDevice(device));
    const size_t cap = std::max<size_t>(n, 1), row_bytes = dim * esize(dtype);
    CUDA_TRY(rep->d_vectors.ensure(cap * ix->row_stride));
    CUDA_TRY(rep->d_status.ensure(cap));
    CUDA_TRY(rep->d_ext_ids.ensure(cap));
    CUDA_TRY(cudaMemset(rep->d_vectors.ptr, 0, cap * ix->row_stride));
    CUDA_TRY(cudaMemset(rep->d_status.ptr, SLOT_EMPTY, cap));
    if (n) {
        CUDA_TRY(cudaMemcpy2D(rep->d_vectors.ptr, ix->row_stride, vectors, row_bytes, row_bytes, n, cudaMemcpyHostToDevice));
        CUDA_TRY(cudaMemcpy(rep->d_status.ptr, ix->status.data(), n, cudaMemcpyHostToDevice));
        CUDA_TRY(cudaMemcpy(rep->d_ext_ids.ptr, ix->ext_ids.data(), n * sizeof(uint64_t), cudaMemcpyHostToDevice));
    }
    ix->device_bytes = slot_bytes(ix, cap);
    *out = h.release();
    return 0;
}

int svsb200_dynamic_flat_destroy(svsb200_dynamic_flat* index) {
    delete index;   // Replica / Scratch destructors release the device memory
    return 0;
}

size_t svsb200_dynamic_flat_size(const svsb200_dynamic_flat* index) { return index ? index->ix->translator.size() : 0; }
size_t svsb200_dynamic_flat_num_slots(const svsb200_dynamic_flat* index) { return index ? index->ix->n : 0; }
size_t svsb200_dynamic_flat_dimensions(const svsb200_dynamic_flat* index) { return index ? index->ix->dim : 0; }
size_t svsb200_dynamic_flat_device_bytes(const svsb200_dynamic_flat* index) { return index ? index->ix->device_bytes : 0; }

int svsb200_dynamic_flat_add(svsb200_dynamic_flat* index, const void* vectors, int dtype, size_t count, const uint64_t* ids,
                             int reuse_empty, uint64_t* slots_out) {
    svsb200_index* ix = index_of(index);
    if (!ix) return fail("svsb200_dynamic_flat_add: NULL index");
    if (count == 0) return 0;
    if (!vectors || !ids) return fail("svsb200_dynamic_flat_add: NULL argument");
    if (dtype != ix->dtype) return fail("svsb200_dynamic_flat_add: the points' dtype differs from the index's");
    // translator_.insert (core/translation.h:105-127), checked before anything changes
    {
        std::unordered_set<uint64_t> seen;
        seen.reserve(count);
        for (size_t i = 0; i < count; ++i) {
            if (ids[i] == ~uint64_t(0)) return fail("svsb200_dynamic_flat_add: external id 2^64 - 1 is reserved");
            if (!seen.insert(ids[i]).second) return fail("svsb200_dynamic_flat_add: External IDs contain repeat elements!");
            if (ix->translator.count(ids[i]))
                return fail("svsb200_dynamic_flat_add: External ID " + std::to_string(ids[i]) + " already exists!");
        }
    }
    // slots (add_points, dynamic_flat.h:214-276): Empty ones from first_empty_ (from 0 with reuse_empty), then appended
    std::vector<uint32_t> slots;
    slots.reserve(count);
    for (size_t s = reuse_empty ? 0 : ix->first_empty; s < ix->status.size() && slots.size() < count; ++s)
        if (ix->status[s] == SLOT_EMPTY) slots.push_back(uint32_t(s));
    const size_t old_n = ix->n, new_n = old_n + (count - slots.size());
    if (new_n >= (size_t(1) << 31)) return fail("svsb200_dynamic_flat_add: more than 2^31-1 slots");
    for (size_t s = old_n; s < new_n; ++s) slots.push_back(uint32_t(s));
    int rc = after_searches(ix,[&](Replica* rep, cudaStream_t stream) -> int {
        // geometric growth: many small calls do not copy the index each time
        const size_t cap = rep->d_status.count;
        if (new_n > cap) {
            const size_t want = std::max(new_n, 2 * cap);
            CUDA_TRY(cudaStreamSynchronize(stream));
            CUDA_TRY(grow(rep->d_vectors, old_n * ix->row_stride, want * ix->row_stride));
            CUDA_TRY(grow(rep->d_status, old_n, want));
            CUDA_TRY(grow(rep->d_ext_ids, old_n, want));
            CUDA_TRY(cudaMemsetAsync(rep->d_status.ptr + old_n, SLOT_EMPTY, want - old_n, stream));
            ix->device_bytes = slot_bytes(ix, want);
        }
        // The slots become Valid (statuses, then the host's state) only once everything else has succeeded; if a step
        // fails after the tiles were touched, they are dropped and the next search tiles the rows again.
        Replica::SlotStaging& st = rep->staging;
        auto stage_and_place = [&]() -> int {
            if (int rc2 = flat_slots_grow(ix, rep, old_n, new_n, stream)) return rc2;
            CUDA_TRY(st.rows.ensure(count * ix->row_stride));
            CUDA_TRY(st.slots.ensure(count));
            CUDA_TRY(st.ids.ensure(count));
            const size_t row_bytes = ix->dim * esize(ix->dtype);
            if (row_bytes == ix->row_stride) {
                CUDA_TRY(cudaMemcpyAsync(st.rows.ptr, vectors, count * row_bytes, cudaMemcpyHostToDevice, stream));
            } else {   // (the row padding stays zero)
                CUDA_TRY(cudaMemsetAsync(st.rows.ptr, 0, count * ix->row_stride, stream));
                CUDA_TRY(cudaMemcpy2DAsync(st.rows.ptr, ix->row_stride, vectors, row_bytes, row_bytes, count,
                                           cudaMemcpyHostToDevice, stream));
            }
            CUDA_TRY(cudaMemcpyAsync(st.slots.ptr, slots.data(), count * sizeof(uint32_t), cudaMemcpyHostToDevice, stream));
            CUDA_TRY(cudaMemcpyAsync(st.ids.ptr, ids, count * sizeof(uint64_t), cudaMemcpyHostToDevice, stream));
            CUDA_TRY(move_rows(st.rows.ptr, nullptr, rep->d_vectors.ptr, st.slots.ptr, count, ix->row_stride, stream));
            if (int rc2 = flat_slots_place(ix, rep, st.rows.ptr, st.slots.ptr, uint32_t(count), stream)) return rc2;
            CUDA_TRY(mark_slots(st.slots.ptr, st.ids.ptr, count, SLOT_VALID, rep, stream));
            CUDA_TRY(cudaStreamSynchronize(stream));
            return 0;
        };
        const int rc2 = stage_and_place();
        if (rc2) flat_slots_reset(rep);
        return rc2;
    });
    if (rc) return rc;
    ix->n = new_n;
    ix->status.resize(new_n, SLOT_EMPTY);
    ix->ext_ids.resize(new_n, ~uint64_t(0));
    for (size_t i = 0; i < count; ++i) {
        ix->status[slots[i]] = SLOT_VALID;
        ix->ext_ids[slots[i]] = ids[i];
        ix->translator.emplace(ids[i], slots[i]);
        if (slots_out) slots_out[i] = slots[i];
    }
    ix->first_empty = std::max<size_t>(ix->first_empty, size_t(slots.back()) + 1);
    return 0;
}

int svsb200_dynamic_flat_delete(svsb200_dynamic_flat* index, const uint64_t* ids, size_t count) {
    svsb200_index* ix = index_of(index);
    if (!ix) return fail("svsb200_dynamic_flat_delete: NULL index");
    if (count && !ids) return fail("svsb200_dynamic_flat_delete: NULL ids");
    // translator_.check_external_exist (core/translation.h:395-407): nothing changes unless every id is present, once
    std::vector<uint32_t> slots;
    slots.reserve(count);
    std::unordered_set<uint64_t> seen;
    seen.reserve(count);
    for (size_t i = 0; i < count; ++i) {
        auto it = ix->translator.find(ids[i]);
        if (it == ix->translator.end() || !seen.insert(ids[i]).second)
            return fail("svsb200_dynamic_flat_delete: External ID " + std::to_string(ids[i]) + " does not exist!");
        slots.push_back(it->second);
    }
    if (count == 0) return 0;
    int rc = after_searches(ix,[&](Replica* rep, cudaStream_t stream) -> int {
        Replica::SlotStaging& st = rep->staging;
        CUDA_TRY(st.slots.ensure(count));
        CUDA_TRY(cudaMemcpyAsync(st.slots.ptr, slots.data(), count * sizeof(uint32_t), cudaMemcpyHostToDevice, stream));
        // (as in add: the statuses change last; a failure after the tiles were touched drops them)
        auto clear = [&]() -> int {
            if (int rc2 = flat_slots_clear(ix, rep, st.slots.ptr, uint32_t(count), stream)) return rc2;
            CUDA_TRY(mark_slots(st.slots.ptr, nullptr, count, SLOT_EMPTY, rep, stream));
            CUDA_TRY(cudaStreamSynchronize(stream));
            return 0;
        };
        const int rc2 = clear();
        if (rc2) flat_slots_reset(rep);
        return rc2;
    });
    if (rc) return rc;
    // delete_entry + translator_.delete_external (dynamic_flat.h:292-307)
    for (size_t i = 0; i < count; ++i) {
        ix->status[slots[i]] = SLOT_EMPTY;
        ix->ext_ids[slots[i]] = ~uint64_t(0);
        ix->translator.erase(ids[i]);
        ix->first_empty = std::min<size_t>(ix->first_empty, slots[i]);
    }
    return 0;
}

int svsb200_dynamic_flat_compact(svsb200_dynamic_flat* index) {
    svsb200_index* ix = index_of(index);
    if (!ix) return fail("svsb200_dynamic_flat_compact: NULL index");
    // nonmissing_indices (dynamic_flat.h:318-327): the Valid slots, ascending
    const size_t n = ix->n;
    std::vector<uint32_t> new_to_old;
    new_to_old.reserve(ix->translator.size());
    for (size_t s = 0; s < n; ++s)
        if (ix->status[s] == SLOT_VALID) new_to_old.push_back(uint32_t(s));
    const size_t m = new_to_old.size(), cap = std::max<size_t>(m, 1);
    std::vector<uint64_t> ext(m);
    for (size_t i = 0; i < m; ++i) ext[i] = ix->ext_ids[new_to_old[i]];
    int rc = after_searches(ix,[&](Replica* rep, cudaStream_t stream) -> int {
        DeviceBuffer<uint32_t> d_n2o;
        DeviceBuffer<unsigned char> vectors;
        DeviceBuffer<uint8_t> status;
        DeviceBuffer<uint64_t> ext_ids;
        CUDA_TRY(d_n2o.ensure(cap));
        CUDA_TRY(vectors.ensure(cap * ix->row_stride));
        CUDA_TRY(status.ensure(cap));
        CUDA_TRY(ext_ids.ensure(cap));
        CUDA_TRY(cudaMemcpyAsync(d_n2o.ptr, new_to_old.data(), m * 4, cudaMemcpyHostToDevice, stream));
        CUDA_TRY(cudaMemcpyAsync(ext_ids.ptr, ext.data(), m * 8, cudaMemcpyHostToDevice, stream));
        CUDA_TRY(cudaMemsetAsync(status.ptr, SLOT_EMPTY, cap, stream));
        CUDA_TRY(cudaMemsetAsync(status.ptr, SLOT_VALID, m, stream));
        CUDA_TRY(cudaMemsetAsync(vectors.ptr, 0, cap * ix->row_stride, stream));
        CUDA_TRY(move_rows(rep->d_vectors.ptr, d_n2o.ptr, vectors.ptr, nullptr, m, ix->row_stride, stream));
        CUDA_TRY(cudaStreamSynchronize(stream));
        rep->d_vectors = std::move(vectors);   // (the old blocks are freed with the locals)
        rep->d_status = std::move(status);
        rep->d_ext_ids = std::move(ext_ids);
        flat_slots_reset(rep);                 // the next search tiles the compacted rows
        return 0;
    });
    if (rc) return rc;
    ix->n = m;
    ix->device_bytes = slot_bytes(ix, cap);
    ix->status.assign(m, SLOT_VALID);
    ix->ext_ids = std::move(ext);
    for (size_t i = 0; i < m; ++i) ix->translator[ix->ext_ids[i]] = uint32_t(i);
    ix->first_empty = m;
    return 0;
}

int svsb200_dynamic_flat_ids(const svsb200_dynamic_flat* index, uint64_t* out_ids, size_t* count) {
    const svsb200_index* ix = index_of(index);
    if (!ix) return fail("svsb200_dynamic_flat_ids: NULL index");
    if (!count) return fail("svsb200_dynamic_flat_ids: NULL count");
    if (out_ids) {
        if (*count < ix->translator.size()) return fail("svsb200_dynamic_flat_ids: output too small");
        size_t o = 0;
        for (size_t s = 0; s < ix->status.size(); ++s)   // slot order (on_ids, dynamic_flat.h:182-189)
            if (ix->status[s] == SLOT_VALID) out_ids[o++] = ix->ext_ids[s];
    }
    *count = ix->translator.size();
    return 0;
}

int svsb200_dynamic_flat_has_id(const svsb200_dynamic_flat* index, uint64_t id, int* out) {
    const svsb200_index* ix = index_of(index);
    if (!ix) return fail("svsb200_dynamic_flat_has_id: NULL index");
    if (!out) return fail("svsb200_dynamic_flat_has_id: NULL output");
    *out = ix->translator.count(id) ? 1 : 0;
    return 0;
}

int svsb200_dynamic_flat_export(const svsb200_dynamic_flat* index, uint8_t* status_out, uint64_t* ext_ids_out) {
    const svsb200_index* ix = index_of(index);
    if (!ix) return fail("svsb200_dynamic_flat_export: NULL index");
    if (status_out) std::copy(ix->status.begin(), ix->status.end(), status_out);
    if (ext_ids_out) std::copy(ix->ext_ids.begin(), ix->ext_ids.end(), ext_ids_out);
    return 0;
}

int svsb200_dynamic_flat_search_device(svsb200_dynamic_flat* index, const void* d_queries, int qdtype, size_t nq, size_t k,
                                       uint64_t* d_out_ids, float* d_out_dists, void* stream, uint32_t* fallback_queries) {
    return flat_search_device("svsb200_dynamic_flat_search_device", index_of(index), d_queries, qdtype, nq, k, d_out_ids,
                              d_out_dists, stream, fallback_queries, flat_max_kc_deep());
}

int svsb200_dynamic_flat_search(svsb200_dynamic_flat* index, const void* queries, int qdtype, size_t nq, size_t k,
                                uint64_t* out_ids, float* out_dists) {
    return flat_search_host("svsb200_dynamic_flat_search", index_of(index), queries, qdtype, nq, k, out_ids, out_dists,
                            flat_max_kc_deep());
}

int svsb200_dynamic_flat_search_filtered_device(svsb200_dynamic_flat* index, const void* d_queries, int qdtype, size_t nq,
                                                size_t k, const uint32_t* d_slot_bitmap, uint64_t* d_out_ids,
                                                float* d_out_dists, void* stream, size_t* out_allowed,
                                                uint32_t* fallback_queries) {
    return flat_search_filtered_device("svsb200_dynamic_flat_search_filtered_device", index_of(index), d_queries, qdtype, nq,
                                       k, d_slot_bitmap, d_out_ids, d_out_dists, stream, out_allowed, fallback_queries);
}

int svsb200_dynamic_flat_search_filtered(svsb200_dynamic_flat* index, const void* queries, int qdtype, size_t nq, size_t k,
                                         const uint32_t* slot_bitmap, uint64_t* out_ids, float* out_dists,
                                         size_t* out_allowed) {
    return flat_search_filtered_host("svsb200_dynamic_flat_search_filtered", index_of(index), queries, qdtype, nq, k,
                                     slot_bitmap, out_ids, out_dists, out_allowed);
}

}  // extern "C"
