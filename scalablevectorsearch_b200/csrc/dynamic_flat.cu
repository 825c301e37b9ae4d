// dynamic_flat.cu -- the dynamic flat index of the C ABI: DynamicFlatIndex (index/flat/dynamic_flat.h), an exact index
// over a mutable set of rows addressed by external ids.  A slot is Valid or Empty (there is no Deleted state and nothing
// to consolidate); status and external ids live in HBM (Replica::d_status / d_ext_ids) with the external -> slot
// translator on the host, as for the dynamic Vamana index; the slot rules are slots.h's.  Searches take the Flat handle's path (flat.cu): the
// tensor-core GEMM over tiles that every mutation keeps exact (a slot that is not Valid is a padding row, which the
// GEMM never offers to a list), then the rescoring and its certificate unchanged, and the exact scan over the Valid
// slots alone for the queries and shapes the GEMM leaves to it.  Ids are mapped to external ids on every route.
#include "host.cuh"

#include <algorithm>

struct svsb200_dynamic_flat {
    std::unique_ptr<svsb200_index> ix;
};

namespace svsb200 {

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
    SlotTable slots;
    if (int rc = slots.assign(who, external_ids, n)) return rc;
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
    ix->slots = std::move(slots);
    ix->reps.push_back(std::make_unique<Replica>());
    Replica* rep = ix->reps.back().get();
    rep->device = device;
    rep->sm_count = prop.multiProcessorCount;
    CUDA_TRY(cudaSetDevice(device));
    const size_t cap = std::max<size_t>(n, 1), row_bytes = dim * esize(dtype);
    CUDA_TRY(rep->d_vectors.ensure(cap * ix->row_stride));
    CUDA_TRY(cudaMemset(rep->d_vectors.ptr, 0, cap * ix->row_stride));
    if (n)
        CUDA_TRY(cudaMemcpy2D(rep->d_vectors.ptr, ix->row_stride, vectors, row_bytes, row_bytes, n, cudaMemcpyHostToDevice));
    if (int rc = upload_slots(rep, ix->slots)) return rc;
    ix->device_bytes = slot_bytes(ix, cap);
    *out = h.release();
    return 0;
}

int svsb200_dynamic_flat_destroy(svsb200_dynamic_flat* index) {
    delete index;   // Replica / Scratch destructors release the device memory
    return 0;
}

size_t svsb200_dynamic_flat_size(const svsb200_dynamic_flat* index) { return index ? index->ix->slots.size() : 0; }
size_t svsb200_dynamic_flat_num_slots(const svsb200_dynamic_flat* index) { return index ? index->ix->n : 0; }
size_t svsb200_dynamic_flat_dimensions(const svsb200_dynamic_flat* index) { return index ? index->ix->dim : 0; }
size_t svsb200_dynamic_flat_device_bytes(const svsb200_dynamic_flat* index) { return index ? index->ix->device_bytes : 0; }

int svsb200_dynamic_flat_add(svsb200_dynamic_flat* index, const void* vectors, int dtype, size_t count, const uint64_t* ids,
                             int reuse_empty, uint64_t* slots_out) {
    const char* who = "svsb200_dynamic_flat_add";
    svsb200_index* ix = index_of(index);
    if (!ix) return fail("svsb200_dynamic_flat_add: NULL index");
    if (count == 0) return 0;
    if (!vectors || !ids) return fail("svsb200_dynamic_flat_add: NULL argument");
    if (dtype != ix->dtype) return fail("svsb200_dynamic_flat_add: the points' dtype differs from the index's");
    if (int rc = ix->slots.check_new(who, ids, count)) return rc;
    // slots (add_points, dynamic_flat.h:214-276): Empty ones from first_empty_ (from 0 with reuse_empty), then appended
    std::vector<uint32_t> slots;
    const size_t old_n = ix->n, new_n = ix->slots.choose(count, reuse_empty ? 0 : ix->slots.first_empty, &slots);
    if (new_n >= (size_t(1) << 31)) return fail("svsb200_dynamic_flat_add: more than 2^31-1 slots");
    int rc = after_searches(ix, [&](Replica* rep, cudaStream_t stream) -> int {
        if (const size_t cap = slot_capacity(rep, new_n)) {   // (the rows first: d_status's size is the capacity)
            CUDA_TRY(cudaStreamSynchronize(stream));
            CUDA_TRY(grow(rep->d_vectors, old_n * ix->row_stride, cap * ix->row_stride));
            if (int rc2 = grow_slots(rep, old_n, cap, stream)) return rc2;
            ix->device_bytes = slot_bytes(ix, cap);
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
            CUDA_TRY(move_rows(st.rows.ptr, nullptr, rep->d_vectors.ptr, st.slots.ptr, nullptr, nullptr, count, ix->row_stride,
                               stream));
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
    ix->slots.commit_add(slots, ids, slots_out);
    return 0;
}

int svsb200_dynamic_flat_delete(svsb200_dynamic_flat* index, const uint64_t* ids, size_t count) {
    svsb200_index* ix = index_of(index);
    if (!ix) return fail("svsb200_dynamic_flat_delete: NULL index");
    if (count && !ids) return fail("svsb200_dynamic_flat_delete: NULL ids");
    std::vector<uint32_t> slots;
    if (int rc = ix->slots.find("svsb200_dynamic_flat_delete", ids, count, &slots)) return rc;
    if (count == 0) return 0;
    int rc = after_searches(ix, [&](Replica* rep, cudaStream_t stream) -> int {
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
    ix->slots.commit_delete(slots, ids, SLOT_EMPTY);
    return 0;
}

int svsb200_dynamic_flat_compact(svsb200_dynamic_flat* index) {
    svsb200_index* ix = index_of(index);
    if (!ix) return fail("svsb200_dynamic_flat_compact: NULL index");
    // nonmissing_indices (dynamic_flat.h:318-327): the Valid slots, ascending
    std::vector<uint64_t> ext;
    const std::vector<uint32_t> new_to_old = ix->slots.valid_slots(&ext);
    const size_t m = new_to_old.size(), cap = std::max<size_t>(m, 1);
    int rc = after_searches(ix, [&](Replica* rep, cudaStream_t stream) -> int {
        DeviceBuffer<uint32_t> d_n2o;
        DeviceBuffer<unsigned char> vectors;
        DeviceBuffer<uint8_t> status;
        DeviceBuffer<uint64_t> ext_ids;
        CUDA_TRY(d_n2o.ensure(cap));
        CUDA_TRY(vectors.ensure(cap * ix->row_stride));
        CUDA_TRY(cudaMemcpyAsync(d_n2o.ptr, new_to_old.data(), m * 4, cudaMemcpyHostToDevice, stream));
        if (int rc2 = compacted_slots(ext, cap, &status, &ext_ids, stream)) return rc2;
        CUDA_TRY(cudaMemsetAsync(vectors.ptr, 0, cap * ix->row_stride, stream));
        CUDA_TRY(move_rows(rep->d_vectors.ptr, d_n2o.ptr, vectors.ptr, nullptr, nullptr, nullptr, m, ix->row_stride, stream));
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
    ix->slots.commit_compact(std::move(ext));
    return 0;
}

int svsb200_dynamic_flat_ids(const svsb200_dynamic_flat* index, uint64_t* out_ids, size_t* count) {
    const svsb200_index* ix = index_of(index);
    if (!ix) return fail("svsb200_dynamic_flat_ids: NULL index");
    return ix->slots.ids("svsb200_dynamic_flat_ids", out_ids, count);   // slot order (on_ids, dynamic_flat.h:182-189)
}

int svsb200_dynamic_flat_has_id(const svsb200_dynamic_flat* index, uint64_t id, int* out) {
    const svsb200_index* ix = index_of(index);
    if (!ix) return fail("svsb200_dynamic_flat_has_id: NULL index");
    return ix->slots.has_id("svsb200_dynamic_flat_has_id", id, out);
}

int svsb200_dynamic_flat_export(const svsb200_dynamic_flat* index, uint8_t* status_out, uint64_t* ext_ids_out) {
    const svsb200_index* ix = index_of(index);
    if (!ix) return fail("svsb200_dynamic_flat_export: NULL index");
    ix->slots.export_to(status_out, ext_ids_out);
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
