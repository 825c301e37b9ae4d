// dynamic.cu -- the dynamic (mutable) Vamana index of the C ABI: MutableVamanaIndex
// (index/vamana/dynamic_index.h) assembled from a graph, data and external ids, with soft deletion.  Every slot has
// a status (Valid / Deleted / Empty) and an external id in HBM; the external -> slot translator
// (core/translation.h) lives on the host.  Searches go through svsb200_search* and run the lean kernel's
// MutableBuffer form (search_fast.cuh, MUT = true).
#include "host.cuh"

#include <algorithm>
#include <unordered_set>

namespace svsb200 {

// status[slots[i]] = value
__global__ void set_status_kernel(const uint32_t* __restrict__ slots, uint32_t count, uint8_t value, uint8_t* __restrict__ status) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < count) status[slots[i]] = value;
}

static int check_dynamic(const svsb200_index* ix, const char* who) {
    if (!ix) return fail(std::string(who) + ": NULL index");
    if (!ix->dynamic) return fail(std::string(who) + ": not a dynamic index (create it with svsb200_dynamic_create)");
    return 0;
}

}  // namespace svsb200

using namespace svsb200;

extern "C" {

int svsb200_dynamic_create(const void* vectors, int dtype, size_t n, size_t dim, const uint32_t* graph_rows,
                           size_t graph_row_len, uint32_t entry_point, int metric, const uint64_t* external_ids, int device,
                           svsb200_index** out) {
    if (!out) return fail("svsb200_dynamic_create: NULL output");
    *out = nullptr;
    if (n && !external_ids) return fail("svsb200_dynamic_create: NULL external ids");
    if (dtype != SVSB200_F32 && dtype != SVSB200_F16) return fail("svsb200_dynamic_create: float32 / float16 data only");
    if (graph_row_len < 2 || graph_row_len - 1 > 32u * kFastMaxGW)
        return fail("svsb200_dynamic_create: graph_max_degree must be in [1, 128]");
    if (n >= (size_t(1) << 30)) return fail("svsb200_dynamic_create: at most 2^30 - 1 slots");
    // IDTranslator::insert (core/translation.h:105-127)
    std::unordered_map<uint64_t, uint32_t> translator;
    translator.reserve(n);
    for (size_t i = 0; i < n; ++i)
        if (external_ids[i] == ~uint64_t(0))   // (marks the padding of short result rows)
            return fail("svsb200_dynamic_create: external id 2^64 - 1 is reserved");
        else if (!translator.emplace(external_ids[i], uint32_t(i)).second)
            return fail("svsb200_dynamic_create: External IDs contain repeat elements!");
    svsb200_index* ix = nullptr;
    if (int rc = svsb200_index_create(vectors, dtype, n, dim, 0, graph_rows, graph_row_len, entry_point, metric, SVSB200_PLAIN,
                                      nullptr, device, &ix))
        return rc;
    std::unique_ptr<svsb200_index, int (*)(svsb200_index*)> owner(ix, svsb200_index_destroy);
    ix->status.assign(n, SLOT_VALID);
    ix->ext_ids.assign(external_ids, external_ids + n);
    ix->translator = std::move(translator);
    Replica* rep = ix->reps[0].get();
    CUDA_TRY(cudaSetDevice(rep->device));
    CUDA_TRY(rep->d_status.ensure(std::max<size_t>(n, 1)));
    CUDA_TRY(rep->d_ext_ids.ensure(std::max<size_t>(n, 1)));
    CUDA_TRY(cudaMemcpy(rep->d_status.ptr, ix->status.data(), n, cudaMemcpyHostToDevice));
    CUDA_TRY(cudaMemcpy(rep->d_ext_ids.ptr, ix->ext_ids.data(), n * sizeof(uint64_t), cudaMemcpyHostToDevice));
    ix->device_bytes += n * (1 + sizeof(uint64_t));
    ix->dynamic = true;
    *out = owner.release();
    return 0;
}

int svsb200_dynamic_delete(svsb200_index* ix, const uint64_t* ids, size_t count) {
    if (int rc = check_dynamic(ix, "svsb200_dynamic_delete")) return rc;
    if (count && !ids) return fail("svsb200_dynamic_delete: NULL ids");
    // translator_.check_external_exist (core/translation.h:395-407): nothing changes unless every id is present
    std::vector<uint32_t> slots;
    slots.reserve(count);
    std::unordered_set<uint64_t> seen;
    for (size_t i = 0; i < count; ++i) {
        auto it = ix->translator.find(ids[i]);
        if (it == ix->translator.end() || !seen.insert(ids[i]).second)
            return fail("svsb200_dynamic_delete: External ID " + std::to_string(ids[i]) + " does not exist!");
        slots.push_back(it->second);
    }
    if (count == 0) return 0;
    Replica* rep = ix->reps[0].get();
    CUDA_TRY(cudaSetDevice(rep->device));
    std::string err;
    Scratch* sc = acquire(rep, &err);
    if (!sc) return fail(err);
    // (mutations must not run concurrently with searches of the same index; once this stream is drained the new status
    // is visible to every later search of it, whatever its stream)
    auto run = [&]() -> int {
        DeviceBuffer<uint32_t> d_slots;
        CUDA_TRY(d_slots.ensure(count));
        CUDA_TRY(cudaMemcpyAsync(d_slots.ptr, slots.data(), count * sizeof(uint32_t), cudaMemcpyHostToDevice, sc->stream));
        set_status_kernel<<<unsigned((count + 255) / 256), 256, 0, sc->stream>>>(d_slots.ptr, uint32_t(count), SLOT_DELETED,
                                                                                  rep->d_status.ptr);
        count_launch();
        CUDA_TRY(cudaGetLastError());
        CUDA_TRY(cudaStreamSynchronize(sc->stream));
        return 0;
    };
    const int rc = run();
    release(rep, sc);
    if (rc) return rc;
    // delete_entry + translator_.delete_external (dynamic_index.h:773-788)
    for (size_t i = 0; i < count; ++i) {
        ix->status[slots[i]] = SLOT_DELETED;
        ix->translator.erase(ids[i]);
    }
    return 0;
}

int svsb200_dynamic_ids(const svsb200_index* ix, uint64_t* out_ids, size_t* count) {
    if (int rc = check_dynamic(ix, "svsb200_dynamic_ids")) return rc;
    if (!count) return fail("svsb200_dynamic_ids: NULL count");
    if (out_ids) {
        if (*count < ix->translator.size()) return fail("svsb200_dynamic_ids: output too small");
        size_t o = 0;
        for (size_t s = 0; s < ix->status.size(); ++s)   // slot order
            if (ix->status[s] == SLOT_VALID) out_ids[o++] = ix->ext_ids[s];
    }
    *count = ix->translator.size();
    return 0;
}

int svsb200_dynamic_has_id(const svsb200_index* ix, uint64_t id, int* out) {
    if (int rc = check_dynamic(ix, "svsb200_dynamic_has_id")) return rc;
    if (!out) return fail("svsb200_dynamic_has_id: NULL output");
    *out = ix->translator.count(id) ? 1 : 0;
    return 0;
}

int svsb200_dynamic_export(const svsb200_index* ix, uint32_t* graph_rows_out, uint8_t* status_out, uint64_t* ext_ids_out,
                           uint32_t* entry_point_out) {
    if (int rc = check_dynamic(ix, "svsb200_dynamic_export")) return rc;
    const size_t n = ix->n, R = ix->max_degree;
    if (graph_rows_out) {
        const Replica* rep = ix->reps[0].get();
        CUDA_TRY(cudaSetDevice(rep->device));
        std::vector<uint32_t> rows(n * size_t(ix->gstride));
        CUDA_TRY(cudaMemcpy(rows.data(), rep->d_graph.ptr, rows.size() * sizeof(uint32_t), cudaMemcpyDeviceToHost));
        // neighbours-first device rows -> the reference's in-memory layout (degree first, core/graph/graph.h:103-114)
        for (size_t v = 0; v < n; ++v) {
            const uint32_t* in = rows.data() + v * ix->gstride;
            uint32_t* o = graph_rows_out + v * (R + 1);
            size_t d = 0;
            while (d < R && in[d] != kNoNeighbor) ++d;
            o[0] = uint32_t(d);
            for (size_t j = 0; j < R; ++j) o[1 + j] = j < d ? in[j] : 0u;
        }
    }
    if (status_out) std::copy(ix->status.begin(), ix->status.end(), status_out);
    if (ext_ids_out) std::copy(ix->ext_ids.begin(), ix->ext_ids.end(), ext_ids_out);
    if (entry_point_out) *entry_point_out = ix->entry_point;
    return 0;
}

}  // extern "C"
