// slots.cu -- the device side of the dynamic indexes' slots (dynamic.cu, dynamic_flat.cu, dynamic_ivf.cu): the
// statuses and external ids in Replica::d_status / d_ext_ids, and the moves of rows between slots or pool positions.
// The host side and the slot rules are slots.h.
#include "host.cuh"

namespace svsb200 {

// status[slots[i]] = value and, with `ids`, ext_ids[slots[i]] = ids[i]
__global__ void mark_slots_kernel(const uint32_t* __restrict__ slots, const uint64_t* __restrict__ ids, uint32_t count,
                                  uint8_t value, uint8_t* __restrict__ status, uint64_t* __restrict__ ext_ids) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= count) return;
    status[slots[i]] = value;
    if (ids) ext_ids[slots[i]] = ids[i];
}

// Row dst_pos[i] of `dst` <- row src_pos[i] of `src` (an index array NULL: i; src NULL: no row moves), and with
// `entries`, entry dst_pos[i] <- vals[i] (vals NULL: all-ones); rows of `words` 16-byte words, one warp per row.  (src
// and dst may be one pool: a dynamic IVF cluster moving to the pool's tail.)
__global__ void move_rows_kernel(const uint4* src, const uint32_t* __restrict__ src_pos, uint4* dst,
                                 const uint32_t* __restrict__ dst_pos, const uint32_t* __restrict__ vals,
                                 uint32_t* __restrict__ entries, uint32_t count, uint32_t words) {
    const uint32_t i = blockIdx.x * (blockDim.x / 32) + threadIdx.x / 32;
    const uint32_t lane = threadIdx.x & 31;
    if (i >= count) return;
    const size_t d = dst_pos ? dst_pos[i] : i;
    if (src) {
        const size_t s = src_pos ? src_pos[i] : i;
        for (uint32_t j = lane; j < words; j += 32) dst[d * words + j] = src[s * words + j];
    }
    if (entries && lane == 0) entries[d] = vals ? vals[i] : 0xFFFFFFFFu;
}

int upload_slots(Replica* rep, const SlotTable& t) {
    const size_t n = t.num_slots(), cap = std::max<size_t>(n, 1);
    CUDA_TRY(rep->d_status.ensure(cap));
    CUDA_TRY(rep->d_ext_ids.ensure(cap));
    CUDA_TRY(cudaMemset(rep->d_status.ptr, SLOT_EMPTY, cap));
    if (n) {
        CUDA_TRY(cudaMemcpy(rep->d_status.ptr, t.status.data(), n, cudaMemcpyHostToDevice));
        CUDA_TRY(cudaMemcpy(rep->d_ext_ids.ptr, t.ext_ids.data(), n * sizeof(uint64_t), cudaMemcpyHostToDevice));
    }
    return 0;
}

int grow_slots(Replica* rep, size_t used, size_t cap, cudaStream_t stream) {
    CUDA_TRY(cudaStreamSynchronize(stream));
    CUDA_TRY(grow(rep->d_ext_ids, used, cap));
    CUDA_TRY(grow(rep->d_status, used, cap));
    CUDA_TRY(cudaMemsetAsync(rep->d_status.ptr + used, SLOT_EMPTY, cap - used, stream));
    return 0;
}

int compacted_slots(const std::vector<uint64_t>& ext, size_t cap, DeviceBuffer<uint8_t>* status,
                    DeviceBuffer<uint64_t>* ext_ids, cudaStream_t stream) {
    const size_t m = ext.size();
    CUDA_TRY(status->ensure(cap));
    CUDA_TRY(ext_ids->ensure(cap));
    CUDA_TRY(cudaMemsetAsync(status->ptr, SLOT_EMPTY, cap, stream));
    CUDA_TRY(cudaMemsetAsync(status->ptr, SLOT_VALID, m, stream));
    if (m) CUDA_TRY(cudaMemcpyAsync(ext_ids->ptr, ext.data(), m * sizeof(uint64_t), cudaMemcpyHostToDevice, stream));
    return 0;
}

cudaError_t mark_slots(const uint32_t* d_slots, const uint64_t* d_ids, size_t count, uint8_t value, Replica* rep,
                       cudaStream_t stream) {
    if (count == 0) return cudaSuccess;
    mark_slots_kernel<<<unsigned((count + 255) / 256), 256, 0, stream>>>(d_slots, d_ids, uint32_t(count), value,
                                                                          rep->d_status.ptr, rep->d_ext_ids.ptr);
    count_launch();
    return cudaGetLastError();
}

cudaError_t move_rows(const void* src, const uint32_t* src_pos, void* dst, const uint32_t* dst_pos, const uint32_t* vals,
                      uint32_t* entries, size_t count, uint32_t row_stride, cudaStream_t stream) {
    if (count == 0) return cudaSuccess;
    move_rows_kernel<<<unsigned((count + 7) / 8), 256, 0, stream>>>(static_cast<const uint4*>(src), src_pos,
                                                                     static_cast<uint4*>(dst), dst_pos, vals, entries,
                                                                     uint32_t(count), row_stride / 16);
    count_launch();
    return cudaGetLastError();
}

}  // namespace svsb200
