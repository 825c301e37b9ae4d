// index.cu -- index life cycle of the C ABI (include/svsb200.h): library-wide state, index creation from host arrays
// or from the reference's files (streamed straight into HBM) on one or several GPUs, options, and the LVQ-8 encoder.
#include "host.cuh"

#include <algorithm>
#include <atomic>
#include <cmath>
#include <cstring>

#include <sys/stat.h>

namespace svsb200 {

static thread_local std::string g_error;
static std::atomic<uint64_t> g_launches{0};
void count_launch() { g_launches.fetch_add(1, std::memory_order_relaxed); }

int fail(const std::string& msg) {
    g_error = msg;
    return 1;
}

int check_device(const char* who, int device, cudaDeviceProp* prop) {
    const int ndev = svsb200_device_count();
    if (ndev == 0) return fail(std::string(who) + ": no CUDA device (there is no CPU fallback)");
    if (device < 0 || device >= ndev) return fail(std::string(who) + ": bad device ordinal");
    CUDA_TRY(cudaGetDeviceProperties(prop, device));
    if (prop->major != 9 || prop->minor != 0)
        return fail(std::string(who) + ": device is not sm_90 (this binary holds sm_90a code only)");
    return 0;
}

// ---------------------------------------------------------------------------------------
// Upload kernels
// ---------------------------------------------------------------------------------------

// Reference adjacency rows (degree first, core/graph/graph.h:103-114) -> HBM layout:
// neighbours first, kNoNeighbor padding, row length a multiple of 4 words so rows stay
// 16-byte aligned.  Repeated ids inside a row keep their first occurrence only: the
// reference's insert() rejects the later copy as a duplicate (search_buffer.h:380-391) or
// drops it off the end, so removing it up front cannot change any result.
__global__ void repack_graph_kernel(const uint32_t* __restrict__ src, size_t row_len, uint32_t n,
                                    uint32_t* __restrict__ dst, uint32_t gstride, uint16_t* __restrict__ ref_degree,
                                    int* __restrict__ bad) {
    const uint32_t row = blockIdx.x * (blockDim.x / 32) + threadIdx.x / 32;
    const int lane = threadIdx.x & 31;
    if (row >= n) return;
    const uint32_t* in = src + size_t(row) * row_len;
    uint32_t* out = dst + size_t(row) * gstride;
    const uint32_t deg = in[0];
    if (deg > row_len - 1) {
        if (lane == 0) atomicExch(bad, 1);
        return;
    }
    if (lane == 0) ref_degree[row] = uint16_t(deg);
    uint32_t written = 0;
    for (uint32_t j0 = 0; j0 < deg; j0 += 32) {
        const uint32_t j = j0 + lane;
        uint32_t id = j < deg ? in[1 + j] : kNoNeighbor;
        bool keep = j < deg;
        if (keep && id >= n) {
            atomicExch(bad, 2);
            keep = false;
        }
        if (keep) {
            for (uint32_t i = 0; i < j; ++i) {
                if (in[1 + i] == id) {
                    keep = false;
                    break;
                }
            }
        }
        const unsigned m = __ballot_sync(0xFFFFFFFFu, keep);
        if (keep) out[written + __popc(m & ((1u << lane) - 1u))] = id;
        written += __popc(m);
    }
    for (uint32_t j = written + lane; j < gstride; j += 32) out[j] = kNoNeighbor;
}

// LVQ-8 encoder (own specification, DESIGN.md §10), one warp per vector:
//   r_i = x_i - mean_i;  lower = min r, upper = max r;  delta = (upper - lower) / 255
//   {delta, lower} are stored as float16 (round to nearest even) and the codes are computed against
//   the *stored* constants:  c_i = clamp(rint((r_i - lower16) / delta16), 0, 255)   (0 when delta16 == 0)
// so that decode y_i = fma(delta16, c_i, lower16) is the nearest representable grid point.
// A row with a residual that is not finite, or whose delta16 or lower16 is not finite, would decode to NaN or -inf: its
// index is recorded in *bad_row (atomicMin, so the host sees the first such row) and the host refuses the data.
__global__ void lvq8_compress_kernel(const float* __restrict__ data, uint32_t n, uint32_t dim,
                                     const float* __restrict__ mean, uint8_t* __restrict__ rows, uint32_t stride,
                                     uint32_t const_offset, uint32_t* __restrict__ bad_row) {
    const uint32_t row = blockIdx.x * (blockDim.x / 32) + threadIdx.x / 32;
    const int lane = threadIdx.x & 31;
    if (row >= n) return;
    const float* x = data + size_t(row) * dim;
    uint8_t* out = rows + size_t(row) * stride;
    float lo = INFINITY, hi = -INFINITY;
    bool finite = true;
    for (uint32_t i = lane; i < dim; i += 32) {
        const float r = __fsub_rn(x[i], mean[i]);
        finite &= isfinite(r);
        lo = fminf(lo, r);
        hi = fmaxf(hi, r);
    }
    for (int o = 16; o; o >>= 1) {
        lo = fminf(lo, __shfl_xor_sync(0xFFFFFFFFu, lo, o));
        hi = fmaxf(hi, __shfl_xor_sync(0xFFFFFFFFu, hi, o));
    }
    const __half dh = __float2half_rn(__fdiv_rn(__fsub_rn(hi, lo), 255.0f));
    const __half lh = __float2half_rn(lo);
    const float d = __half2float(dh), l = __half2float(lh);
    if (!__all_sync(0xFFFFFFFFu, finite) || !isfinite(d) || !isfinite(l)) {
        if (lane == 0) atomicMin(bad_row, row);
        return;
    }
    for (uint32_t i = lane; i < stride; i += 32) {
        uint8_t c = 0;
        if (i < dim && d > 0.0f) {
            const float r = __fsub_rn(x[i], mean[i]);
            float q = rintf(__fdiv_rn(__fsub_rn(r, l), d));
            q = fminf(fmaxf(q, 0.0f), 255.0f);
            c = uint8_t(int(q));
        }
        if (i < const_offset || i >= const_offset + 4) out[i] = c;
    }
    if (lane == 0) {
        __half2 h = __halves2half2(dh, lh);
        *reinterpret_cast<__half2*>(out + const_offset) = h;
    }
}

// ---------------------------------------------------------------------------------------
// Index construction, shared by svsb200_index_create_multi and svsb200_index_assemble
// ---------------------------------------------------------------------------------------

// Checks the element type, metric, shape and device list (ordinals, repeats, sm_90) of a new index and makes it, with its
// layout and one empty replica per listed device.  Errors read "<who>: ...".
static int new_index(const char* who, int dtype, int metric, int storage, size_t n, size_t dim, size_t graph_row_len,
                     int64_t entry_point, const int* devices, size_t ndevices, std::unique_ptr<svsb200_index>* out) {
    const std::string w(who);
    if (!devices || ndevices == 0) return fail(w + ": empty device list");
    if (dtype < SVSB200_F32 || dtype > SVSB200_U8) return fail(w + ": bad dtype");
    if (metric < SVSB200_L2 || metric > SVSB200_COSINE) return fail(w + ": bad metric");
    if (n == 0 || dim == 0) return fail(w + ": empty dataset");
    if (n >= (size_t(1) << 31)) return fail(w + ": more than 2^31-1 vectors per index");
    if (graph_row_len < 2) return fail(w + ": graph rows need a degree word and one slot");
    if (graph_row_len > 65536) return fail(w + ": max_degree above 65535");
    if (entry_point < 0 || uint64_t(entry_point) >= n) return fail(w + ": entry point out of range");

    auto ix = std::make_unique<svsb200_index>();
    ix->dtype = dtype;
    ix->metric = metric;
    ix->storage = storage;
    ix->n = n;
    ix->dim = dim;
    ix->max_degree = graph_row_len - 1;
    ix->entry_point = uint32_t(entry_point);
    if (storage == SVSB200_LVQ8) ix->lvq_const_offset = uint32_t(round_up(dim, 4));
    ix->row_stride = data_row_stride(storage, dtype, dim);
    ix->gstride = graph_stride(ix->max_degree);
    for (size_t r = 0; r < ndevices; ++r) {
        cudaDeviceProp prop;
        if (int rc = check_device(who, devices[r], &prop)) return rc;
        for (size_t j = 0; j < r; ++j)
            if (devices[j] == devices[r]) return fail(w + ": device listed twice");
        ix->reps.push_back(std::make_unique<Replica>());
        ix->reps.back()->device = devices[r];
        ix->reps.back()->sm_count = prop.multiProcessorCount;
    }
    *out = std::move(ix);
    return 0;
}

// Copies an uploaded replica device to device (NVLink when peer access exists).
static int clone_replica(svsb200_index* ix, const Replica* src, Replica* dst) {
    const size_t n = ix->n;
    CUDA_TRY(cudaSetDevice(dst->device));
    const size_t vbytes = n * size_t(ix->row_stride);
    const size_t gbytes = n * size_t(ix->gstride) * sizeof(uint32_t);
    CUDA_TRY(dst->d_vectors.ensure(vbytes));
    CUDA_TRY(dst->d_graph.ensure(n * size_t(ix->gstride)));
    CUDA_TRY(dst->d_ref_degree.ensure(n));
    CUDA_TRY(cudaMemcpyPeer(dst->d_vectors.ptr, dst->device, src->d_vectors.ptr, src->device, vbytes));
    CUDA_TRY(cudaMemcpyPeer(dst->d_graph.ptr, dst->device, src->d_graph.ptr, src->device, gbytes));
    CUDA_TRY(cudaMemcpyPeer(dst->d_ref_degree.ptr, dst->device, src->d_ref_degree.ptr, src->device, n * sizeof(uint16_t)));
    if (src->d_mean.ptr) {
        CUDA_TRY(dst->d_mean.ensure(ix->dim));
        CUDA_TRY(cudaMemcpyPeer(dst->d_mean.ptr, dst->device, src->d_mean.ptr, src->device, ix->dim * sizeof(float)));
    }
    return 0;
}

// Fills the first replica, then copies it to the others.  `upload(rep, rows)` brings the data rows into rep->d_vectors
// (zeroed, row_stride apart) and the reference's adjacency rows (degree first, max_degree + 1 words) into the device
// staging block `rows`; those are then repacked into the HBM layout.
template <typename Upload> static int fill_replicas(const char* who, svsb200_index* ix, Upload upload) {
    const size_t n = ix->n, graph_row_len = ix->max_degree + 1;
    Replica* rep = ix->reps[0].get();
    CUDA_TRY(cudaSetDevice(rep->device));
    const size_t vbytes = n * size_t(ix->row_stride);
    CUDA_TRY(rep->d_vectors.ensure(vbytes));
    CUDA_TRY(rep->d_graph.ensure(n * size_t(ix->gstride)));
    CUDA_TRY(rep->d_ref_degree.ensure(n));
    ix->device_bytes = vbytes + n * size_t(ix->gstride) * sizeof(uint32_t) + n * sizeof(uint16_t);
    CUDA_TRY(cudaMemset(rep->d_vectors.ptr, 0, vbytes));
    {
        DeviceBuffer<uint32_t> rows;
        DeviceBuffer<int> d_bad;
        CUDA_TRY(rows.ensure(n * graph_row_len));
        CUDA_TRY(d_bad.ensure(1));
        CUDA_TRY(cudaMemset(d_bad.ptr, 0, sizeof(int)));
        if (int rc = upload(rep, rows.ptr)) return rc;
        const int warps = 8;
        repack_graph_kernel<<<unsigned((n + warps - 1) / warps), warps * 32>>>(rows.ptr, graph_row_len, uint32_t(n),
                                                                              rep->d_graph.ptr, ix->gstride,
                                                                              rep->d_ref_degree.ptr, d_bad.ptr);
        count_launch();
        CUDA_TRY(cudaGetLastError());
        int bad = 0;
        CUDA_TRY(cudaMemcpy(&bad, d_bad.ptr, sizeof(int), cudaMemcpyDeviceToHost));
        if (bad)
            return fail(std::string(who) + (bad == 1 ? ": adjacency row with degree > max_degree" : ": neighbour id out of range"));
    }
    for (size_t r = 1; r < ix->reps.size(); ++r)
        if (int rc = clone_replica(ix, rep, ix->reps[r].get())) return rc;
    return 0;
}

// -----------------------------------------------------------------------------------------------------------------
// Assembling an index from files, streamed straight into HBM (SURVEY.md 8 f3).  Replaces
// index::vamana::auto_assemble (index/vamana/index.h:1022-1050) + the native / vecs readers
// (core/io/native.h:315-345, core/io/vecs.h:137-273) + the TOML load of VamanaIndexParameters
// (index/vamana/index.h:53-178, lib/saveload/load.h:829-878).
// -----------------------------------------------------------------------------------------------------------------
namespace {

// A TOML subset sufficient for the reference's saved configurations: comments, [tables] with dotted names,
// [[arrays of tables]] (skipped), key = value with integers, floats, booleans, 'literal' / "basic" strings,
// dates as bare tokens.  Returns "table.key" -> raw value text (strings unquoted).
bool parse_toml_subset(const std::string& text, std::map<std::string, std::string>& out, std::string& err) {
    std::string table;
    bool skip = false;
    size_t line_no = 0, pos = 0;
    while (pos <= text.size()) {
        size_t eol = text.find('\n', pos);
        if (eol == std::string::npos) eol = text.size();
        std::string line = text.substr(pos, eol - pos);
        pos = eol + 1;
        ++line_no;
        // strip comments outside strings
        bool in_s = false, in_d = false;
        for (size_t i = 0; i < line.size(); ++i) {
            const char c = line[i];
            if (c == '\'' && !in_d) in_s = !in_s;
            else if (c == '"' && !in_s && (i == 0 || line[i - 1] != '\\')) in_d = !in_d;
            else if (c == '#' && !in_s && !in_d) {
                line.resize(i);
                break;
            }
        }
        auto trim = [](std::string& v) {
            const size_t b = v.find_first_not_of(" \t\r");
            if (b == std::string::npos) {
                v.clear();
                return;
            }
            v = v.substr(b, v.find_last_not_of(" \t\r") - b + 1);
        };
        trim(line);
        if (line.empty()) continue;
        if (line[0] == '[') {
            if (line.size() > 1 && line[1] == '[') {   // array of tables: not needed for index parameters
                skip = true;
                continue;
            }
            const size_t close = line.find(']');
            if (close == std::string::npos) {
                err = "line " + std::to_string(line_no) + ": unterminated table header";
                return false;
            }
            table = line.substr(1, close - 1);
            trim(table);
            skip = false;
            continue;
        }
        if (skip) continue;
        const size_t eq = line.find('=');
        if (eq == std::string::npos) {
            err = "line " + std::to_string(line_no) + ": expected key = value";
            return false;
        }
        std::string key = line.substr(0, eq), value = line.substr(eq + 1);
        trim(key);
        trim(value);
        if (key.size() >= 2 && (key.front() == '"' || key.front() == '\'')) key = key.substr(1, key.size() - 2);
        if (value.size() >= 2 && (value.front() == '\'' || value.front() == '"') && value.back() == value.front())
            value = value.substr(1, value.size() - 2);
        if (key.empty() || value.empty()) {
            err = "line " + std::to_string(line_no) + ": empty key or value";
            return false;
        }
        out[table.empty() ? key : table + "." + key] = value;
    }
    return true;
}

// Reads and parses a whole TOML file.
int read_toml(const std::string& path, std::map<std::string, std::string>& cfg) {
    FILE* f = fopen(path.c_str(), "rb");
    if (!f) return fail("cannot open " + path);
    std::string text;
    char buf[4096];
    size_t got;
    while ((got = fread(buf, 1, sizeof(buf), f)) > 0) text.append(buf, got);
    fclose(f);
    std::string err;
    if (!parse_toml_subset(text, cfg, err)) return fail(path + ": " + err);
    return 0;
}

struct RowFile {
    FILE* f = nullptr;
    size_t n = 0, dim = 0, esize = 0;
    size_t row_prefix = 0;     // bytes in front of every row (vecs formats: the int32 dimension)
    ~RowFile() {
        if (f) fclose(f);
    }
};

std::string resolve(const std::string& path, const char* inside) {
    struct stat st;
    if (stat(path.c_str(), &st) == 0 && S_ISDIR(st.st_mode)) return path + "/" + inside;
    return path;
}

// Opens a native v1 .svs container or a [fibh]vecs file; `esize` is the element size the caller expects.
int open_rows(const std::string& path, size_t esize, RowFile& rf) {
    rf.f = fopen(path.c_str(), "rb");
    if (!rf.f) return fail("cannot open " + path);
    rf.esize = esize;
    const size_t dot = path.rfind('.');
    const std::string ext = dot == std::string::npos ? "" : path.substr(dot);
    fseek(rf.f, 0, SEEK_END);
    const size_t bytes = size_t(ftell(rf.f));
    fseek(rf.f, 0, SEEK_SET);
    if (ext == ".fvecs" || ext == ".ivecs" || ext == ".bvecs" || ext == ".hvecs") {
        int32_t d = 0;
        if (fread(&d, 4, 1, rf.f) != 1 || d <= 0) return fail(path + ": empty or malformed vecs file");
        rf.dim = size_t(d);
        rf.row_prefix = 4;
        const size_t row = 4 + rf.dim * esize;
        if (bytes % row) return fail(path + ": size is not a multiple of the row size");
        rf.n = bytes / row;
        fseek(rf.f, 0, SEEK_SET);
        return 0;
    }
    unsigned char header[1024];
    if (fread(header, 1, 1024, rf.f) != 1024) return fail(path + ": truncated header");
    uint64_t magic, n, dims;
    memcpy(&magic, header, 8);
    memcpy(&n, header + 24, 8);
    memcpy(&dims, header + 32, 8);
    if (magic != 0xcad4a6b2579980feull) return fail(path + ": not a native v1 .svs file (bad magic)");
    if (bytes < 1024 + n * dims * esize) return fail(path + ": truncated body");
    rf.n = n;
    rf.dim = dims;
    return 0;
}

// Streams the rows of `rf` through two pinned staging buffers: while chunk i is copied host->device (asynchronously,
// strided into the padded HBM rows), chunk i+1 is read from the file.  Rows land at dst + row * dst_stride.
int stream_rows_to_device(RowFile& rf, char* dst, size_t dst_stride, cudaStream_t stream) {
    const size_t src_row = rf.row_prefix + rf.dim * rf.esize;
    const size_t chunk_rows = std::max<size_t>(1, (size_t(32) << 20) / src_row);
    struct Staging {   // released once every copy out of the buffers is done
        cudaStream_t stream;
        char* pinned[2] = {nullptr, nullptr};
        cudaEvent_t done[2] = {nullptr, nullptr};
        ~Staging() {
            cudaStreamSynchronize(stream);
            for (int i = 0; i < 2; ++i) {
                if (pinned[i]) cudaFreeHost(pinned[i]);
                if (done[i]) cudaEventDestroy(done[i]);
            }
        }
    } st{stream};
    for (int i = 0; i < 2; ++i) {
        if (cudaMallocHost(&st.pinned[i], chunk_rows * src_row) != cudaSuccess || cudaEventCreate(&st.done[i]) != cudaSuccess)
            return fail("pinned staging buffer allocation failed");
    }
    for (size_t r0 = 0, c = 0; r0 < rf.n; r0 += chunk_rows, ++c) {
        const int b = int(c & 1);
        const size_t rows = std::min(chunk_rows, rf.n - r0);
        if (c >= 2 && cudaEventSynchronize(st.done[b]) != cudaSuccess) return fail("cudaEventSynchronize failed");
        if (fread(st.pinned[b], src_row, rows, rf.f) != rows) return fail("short read");
        if (cudaMemcpy2DAsync(dst + r0 * dst_stride, dst_stride, st.pinned[b] + rf.row_prefix, src_row, rf.dim * rf.esize, rows,
                              cudaMemcpyHostToDevice, stream) != cudaSuccess)
            return fail("cudaMemcpy2DAsync failed");
        cudaEventRecord(st.done[b], stream);
    }
    if (cudaStreamSynchronize(stream) != cudaSuccess) return fail("stream synchronisation failed");
    return 0;
}

}  // namespace

}  // namespace svsb200

using namespace svsb200;

// =========================================================================================
// C ABI
// =========================================================================================
extern "C" {

const char* svsb200_last_error(void) { return g_error.c_str(); }
int svsb200_version(void) { return SVSB200_VERSION; }
uint64_t svsb200_launch_count(void) { return g_launches.load(); }

int svsb200_device_count(void) {
    int n = 0;
    if (cudaGetDeviceCount(&n) != cudaSuccess) {
        cudaGetLastError();
        return 0;
    }
    return n;
}

int svsb200_device_sm(int device, int* sm) {
    cudaDeviceProp prop;
    CUDA_TRY(cudaGetDeviceProperties(&prop, device));
    if (sm) *sm = prop.major * 10 + prop.minor;
    return 0;
}

int svsb200_index_create_multi(const void* vectors, int dtype, size_t n, size_t dim, size_t row_stride_bytes,
                               const uint32_t* graph_rows, size_t graph_row_len, uint32_t entry_point, int metric,
                               int storage, const float* aux, const int* devices, size_t ndevices, svsb200_index** out) {
    const char* who = "svsb200_index_create";
    if (!out) return fail("svsb200_index_create: out is NULL");
    *out = nullptr;
    if (!vectors || !graph_rows) return fail("svsb200_index_create: NULL input");
    if (storage == SVSB200_SQ) {
        if (dtype != SVSB200_I8 && dtype != SVSB200_U8) return fail("svsb200_index_create: SQ codes must be int8/uint8");
        if (!aux) return fail("svsb200_index_create: SQ needs aux = {scale, bias}");
    } else if (storage == SVSB200_LVQ8) {
        if (dtype != SVSB200_U8) return fail("svsb200_index_create: LVQ-8 rows are uint8 codes (dtype SVSB200_U8)");
        if (!aux) return fail("svsb200_index_create: LVQ-8 needs aux = mean[dim]");
        if (row_stride_bytes != svsb200_lvq8_row_stride(dim))
            return fail("svsb200_index_create: LVQ-8 rows must use svsb200_lvq8_row_stride(dim)");
    } else if (storage != SVSB200_PLAIN) {
        return fail("svsb200_index_create: unsupported storage kind");
    }
    std::unique_ptr<svsb200_index> ix;
    if (int rc = new_index(who, dtype, metric, storage, n, dim, graph_row_len, entry_point, devices, ndevices, &ix)) return rc;
    if (storage == SVSB200_SQ) {
        ix->scale = aux[0];
        ix->bias = aux[1];
    }
    const size_t row_bytes = storage == SVSB200_LVQ8 ? ix->lvq_const_offset + 4 : dim * esize(dtype);
    const size_t src_stride = row_stride_bytes ? row_stride_bytes : row_bytes;
    int rc = fill_replicas(who, ix.get(), [&](Replica* rep, uint32_t* rows) -> int {
        CUDA_TRY(cudaMemcpy2D(rep->d_vectors.ptr, ix->row_stride, vectors, src_stride, row_bytes, n, cudaMemcpyHostToDevice));
        CUDA_TRY(cudaMemcpy(rows, graph_rows, n * graph_row_len * sizeof(uint32_t), cudaMemcpyHostToDevice));
        if (storage == SVSB200_LVQ8) {
            CUDA_TRY(rep->d_mean.ensure(dim));
            CUDA_TRY(cudaMemcpy(rep->d_mean.ptr, aux, dim * sizeof(float), cudaMemcpyHostToDevice));
        }
        return 0;
    });
    if (rc) return rc;
    *out = ix.release();
    return 0;
}

int svsb200_index_create(const void* vectors, int dtype, size_t n, size_t dim, size_t row_stride_bytes,
                         const uint32_t* graph_rows, size_t graph_row_len, uint32_t entry_point, int metric, int storage,
                         const float* aux, int device, svsb200_index** out) {
    return svsb200_index_create_multi(vectors, dtype, n, dim, row_stride_bytes, graph_rows, graph_row_len, entry_point,
                                      metric, storage, aux, &device, 1, out);
}

int svsb200_toml_get(const char* path, const char* dotted_key, char* out, size_t capacity) {
    if (!path || !dotted_key || !out || capacity == 0) return fail("svsb200_toml_get: NULL argument");
    std::map<std::string, std::string> cfg;
    if (int rc = read_toml(path, cfg)) return rc;
    auto it = cfg.find(dotted_key);
    if (it == cfg.end()) return fail(std::string(path) + ": no key " + dotted_key);
    if (it->second.size() + 1 > capacity) return fail("svsb200_toml_get: value does not fit");
    memcpy(out, it->second.c_str(), it->second.size() + 1);
    return 0;
}

int svsb200_index_assemble(const char* config_path, const char* graph_path, const char* data_path, int dtype,
                           size_t expected_dims, int metric, const int* devices, size_t ndevices, svsb200_index** out) {
    const char* who = "svsb200_index_assemble";
    if (!out) return fail("svsb200_index_assemble: out is NULL");
    *out = nullptr;
    if (!config_path || !graph_path || !data_path) return fail("svsb200_index_assemble: NULL path");
    // ---- VamanaIndexParameters from TOML ----
    const std::string cfg_file = resolve(config_path, "svs_config.toml");
    std::map<std::string, std::string> cfg;
    if (int rc = read_toml(cfg_file, cfg)) return rc;
    auto cfg_long = [&](const char* key, long dflt) {
        auto it = cfg.find(key);
        if (it == cfg.end()) return dflt;
        if (it->second == "true") return 1l;
        if (it->second == "false") return 0l;
        return strtol(it->second.c_str(), nullptr, 10);
    };
    if (cfg.find("object.entry_point") == cfg.end()) return fail(cfg_file + ": no entry_point in [object]");
    // ---- files ----
    RowFile data, graph;
    if (int rc = open_rows(resolve(data_path, "data_0.svs"), esize(dtype), data)) return rc;
    if (int rc = open_rows(resolve(graph_path, "graph_0.svs"), 4, graph)) return rc;
    if (expected_dims && data.dim != expected_dims)
        return fail("svsb200_index_assemble: the data file holds " + std::to_string(data.dim) + "-dimensional vectors, " +
                    std::to_string(expected_dims) + " expected");
    if (graph.n != data.n) return fail("Wrong sizes!");   // index/vamana/index.h:417-419
    std::unique_ptr<svsb200_index> ix;
    if (int rc = new_index(who, dtype, metric, SVSB200_PLAIN, data.n, data.dim, graph.dim, cfg_long("object.entry_point", 0),
                           devices, ndevices, &ix))
        return rc;
    ix->cfg_window = cfg_long("object.search_parameters.search_window_size", 0);
    ix->cfg_capacity = cfg_long("object.search_parameters.search_buffer_capacity", 0);
    ix->cfg_visited = cfg_long("object.search_parameters.search_buffer_visited_set", 0);
    // both files are streamed on the default stream, like the host-array upload; the graph goes to the staging block
    int rc = fill_replicas(who, ix.get(), [&](Replica* rep, uint32_t* rows) -> int {
        if (int rc2 = stream_rows_to_device(data, reinterpret_cast<char*>(rep->d_vectors.ptr), ix->row_stride, nullptr))
            return rc2;
        return stream_rows_to_device(graph, reinterpret_cast<char*>(rows), graph.dim * sizeof(uint32_t), nullptr);
    });
    if (rc) return rc;
    *out = ix.release();
    return 0;
}

int svsb200_index_destroy(svsb200_index* ix) {
    delete ix;   // Replica / Scratch destructors release the device memory
    return 0;
}

size_t svsb200_index_size(const svsb200_index* ix) { return ix ? ix->n : 0; }
size_t svsb200_index_dimensions(const svsb200_index* ix) { return ix ? ix->dim : 0; }
size_t svsb200_index_max_degree(const svsb200_index* ix) { return ix ? ix->max_degree : 0; }
size_t svsb200_index_device_bytes(const svsb200_index* ix) { return ix ? ix->device_bytes : 0; }
int svsb200_index_device(const svsb200_index* ix) { return ix && !ix->reps.empty() ? ix->reps[0]->device : -1; }
size_t svsb200_index_num_devices(const svsb200_index* ix) { return ix ? ix->reps.size() : 0; }

int svsb200_set_counting(svsb200_index* ix, int enabled) {
    if (!ix) return fail("svsb200_set_counting: NULL index");
    ix->counting = enabled;
    return 0;
}

int svsb200_set_entry_points(svsb200_index* ix, const uint32_t* entry_points, size_t count) {
    if (!ix || !entry_points) return fail("svsb200_set_entry_points: NULL argument");
    if (count == 0 || count > 32) return fail("svsb200_set_entry_points: 1..32 entry points");
    // MutableVamanaIndex keeps exactly one entry point (dynamic_index.h:790-793)
    if (ix->dynamic) return fail("svsb200_set_entry_points: a dynamic index has a single entry point");
    for (size_t i = 0; i < count; ++i)
        if (entry_points[i] >= ix->n) return fail("svsb200_set_entry_points: entry point out of range");
    for (auto& rep : ix->reps) {
        CUDA_TRY(cudaSetDevice(rep->device));
        CUDA_TRY(cudaDeviceSynchronize());
        CUDA_TRY(rep->d_entry.ensure(32));
        CUDA_TRY(cudaMemcpy(rep->d_entry.ptr, entry_points, count * sizeof(uint32_t), cudaMemcpyHostToDevice));
    }
    ix->entry_point = entry_points[0];
    ix->n_entry = uint32_t(count);
    return 0;
}

int svsb200_set_id_offset(svsb200_index* ix, uint64_t offset) {
    if (!ix) return fail("svsb200_set_id_offset: NULL index");
    if (ix->dynamic) return fail("svsb200_set_id_offset: a dynamic index cannot be a shard");
    ix->id_offset = offset;
    return 0;
}

int svsb200_set_option(svsb200_index* ix, const char* name, long value) {
    if (!ix || !name) return fail("svsb200_set_option: NULL argument");
    const std::string key(name);
    if (key == "warps_per_cta") {
        if (value < 0 || value > 8) return fail("warps_per_cta must be in [0, 8]");
        ix->warps_per_cta = value;
    } else if (key == "ctas_per_sm") {
        if (value < 0 || value > 32) return fail("ctas_per_sm must be in [0, 32]");
        ix->ctas_per_sm = value;
    } else if (key == "rows_in_flight") {
        if (value < 0 || value > 2) return fail("rows_in_flight must be in [0, 2]");
        ix->rows_in_flight = value;
    } else if (key == "no_split") {
        ix->no_split = value;
    } else if (key == "filter_tag16") {
        ix->filter_tag16 = value;
    } else if (key == "generic_kernel") {
        ix->generic_kernel = value;
    } else if (key == "host_chunks") {
        if (value < 0 || value > 16) return fail("host_chunks must be in [0, 16]");
        ix->host_chunks = value;
    } else if (key == "visited_filter_slots") {
        // -1 = default; 0 = off; otherwise a power of two
        if (value > 0 && (value & (value - 1))) return fail("visited_filter_slots must be a power of two");
        // the filter words sit in front of 16-byte aligned arrays in shared memory
        if (value > 0 && value < 8) return fail("visited_filter_slots must be 0 (off) or at least 8");
        if (value > 16384) return fail("visited_filter_slots must be <= 16384");
        ix->filter_slots = value;
    } else if (key == "dynamic_slack") {
        // dynamic index: buffer entries held beyond the capacity for Deleted ones (-1 = default); results never change,
        // a query that needs more is re-run with more room
        if (value < -1 || value > (1 << 20)) return fail("dynamic_slack must be in [-1, 2^20]");
        ix->dyn_slack = value;
    } else {
        return fail("svsb200_set_option: unknown option " + key);
    }
    return 0;
}

int svsb200_get_option(svsb200_index* ix, const char* name, long* value) {
    if (!ix || !name || !value) return fail("svsb200_get_option: NULL argument");
    const std::string key(name);
    if (key == "last_kernel") {          // 1 = lean kernel, 0 = generic kernel
        std::lock_guard<std::mutex> lock(ix->mu);
        *value = ix->last ? ix->last->last_kernel : 0;
    } else if (key == "warps_per_cta") *value = ix->warps_per_cta;
    else if (key == "ctas_per_sm") *value = ix->ctas_per_sm;
    else if (key == "rows_in_flight") *value = ix->rows_in_flight;
    else if (key == "visited_filter_slots") *value = ix->filter_slots;
    else if (key == "generic_kernel") *value = ix->generic_kernel;
    else if (key == "host_chunks") *value = ix->host_chunks;
    else if (key == "config_search_window_size") *value = ix->cfg_window;
    else if (key == "config_search_buffer_capacity") *value = ix->cfg_capacity;
    else if (key == "config_search_buffer_visited_set") *value = ix->cfg_visited;
    else if (key == "entry_point") *value = long(ix->entry_point);
    else if (key == "dynamic_slack") *value = ix->dyn_slack;
    else if (key == "dynamic_reruns") *value = long(ix->dyn_reruns);
    else if (key == "streams") {         // scratch sets (= streams) created so far over all replicas
        long c = 0;
        for (auto& rep : ix->reps) {
            std::lock_guard<std::mutex> lock(rep->mu);
            c += long(rep->all.size());
        }
        *value = c;
    } else return fail("svsb200_get_option: unknown option " + key);
    return 0;
}

size_t svsb200_lvq8_row_stride(size_t dim) { return round_up(round_up(dim, 4) + 4, 32); }

int svsb200_lvq8_compress(const float* data, size_t n, size_t dim, const float* mean, void* out_rows, int device) {
    if (!data || !mean || !out_rows) return fail("svsb200_lvq8_compress: NULL argument");
    if (n == 0 || dim == 0 || n >= (size_t(1) << 31)) return fail("svsb200_lvq8_compress: bad shape");
    if (svsb200_device_count() == 0) return fail("svsb200_lvq8_compress: no CUDA device (there is no CPU fallback)");
    CUDA_TRY(cudaSetDevice(device));
    const size_t stride = svsb200_lvq8_row_stride(dim);
    DeviceBuffer<float> d_data, d_mean;
    DeviceBuffer<uint8_t> d_rows;
    DeviceBuffer<uint32_t> d_bad;
    CUDA_TRY(d_data.ensure(n * dim));
    CUDA_TRY(d_mean.ensure(dim));
    CUDA_TRY(d_rows.ensure(n * stride));
    CUDA_TRY(d_bad.ensure(1));
    CUDA_TRY(cudaMemcpy(d_data.ptr, data, n * dim * sizeof(float), cudaMemcpyHostToDevice));
    CUDA_TRY(cudaMemcpy(d_mean.ptr, mean, dim * sizeof(float), cudaMemcpyHostToDevice));
    CUDA_TRY(cudaMemset(d_bad.ptr, 0xFF, sizeof(uint32_t)));
    const int warps = 8;
    lvq8_compress_kernel<<<unsigned((n + warps - 1) / warps), warps * 32>>>(d_data.ptr, uint32_t(n), uint32_t(dim), d_mean.ptr,
                                                                          d_rows.ptr, uint32_t(stride),
                                                                          uint32_t(round_up(dim, 4)), d_bad.ptr);
    count_launch();
    CUDA_TRY(cudaGetLastError());
    uint32_t bad = 0;
    CUDA_TRY(cudaMemcpy(&bad, d_bad.ptr, sizeof(uint32_t), cudaMemcpyDeviceToHost));
    if (bad != 0xFFFFFFFFu)
        return fail("svsb200_lvq8_compress: row " + std::to_string(bad) +
                    " holds a value that is not finite, or a delta or lower bound that float16 cannot hold");
    CUDA_TRY(cudaMemcpy(out_rows, d_rows.ptr, n * stride, cudaMemcpyDeviceToHost));
    return 0;
}

}  // extern "C"
