// shine_host_pool.cu — the batch-mode sample pool in pinned host memory, for maps of more scans than the device holds.
// Reference: dataset/lidar_dataset.py:94-101 moves the pools to CPU memory once a batch run uses more than
// `pc_count_gpu_limit` scans; get_batch (:431-448) then indexes on the CPU and copies each batch to the GPU.  Here the pool
// is a list of pinned host chunks the kernels read and write through unified addressing: a frame is packed into records
// by one launch, and a batch is gathered straight from host memory over PCIe by one launch (graph-capturable).
//
// Record: 32 bytes, 32-byte aligned, {x, y, z, label, weight, 0, 0, 0} fp32 — one sector, so a drawn sample costs one
// PCIe read request (read as two 16-byte loads of the same sector).  Record i lives in chunk i >> chunk_shift at offset
// (i & mask) * 32; chunks hold 2^chunk_shift records.
#include "shine_device.cuh"

namespace {

constexpr int kHostPoolThreads = 256;
constexpr int kHostPoolMinShift = 5;    // a chunk holds at least one warp's 32 records (1 KB)
constexpr int kHostPoolMaxShift = 31;   // 64 GB chunks

struct HostRecord {
    float4 lo;                          // x, y, z, label
    float4 hi;                          // weight, pad, pad, pad
};
static_assert(sizeof(HostRecord) == 32, "one record is one 32-byte sector");

__device__ __forceinline__ HostRecord* record_at(void* const* chunks, int shift, int64_t i) {
    const int64_t chunk = i >> shift;
    const int64_t offset = i & ((int64_t(1) << shift) - 1);
    return static_cast<HostRecord*>(chunks[chunk]) + offset;
}

// Thread t packs frame sample t into record at + t: a warp writes 32 consecutive records (1 KB; two when the run
// crosses a chunk boundary).
__global__ void __launch_bounds__(kHostPoolThreads)
host_pool_append_kernel(void* const* __restrict__ chunks, int shift, int64_t at, const float* __restrict__ coord,
                        const float* __restrict__ label, const float* __restrict__ weight, int64_t n) {
    for (int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; t < n; t += (int64_t)gridDim.x * blockDim.x) {
        HostRecord r;
        r.lo = make_float4(coord[3 * t], coord[3 * t + 1], coord[3 * t + 2], label[t]);
        r.hi = make_float4(weight[t], 0.f, 0.f, 0.f);
        HostRecord* dst = record_at(chunks, shift, at + t);
        dst->lo = r.lo;
        dst->hi = r.hi;
    }
}

// One thread per drawn sample: both 16-byte loads of its record are issued before either is used, so a warp has 64
// PCIe reads in flight.  An index outside [0, size) reads nothing and yields NaN coordinates with label and weight 0.
__global__ void __launch_bounds__(kHostPoolThreads)
host_pool_gather_kernel(void* const* __restrict__ chunks, int shift, int64_t size, const int64_t* __restrict__ index,
                        int64_t n, float* __restrict__ coord_out, float* __restrict__ label_out,
                        float* __restrict__ weight_out) {
    for (int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; t < n; t += (int64_t)gridDim.x * blockDim.x) {
        const int64_t i = index[t];
        float4 lo = make_float4(__int_as_float(0x7fc00000), __int_as_float(0x7fc00000), __int_as_float(0x7fc00000), 0.f);
        float4 hi = make_float4(0.f, 0.f, 0.f, 0.f);
        if (i >= 0 && i < size) {
            const HostRecord* src = record_at(chunks, shift, i);
            lo = src->lo;
            hi = src->hi;
        }
        coord_out[3 * t] = lo.x; coord_out[3 * t + 1] = lo.y; coord_out[3 * t + 2] = lo.z;
        label_out[t] = lo.w;
        weight_out[t] = hi.x;
    }
}

unsigned host_pool_blocks(int64_t n) {
    const int64_t blocks = (n + kHostPoolThreads - 1) / kHostPoolThreads;
    const int64_t cap = (int64_t)sm_count() * 64;          // grid-stride beyond this: still 8 resident blocks per SM
    return (unsigned)(blocks < cap ? blocks : cap);
}

bool on_device(const void* p, int dev) {
    cudaPointerAttributes at;
    if (cudaPointerGetAttributes(&at, p) != cudaSuccess) { (void)cudaGetLastError(); return false; }
    return (at.type == cudaMemoryTypeDevice || at.type == cudaMemoryTypeManaged) && at.device == dev;
}

int check_pool(const shine_host_pool* pool) {
    if (!pool || !pool->chunks) return SHINE_ERR_INVALID_ARG;
    if (pool->chunk_shift < kHostPoolMinShift || pool->chunk_shift > kHostPoolMaxShift) return SHINE_ERR_INVALID_ARG;
    if (pool->num_chunks < 0 || pool->size < 0) return SHINE_ERR_INVALID_ARG;
    if (pool->size > ((int64_t)pool->num_chunks << pool->chunk_shift)) return SHINE_ERR_INVALID_ARG;
    return SHINE_OK;
}

}  // namespace

extern "C" {

int shine_host_pool_append(const shine_host_pool* pool, int64_t at, const float* coord, const float* label,
                           const float* weight, int64_t n, void* stream) {
    const int rc = check_pool(pool);
    if (rc != SHINE_OK) return rc;
    if (at < 0 || n < 0 || at > ((int64_t)pool->num_chunks << pool->chunk_shift) - n) return SHINE_ERR_INVALID_ARG;
    if (n == 0) return SHINE_OK;
    if (!coord || !label || !weight) return SHINE_ERR_INVALID_ARG;
    const int dev = device_of(pool->chunks);
    if (dev < 0 || !on_device(coord, dev) || !on_device(label, dev) || !on_device(weight, dev))
        return SHINE_ERR_INVALID_ARG;
    DeviceGuard guard(pool->chunks);
    host_pool_append_kernel<<<host_pool_blocks(n), kHostPoolThreads, 0, (cudaStream_t)stream>>>(
        pool->chunks, pool->chunk_shift, at, coord, label, weight, n);
    return (int)cudaGetLastError();
}

int shine_host_pool_gather(const shine_host_pool* pool, const int64_t* index, int64_t n, float* coord_out,
                           float* label_out, float* weight_out, void* stream) {
    const int rc = check_pool(pool);
    if (rc != SHINE_OK) return rc;
    if (n < 0) return SHINE_ERR_INVALID_ARG;
    if (n == 0) return SHINE_OK;
    if (!index || !coord_out || !label_out || !weight_out) return SHINE_ERR_INVALID_ARG;
    const int dev = device_of(pool->chunks);
    if (dev < 0 || !on_device(index, dev) || !on_device(coord_out, dev) || !on_device(label_out, dev) ||
        !on_device(weight_out, dev))
        return SHINE_ERR_INVALID_ARG;
    DeviceGuard guard(pool->chunks);
    host_pool_gather_kernel<<<host_pool_blocks(n), kHostPoolThreads, 0, (cudaStream_t)stream>>>(
        pool->chunks, pool->chunk_shift, pool->size, index, n, coord_out, label_out, weight_out);
    return (int)cudaGetLastError();
}

}  // extern "C"
