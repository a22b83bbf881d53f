// shine_scan.cu — one LiDAR frame from the records of its file to training samples, on the GPU.
// Reference: dataset/lidar_dataset.py:115-218 (process_frame) with preprocess_kitti (:334-339), open3d's crop,
// voxel_down_sample, transform and scale, and utils/data_sampler.py:18-139 (dataSampler.sample).
//
//   shine_scan_filter_keys         z > min_z, range >= min_range, inclusive crop (fp64); per-axis bounds of the kept
//                                  points (integer atomics on an order-preserving image of the doubles); voxel keys
//   shine_scan_sort_voxels         stable radix sort of (key, input index); run heads, their exclusive scan, the count
//   shine_scan_average_transform   per voxel the fp64 sum of its points in input order / count; T·[p,1], / w, * scale,
//                                  rounded to fp32
//   shine_scan_sample              the sampler, operation for operation in fp32 without contraction
//
// The caller reads the voxel count back once (it sizes every later buffer); nothing else crosses to the host.
#include <cub/device/device_radix_sort.cuh>
#include <cub/device/device_scan.cuh>

#include "shine_device.cuh"

namespace {

constexpr int kScanThreads = 256;
constexpr int kAxisBits = 21;
constexpr unsigned long long kDropped = ~0ull;       // key of a point the filters drop: sorts behind every voxel
constexpr int64_t kAlign = 256;

// order-preserving unsigned image of a double: a < b (IEEE, not NaN) <=> img(a) < img(b)
__device__ __forceinline__ unsigned long long ordered_bits(double v) {
    const unsigned long long b = (unsigned long long)__double_as_longlong(v);
    return (b >> 63) ? ~b : (b | (1ull << 63));
}
__device__ __forceinline__ double from_ordered_bits(unsigned long long o) {
    return __longlong_as_double((long long)((o >> 63) ? (o & ~(1ull << 63)) : ~o));
}

struct ScanLayout {            // byte offsets into the caller's scratch, for n records
    int64_t bounds, keys_in, keys_out, idx_in, idx_out, pos, cub, total;
    size_t cub_bytes;
};

int64_t align_up(int64_t v) { return (v + kAlign - 1) / kAlign * kAlign; }

ScanLayout scan_layout(int64_t n) {
    ScanLayout l;
    const int m = (int)(n > 0 ? n : 1);
    size_t sort_bytes = 0, scan_bytes = 0;
    cub::DeviceRadixSort::SortPairs(nullptr, sort_bytes, (const unsigned long long*)nullptr, (unsigned long long*)nullptr,
                                    (const int*)nullptr, (int*)nullptr, m);
    cub::DeviceScan::ExclusiveSum(nullptr, scan_bytes, (int*)nullptr, (int*)nullptr, m);
    l.cub_bytes = sort_bytes > scan_bytes ? sort_bytes : scan_bytes;
    l.bounds = 0;                                     // 6 x u64: ordered min x y z, ordered max x y z
    l.keys_in = kAlign;
    l.keys_out = l.keys_in + align_up(8 * (int64_t)m);
    l.idx_in = l.keys_out + align_up(8 * (int64_t)m);
    l.idx_out = l.idx_in + align_up(4 * (int64_t)m);
    l.pos = l.idx_out + align_up(4 * (int64_t)m);
    l.cub = l.pos + align_up(4 * (int64_t)m);
    l.total = l.cub + align_up((int64_t)l.cub_bytes);
    return l;
}

template <typename T>
T* at(void* scratch, int64_t off) { return reinterpret_cast<T*>(static_cast<char*>(scratch) + off); }

unsigned scan_blocks(int64_t n) {
    int64_t b = (n + kScanThreads - 1) / kScanThreads;
    const int64_t cap = (int64_t)sm_count() * 8;
    if (b > cap) b = cap;
    return (unsigned)(b > 0 ? b : 1);
}

struct Records {
    const char* base;
    int64_t n;
    int32_t stride;
    int32_t fp64;
};

__device__ __forceinline__ void load_point(const Records& r, int64_t i, double& x, double& y, double& z) {
    const char* p = r.base + i * (int64_t)r.stride;
    if (r.fp64) {
        const double* d = reinterpret_cast<const double*>(p);
        x = d[0]; y = d[1]; z = d[2];
    } else {
        const float* f = reinterpret_cast<const float*>(p);
        x = (double)f[0]; y = (double)f[1]; z = (double)f[2];
    }
}

struct FilterParams {
    double min_z, max_z, min_range, radius, voxel;
};

// preprocess_kitti (`z > z_th`, then `np.linalg.norm(points, axis=1) >= min_range`: ((x*x + y*y) + z*z), sqrt) and the
// inclusive crop of AxisAlignedBoundingBox([-r, -r, min_z], [r, r, max_z]).  NaN fails every comparison; inf fails the crop.
__device__ __forceinline__ bool kept(double x, double y, double z, const FilterParams& f) {
    if (!(z > f.min_z)) return false;
    const double r2 = __dadd_rn(__dadd_rn(__dmul_rn(x, x), __dmul_rn(y, y)), __dmul_rn(z, z));
    if (!(__dsqrt_rn(r2) >= f.min_range)) return false;
    return x >= -f.radius && x <= f.radius && y >= -f.radius && y <= f.radius && z >= f.min_z && z <= f.max_z;
}

__global__ void __launch_bounds__(kScanThreads) scan_bounds_kernel(const Records r, const FilterParams f,
                                                                   unsigned long long* bounds) {
    unsigned long long lo[3] = {kDropped, kDropped, kDropped}, hi[3] = {0ull, 0ull, 0ull};
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < r.n; i += (int64_t)gridDim.x * blockDim.x) {
        double p[3];
        load_point(r, i, p[0], p[1], p[2]);
        if (!kept(p[0], p[1], p[2], f)) continue;
#pragma unroll
        for (int a = 0; a < 3; ++a) {
            const unsigned long long o = ordered_bits(p[a]);
            lo[a] = o < lo[a] ? o : lo[a];
            hi[a] = o > hi[a] ? o : hi[a];
        }
    }
#pragma unroll
    for (int a = 0; a < 3; ++a) {
#pragma unroll
        for (int s = 16; s > 0; s >>= 1) {
            const unsigned long long l = __shfl_xor_sync(kFull, lo[a], s), h = __shfl_xor_sync(kFull, hi[a], s);
            lo[a] = l < lo[a] ? l : lo[a];
            hi[a] = h > hi[a] ? h : hi[a];
        }
    }
    if ((threadIdx.x & 31) == 0 && lo[0] != kDropped) {
#pragma unroll
        for (int a = 0; a < 3; ++a) {
            atomicMin(bounds + a, lo[a]);
            atomicMax(bounds + 3 + a, hi[a]);
        }
    }
}

// open3d VoxelDownSample: voxel_min_bound = min_bound - v/2, index floor((p - voxel_min_bound) / v) per axis
__global__ void __launch_bounds__(kScanThreads) scan_keys_kernel(const Records r, const FilterParams f,
                                                                 const unsigned long long* bounds,
                                                                 unsigned long long* keys, int* idx) {
    const double half = f.voxel * 0.5;
    double vmin[3];
#pragma unroll
    for (int a = 0; a < 3; ++a) vmin[a] = __dsub_rn(from_ordered_bits(bounds[a]), half);
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < r.n; i += (int64_t)gridDim.x * blockDim.x) {
        double p[3];
        load_point(r, i, p[0], p[1], p[2]);
        unsigned long long key = kDropped;
        if (kept(p[0], p[1], p[2], f)) {
            key = 0ull;
#pragma unroll
            for (int a = 0; a < 3; ++a)
                key = (key << kAxisBits) | (unsigned long long)(long long)floor(__ddiv_rn(__dsub_rn(p[a], vmin[a]), f.voxel));
        }
        keys[i] = key;
        idx[i] = (int)i;
    }
}

__device__ __forceinline__ bool run_head(const unsigned long long* keys, int64_t i) {
    return keys[i] != kDropped && (i == 0 || keys[i] != keys[i - 1]);
}

__global__ void __launch_bounds__(kScanThreads) scan_heads_kernel(const unsigned long long* keys, int64_t n, int* head) {
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x)
        head[i] = run_head(keys, i) ? 1 : 0;
}

__global__ void scan_count_kernel(const unsigned long long* keys, const int* pos, int64_t n, int64_t* count) {
    *count = (int64_t)pos[n - 1] + (run_head(keys, n - 1) ? 1 : 0);
}

struct TransformParams {
    double m[16];          // row-major 4x4
    double scale;
};

// One thread per run head: sum the run's points in input order (the sort is stable), divide by the count, then
// open3d's TransformPoints (T·[p,1] per row as ((m0*x + m1*y) + m2*z) + m3, / w), ScalePoints about the origin
// ((p - 0)*s + 0) and the fp32 rounding of torch.tensor(np.asarray(points), dtype=float32).
__global__ void __launch_bounds__(kScanThreads) scan_average_kernel(const Records r, const unsigned long long* keys,
                                                                    const int* idx, const int* pos,
                                                                    const TransformParams t, double* voxels,
                                                                    float* points) {
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < r.n; i += (int64_t)gridDim.x * blockDim.x) {
        if (!run_head(keys, i)) continue;
        const unsigned long long key = keys[i];
        double s[3] = {0.0, 0.0, 0.0};
        int64_t j = i;
        for (; j < r.n && keys[j] == key; ++j) {
            double x, y, z;
            load_point(r, idx[j], x, y, z);
            s[0] = __dadd_rn(s[0], x); s[1] = __dadd_rn(s[1], y); s[2] = __dadd_rn(s[2], z);
        }
        const double c = (double)(j - i);
        double p[3];
#pragma unroll
        for (int a = 0; a < 3; ++a) p[a] = __ddiv_rn(s[a], c);
        const int64_t o = pos[i];
        if (voxels) { voxels[3 * o] = p[0]; voxels[3 * o + 1] = p[1]; voxels[3 * o + 2] = p[2]; }
        double q[4];
#pragma unroll
        for (int row = 0; row < 4; ++row) {
            const double* m = t.m + 4 * row;
            q[row] = __dadd_rn(__dadd_rn(__dadd_rn(__dmul_rn(m[0], p[0]), __dmul_rn(m[1], p[1])), __dmul_rn(m[2], p[2])), m[3]);
        }
#pragma unroll
        for (int a = 0; a < 3; ++a)
            points[3 * o + a] = __double2float_rn(__dadd_rn(__dmul_rn(__dsub_rn(__ddiv_rn(q[a], q[3]), 0.0), t.scale), 0.0));
    }
}

struct SampleParams {
    const float* points;
    const float* u_surface;    // [ns * R], sample-major
    const float* u_free;       // [nf * R]
    float* coord;
    float* label;
    float* weight;
    int64_t rays;
    int32_t ns, nf;
    float ox, oy, oz, range, free_end, free_begin;
};

__global__ void __launch_bounds__(kScanThreads) scan_sample_kernel(const SampleParams a) {
    const int per_ray = a.ns + a.nf;
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < a.rays; i += (int64_t)gridDim.x * blockDim.x) {
        const float sx = __fsub_rn(a.points[3 * i], a.ox), sy = __fsub_rn(a.points[3 * i + 1], a.oy),
                    sz = __fsub_rn(a.points[3 * i + 2], a.oz);
        const float dist = __fsqrt_rn(__fadd_rn(__fadd_rn(__fmul_rn(sx, sx), __fmul_rn(sy, sy)), __fmul_rn(sz, sz)));
        // free_max_ratio = end / dist + 1: torch's scalar / tensor is reciprocal() * scalar
        const float free_max = __fadd_rn(__fmul_rn(__frcp_rn(dist), a.free_end), 1.0f);
        const float free_diff = __fsub_rn(free_max, a.free_begin);
        for (int s = 0; s < per_ray; ++s) {
            float disp, ratio;
            if (s < a.ns) {
                const float u = a.u_surface[(int64_t)s * a.rays + i];
                disp = __fmul_rn(__fmul_rn(__fsub_rn(u, 0.5f), 2.0f), a.range);
                ratio = __fadd_rn(__fdiv_rn(disp, dist), 1.0f);
            } else {
                const float u = a.u_free[(int64_t)(s - a.ns) * a.rays + i];
                ratio = __fadd_rn(__fmul_rn(u, free_diff), a.free_begin);
                disp = __fmul_rn(__fsub_rn(ratio, 1.0f), dist);
            }
            const int64_t o = i * per_ray + s;
            a.coord[3 * o] = __fadd_rn(__fmul_rn(sx, ratio), a.ox);
            a.coord[3 * o + 1] = __fadd_rn(__fmul_rn(sy, ratio), a.oy);
            a.coord[3 * o + 2] = __fadd_rn(__fmul_rn(sz, ratio), a.oz);
            a.label[o] = disp;
            a.weight[o] = s < a.ns ? 1.0f : -1.0f;
        }
    }
}

int check_input(const shine_scan_input* in) {
    if (!in || in->n < 0) return SHINE_ERR_INVALID_ARG;
    if (in->n > 0x7fffffffLL) return SHINE_ERR_UNSUPPORTED;     // CUB sorts int-counted sequences
    const int need = in->fp64 ? 24 : 12;
    if ((in->fp64 != 0 && in->fp64 != 1) || in->stride_bytes < need || in->stride_bytes % (in->fp64 ? 8 : 4))
        return SHINE_ERR_INVALID_ARG;
    if (in->n > 0 && (!in->records || ((uintptr_t)in->records % (in->fp64 ? 8 : 4)))) return SHINE_ERR_INVALID_ARG;
    return SHINE_OK;
}

int check_scratch(const void* scratch, int64_t scratch_bytes, int64_t n) {
    if (!scratch || ((uintptr_t)scratch % kAlign) || scratch_bytes < scan_layout(n).total) return SHINE_ERR_INVALID_ARG;
    return SHINE_OK;
}

Records records_of(const shine_scan_input* in) {
    Records r;
    r.base = static_cast<const char*>(in->records);
    r.n = in->n; r.stride = in->stride_bytes; r.fp64 = in->fp64;
    return r;
}

}  // namespace

extern "C" {

int64_t shine_scan_scratch_bytes(int64_t n) {
    if (n < 0) return SHINE_ERR_INVALID_ARG;
    if (n > 0x7fffffffLL) return SHINE_ERR_UNSUPPORTED;
    return scan_layout(n).total;
}

int shine_scan_filter_keys(const shine_scan_input* in, double min_z, double max_z, double min_range, double pc_radius,
                           double voxel, void* scratch, int64_t scratch_bytes, void* stream) {
    int rc = check_input(in);
    if (rc) return rc;
    if (check_scratch(scratch, scratch_bytes, in->n)) return SHINE_ERR_INVALID_ARG;
    if (!(voxel > 0.0) || !isfinite(voxel) || !isfinite(min_z) || !isfinite(max_z) || !isfinite(pc_radius) ||
        !(min_range == min_range))
        return SHINE_ERR_INVALID_ARG;
    // every kept point lies in the crop box, so its voxel index on an axis is at most extent / v + 1
    const double limit = (double)(1 << kAxisBits) - 2.0;
    if (2.0 * pc_radius / voxel >= limit || (max_z - min_z) / voxel >= limit) return SHINE_ERR_INVALID_ARG;
    DeviceGuard guard(scratch);
    cudaStream_t st = (cudaStream_t)stream;
    const ScanLayout l = scan_layout(in->n);
    cudaError_t e = cudaMemsetAsync(scratch, 0xff, 24, st);                       // ordered minima
    if (e == cudaSuccess) e = cudaMemsetAsync(at<char>(scratch, 24), 0, 24, st);  // ordered maxima
    if (e != cudaSuccess || in->n == 0) return (int)e;
    const Records r = records_of(in);
    FilterParams f;
    f.min_z = min_z; f.max_z = max_z; f.min_range = min_range; f.radius = pc_radius; f.voxel = voxel;
    unsigned long long* bounds = at<unsigned long long>(scratch, l.bounds);
    const unsigned blocks = scan_blocks(in->n);
    scan_bounds_kernel<<<blocks, kScanThreads, 0, st>>>(r, f, bounds);
    scan_keys_kernel<<<blocks, kScanThreads, 0, st>>>(r, f, bounds, at<unsigned long long>(scratch, l.keys_in),
                                                      at<int>(scratch, l.idx_in));
    return (int)cudaGetLastError();
}

int shine_scan_sort_voxels(int64_t n, int64_t* voxel_count, void* scratch, int64_t scratch_bytes, void* stream) {
    if (n < 0 || !voxel_count) return SHINE_ERR_INVALID_ARG;
    if (n > 0x7fffffffLL) return SHINE_ERR_UNSUPPORTED;
    if (check_scratch(scratch, scratch_bytes, n)) return SHINE_ERR_INVALID_ARG;
    DeviceGuard guard(scratch);
    cudaStream_t st = (cudaStream_t)stream;
    if (n == 0) return (int)cudaMemsetAsync(voxel_count, 0, sizeof(int64_t), st);
    const ScanLayout l = scan_layout(n);
    size_t bytes = l.cub_bytes;
    unsigned long long* keys = at<unsigned long long>(scratch, l.keys_out);
    int* pos = at<int>(scratch, l.pos);
    cudaError_t e = cub::DeviceRadixSort::SortPairs(at<void>(scratch, l.cub), bytes,
                                                    at<const unsigned long long>(scratch, l.keys_in), keys,
                                                    at<const int>(scratch, l.idx_in), at<int>(scratch, l.idx_out),
                                                    (int)n, 0, 64, st);
    if (e != cudaSuccess) return (int)e;
    scan_heads_kernel<<<scan_blocks(n), kScanThreads, 0, st>>>(keys, n, pos);
    bytes = l.cub_bytes;
    e = cub::DeviceScan::ExclusiveSum(at<void>(scratch, l.cub), bytes, pos, pos, (int)n, st);
    if (e != cudaSuccess) return (int)e;
    scan_count_kernel<<<1, 1, 0, st>>>(keys, pos, n, voxel_count);
    return (int)cudaGetLastError();
}

int shine_scan_average_transform(const shine_scan_input* in, const double* pose, double scale, int64_t n_voxels,
                                 double* voxels_out, float* points_out, void* scratch, int64_t scratch_bytes,
                                 void* stream) {
    int rc = check_input(in);
    if (rc) return rc;
    if (!pose || n_voxels < 0 || n_voxels > in->n || (n_voxels > 0 && !points_out)) return SHINE_ERR_INVALID_ARG;
    if (check_scratch(scratch, scratch_bytes, in->n)) return SHINE_ERR_INVALID_ARG;
    if (n_voxels == 0) return SHINE_OK;
    DeviceGuard guard(scratch);
    const ScanLayout l = scan_layout(in->n);
    TransformParams t;
    for (int k = 0; k < 16; ++k) t.m[k] = pose[k];
    t.scale = scale;
    scan_average_kernel<<<scan_blocks(in->n), kScanThreads, 0, (cudaStream_t)stream>>>(
        records_of(in), at<const unsigned long long>(scratch, l.keys_out), at<const int>(scratch, l.idx_out),
        at<const int>(scratch, l.pos), t, voxels_out, points_out);
    return (int)cudaGetLastError();
}

int shine_scan_sample(const float* points, int64_t n_rays, float ox, float oy, float oz, const float* u_surface,
                      int32_t surface_n, const float* u_free, int32_t free_n, float surface_range, float free_end,
                      float free_begin_ratio, float* coord, float* label, float* weight, void* stream) {
    if (n_rays < 0 || surface_n < 0 || free_n < 0) return SHINE_ERR_INVALID_ARG;
    if (n_rays == 0 || surface_n + free_n == 0) return SHINE_OK;
    if (!points || !coord || !label || !weight || (surface_n && !u_surface) || (free_n && !u_free))
        return SHINE_ERR_INVALID_ARG;
    DeviceGuard guard(coord);
    SampleParams a;
    a.points = points; a.u_surface = u_surface; a.u_free = u_free;
    a.coord = coord; a.label = label; a.weight = weight;
    a.rays = n_rays; a.ns = surface_n; a.nf = free_n;
    a.ox = ox; a.oy = oy; a.oz = oz; a.range = surface_range; a.free_end = free_end; a.free_begin = free_begin_ratio;
    scan_sample_kernel<<<scan_blocks(n_rays), kScanThreads, 0, (cudaStream_t)stream>>>(a);
    return (int)cudaGetLastError();
}

}  // extern "C"
