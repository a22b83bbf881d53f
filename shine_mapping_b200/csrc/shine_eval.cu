// shine_eval.cu — mesh evaluation (reference eval/eval_utils.py eval_mesh, crop_intersection): uniform sampling of a
// triangle mesh and exact nearest neighbours within a radius.
//
//   shine_mesh_sample_areas    per-triangle crop test and fp64 area, then a deterministic chunked fp64 inclusive scan of
//                              the areas (the CDF ends); the total area goes to a device double (the caller's one read)
//   shine_mesh_sample_points   one thread per sample: binary search of its triangle over round(C_t N), a Philox4x32-10
//                              draw keyed by (seed, sample index), the barycentric point in fp64 without contraction
//   shine_nn_build             Morton-sorted reference points in leaf buckets of kNnBucket, an implicit complete binary tree
//                              of fp32 boxes rounded outward over the buckets
//   shine_nn_query             queries in Morton order; depth-first traversal pruned by min(best, r)^2, exact fp64 at leaves
#include <cub/device/device_radix_sort.cuh>

#include "shine_device.cuh"

namespace {

constexpr int kThreads = 256;
constexpr int kScanChunk = 256;     // triangles summed sequentially by one thread of the area scan
constexpr int kNnBucket = 8;        // reference points per leaf
constexpr int kNnStack = 32;        // >= tree depth + 1 (depth <= 28 for 2^31 points)
constexpr int kMortonBits = 21;
constexpr int64_t kAlign = 256;

int64_t align_up(int64_t v) { return (v + kAlign - 1) / kAlign * kAlign; }

template <typename T>
T* at(void* base, int64_t off) { return reinterpret_cast<T*>(static_cast<char*>(base) + off); }
template <typename T>
const T* at(const void* base, int64_t off) { return reinterpret_cast<const T*>(static_cast<const char*>(base) + off); }

unsigned blocks_for(int64_t n) {
    int64_t b = (n + kThreads - 1) / kThreads;
    const int64_t cap = (int64_t)sm_count() * 16;
    if (b > cap) b = cap;
    return (unsigned)(b > 0 ? b : 1);
}

// ---- sampling ------------------------------------------------------------------------------------------------------

struct SampleLayout {          // byte offsets into the sampling scratch, for nt triangles
    int64_t cum, chunk, total;
};

SampleLayout sample_layout(int64_t nt) {
    const int64_t m = nt > 0 ? nt : 1;
    SampleLayout l;
    l.cum = 0;
    l.chunk = align_up(8 * m);
    l.total = l.chunk + align_up(8 * ((m + kScanChunk - 1) / kScanChunk));
    return l;
}

__device__ __forceinline__ void load_vertex(const double* v, int i, double (&p)[3]) {
    p[0] = v[3 * (int64_t)i]; p[1] = v[3 * (int64_t)i + 1]; p[2] = v[3 * (int64_t)i + 2];
}

__device__ __forceinline__ bool in_box(const double (&p)[3], const double* box) {
    return p[0] >= box[0] && p[0] <= box[3] && p[1] >= box[1] && p[1] <= box[4] && p[2] >= box[2] && p[2] <= box[5];
}

// Open3D GetTriangleArea: 0.5 * |(p0 - p1) x (p0 - p2)|, the norm as sqrt((x*x + y*y) + z*z).  A triangle with a vertex
// outside the crop box (TriangleMesh::Crop keeps a triangle iff its three vertices are inside, bounds inclusive) has area 0.
__device__ double triangle_area(const double* verts, const int32_t* tri, const double* crop) {
    double p0[3], p1[3], p2[3];
    load_vertex(verts, tri[0], p0); load_vertex(verts, tri[1], p1); load_vertex(verts, tri[2], p2);
    if (crop && !(in_box(p0, crop) && in_box(p1, crop) && in_box(p2, crop))) return 0.0;
    double a[3], b[3];
#pragma unroll
    for (int k = 0; k < 3; ++k) { a[k] = __dsub_rn(p0[k], p1[k]); b[k] = __dsub_rn(p0[k], p2[k]); }
    const double cx = __dsub_rn(__dmul_rn(a[1], b[2]), __dmul_rn(a[2], b[1]));
    const double cy = __dsub_rn(__dmul_rn(a[2], b[0]), __dmul_rn(a[0], b[2]));
    const double cz = __dsub_rn(__dmul_rn(a[0], b[1]), __dmul_rn(a[1], b[0]));
    return __dmul_rn(0.5, __dsqrt_rn(__dadd_rn(__dadd_rn(__dmul_rn(cx, cx), __dmul_rn(cy, cy)), __dmul_rn(cz, cz))));
}

// Pass 1: areas, and per chunk the sequential sum of its areas.
__global__ void __launch_bounds__(kThreads) area_chunk_kernel(const double* __restrict__ verts,
                                                              const int32_t* __restrict__ tris, int64_t nt,
                                                              const double* crop, double* __restrict__ area,
                                                              double* __restrict__ chunk) {
    const int64_t nc = (nt + kScanChunk - 1) / kScanChunk;
    for (int64_t c = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; c < nc; c += (int64_t)gridDim.x * blockDim.x) {
        const int64_t end = min(nt, (c + 1) * kScanChunk);
        double s = 0.0;
        for (int64_t t = c * kScanChunk; t < end; ++t) {
            const double a = triangle_area(verts, tris + 3 * t, crop);
            area[t] = a;
            s = __dadd_rn(s, a);
        }
        chunk[c] = s;
    }
}

// Pass 2 (one thread): the chunk sums to exclusive prefixes, in sequence; the total area.
__global__ void chunk_prefix_kernel(double* chunk, int64_t nc, double* total) {
    double p = 0.0;
    for (int64_t c = 0; c < nc; ++c) {
        const double s = chunk[c];
        chunk[c] = p;
        p = __dadd_rn(p, s);
    }
    *total = p;
}

// Pass 3: area -> inclusive prefix, chunk prefix + the chunk's running sum.  The last value of a chunk is then exactly the
// next chunk's prefix, so the ends are non-decreasing and a triangle of area 0 has the same end as the one before it.
__global__ void __launch_bounds__(kThreads) area_scan_kernel(double* __restrict__ cum, int64_t nt,
                                                             const double* __restrict__ chunk) {
    const int64_t nc = (nt + kScanChunk - 1) / kScanChunk;
    for (int64_t c = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; c < nc; c += (int64_t)gridDim.x * blockDim.x) {
        const int64_t end = min(nt, (c + 1) * kScanChunk);
        const double p = chunk[c];
        double s = 0.0;
        for (int64_t t = c * kScanChunk; t < end; ++t) {
            s = __dadd_rn(s, cum[t]);
            cum[t] = __dadd_rn(p, s);
        }
    }
}

// Philox4x32-10 (Salmon et al., SC 2011): counter (lo, hi, 0, 0) = sample index, key (lo, hi) = seed.
__device__ __forceinline__ uint4 philox4x32_10(unsigned long long ctr, unsigned long long seed) {
    uint32_t c0 = (uint32_t)ctr, c1 = (uint32_t)(ctr >> 32), c2 = 0u, c3 = 0u;
    uint32_t k0 = (uint32_t)seed, k1 = (uint32_t)(seed >> 32);
#pragma unroll
    for (int r = 0; r < 10; ++r) {
        if (r) { k0 += 0x9E3779B9u; k1 += 0xBB67AE85u; }
        const uint32_t lo0 = 0xD2511F53u * c0, hi0 = __umulhi(0xD2511F53u, c0);
        const uint32_t lo1 = 0xCD9E8D57u * c2, hi1 = __umulhi(0xCD9E8D57u, c2);
        const uint32_t n0 = hi1 ^ c1 ^ k0, n2 = hi0 ^ c3 ^ k1;
        c0 = n0; c1 = lo1; c2 = n2; c3 = lo0;
    }
    return make_uint4(c0, c1, c2, c3);
}

// two words -> a double in [0, 1) with 53 random bits: ((a >> 5) 2^26 + (b >> 6)) 2^-53
__device__ __forceinline__ double unit53(uint32_t a, uint32_t b) {
    return (double)(((unsigned long long)(a >> 5) << 26) | (unsigned long long)(b >> 6)) * 0x1.0p-53;
}

// SamplePointsUniformlyImpl: triangle t gets the samples [round(C_{t-1} N), round(C_t N)), C_t = cum_t / S, the last end N.
__device__ __forceinline__ int64_t cdf_end(const double* cum, int64_t t, int64_t nt, double total, int64_t n) {
    if (t == nt - 1) return n;
    return (int64_t)round(__dmul_rn(__ddiv_rn(cum[t], total), (double)n));
}

__global__ void __launch_bounds__(kThreads) sample_kernel(const double* __restrict__ verts,
                                                          const int32_t* __restrict__ tris, int64_t nt,
                                                          const double* __restrict__ cum, const double* total_ptr,
                                                          int64_t n, unsigned long long seed, double* __restrict__ points,
                                                          int32_t* __restrict__ tri_ids) {
    const double total = *total_ptr;
    for (int64_t k = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; k < n; k += (int64_t)gridDim.x * blockDim.x) {
        int64_t lo = 0, hi = nt - 1;          // the first t with end_t > k (end_{nt-1} = n > k)
        while (lo < hi) {
            const int64_t mid = (lo + hi) >> 1;
            if (cdf_end(cum, mid, nt, total, n) > k) hi = mid; else lo = mid + 1;
        }
        const uint4 r = philox4x32_10((unsigned long long)k, seed);
        const double r1 = unit53(r.x, r.y), r2 = unit53(r.z, r.w);
        const double s = __dsqrt_rn(r1);
        const double a = __dsub_rn(1.0, s), b = __dmul_rn(s, __dsub_rn(1.0, r2)), c = __dmul_rn(s, r2);
        double p0[3], p1[3], p2[3];
        load_vertex(verts, tris[3 * lo], p0); load_vertex(verts, tris[3 * lo + 1], p1); load_vertex(verts, tris[3 * lo + 2], p2);
#pragma unroll
        for (int ax = 0; ax < 3; ++ax)
            points[3 * k + ax] = __dadd_rn(__dadd_rn(__dmul_rn(a, p0[ax]), __dmul_rn(b, p1[ax])), __dmul_rn(c, p2[ax]));
        if (tri_ids) tri_ids[k] = (int32_t)lo;
    }
}

// ---- nearest neighbours --------------------------------------------------------------------------------------------

// order-preserving unsigned image of a double: a < b (IEEE, not NaN) <=> img(a) < img(b)
__device__ __forceinline__ unsigned long long ordered_bits(double v) {
    const unsigned long long b = (unsigned long long)__double_as_longlong(v);
    return (b >> 63) ? ~b : (b | (1ull << 63));
}
__device__ __forceinline__ double from_ordered_bits(unsigned long long o) {
    return __longlong_as_double((long long)((o >> 63) ? (o & ~(1ull << 63)) : ~o));
}

struct TreeHeader {            // first bytes of the tree buffer
    unsigned long long bounds[6];   // ordered min x y z, ordered max x y z of the reference points
    int64_t n, leaves;              // points, leaves of the complete tree (a power of two)
};

struct TreeLayout {            // byte offsets into the tree buffer for n reference points
    int64_t points, ids, boxes, total, leaves;
};

int64_t next_pow2(int64_t v) {
    int64_t p = 1;
    while (p < v) p <<= 1;
    return p;
}

TreeLayout tree_layout(int64_t n) {
    TreeLayout l;
    l.leaves = next_pow2((n + kNnBucket - 1) / kNnBucket);
    l.points = align_up((int64_t)sizeof(TreeHeader));
    l.ids = l.points + align_up(24 * n);
    l.boxes = l.ids + align_up(4 * n);
    l.total = l.boxes + align_up(24 * 2 * l.leaves);        // node i (heap order, root 1) at 6 floats: lo x y z, hi x y z
    return l;
}

struct SortLayout {            // byte offsets into the build / query scratch for n points
    int64_t keys_in, keys_out, idx_in, idx_out, cub, total;
    size_t cub_bytes;
};

SortLayout sort_layout(int64_t n) {
    SortLayout l;
    const int m = (int)(n > 0 ? n : 1);
    l.cub_bytes = 0;
    cub::DeviceRadixSort::SortPairs(nullptr, l.cub_bytes, (const unsigned long long*)nullptr, (unsigned long long*)nullptr,
                                    (const int*)nullptr, (int*)nullptr, m);
    l.keys_in = 0;
    l.keys_out = align_up(8 * (int64_t)m);
    l.idx_in = l.keys_out + align_up(8 * (int64_t)m);
    l.idx_out = l.idx_in + align_up(4 * (int64_t)m);
    l.cub = l.idx_out + align_up(4 * (int64_t)m);
    l.total = l.cub + align_up((int64_t)l.cub_bytes);
    return l;
}

__global__ void __launch_bounds__(kThreads) nn_bounds_kernel(const double* __restrict__ p, int64_t n, TreeHeader* h) {
    unsigned long long lo[3] = {~0ull, ~0ull, ~0ull}, hi[3] = {0ull, 0ull, 0ull};
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
#pragma unroll
        for (int a = 0; a < 3; ++a) {
            const unsigned long long o = ordered_bits(p[3 * i + a]);
            lo[a] = o < lo[a] ? o : lo[a];
            hi[a] = o > hi[a] ? o : hi[a];
        }
    }
#pragma unroll
    for (int a = 0; a < 3; ++a) {
#pragma unroll
        for (int s = 16; s > 0; s >>= 1) {
            const unsigned long long l = __shfl_xor_sync(kFull, lo[a], s), u = __shfl_xor_sync(kFull, hi[a], s);
            lo[a] = l < lo[a] ? l : lo[a];
            hi[a] = u > hi[a] ? u : hi[a];
        }
    }
    if ((threadIdx.x & 31) == 0) {
#pragma unroll
        for (int a = 0; a < 3; ++a) {
            atomicMin(h->bounds + a, lo[a]);
            atomicMax(h->bounds + 3 + a, hi[a]);
        }
    }
}

// bit i of a 21-bit v -> bit 3i
__device__ __forceinline__ unsigned long long spread21(unsigned long long x) {
    x &= 0x1FFFFFull;
    x = (x | (x << 32)) & 0x1F00000000FFFFull;
    x = (x | (x << 16)) & 0x1F0000FF0000FFull;
    x = (x | (x << 8)) & 0x100F00F00F00F00Full;
    x = (x | (x << 4)) & 0x10C30C30C30C30C3ull;
    x = (x | (x << 2)) & 0x1249249249249249ull;
    return x;
}

// Morton key of p on a 2^21 grid over the reference bounds (clamped: queries may lie outside).  It only orders points.
__global__ void __launch_bounds__(kThreads) nn_keys_kernel(const double* __restrict__ p, int64_t n,
                                                           const TreeHeader* h, unsigned long long* __restrict__ keys,
                                                           int* __restrict__ idx) {
    double lo[3], scale[3];
#pragma unroll
    for (int a = 0; a < 3; ++a) {
        lo[a] = from_ordered_bits(h->bounds[a]);
        const double ext = from_ordered_bits(h->bounds[3 + a]) - lo[a];
        scale[a] = ext > 0.0 ? (double)((1 << kMortonBits) - 1) / ext : 0.0;
    }
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
        unsigned long long key = 0ull;
#pragma unroll
        for (int a = 0; a < 3; ++a) {
            double g = (p[3 * i + a] - lo[a]) * scale[a];
            g = fmin(fmax(g, 0.0), (double)((1 << kMortonBits) - 1));      // NaN -> 0
            key |= spread21((unsigned long long)g) << (2 - a);
        }
        keys[i] = key;
        idx[i] = (int)i;
    }
}

__global__ void __launch_bounds__(kThreads) nn_gather_kernel(const double* __restrict__ p, int64_t n,
                                                             const int* __restrict__ order, double* __restrict__ sorted,
                                                             int32_t* __restrict__ ids) {
    for (int64_t j = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; j < n; j += (int64_t)gridDim.x * blockDim.x) {
        const int i = order[j];
        sorted[3 * j] = p[3 * (int64_t)i]; sorted[3 * j + 1] = p[3 * (int64_t)i + 1]; sorted[3 * j + 2] = p[3 * (int64_t)i + 2];
        ids[j] = i;
    }
}

// Leaf boxes in fp32, rounded outward so that every point of the bucket lies inside; a leaf past the last point is empty
// (lo +inf, hi -inf), which every query prunes.
__global__ void __launch_bounds__(kThreads) nn_leaf_kernel(const double* __restrict__ sorted, int64_t n, int64_t leaves,
                                                           float* __restrict__ boxes) {
    for (int64_t L = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; L < leaves; L += (int64_t)gridDim.x * blockDim.x) {
        float lo[3] = {INFINITY, INFINITY, INFINITY}, hi[3] = {-INFINITY, -INFINITY, -INFINITY};
        const int64_t end = min(n, (L + 1) * kNnBucket);
        for (int64_t j = L * kNnBucket; j < end; ++j) {
#pragma unroll
            for (int a = 0; a < 3; ++a) {
                lo[a] = fminf(lo[a], __double2float_rd(sorted[3 * j + a]));
                hi[a] = fmaxf(hi[a], __double2float_ru(sorted[3 * j + a]));
            }
        }
        float* b = boxes + 6 * (leaves + L);
#pragma unroll
        for (int a = 0; a < 3; ++a) { b[a] = lo[a]; b[3 + a] = hi[a]; }
    }
}

__global__ void __launch_bounds__(kThreads) nn_level_kernel(float* __restrict__ boxes, int64_t first) {
    for (int64_t i = first + blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < 2 * first;
         i += (int64_t)gridDim.x * blockDim.x) {
        const float* l = boxes + 6 * (2 * i);
        const float* r = l + 6;
        float* b = boxes + 6 * i;
#pragma unroll
        for (int a = 0; a < 3; ++a) { b[a] = fminf(l[a], r[a]); b[3 + a] = fmaxf(l[3 + a], r[3 + a]); }
    }
}

// A lower bound of the squared distance from q to any point of the box: every operation rounds toward -inf.
__device__ __forceinline__ double box_lower_bound(const float* b, const double (&q)[3]) {
    double d2 = 0.0;
#pragma unroll
    for (int a = 0; a < 3; ++a) {
        const double d = fmax(fmax(__dsub_rd((double)b[a], q[a]), __dsub_rd(q[a], (double)b[3 + a])), 0.0);
        d2 = __dadd_rd(d2, __dmul_rd(d, d));
    }
    return d2;
}

__device__ __forceinline__ double dist2(const double (&q)[3], const double* p) {
    const double dx = __dsub_rn(q[0], p[0]), dy = __dsub_rn(q[1], p[1]), dz = __dsub_rn(q[2], p[2]);
    return __dadd_rn(__dadd_rn(__dmul_rn(dx, dx), __dmul_rn(dy, dy)), __dmul_rn(dz, dz));
}

__global__ void __launch_bounds__(128) nn_query_kernel(const double* __restrict__ sorted, const int32_t* __restrict__ ids,
                                                       const float* __restrict__ boxes, int64_t n, int64_t leaves,
                                                       const double* __restrict__ queries, const int* __restrict__ order,
                                                       int64_t m, double r2, double* __restrict__ dist,
                                                       int32_t* __restrict__ index) {
    for (int64_t j = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; j < m; j += (int64_t)gridDim.x * blockDim.x) {
        const int64_t qi = order[j];
        const double q[3] = {queries[3 * qi], queries[3 * qi + 1], queries[3 * qi + 2]};
        double best = r2;
        int64_t best_j = -1;
        int64_t stack[kNnStack];
        double bound[kNnStack];
        int sp = 0;
        stack[sp] = 1; bound[sp] = box_lower_bound(boxes + 6, q); ++sp;
        while (sp > 0) {
            --sp;
            const int64_t node = stack[sp];
            if (!(bound[sp] < best)) continue;
            if (node >= leaves) {
                const int64_t L = node - leaves, end = min(n, (L + 1) * kNnBucket);
                for (int64_t k = L * kNnBucket; k < end; ++k) {
                    const double d2 = dist2(q, sorted + 3 * k);
                    if (d2 < best) { best = d2; best_j = k; }
                }
                continue;
            }
            const double bl = box_lower_bound(boxes + 6 * (2 * node), q);
            const double br = box_lower_bound(boxes + 6 * (2 * node + 1), q);
            const bool left_near = bl <= br;
            const double bn = left_near ? bl : br, bf = left_near ? br : bl;
            const int64_t cn = left_near ? 2 * node : 2 * node + 1;
            if (bf < best) { stack[sp] = 4 * node + 1 - cn; bound[sp] = bf; ++sp; }      // the other child
            if (bn < best) { stack[sp] = cn; bound[sp] = bn; ++sp; }
        }
        dist[qi] = best_j >= 0 ? __dsqrt_rn(best) : INFINITY;
        index[qi] = best_j >= 0 ? ids[best_j] : -1;
    }
}

__global__ void nn_empty_kernel(int64_t m, double* dist, int32_t* index) {
    for (int64_t j = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; j < m; j += (int64_t)gridDim.x * blockDim.x) {
        dist[j] = INFINITY;
        index[j] = -1;
    }
}

bool aligned(const void* p) { return ((uintptr_t)p % kAlign) == 0; }

int sort_keys(void* scratch, const SortLayout& l, int64_t n, cudaStream_t st) {
    size_t bytes = l.cub_bytes;
    return (int)cub::DeviceRadixSort::SortPairs(at<void>(scratch, l.cub), bytes, at<const unsigned long long>(scratch, l.keys_in),
                                                at<unsigned long long>(scratch, l.keys_out), at<const int>(scratch, l.idx_in),
                                                at<int>(scratch, l.idx_out), (int)n, 0, 3 * kMortonBits, st);
}

}  // namespace

extern "C" {

int64_t shine_mesh_sample_scratch_bytes(int64_t num_tris) {
    if (num_tris < 0) return SHINE_ERR_INVALID_ARG;
    if (num_tris > 0x7fffffffLL) return SHINE_ERR_UNSUPPORTED;
    return sample_layout(num_tris).total;
}

int shine_mesh_sample_areas(const double* verts, int64_t num_verts, const int32_t* tris, int64_t num_tris,
                            const double* crop_box, double* total_area, void* scratch, int64_t scratch_bytes,
                            void* stream) {
    if (num_verts < 0 || num_tris < 0 || !total_area) return SHINE_ERR_INVALID_ARG;
    if (num_tris > 0x7fffffffLL || num_verts > 0x7fffffffLL) return SHINE_ERR_UNSUPPORTED;
    if (num_tris > 0 && (!verts || !tris || num_verts == 0)) return SHINE_ERR_INVALID_ARG;
    if (!scratch || !aligned(scratch) || scratch_bytes < sample_layout(num_tris).total) return SHINE_ERR_INVALID_ARG;
    DeviceGuard guard(scratch);
    const cudaStream_t st = (cudaStream_t)stream;
    if (num_tris == 0) return (int)cudaMemsetAsync(total_area, 0, sizeof(double), st);
    const SampleLayout l = sample_layout(num_tris);
    const int64_t nc = (num_tris + kScanChunk - 1) / kScanChunk;
    double* cum = at<double>(scratch, l.cum);
    double* chunk = at<double>(scratch, l.chunk);
    area_chunk_kernel<<<blocks_for(nc), kThreads, 0, st>>>(verts, tris, num_tris, crop_box, cum, chunk);
    chunk_prefix_kernel<<<1, 1, 0, st>>>(chunk, nc, total_area);
    area_scan_kernel<<<blocks_for(nc), kThreads, 0, st>>>(cum, num_tris, chunk);
    return (int)cudaGetLastError();
}

int shine_mesh_sample_points(const double* verts, const int32_t* tris, int64_t num_tris, const double* total_area,
                             int64_t num_samples, uint64_t seed, const void* scratch, int64_t scratch_bytes,
                             double* points, int32_t* tri_ids, void* stream) {
    if (num_tris < 0 || num_samples < 0 || !total_area) return SHINE_ERR_INVALID_ARG;
    if (num_tris > 0x7fffffffLL) return SHINE_ERR_UNSUPPORTED;
    if (!scratch || !aligned(scratch) || scratch_bytes < sample_layout(num_tris).total) return SHINE_ERR_INVALID_ARG;
    if (num_samples == 0) return SHINE_OK;
    if (num_tris == 0 || !verts || !tris || !points) return SHINE_ERR_INVALID_ARG;
    DeviceGuard guard(points);
    const SampleLayout l = sample_layout(num_tris);
    sample_kernel<<<blocks_for(num_samples), kThreads, 0, (cudaStream_t)stream>>>(
        verts, tris, num_tris, at<double>(scratch, l.cum), total_area, num_samples, (unsigned long long)seed, points, tri_ids);
    return (int)cudaGetLastError();
}

int64_t shine_nn_tree_bytes(int64_t n) {
    if (n < 0) return SHINE_ERR_INVALID_ARG;
    if (n > 0x7fffffffLL) return SHINE_ERR_UNSUPPORTED;
    return tree_layout(n).total;
}

int64_t shine_nn_scratch_bytes(int64_t n) {
    if (n < 0) return SHINE_ERR_INVALID_ARG;
    if (n > 0x7fffffffLL) return SHINE_ERR_UNSUPPORTED;
    return sort_layout(n).total;
}

int shine_nn_build(const double* points, int64_t n, void* tree, int64_t tree_bytes, void* scratch, int64_t scratch_bytes,
                   void* stream) {
    if (n < 0 || (n > 0 && !points)) return SHINE_ERR_INVALID_ARG;
    if (n > 0x7fffffffLL) return SHINE_ERR_UNSUPPORTED;
    if (!tree || !aligned(tree) || tree_bytes < tree_layout(n).total) return SHINE_ERR_INVALID_ARG;
    if (!scratch || !aligned(scratch) || scratch_bytes < sort_layout(n).total) return SHINE_ERR_INVALID_ARG;
    DeviceGuard guard(tree);
    const cudaStream_t st = (cudaStream_t)stream;
    const TreeLayout t = tree_layout(n);
    TreeHeader h;
    for (int a = 0; a < 3; ++a) { h.bounds[a] = ~0ull; h.bounds[3 + a] = 0ull; }
    h.n = n; h.leaves = t.leaves;
    cudaError_t e = cudaMemcpyAsync(tree, &h, sizeof(h), cudaMemcpyHostToDevice, st);
    if (e != cudaSuccess || n == 0) return (int)e;
    auto* hd = at<TreeHeader>(tree, 0);
    const SortLayout l = sort_layout(n);
    nn_bounds_kernel<<<blocks_for(n), kThreads, 0, st>>>(points, n, hd);
    nn_keys_kernel<<<blocks_for(n), kThreads, 0, st>>>(points, n, hd, at<unsigned long long>(scratch, l.keys_in),
                                                       at<int>(scratch, l.idx_in));
    int rc = sort_keys(scratch, l, n, st);
    if (rc) return rc;
    double* sorted = at<double>(tree, t.points);
    float* boxes = at<float>(tree, t.boxes);
    nn_gather_kernel<<<blocks_for(n), kThreads, 0, st>>>(points, n, at<const int>(scratch, l.idx_out), sorted,
                                                         at<int32_t>(tree, t.ids));
    nn_leaf_kernel<<<blocks_for(t.leaves), kThreads, 0, st>>>(sorted, n, t.leaves, boxes);
    for (int64_t first = t.leaves / 2; first >= 1; first /= 2)
        nn_level_kernel<<<blocks_for(first), kThreads, 0, st>>>(boxes, first);
    return (int)cudaGetLastError();
}

int shine_nn_query(const void* tree, int64_t n, const double* queries, int64_t m, double radius2, double* dist,
                   int32_t* index, void* scratch, int64_t scratch_bytes, void* stream) {
    if (n < 0 || m < 0 || !(radius2 >= 0.0)) return SHINE_ERR_INVALID_ARG;
    if (n > 0x7fffffffLL || m > 0x7fffffffLL) return SHINE_ERR_UNSUPPORTED;
    if (!tree || !aligned(tree)) return SHINE_ERR_INVALID_ARG;
    if (m == 0) return SHINE_OK;
    if (!queries || !dist || !index) return SHINE_ERR_INVALID_ARG;
    if (!scratch || !aligned(scratch) || scratch_bytes < sort_layout(m).total) return SHINE_ERR_INVALID_ARG;
    DeviceGuard guard(dist);
    const cudaStream_t st = (cudaStream_t)stream;
    if (n == 0) {
        nn_empty_kernel<<<blocks_for(m), kThreads, 0, st>>>(m, dist, index);
        return (int)cudaGetLastError();
    }
    const TreeLayout t = tree_layout(n);
    const SortLayout l = sort_layout(m);
    nn_keys_kernel<<<blocks_for(m), kThreads, 0, st>>>(queries, m, at<TreeHeader>(tree, 0),
                                                       at<unsigned long long>(scratch, l.keys_in), at<int>(scratch, l.idx_in));
    int rc = sort_keys(scratch, l, m, st);
    if (rc) return rc;
    const int64_t qb = (m + 127) / 128;
    nn_query_kernel<<<(unsigned)(qb < (int64_t)sm_count() * 64 ? qb : (int64_t)sm_count() * 64), 128, 0, st>>>(
        at<double>(tree, t.points), at<int32_t>(tree, t.ids), at<float>(tree, t.boxes), n, t.leaves, queries,
        at<int>(scratch, l.idx_out), m, radius2, dist, index);
    return (int)cudaGetLastError();
}

}  // extern "C"
