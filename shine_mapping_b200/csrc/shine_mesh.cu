// shine_mesh.cu — the mesher (reference utils/mesher.py): block-sparse SDF grid, masked marching cubes, vertex normals
// the connected-cluster filter, and the save_map point records.  The grid query is shine_sdf_infer's kernel (shine_internal::launch_sdf_grid);
// this file holds what follows it.

#include <cuda_runtime.h>
#include <stdint.h>

#include <cub/block/block_scan.cuh>

#include "shine_b200.h"
#include "shine_device.cuh"
#include "shine_mc_table.cuh"

namespace {

constexpr int kMaxGrid = 1 << 20;   // grid indices per axis (20 bits each in an edge key)

struct EdgeSlot {                   // 16 bytes; key kEmptyKey when free
    unsigned long long key;
    uint32_t val;
    uint32_t pad;
};

__device__ __forceinline__ int64_t brick_key(int x, int y, int z) {
    return ((int64_t)x << 42) | ((int64_t)y << 21) | (int64_t)z;
}

__device__ bool has_brick(const int64_t* keys, int64_t n, int64_t key) {
    int64_t a = 0, b = n;
    while (a < b) {
        const int64_t m = (a + b) >> 1;
        const int64_t k = __ldg(keys + m);
        if (k == key) return true;
        if (k < key) a = m + 1; else b = m;
    }
    return false;
}

// +1 face points of bricks that are not in the map: sdf `missing`, mask 0 (utils/mesher.py:323-324 zero-initialises)
__global__ void halo_fixup_kernel(const __grid_constant__ shine_brick_grid g) {
    const int n1 = g.n + 1, per = n1 * n1 * n1;
    const int64_t p = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (p >= g.num_bricks * per) return;
    const int64_t b = p / per;
    const int r = (int)(p - b * per);
    const int i = r / (n1 * n1), j = (r / n1) % n1, k = r % n1;
    if (i < g.n && j < g.n && k < g.n) return;
    const int64_t key = brick_key(g.bricks[3 * b] + (i == g.n), g.bricks[3 * b + 1] + (j == g.n), g.bricks[3 * b + 2] + (k == g.n));
    if (!has_brick(g.all_keys, g.num_all, key)) {
        g.sdf[p] = g.missing_sdf;
        g.mask[p] = 0;
    }
}

// Insert `key` (or find it).  Returns the slot, -1 when the table is full.  `fresh` tells whether this call inserted it.
__device__ int edge_insert(EdgeSlot* slots, uint32_t mask, unsigned long long key, bool& fresh) {
    const uint32_t h0 = hash_key(key) & mask;
    for (uint32_t it = 0; it <= mask; ++it) {
        const uint32_t h = (h0 + it) & mask;
        const unsigned long long prev = atomicCAS(&slots[h].key, kEmptyKey, key);
        if (prev == kEmptyKey || prev == key) { fresh = prev == kEmptyKey; return (int)h; }
    }
    fresh = false;
    return -1;
}

__device__ int edge_find(const EdgeSlot* slots, uint32_t mask, unsigned long long key) {
    const uint32_t h0 = hash_key(key) & mask;
    for (uint32_t it = 0; it <= mask; ++it) {
        const uint32_t h = (h0 + it) & mask;
        const unsigned long long k = slots[h].key;
        if (k == key) return (int)h;
        if (k == kEmptyKey) return -1;
    }
    return -1;
}

// One thread per cube of the chunk: cube (i, j, k) of brick b, its corners read from the brick's (n+1)^3 points.
struct Cube {
    float v[8];
    int gx, gy, gz;      // grid index of the lowest corner
    int local;           // its point index in the brick
    int64_t base;        // first point of the brick
    bool active;         // processed (mask at the lowest corner, inside hi)
    int ntri;            // triangles without two coincident vertices (processed cubes only)
    int cls;
};

__device__ __forceinline__ void edge_vertex(const shine_brick_grid& g, const Cube& c, int e, float (&pos)[3],
                                            unsigned long long& key) {
    const int a = e >> 2, c0 = kMcEdgeCorner[e], c1 = c0 + (1 << a);
    const float v0 = c.v[c0], v1 = c.v[c1];
    const float t = __fdiv_rn(v0, __fsub_rn(v0, v1));
    const int ex = c.gx + (c0 & 1), ey = c.gy + ((c0 >> 1) & 1), ez = c.gz + ((c0 >> 2) & 1);
    pos[0] = (float)(ex - g.lo[0]); pos[1] = (float)(ey - g.lo[1]); pos[2] = (float)(ez - g.lo[2]);
    pos[a] = __fadd_rn(pos[a], t);
    key = ((((unsigned long long)ex << 20 | (unsigned long long)ey) << 20 | (unsigned long long)ez) << 2) | (unsigned)a;
}

__device__ void load_cube(const shine_brick_grid& g, int64_t q, Cube& c) {
    const int n = g.n, n1 = n + 1, per = n * n * n;
    const int64_t b = q / per;
    const int r = (int)(q - b * per);
    const int i = r / (n * n), j = (r / n) % n, k = r % n;
    c.gx = g.bricks[3 * b] * n + i; c.gy = g.bricks[3 * b + 1] * n + j; c.gz = g.bricks[3 * b + 2] * n + k;
    c.base = b * (int64_t)(n1 * n1 * n1);
    c.local = (i * n1 + j) * n1 + k;
    c.active = g.mask[c.base + c.local] != 0 && c.gx + 1 < g.hi[0] && c.gy + 1 < g.hi[1] && c.gz + 1 < g.hi[2];
    c.cls = 0;
    c.ntri = 0;
    if (!c.active) return;
#pragma unroll
    for (int cc = 0; cc < 8; ++cc) {
        const int o = ((cc & 1) * n1 + ((cc >> 1) & 1)) * n1 + ((cc >> 2) & 1);
        c.v[cc] = g.sdf[c.base + c.local + o];
        if (c.v[cc] < 0.f) c.cls |= 1 << cc;
    }
}

__device__ __forceinline__ bool same3(const float (&a)[3], const float (&b)[3]) {
    return a[0] == b[0] && a[1] == b[1] && a[2] == b[2];
}

template <bool EMIT>
__global__ void __launch_bounds__(256) mc_kernel(const __grid_constant__ shine_brick_grid g, EdgeSlot* __restrict__ slots,
                                                 uint32_t smask, int32_t* __restrict__ counters, float* __restrict__ verts,
                                                 int64_t vcap, int32_t* __restrict__ tris, int64_t tcap) {
    using Scan = cub::BlockScan<int, 256>;
    __shared__ typename Scan::TempStorage scan_tmp;
    __shared__ int block_base;
    const int64_t cubes = g.num_bricks * (int64_t)g.n * g.n * g.n;
    const int64_t q = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    Cube c;
    c.active = false; c.ntri = 0; c.cls = 0;
    if (q < cubes) load_cube(g, q, c);
    const uint32_t emask = c.active ? kMcEdgeMask[c.cls] : 0u;
    float pos[12][3];
    int ids[12];
#pragma unroll
    for (int e = 0; e < 12; ++e) {
        ids[e] = -1;
        if (emask & (1u << e)) {
            unsigned long long key;
            edge_vertex(g, c, e, pos[e], key);
            if (!EMIT) {
                bool fresh;
                const int s = edge_insert(slots, smask, key, fresh);
                if (s < 0) atomicAdd(counters + 3, 1);
                else if (fresh) atomicExch(&slots[s].val, (uint32_t)atomicAdd(counters, 1));
            } else {
                const int s = edge_find(slots, smask, key);
                ids[e] = s < 0 ? -1 : (int)slots[s].val;
                if (ids[e] >= 0 && ids[e] < vcap) {
                    verts[3 * (int64_t)ids[e]] = pos[e][0];
                    verts[3 * (int64_t)ids[e] + 1] = pos[e][1];
                    verts[3 * (int64_t)ids[e] + 2] = pos[e][2];
                }
            }
        }
    }
    if (c.active) {
        for (int t = 0; t < SHINE_MC_TRI_WIDTH - 1 && kMcTri[c.cls][t] >= 0; t += 3) {
            const int a = kMcTri[c.cls][t], b = kMcTri[c.cls][t + 1], d = kMcTri[c.cls][t + 2];
            if (!same3(pos[a], pos[b]) && !same3(pos[b], pos[d]) && !same3(pos[a], pos[d])) ++c.ntri;
        }
    }
    if (!EMIT) {
        const int tot = __reduce_add_sync(kFull, c.ntri);
        if ((threadIdx.x & 31) == 0 && tot) atomicAdd(counters + 1, tot);
        return;
    }
    int off, total;
    Scan(scan_tmp).ExclusiveSum(c.ntri, off, total);
    if (threadIdx.x == 0) block_base = total ? atomicAdd(counters + 2, total) : 0;
    __syncthreads();
    if (!c.ntri) return;
    int64_t row = (int64_t)block_base + off;
    for (int t = 0; t < SHINE_MC_TRI_WIDTH - 1 && kMcTri[c.cls][t] >= 0; t += 3) {
        const int a = kMcTri[c.cls][t], b = kMcTri[c.cls][t + 1], d = kMcTri[c.cls][t + 2];
        if (same3(pos[a], pos[b]) || same3(pos[b], pos[d]) || same3(pos[a], pos[d])) continue;
        if (row < tcap) {
            tris[3 * row] = ids[a]; tris[3 * row + 1] = ids[b]; tris[3 * row + 2] = ids[d];
        }
        ++row;
    }
}

// ---- clusters of edge-connected triangles (Open3D cluster_connected_triangles) and vertex normals --------------------

__device__ __forceinline__ unsigned long long tri_edge_key(int a, int b, int64_t nv) {
    return a < b ? (unsigned long long)a * (unsigned long long)nv + (unsigned)b
                 : (unsigned long long)b * (unsigned long long)nv + (unsigned)a;
}

// per edge the smallest triangle id that has it; parent[t] = t
__global__ void cluster_edges_kernel(const int32_t* __restrict__ tris, int64_t nt, int64_t nv, EdgeSlot* slots,
                                     uint32_t smask, int32_t* parent) {
    const int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= nt) return;
    parent[t] = (int32_t)t;
    for (int e = 0; e < 3; ++e) {
        bool fresh;
        const int s = edge_insert(slots, smask, tri_edge_key(tris[3 * t + e], tris[3 * t + (e + 1) % 3], nv), fresh);
        if (s >= 0) atomicMin(&slots[s].val, (uint32_t)t);
    }
}

__device__ int uf_find(int32_t* parent, int x) {
    while (true) {
        const int p = ((volatile int32_t*)parent)[x];
        if (p == x) return x;
        const int gp = ((volatile int32_t*)parent)[p];
        if (gp != p) atomicCAS(parent + x, p, gp);   // path halving; any ancestor is a valid parent
        x = p;
    }
}

__device__ void uf_union(int32_t* parent, int a, int b) {
    while (true) {
        a = uf_find(parent, a);
        b = uf_find(parent, b);
        if (a == b) return;
        if (a < b) { const int s = a; a = b; b = s; }   // link the larger root under the smaller
        if (atomicCAS(parent + a, a, b) == a) return;
    }
}

__global__ void cluster_union_kernel(const int32_t* __restrict__ tris, int64_t nt, int64_t nv, const EdgeSlot* slots,
                                     uint32_t smask, int32_t* parent) {
    const int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= nt) return;
    for (int e = 0; e < 3; ++e) {
        const int s = edge_find(slots, smask, tri_edge_key(tris[3 * t + e], tris[3 * t + (e + 1) % 3], nv));
        if (s >= 0 && slots[s].val != (uint32_t)t) uf_union(parent, (int)t, (int)slots[s].val);
    }
}

__global__ void cluster_count_kernel(int64_t nt, int32_t* parent, int32_t* count) {
    const int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= nt) return;
    const int r = uf_find(parent, (int)t);
    atomicAdd(count + r, 1);
}

__global__ void cluster_keep_kernel(int64_t nt, int32_t* parent, const int32_t* count, int32_t min_tris,
                                    uint8_t* keep) {
    const int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= nt) return;
    keep[t] = count[uf_find(parent, (int)t)] >= min_tris;
}

__global__ void face_normal_kernel(const float* __restrict__ verts, const int32_t* __restrict__ tris, int64_t nt,
                                   float* normals) {
    const int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= nt) return;
    const int a = tris[3 * t], b = tris[3 * t + 1], c = tris[3 * t + 2];
    const float ux = verts[3 * b] - verts[3 * a], uy = verts[3 * b + 1] - verts[3 * a + 1], uz = verts[3 * b + 2] - verts[3 * a + 2];
    const float wx = verts[3 * c] - verts[3 * a], wy = verts[3 * c + 1] - verts[3 * a + 1], wz = verts[3 * c + 2] - verts[3 * a + 2];
    float nx = uy * wz - uz * wy, ny = uz * wx - ux * wz, nz = ux * wy - uy * wx;
    const float len = sqrtf(nx * nx + ny * ny + nz * nz);
    if (len == 0.f) return;
    nx /= len; ny /= len; nz /= len;
    for (const int v : {a, b, c}) {
        atomicAdd(normals + 3 * v, nx); atomicAdd(normals + 3 * v + 1, ny); atomicAdd(normals + 3 * v + 2, nz);
    }
}

__global__ void normalize_kernel(float* normals, int64_t nv) {
    const int64_t v = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (v >= nv) return;
    const float x = normals[3 * v], y = normals[3 * v + 1], z = normals[3 * v + 2];
    const float len = sqrtf(x * x + y * y + z * z);
    if (len > 0.f) { normals[3 * v] = x / len; normals[3 * v + 1] = y / len; normals[3 * v + 2] = z / len; }
}

// ---- save_map: the owned grid points of a chunk as PLY records (utils/mesher.py:152-173 generate_sdf_map) ------------

struct ExportParams {
    double origin[3];   // metres, position of grid index lo
    double voxel;
    double t[12];       // 3x4, row-major
    float factor;
    int masked_only;
};

// One thread per owned point (i, j, k < n) of the chunk.  A warp's passing points take consecutive records: one ballot,
// one atomic by the first passing lane.  Records past `capacity` are counted, not written.
__global__ void __launch_bounds__(256) export_points_kernel(const __grid_constant__ shine_brick_grid g,
                                                            const __grid_constant__ ExportParams P,
                                                            uint8_t* __restrict__ records, int64_t capacity,
                                                            unsigned long long* __restrict__ counter) {
    const int n = g.n, n1 = n + 1, per = n * n * n;
    const int64_t q = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    bool pass = false;
    int gi[3] = {0, 0, 0};
    int64_t p = 0;
    int m = 0;
    if (q < g.num_bricks * per) {
        const int64_t b = q / per;
        const int r = (int)(q - b * per);
        const int i = r / (n * n), j = (r / n) % n, k = r % n;
        gi[0] = g.bricks[3 * b] * n + i; gi[1] = g.bricks[3 * b + 1] * n + j; gi[2] = g.bricks[3 * b + 2] * n + k;
        p = b * (int64_t)(n1 * n1 * n1) + (i * n1 + j) * n1 + k;
        m = g.mask[p] != 0;
        pass = gi[0] < g.hi[0] && gi[1] < g.hi[1] && gi[2] < g.hi[2] && (m || !P.masked_only);
    }
    const unsigned ballot = __ballot_sync(kFull, pass);
    if (!ballot) return;
    const int lane = threadIdx.x & 31, leader = __ffs(ballot) - 1;
    unsigned long long base = 0;
    if (lane == leader) base = atomicAdd(counter, (unsigned long long)__popc(ballot));
    base = __shfl_sync(kFull, base, leader);
    if (!pass) return;
    const int64_t row = (int64_t)base + __popc(ballot & ((1u << lane) - 1u));
    if (row >= capacity) return;
    double x[3];
#pragma unroll
    for (int a = 0; a < 3; ++a) x[a] = __dadd_rn(P.origin[a], __dmul_rn(P.voxel, (double)(gi[a] - g.lo[a])));
    float* rec = reinterpret_cast<float*>(records + row * 20);
#pragma unroll
    for (int a = 0; a < 3; ++a) {   // ((t0 x + t1 y) + t2 z) + t3, every product and sum rounded on its own
        const double* t = P.t + 4 * a;
        rec[a] = (float)__dadd_rn(__dadd_rn(__dadd_rn(__dmul_rn(t[0], x[0]), __dmul_rn(t[1], x[1])), __dmul_rn(t[2], x[2])), t[3]);
    }
    rec[3] = __fmul_rn(g.sdf[p], P.factor);
    reinterpret_cast<int32_t*>(rec)[4] = m;
}

int check_grid(const shine_brick_grid* g) {
    if (!g || g->num_bricks < 0 || g->n < 1 || g->n > 64) return SHINE_ERR_INVALID_ARG;
    if (g->num_bricks > 0 && (!g->bricks || !g->sdf || !g->mask)) return SHINE_ERR_INVALID_ARG;
    if (g->all_keys == nullptr && g->num_all != 0) return SHINE_ERR_INVALID_ARG;
    for (int a = 0; a < 3; ++a)
        if (g->lo[a] < 0 || g->hi[a] > kMaxGrid || g->lo[a] > g->hi[a]) return SHINE_ERR_INVALID_ARG;
    if (g->num_bricks * (int64_t)(g->n + 1) * (g->n + 1) * (g->n + 1) > (int64_t)INT32_MAX * 8) return SHINE_ERR_UNSUPPORTED;
    return SHINE_OK;
}

inline unsigned blocks_for(int64_t n) { return (unsigned)((n + 255) / 256); }

}  // namespace

extern "C" {

int shine_mesh_grid(const shine_octree* oct, const shine_decoder* dec, const shine_brick_grid* grid, int32_t mask_level,
                    uint32_t flags, void* stream) {
    int rc = check_octree(oct, false);
    if (rc) return rc;
    if ((rc = check_grid(grid))) return rc;
    if (!dec || mask_level < 0 || mask_level >= oct->num_levels) return SHINE_ERR_INVALID_ARG;
    if (grid->num_bricks == 0) return SHINE_OK;
    if ((rc = check_same_device(oct, grid->sdf))) return rc;
    DeviceGuard guard(oct->lv[0].features);
    const int64_t n1 = grid->n + 1, points = grid->num_bricks * n1 * n1 * n1;
    shine_internal::StepParams P{};
    P.oct = *oct; P.dec = *dec; P.n = points;
    P.num_tiles = (int32_t)((points + kTile - 1) / kTile);
    P.pred = grid->sdf; P.mask = grid->mask; P.mask_level = mask_level;
    P.sigma = 1.f; P.loss_scale = 1.f;
    shine_internal::BrickGrid bg;
    bg.bricks = grid->bricks; bg.spacing = grid->spacing; bg.n = grid->n;
    for (int a = 0; a < 3; ++a) bg.origin[a] = grid->origin[a];
    const cudaStream_t st = (cudaStream_t)stream;
    if ((rc = shine_internal::launch_sdf_grid(P, bg, flags, st))) return rc;
    if (grid->all_keys) halo_fixup_kernel<<<blocks_for(points), 256, 0, st>>>(*grid);
    return (int)cudaGetLastError();
}

int shine_marching_cubes(const shine_brick_grid* grid, void* edge_slots, uint32_t edge_capacity, int32_t* counters,
                         float* verts, int64_t vert_capacity, int32_t* tris, int64_t tri_capacity, void* stream) {
    int rc = check_grid(grid);
    if (rc) return rc;
    if (!edge_slots || !is_pow2(edge_capacity) || !counters) return SHINE_ERR_INVALID_ARG;
    if (verts && (!tris || vert_capacity < 0 || tri_capacity < 0)) return SHINE_ERR_INVALID_ARG;
    if (grid->num_bricks == 0) return SHINE_OK;
    DeviceGuard guard(grid->sdf);
    const int64_t cubes = grid->num_bricks * (int64_t)grid->n * grid->n * grid->n;
    auto* slots = reinterpret_cast<EdgeSlot*>(edge_slots);
    const cudaStream_t st = (cudaStream_t)stream;
    if (verts)
        mc_kernel<true><<<blocks_for(cubes), 256, 0, st>>>(*grid, slots, edge_capacity - 1, counters, verts, vert_capacity,
                                                            tris, tri_capacity);
    else
        mc_kernel<false><<<blocks_for(cubes), 256, 0, st>>>(*grid, slots, edge_capacity - 1, counters, nullptr, 0,
                                                             nullptr, 0);
    return (int)cudaGetLastError();
}

int shine_mesh_export_points(const shine_brick_grid* grid, const double* origin_m, double voxel_m, const double* transform,
                             float sdf_factor, int32_t masked_only, void* records, int64_t capacity, int64_t* counter,
                             int64_t* count_out, void* stream) {
    int rc = check_grid(grid);
    if (rc) return rc;
    if (!origin_m || !transform || !counter || capacity < 0 || (capacity > 0 && !records)) return SHINE_ERR_INVALID_ARG;
    if ((uintptr_t)records & 3u) return SHINE_ERR_INVALID_ARG;
    const int dev = device_of(counter);
    if (dev < 0 || (capacity > 0 && device_of(records) != dev)) return SHINE_ERR_INVALID_ARG;
    if (grid->num_bricks > 0 && device_of(grid->sdf) != dev) return SHINE_ERR_INVALID_ARG;
    DeviceGuard guard(counter);
    const cudaStream_t st = (cudaStream_t)stream;
    if (grid->num_bricks > 0) {
        ExportParams P;
        for (int a = 0; a < 3; ++a) P.origin[a] = origin_m[a];
        for (int a = 0; a < 12; ++a) P.t[a] = transform[a];
        P.voxel = voxel_m; P.factor = sdf_factor; P.masked_only = masked_only != 0;
        const int64_t owned = grid->num_bricks * (int64_t)grid->n * grid->n * grid->n;
        export_points_kernel<<<blocks_for(owned), 256, 0, st>>>(*grid, P, static_cast<uint8_t*>(records), capacity,
                                                                 reinterpret_cast<unsigned long long*>(counter));
        if (cudaError_t e = cudaGetLastError()) return (int)e;
    }
    int64_t count = 0;
    cudaError_t e = cudaMemcpyAsync(&count, counter, sizeof(count), cudaMemcpyDeviceToHost, st);
    if (e == cudaSuccess) e = cudaStreamSynchronize(st);
    if (e != cudaSuccess) return (int)e;
    if (count_out) *count_out = count;
    return count > capacity ? SHINE_ERR_CAPACITY : SHINE_OK;
}

int shine_mesh_clusters(const float* verts, int64_t nv, const int32_t* tris, int64_t nt, int32_t min_tris,
                        void* edge_slots, uint32_t edge_capacity, int32_t* scratch, uint8_t* keep, float* normals,
                        void* stream) {
    if (nv < 0 || nt < 0 || nt > INT32_MAX / 2 || nv > INT32_MAX) return SHINE_ERR_INVALID_ARG;
    if (nt > 0 && (!verts || !tris || !edge_slots || !scratch || !keep || !normals)) return SHINE_ERR_INVALID_ARG;
    if (nt > 0 && (!is_pow2(edge_capacity) || (int64_t)edge_capacity < 2 * 3 * nt)) return SHINE_ERR_INVALID_ARG;
    if (nv > 0 && !normals) return SHINE_ERR_INVALID_ARG;
    if (nv == 0) return SHINE_OK;
    DeviceGuard guard(normals);
    const cudaStream_t st = (cudaStream_t)stream;
    cudaError_t e = cudaMemsetAsync(normals, 0, (size_t)nv * 3 * sizeof(float), st);
    if (e != cudaSuccess) return (int)e;
    if (nt > 0) {
        auto* slots = reinterpret_cast<EdgeSlot*>(edge_slots);
        int32_t* parent = scratch;
        int32_t* count = scratch + nt;
        e = cudaMemsetAsync(count, 0, (size_t)nt * sizeof(int32_t), st);
        if (e != cudaSuccess) return (int)e;
        cluster_edges_kernel<<<blocks_for(nt), 256, 0, st>>>(tris, nt, nv, slots, edge_capacity - 1, parent);
        cluster_union_kernel<<<blocks_for(nt), 256, 0, st>>>(tris, nt, nv, slots, edge_capacity - 1, parent);
        cluster_count_kernel<<<blocks_for(nt), 256, 0, st>>>(nt, parent, count);
        cluster_keep_kernel<<<blocks_for(nt), 256, 0, st>>>(nt, parent, count, min_tris, keep);
        face_normal_kernel<<<blocks_for(nt), 256, 0, st>>>(verts, tris, nt, normals);
    }
    normalize_kernel<<<blocks_for(nv), 256, 0, st>>>(normals, nv);
    return (int)cudaGetLastError();
}

}  // extern "C"
