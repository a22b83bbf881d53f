// shine_device.cuh — device helpers shared by every translation unit of libshine_b200.so: the hash-slot format,
// Morton / quantise / interpolation arithmetic of the reference (model/feature_octree.py:172-218) and small PTX wrappers.
// Everything lives in an anonymous namespace (one private copy per .cu file).
#pragma once

#include <cuda_runtime.h>
#include <math.h>
#include <stdint.h>

#include "shine_b200.h"

// types / functions shared ACROSS translation units (external linkage)
namespace shine_internal {

struct StepParams {
    shine_octree oct;
    shine_decoder dec;
    const float* coord;
    const float* label;
    const float* weight;     // nullable (ignored unless weighted)
    const float* d_loss;     // nullable device scalar
    float* pred;             // nullable
    float* loss;             // nullable, accumulated
    uint8_t* mask;           // nullable (infer only)
    int64_t n;
    int32_t num_tiles;
    int32_t mask_level;
    float sigma;
    float loss_scale;
    int32_t weighted;
    float scale;             // sdf_diff_loss (L1 / L2 steps): config.scale, map units per metre
};

// The mesher's block-sparse grid (shine_mesh.cu): point p of a query is point r = p % (n+1)^3 of brick b = p / (n+1)^3,
// r = (i (n+1) + j) (n+1) + k, at grid index G = bricks[b] * n + (i, j, k) and coordinate origin + spacing * G (fp32).
struct BrickGrid {
    const int32_t* bricks;   // [bricks, 3]
    float origin[3];
    float spacing;
    int32_t n;
};

// shine_sdf_infer's kernel over the points of a BrickGrid instead of a coordinate array; out_pred gets -Decoder.sdf
// (the mesher's sign, utils/mesher.py:72).  Checks the decoder and the flags; P.n / P.num_tiles count the grid's points.
int launch_sdf_grid(const StepParams& P, const BrickGrid& grid, uint32_t flags, cudaStream_t st);

}  // namespace shine_internal

namespace {

// ------------------------------------------------------------------------------------------------------
// constants / small helpers
// ------------------------------------------------------------------------------------------------------

constexpr int kTile = 16;          // points per warp tile
constexpr int kF = 8;              // fused path: feature_dim
constexpr int kH = 32;             // fused path: hidden width
constexpr int kWS = 40;            // padded row stride (floats) of 32-wide smem matrices: conflict-free frags
constexpr unsigned long long kEmptyKey = 0xFFFFFFFFFFFFFFFFull;
constexpr unsigned kFull = 0xFFFFFFFFu;

// One node of `nodes_lookup_tables[level]` (model/feature_octree.py:162-166) = one 64-byte slot made of two
// self-contained 32-byte sectors: sector z holds a copy of the key and the rows of the 4 corners whose z bit is z.
// The two lanes that share a point each read ONE sector with ONE 256-bit load and get key + their 4 corner rows at
// once: a first-probe hit costs a single memory round trip before the feature rows can be requested.
struct __align__(64) HashSlot {
    unsigned long long key;   // Morton code of the voxel, kEmptyKey when free
    int32_t node;             // insertion ordinal = index in node_keys, the reference's order (Morton order within a frame)
    int32_t maxdisp;          // as HOME slot: largest probe index of any key whose probe sequence starts here (<= 0: none
                              // was displaced) — a lookup that does not find its key in its home slot stops right there
                              // unless this says that some key of this home lives further along
    int32_t ids0[4];          // rows of corners c0 c2 c4 c6 (z bit 0)
    unsigned long long key2;  // copy of key (written after the slot is claimed through `key`)
    int32_t pad1;
    int32_t maxdisp2;         // copy of maxdisp for the lane that reads sector 1
    int32_t ids1[4];          // rows of corners c1 c3 c5 c7 (z bit 1)
};
static_assert(sizeof(HashSlot) == SHINE_HASH_SLOT_BYTES, "slot must be 64 bytes");

// the 4 corner rows with z bit == half of slot s
__device__ __forceinline__ const int32_t* slot_ids(const HashSlot* slots, int s, int half) {
    return reinterpret_cast<const int32_t*>(slots + s) + 8 * half + 4;
}

// 64-bit mix (two multiplies).  A cheaper 32-bit fmix32 of the folded key was measured and rejected: more first-probe
// collisions (gather-only kernel 0.111 -> 0.137 ms).
__host__ __device__ __forceinline__ uint32_t hash_key(unsigned long long k) {
    k ^= k >> 31; k *= 0x9E3779B97F4A7C15ull;
    k ^= k >> 29; k *= 0xBF58476D1CE4E5B9ull;
    k ^= k >> 32;
    return (uint32_t)k;
}

// bit i of v -> bit 3i (16 significant bits, as kaolin's int16 coordinates)
__device__ __forceinline__ unsigned long long spread3(uint32_t v) {
    unsigned long long x = v & 0xFFFFull;
    x = (x | (x << 16)) & 0x0000FF0000FFull;
    x = (x | (x << 8)) & 0x00F00F00F00Full;
    x = (x | (x << 4)) & 0x0C30C30C30C3ull;
    x = (x | (x << 2)) & 0x249249249249ull;
    return x;
}

// kal.ops.spc.quantize_points (model/feature_octree.py:203): floor(clamp(res*(x+1)/2, 0, res-1)), fp32 op order kept
__device__ __forceinline__ uint32_t quantize1(float x, float res) {
    float v = __fmul_rn(__fmul_rn(res, __fadd_rn(x, 1.0f)), 0.5f);
    v = fminf(fmaxf(v, 0.0f), res - 1.0f);
    return (uint32_t)(int)floorf(v);
}

// kal.ops.spc.points_to_morton (model/feature_octree.py:204): x -> bit 3i+2, y -> 3i+1, z -> 3i
__device__ __forceinline__ unsigned long long morton_of(float x, float y, float z, int level) {
    const float res = (float)(1u << level);
    return (spread3(quantize1(x, res)) << 2) | (spread3(quantize1(y, res)) << 1) | spread3(quantize1(z, res));
}

// FeatureOctree.interpolat (model/feature_octree.py:172-185): per-axis blend factor at `level`
__device__ __forceinline__ float axis_t(float x, float res, bool poly) {
    const float c = __fmul_rn(res, __fmaf_rn(x, 0.5f, 0.5f));   // x*0.5 is exact, so the fma rounds like mul+add
    const float d = c - truncf(c);                              // torch.frac
    if (!poly) return d;
    const float d2 = __fmul_rn(d, d);
    const float d3 = __fmul_rn(d2, d);
    return __fsub_rn(__fmul_rn(3.0f, d2), __fmul_rn(2.0f, d3));
}

struct Blend {   // the 8 weights of model/feature_octree.py:186-193, corner c = (x bit2, y bit1, z bit0)
    float tx, ty, tz, ux, uy, uz;
    __device__ __forceinline__ void init(float x, float y, float z, int level, bool poly) {
        const float res = (float)(1u << level);
        tx = axis_t(x, res, poly); ty = axis_t(y, res, poly); tz = axis_t(z, res, poly);
        ux = __fsub_rn(1.0f, tx); uy = __fsub_rn(1.0f, ty); uz = __fsub_rn(1.0f, tz);
    }
    __device__ __forceinline__ float w(int c) const {
        const float a = (c & 4) ? tx : ux, b = (c & 2) ? ty : uy, d = (c & 1) ? tz : uz;
        return __fmul_rn(__fmul_rn(a, b), d);
    }
};

// t and dt/dx of one axis: t = smoothstep(frac(res*(0.5x+0.5))) or the linear fraction; dt/dx = t'(d) * res * 0.5
__device__ __forceinline__ void axis_td(float x, float res, bool poly, float& t, float& dt) {
    const float c = __fmul_rn(res, __fmaf_rn(x, 0.5f, 0.5f));
    const float d = c - truncf(c);
    const float s = res * 0.5f;
    if (!poly) { t = d; dt = s; return; }
    const float d2 = __fmul_rn(d, d);
    t = __fsub_rn(__fmul_rn(3.0f, d2), __fmul_rn(2.0f, __fmul_rn(d2, d)));
    dt = (6.0f * d - 6.0f * d2) * s;
}

struct BlendD {   // weights of model/feature_octree.py:186-193 and their derivatives w.r.t. x, y, z
    float t[3], u[3], dt[3];
    __device__ __forceinline__ void init(float x, float y, float z, int level, bool poly) {
        const float res = (float)(1u << level);
        axis_td(x, res, poly, t[0], dt[0]); axis_td(y, res, poly, t[1], dt[1]); axis_td(z, res, poly, t[2], dt[2]);
#pragma unroll
        for (int a = 0; a < 3; ++a) u[a] = 1.0f - t[a];
    }
    // dw_c/da for a = 0,1,2
    __device__ __forceinline__ void dw(int c, float (&g)[3]) const {
        const float X = (c & 4) ? t[0] : u[0], Y = (c & 2) ? t[1] : u[1], Z = (c & 1) ? t[2] : u[2];
        const float dX = (c & 4) ? dt[0] : -dt[0], dY = (c & 2) ? dt[1] : -dt[1], dZ = (c & 1) ? dt[2] : -dt[2];
        g[0] = dX * Y * Z; g[1] = X * dY * Z; g[2] = X * Y * dZ;
    }
};

__device__ __forceinline__ float4 ldg_f4(const float* p) {
    return __ldg(reinterpret_cast<const float4*>(p));
}
// a full 32-byte feature row as two 16-byte non-coherent loads (the widest global load of sm_90a); the pair lands in
// one sector
__device__ __forceinline__ void ldg_row8(const float* p, float (&v)[8]) {
    asm volatile("ld.global.nc.v4.f32 {%0,%1,%2,%3}, [%4];" : "=f"(v[0]), "=f"(v[1]), "=f"(v[2]), "=f"(v[3]) : "l"(p));
    asm volatile("ld.global.nc.v4.f32 {%0,%1,%2,%3}, [%4];" : "=f"(v[4]), "=f"(v[5]), "=f"(v[6]), "=f"(v[7]) : "l"(p + 4));
}
__device__ __forceinline__ int4 ldg_i4(const int32_t* p) {
    return __ldg(reinterpret_cast<const int4*>(p));
}
__device__ __forceinline__ void red_add_f4(float* p, float a, float b, float c, float d) {
    asm volatile("red.global.add.v4.f32 [%0], {%1,%2,%3,%4};" ::"l"(p), "f"(a), "f"(b), "f"(c), "f"(d) : "memory");
}

// gradient privatisation: replica 0 is the caller's grad table, replicas 1.. live in lv.grad_replicas
__device__ __forceinline__ float* grad_base(const shine_level& lv, uint32_t warp_id, int F) {
    const uint32_t r = lv.num_replicas > 1 ? (warp_id & (uint32_t)(lv.num_replicas - 1)) : 0u;
    return r == 0 ? lv.feature_grads : lv.grad_replicas + (size_t)(r - 1) * (size_t)lv.rows * F;
}

// Probe sequence of key k in a table of mask+1 slots: p0 = hash & mask, p1 = p0 ^ 1 (the buddy slot in the same
// 128-byte line: a second probe that hits L1), then linearly from the next pair on.  Visits every slot once.
__host__ __device__ __forceinline__ uint32_t probe_pos(uint32_t h0, uint32_t k, uint32_t mask) {
    return k == 0 ? h0 : (k == 1 ? (h0 ^ 1u) : (((h0 & ~1u) + k) & mask));
}

// nodes_lookup_tables[level].get(morton, [-1]*8)  (model/feature_octree.py:205-209) as an open-addressing probe.
// Returns the slot index or -1.  The home slot's `maxdisp` bounds the walk: most misses end at the first probe.
__device__ __forceinline__ int probe_slot(const HashSlot* __restrict__ slots, uint32_t mask, unsigned long long key) {
    const uint32_t h0 = hash_key(key) & mask;
    const uint4 first = __ldg(reinterpret_cast<const uint4*>(slots + h0));        // {key lo, key hi, node, maxdisp}
    const unsigned long long k0 = ((unsigned long long)first.y << 32) | first.x;
    if (k0 == key) return (int)h0;
    const int last = (int)first.w;
    if (k0 == kEmptyKey || last <= 0) return -1;
#pragma unroll 1
    for (int n = 1; n <= last; ++n) {
        const uint32_t h = probe_pos(h0, (uint32_t)n, mask);
        const unsigned long long k = __ldg(&slots[h].key);
        if (k == key) return (int)h;
        if (k == kEmptyKey) return -1;
    }
    return -1;
}

// continuation of a walk whose home slot h0 was neither the key nor empty: probes 1 .. last
__device__ __noinline__ int probe_slot_from(const HashSlot* __restrict__ slots, uint32_t mask, unsigned long long key,
                                            uint32_t h0, int last) {
#pragma unroll 1
    for (int n = 1; n <= last; ++n) {
        const uint32_t h = probe_pos(h0, (uint32_t)n, mask);
        const unsigned long long k = __ldg(&slots[h].key);
        if (k == key) return (int)h;
        if (k == kEmptyKey) return -1;
    }
    return -1;
}

// insertion side: record that a key of home h0 went to probe index `it`
__device__ __forceinline__ void note_displacement(HashSlot* slots, uint32_t h0, uint32_t it) {
    if (it > 0) { atomicMax(&slots[h0].maxdisp, (int32_t)it); atomicMax(&slots[h0].maxdisp2, (int32_t)it); }
}

// one 32-byte sector of a slot: {key (2 words), 2 words of padding / ordinal, 4 corner rows}
struct SlotSector { unsigned long long key; int32_t maxdisp; int32_t ids[4]; };
__device__ __forceinline__ SlotSector ldg_sector(const HashSlot* slots, uint32_t s, int half) {
    uint32_t w[8];
    const void* p = reinterpret_cast<const char*>(slots + s) + 32 * half;
    asm volatile("ld.global.nc.v4.b32 {%0,%1,%2,%3}, [%4];" : "=r"(w[0]), "=r"(w[1]), "=r"(w[2]), "=r"(w[3]) : "l"(p));
    asm volatile("ld.global.nc.v4.b32 {%0,%1,%2,%3}, [%4];"
                 : "=r"(w[4]), "=r"(w[5]), "=r"(w[6]), "=r"(w[7]) : "l"(reinterpret_cast<const char*>(p) + 16));
    SlotSector r;
    r.key = ((unsigned long long)w[1] << 32) | w[0];
    r.maxdisp = (int32_t)w[3];
    r.ids[0] = (int32_t)w[4]; r.ids[1] = (int32_t)w[5]; r.ids[2] = (int32_t)w[6]; r.ids[3] = (int32_t)w[7];
    return r;
}

// Full lookup as the pair-split kernels do it: lane `half` of a point reads sector `half` of the first-probe slot; on
// a first-probe collision it walks on and fetches its 4 rows separately.  hit == false: ids are -1.
__device__ __forceinline__ bool resolve_sector(const HashSlot* slots, uint32_t mask, unsigned long long key, int half,
                                               SlotSector& sec) {
    if (sec.key == key) return true;
    int s = -1;
    if (sec.key != kEmptyKey && sec.maxdisp > 0) s = probe_slot_from(slots, mask, key, hash_key(key) & mask, sec.maxdisp);
    if (s >= 0) {
        const int4 v = __ldg(reinterpret_cast<const int4*>(slot_ids(slots, s, half)));
        sec.ids[0] = v.x; sec.ids[1] = v.y; sec.ids[2] = v.z; sec.ids[3] = v.w;
        return true;
    }
    sec.ids[0] = sec.ids[1] = sec.ids[2] = sec.ids[3] = -1;
    return false;
}

// pred = Decoder.sdf(f(q)) and its input gradient dpred/dq at q = (x, y, z), fp32 (shine_register.cu's normal equations,
// shine_render's normals):
//     f = sum_c w_c F_c,  J = df/dq = sum_c F_c (x) grad w_c         (one gather over the 8 x L corner rows)
//     pred as fp32 FMA chains (decoder in shared memory), masks D1, D2 of the two ReLUs
//     dq = W1^T D1 W2^T D2 w3 = dpred/df,  grad = J^T dq
// Returns whether q's voxel exists at lv[0].  With kNeedLeaf, a q without it returns false right after the gather, and
// pred and grad are not formed.  S holds W1 [32][8], W2 [32][32] (W2[j][n]), its transpose W2T, b1, b2, w3 and b3.
template <bool kNeedLeaf, class S>
__device__ __forceinline__ bool sdf_grad_at(const shine_octree& oct, const S& sm, float x, float y, float z, float& pred,
                                            float (&grad)[3]) {
    const bool poly = oct.poly_interp != 0;
    const int L = oct.num_levels;
    float f[8], J[8][3];
#pragma unroll
    for (int k = 0; k < 8; ++k) { f[k] = 0.f; J[k][0] = J[k][1] = J[k][2] = 0.f; }
    bool valid = false;
#pragma unroll 1
    for (int i = 0; i < L; ++i) {
        const shine_level& lv = oct.lv[i];
        const HashSlot* slots = reinterpret_cast<const HashSlot*>(lv.hash_slots);
        const int s = probe_slot(slots, lv.hash_capacity - 1, morton_of(x, y, z, lv.level));
        if (s < 0) continue;
        if (i == 0) valid = true;
        const int4 ia = ldg_i4(slots[s].ids0), ib = ldg_i4(slots[s].ids1);
        const int ids[8] = {ia.x, ib.x, ia.y, ib.y, ia.z, ib.z, ia.w, ib.w};
        BlendD b; b.init(x, y, z, lv.level, poly);
#pragma unroll
        for (int c = 0; c < 8; ++c) {
            float row[8];
            ldg_row8(lv.features + (int64_t)ids[c] * kF, row);
            const float X = (c & 4) ? b.t[0] : b.u[0], Y = (c & 2) ? b.t[1] : b.u[1], Z = (c & 1) ? b.t[2] : b.u[2];
            const float w = __fmul_rn(__fmul_rn(X, Y), Z);
            float dw[3]; b.dw(c, dw);
#pragma unroll
            for (int k = 0; k < 8; ++k) {
                f[k] = fmaf(w, row[k], f[k]);
                J[k][0] = fmaf(dw[0], row[k], J[k][0]); J[k][1] = fmaf(dw[1], row[k], J[k][1]);
                J[k][2] = fmaf(dw[2], row[k], J[k][2]);
            }
        }
    }
    if (kNeedLeaf && !valid) return false;

    // Decoder.sdf forward (model/decoder.py:49-63), fp32 FMA chains
    float h1[32];
    uint32_t m1 = 0, m2 = 0;
#pragma unroll
    for (int n = 0; n < 32; ++n) {
        const float4 wa = *reinterpret_cast<const float4*>(sm.W1 + n * 8), wb = *reinterpret_cast<const float4*>(sm.W1 + n * 8 + 4);
        float a = sm.b1[n];
        a = fmaf(wa.x, f[0], a); a = fmaf(wa.y, f[1], a); a = fmaf(wa.z, f[2], a); a = fmaf(wa.w, f[3], a);
        a = fmaf(wb.x, f[4], a); a = fmaf(wb.y, f[5], a); a = fmaf(wb.z, f[6], a); a = fmaf(wb.w, f[7], a);
        m1 |= (a > 0.f ? 1u : 0u) << n;
        h1[n] = fmaxf(a, 0.f);
    }
    float pr = sm.b3;
#pragma unroll 1
    for (int j = 0; j < 32; ++j) {
        float a = sm.b2[j];
#pragma unroll
        for (int n = 0; n < 32; n += 4) {
            const float4 w = *reinterpret_cast<const float4*>(sm.W2 + j * 32 + n);
            a = fmaf(w.x, h1[n], a); a = fmaf(w.y, h1[n + 1], a); a = fmaf(w.z, h1[n + 2], a); a = fmaf(w.w, h1[n + 3], a);
        }
        m2 |= (a > 0.f ? 1u : 0u) << j;
        pr = fmaf(fmaxf(a, 0.f), sm.w3[j], pr);
    }

    // dq = W1^T D1 W2^T D2 w3 = dpred/df, grad = J^T dq
    float dq[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
#pragma unroll 1
    for (int n = 0; n < 32; ++n) {
        if (!((m1 >> n) & 1u)) continue;
        float a = 0.f;
#pragma unroll
        for (int j = 0; j < 32; j += 4) {
            const float4 w = *reinterpret_cast<const float4*>(sm.W2T + n * 32 + j);
            a = fmaf(w.x, ((m2 >> j) & 1u) ? sm.w3[j] : 0.f, a);
            a = fmaf(w.y, ((m2 >> (j + 1)) & 1u) ? sm.w3[j + 1] : 0.f, a);
            a = fmaf(w.z, ((m2 >> (j + 2)) & 1u) ? sm.w3[j + 2] : 0.f, a);
            a = fmaf(w.w, ((m2 >> (j + 3)) & 1u) ? sm.w3[j + 3] : 0.f, a);
        }
        const float4 wa = *reinterpret_cast<const float4*>(sm.W1 + n * 8), wb = *reinterpret_cast<const float4*>(sm.W1 + n * 8 + 4);
        dq[0] = fmaf(a, wa.x, dq[0]); dq[1] = fmaf(a, wa.y, dq[1]); dq[2] = fmaf(a, wa.z, dq[2]); dq[3] = fmaf(a, wa.w, dq[3]);
        dq[4] = fmaf(a, wb.x, dq[4]); dq[5] = fmaf(a, wb.y, dq[5]); dq[6] = fmaf(a, wb.z, dq[6]); dq[7] = fmaf(a, wb.w, dq[7]);
    }
#pragma unroll
    for (int a = 0; a < 3; ++a) {
        float s = 0.f;
#pragma unroll
        for (int k = 0; k < 8; ++k) s = fmaf(J[k][a], dq[k], s);
        grad[a] = s;
    }
    pred = pr;
    return valid;
}

// ------------------------------------------------------------------------------------------------------
// tensor-core helpers: mma.sync m16n8k8 TF32, fp32 accumulate, optional 3xTF32 error compensation
// ------------------------------------------------------------------------------------------------------

__device__ __forceinline__ uint32_t f2tf32(float x) {
    uint32_t r;
    asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(r) : "f"(x));
    return r;
}
__device__ __forceinline__ void split_tf32(float x, uint32_t& hi, uint32_t& lo) {
    hi = f2tf32(x);
    lo = f2tf32(x - __uint_as_float(hi));
}
__device__ __forceinline__ void mma_tf32(float (&d)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
    asm volatile(
        "mma.sync.aligned.m16n8k8.row.col.f32.tf32.tf32.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
        : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}

// A operand: fp32 values in A-fragment order, split on demand.  NTF == 3: D += Al*Bh + Ah*Bl + Ah*Bh.
// activation split for 3xTF32: hi = x with the low 13 mantissa bits cleared (1 LOP), lo = x - hi (exact; the MMA
// reads its top 19 bits).  x*w = hi*wh + hi*wl + lo*wh + O(2^-20 |x w|): same order as the cvt.rna split, one
// instruction less per element.
// The mask lives in constant memory on purpose: with a literal, ptxas knows that HMMA ignores the bits the AND clears, feeds
// the unmasked value to the tensor core instead, and then re-assembles that operand quad with four MOVs before every use.
__constant__ uint32_t g_tf32_mask = 0xFFFFE000u;
__device__ __forceinline__ void split_fast(float x, uint32_t& hi, uint32_t& lo) {
    hi = __float_as_uint(x) & g_tf32_mask;
    lo = __float_as_uint(x - __uint_as_float(hi));
}
// fp32 pairs.  Every operation rounds once, like its scalar form (the _rn intrinsics keep the compiler from contracting
// a multiply and an add into one FMA), so the results are those of the element-wise scalar code.
typedef float2 f2_t;
__device__ __forceinline__ f2_t f2_pack(float a, float b) { return make_float2(a, b); }
__device__ __forceinline__ void f2_unpack(f2_t r, float& a, float& b) { a = r.x; b = r.y; }
__device__ __forceinline__ f2_t f2_fma(f2_t a, f2_t b, f2_t c) { return make_float2(__fmaf_rn(a.x, b.x, c.x), __fmaf_rn(a.y, b.y, c.y)); }
__device__ __forceinline__ f2_t f2_mul(f2_t a, f2_t b) { return make_float2(__fmul_rn(a.x, b.x), __fmul_rn(a.y, b.y)); }
__device__ __forceinline__ f2_t f2_add(f2_t a, f2_t b) { return make_float2(__fadd_rn(a.x, b.x), __fadd_rn(a.y, b.y)); }
__device__ __forceinline__ f2_t f2_sub(f2_t a, f2_t b) { return make_float2(__fsub_rn(a.x, b.x), __fsub_rn(a.y, b.y)); }
// split_fast of two values
__device__ __forceinline__ void split_fast2(float a, float b, uint32_t& ha, uint32_t& hb, uint32_t& la, uint32_t& lb) {
    ha = __float_as_uint(a) & g_tf32_mask; hb = __float_as_uint(b) & g_tf32_mask;
    float x, y;
    f2_unpack(f2_sub(f2_pack(a, b), f2_pack(__uint_as_float(ha), __uint_as_float(hb))), x, y);
    la = __float_as_uint(x); lb = __float_as_uint(y);
}
template <int NTF>
struct AFrag {
    uint32_t hi[4], lo[4];
    __device__ __forceinline__ void set(float a0, float a1, float a2, float a3) {
        if (NTF == 3) {
            split_fast(a0, hi[0], lo[0]); split_fast(a1, hi[1], lo[1]);
            split_fast(a2, hi[2], lo[2]); split_fast(a3, hi[3], lo[3]);
        } else {
            hi[0] = f2tf32(a0); hi[1] = f2tf32(a1); hi[2] = f2tf32(a2); hi[3] = f2tf32(a3);
        }
    }
    // same, for operands that come straight from shared memory (no register-placement constraints): packed split
    __device__ __forceinline__ void set_packed(float a0, float a1, float a2, float a3) {
        if (NTF == 3) {
            split_fast2(a0, a1, hi[0], hi[1], lo[0], lo[1]);
            split_fast2(a2, a3, hi[2], hi[3], lo[2], lo[3]);
        } else {
            set(a0, a1, a2, a3);
        }
    }
};
template <int NTF>
__device__ __forceinline__ void mma3(float (&d)[4], const AFrag<NTF>& a, uint2 bh, uint2 bl) {
    if (NTF == 3) {
        mma_tf32(d, a.lo, bh.x, bh.y);
        mma_tf32(d, a.hi, bl.x, bl.y);
    }
    mma_tf32(d, a.hi, bh.x, bh.y);
}

// acc[q] = fma(w3, r3[q], fma(w2, r2[q], fma(w1, r1[q], fma(w0, r0[q], acc[q])))) for the 8 channels
__device__ __forceinline__ void blend4(float (&acc)[8], const float (&r0)[8], const float (&r1)[8], const float (&r2)[8],
                                       const float (&r3)[8], float w0, float w1, float w2, float w3) {
    const f2_t p0 = f2_pack(w0, w0), p1 = f2_pack(w1, w1), p2 = f2_pack(w2, w2), p3 = f2_pack(w3, w3);
#pragma unroll
    for (int q = 0; q < 8; q += 2) {
        f2_t a = f2_pack(acc[q], acc[q + 1]);
        a = f2_fma(p0, f2_pack(r0[q], r0[q + 1]), a); a = f2_fma(p1, f2_pack(r1[q], r1[q + 1]), a);
        a = f2_fma(p2, f2_pack(r2[q], r2[q + 1]), a); a = f2_fma(p3, f2_pack(r3[q], r3[q + 1]), a);
        f2_unpack(a, acc[q], acc[q + 1]);
    }
}

// the same three products for four independent accumulators sharing one A fragment, issued term by term: consecutive
// HMMAs never depend on each other (the per-accumulator order, hence the result, is that of four mma3 calls)
template <int NTF>
__device__ __forceinline__ void mma3x4(float (&d)[4][4], const AFrag<NTF>& a, const uint2 (&bh)[4], const uint2 (&bl)[4]) {
    if (NTF == 3) {
#pragma unroll
        for (int j = 0; j < 4; ++j) mma_tf32(d[j], a.lo, bh[j].x, bh[j].y);
#pragma unroll
        for (int j = 0; j < 4; ++j) mma_tf32(d[j], a.hi, bl[j].x, bl[j].y);
    }
#pragma unroll
    for (int j = 0; j < 4; ++j) mma_tf32(d[j], a.hi, bh[j].x, bh[j].y);
}
// two accumulators, two A fragments, one B fragment pair each
template <int NTF>
__device__ __forceinline__ void mma3x2(float (&d0)[4], float (&d1)[4], const AFrag<NTF>& a0, const AFrag<NTF>& a1,
                                       uint2 bh0, uint2 bl0, uint2 bh1, uint2 bl1) {
    if (NTF == 3) {
        mma_tf32(d0, a0.lo, bh0.x, bh0.y); mma_tf32(d1, a1.lo, bh1.x, bh1.y);
        mma_tf32(d0, a0.hi, bl0.x, bl0.y); mma_tf32(d1, a1.hi, bl1.x, bl1.y);
    }
    mma_tf32(d0, a0.hi, bh0.x, bh0.y); mma_tf32(d1, a1.hi, bh1.x, bh1.y);
}
// The same for an operand that is exact in tf32 (a 0/1 ReLU mask): its lo word is zero, so 3xTF32 takes two products.
// 1.0f as an mma operand word
constexpr uint32_t kTf32One = 0x3f800000u;
// exact A (one word per element), four accumulators: D[j] += A Bh[j] + A Bl[j]
template <int NTF>
__device__ __forceinline__ void mma2x4_exact_a(float (&d)[4][4], const uint32_t (&a)[4], const uint2 (&bh)[4], const uint2 (&bl)[4]) {
    if (NTF == 3) {
#pragma unroll
        for (int j = 0; j < 4; ++j) mma_tf32(d[j], a, bl[j].x, bl[j].y);
    }
#pragma unroll
    for (int j = 0; j < 4; ++j) mma_tf32(d[j], a, bh[j].x, bh[j].y);
}
// exact B, four accumulators sharing one A fragment: D[j] += Al B[j] + Ah B[j]
template <int NTF>
__device__ __forceinline__ void mma2x4_exact_b(float (&d)[4][4], const AFrag<NTF>& a, const uint2 (&b)[4]) {
    if (NTF == 3) {
#pragma unroll
        for (int j = 0; j < 4; ++j) mma_tf32(d[j], a.lo, b[j].x, b[j].y);
    }
#pragma unroll
    for (int j = 0; j < 4; ++j) mma_tf32(d[j], a.hi, b[j].x, b[j].y);
}

// ------------------------------------------------------------------------------------------------------
// host-side helpers shared by the entry points
// ------------------------------------------------------------------------------------------------------

constexpr int kMaxDevices = 64;

inline bool is_pow2(uint32_t v) { return v && !(v & (v - 1)); }

// Every entry point launches on the device that OWNS its buffers, not on whatever device happens to be current:
// the guard looks the device up from a representative device pointer and restores the previous device on exit.
// Pinned-host / unregistered pointers leave the current device alone.
struct DeviceGuard {
    int prev = -1, dev = -1;
    bool switched = false;
    explicit DeviceGuard(const void* p) {
        if (cudaGetDevice(&prev) != cudaSuccess) { prev = -1; (void)cudaGetLastError(); }
        dev = prev;
        if (!p) return;
        cudaPointerAttributes a;
        if (cudaPointerGetAttributes(&a, p) != cudaSuccess) { (void)cudaGetLastError(); return; }
        if (a.type != cudaMemoryTypeDevice && a.type != cudaMemoryTypeManaged) return;
        dev = a.device;
        if (dev != prev && cudaSetDevice(dev) == cudaSuccess) switched = true;
    }
    ~DeviceGuard() { if (switched) (void)cudaSetDevice(prev); }
    DeviceGuard(const DeviceGuard&) = delete;
    DeviceGuard& operator=(const DeviceGuard&) = delete;
};

// device ordinal that owns `p`, or -1 for host / unknown pointers
inline int device_of(const void* p) {
    if (!p) return -1;
    cudaPointerAttributes a;
    if (cudaPointerGetAttributes(&a, p) != cudaSuccess) { (void)cudaGetLastError(); return -1; }
    return (a.type == cudaMemoryTypeDevice || a.type == cudaMemoryTypeManaged) ? a.device : -1;
}

inline int current_device() {
    int dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= kMaxDevices) return 0;
    return dev;
}

inline int sm_count() {
    static int cached[kMaxDevices] = {0};
    const int dev = current_device();
    if (cached[dev] == 0) {
        int n = 0;
        if (cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || n <= 0) n = 132;
        cached[dev] = n;
    }
    return cached[dev];
}

inline int check_octree(const shine_octree* o, bool need_grads) {
    if (!o) return SHINE_ERR_INVALID_ARG;
    if (o->num_levels < 1 || o->num_levels > SHINE_MAX_LEVELS) return SHINE_ERR_INVALID_ARG;
    if (o->feature_dim < 4 || (o->feature_dim & 3)) return SHINE_ERR_UNSUPPORTED;
    for (int i = 0; i < o->num_levels; ++i) {
        const shine_level& lv = o->lv[i];
        if (!lv.hash_slots || !lv.features || !is_pow2(lv.hash_capacity) || lv.rows < 1) return SHINE_ERR_INVALID_ARG;
        if (lv.level < 1 || lv.level > 16) return SHINE_ERR_INVALID_ARG;
        if (need_grads && !lv.feature_grads) return SHINE_ERR_INVALID_ARG;
        if (lv.num_replicas > 1 && (!is_pow2((uint32_t)lv.num_replicas) || lv.num_replicas > 64 || !lv.grad_replicas))
            return SHINE_ERR_INVALID_ARG;
    }
    return SHINE_OK;
}

// the batch must live on the same device as the tables (pinned host memory is allowed: the kernels can read it
// through the unified address space)
inline int check_same_device(const shine_octree* o, const void* batch_ptr) {
    const int d = device_of(batch_ptr);
    return (d >= 0 && d != device_of(o->lv[0].features)) ? SHINE_ERR_INVALID_ARG : SHINE_OK;
}

// the decoder of the fused kernels: F -> 32 -> 32 -> 1 with F = 8.  With dec_grad: its gradient buffers gw1, gw2, gw3 are
// all set or all NULL (a frozen decoder), and *dec_grad says which.
inline int check_decoder(const shine_decoder* d, const shine_octree* o, bool* dec_grad = nullptr) {
    if (!d) return SHINE_ERR_INVALID_ARG;
    if (d->in_dim != kF || d->hidden != kH || d->mlp_level != 2 || o->feature_dim != kF) return SHINE_ERR_UNSUPPORTED;
    if (!d->w1 || !d->w2 || !d->w3) return SHINE_ERR_INVALID_ARG;
    if (dec_grad) {
        *dec_grad = d->gw1 || d->gw2 || d->gw3;
        if (*dec_grad && !(d->gw1 && d->gw2 && d->gw3)) return SHINE_ERR_INVALID_ARG;
    }
    return SHINE_OK;
}

// The per-sample loss of the training kernels, a template parameter: sdf_bce_loss (utils/loss.py:17-24), or sdf_diff_loss
// (utils/loss.py:6-14) with l2_loss False (L1) or True (L2).
enum SdfLoss : int { kLossBce = 0, kLossL1 = 1, kLossL2 = 2 };

// One sample of sdf_diff_loss with diff_m = (pred - label) / scale (back to metres): the unweighted term li (|diff_m| or
// diff_m^2) and its derivative with respect to pred (sign(diff_m) / scale, torch's sign(0) = 0, or 2 diff_m / scale).
// IEEE divisions as torch rounds them.  (A product with a rounded 1 / scale was tried: the Morton-ordered training kernel
// then spills 12 bytes instead of the BCE kernel's 4.)
template <int LOSS>
__device__ __forceinline__ void diff_point(float pv, float lb, float scale, float& li, float& dli) {
    static_assert(LOSS == kLossL1 || LOSS == kLossL2, "sdf_diff_loss is L1 or L2");
    const float dm = __fdiv_rn(__fsub_rn(pv, lb), scale);
    if (LOSS == kLossL2) {
        li = __fmul_rn(dm, dm);
        dli = __fdiv_rn(__fmul_rn(2.0f, dm), scale);
    } else {
        li = fabsf(dm);
        dli = __fdiv_rn(dm > 0.f ? 1.0f : (dm < 0.f ? -1.0f : 0.0f), scale);
    }
}

// sdf_l1 / sdf_l2: the scale a caller passes must be a positive finite number
inline bool valid_scale(float scale) { return scale > 0.f && scale <= 3.402823466e38f; }

// The loss the loss bits of a shine_sdf_fwd / _step / _eikonal_step flag word pick (neither: sdf_bce), or -1 when the call
// refuses the word: both loss bits, or a bit outside those it accepts with that loss (bce_flags / diff_flags).
inline int sdf_loss_of(uint32_t flags, uint32_t bce_flags, uint32_t diff_flags) {
    const uint32_t bits = flags & (SHINE_FLAG_LOSS_L1 | SHINE_FLAG_LOSS_L2);
    if (bits == (SHINE_FLAG_LOSS_L1 | SHINE_FLAG_LOSS_L2)) return -1;
    const int loss = bits == SHINE_FLAG_LOSS_L1 ? kLossL1 : bits == SHINE_FLAG_LOSS_L2 ? kLossL2 : kLossBce;
    return (flags & ~(bits | (loss == kLossBce ? bce_flags : diff_flags))) ? -1 : loss;
}

}  // namespace
