// shine_b200.cu — hand-written sm_90a kernels + the C ABI of include/shine_b200.h.
//
// Hot path (reference PRBonn/SHINE_mapping, shine_batch.py:123-209):
//   FeatureOctree.query_feature  (model/feature_octree.py:199-244)   Morton hash walk + 8-corner blend, L levels
//   Decoder.sdf                  (model/decoder.py:49-63)            8 -> 32 -> 32 -> 1 MLP
//   sdf_bce_loss                 (utils/loss.py:17-24)               BCE-with-logits vs sigmoid(label/sigma)
//   cur_loss.backward()          (shine_batch.py:209)                scatter-add into corner table + decoder grads
//
// Work decomposition of every per-point kernel here: a warp owns a TILE of 16 points (the M of
// mma.m16n8k8).  Lane (g = lane>>2, t = lane&3) owns point  g + 8*(t&1)  and feature half  t>>1
// (4 of the F=8 channels = one 16-byte half of a 32-byte table row).  The two lanes that share a row
// are served by the same 32-byte sector, so every sector that comes back from L2/HBM is fully used.
// That "row-half" layout converts to / from the mma A-fragment / C-fragment layouts with two
// shfl.xor(1) each (see to_afrag / from_cfrag), so activations never touch shared memory in the forward.
//
// Built with: nvcc -gencode arch=compute_90a,code=sm_90a -lineinfo -O3 (see __graft_entry__.build()).

#include <cuda_runtime.h>
#include <math.h>
#include <stdint.h>

#include <type_traits>

#include "shine_b200.h"

// tuning constants
#ifndef SHINE_GATHER_GROUP
#define SHINE_GATHER_GROUP 2  // levels whose first-probe sectors are in flight together (register pressure vs parallelism)
#endif
#ifndef SHINE_TRAIN_MINB
#define SHINE_TRAIN_MINB 2    // min resident blocks/SM of the training kernels (register cap 65536/(256*MINB))
#endif
// The per-point training kernels with decoder gradients keep 56 accumulators per lane live through the whole tile: at 2
// blocks/SM (128 registers) they spill ~0.5 KB per thread, at 1 block/SM (255) they do not, and on H100 the spill-free
// build is faster (C2 batch in the order drawn, kernel: 0.460 vs 0.564 ms).  The grouped kernel timed on Morton-ordered batches
// keeps its dW2 partial in shared memory and fits SHINE_TRAIN_MINB with a 4-byte spill.
#ifndef SHINE_TRAIN_DECGRAD_MINB
#define SHINE_TRAIN_DECGRAD_MINB 1
#endif
#ifndef SHINE_INFER_MINB
#define SHINE_INFER_MINB 3
#endif

#include "shine_device.cuh"

namespace {

// ------------------------------------------------------------------------------------------------------
// hash build (model/feature_octree.py:162-166)
// ------------------------------------------------------------------------------------------------------

__global__ void hash_insert_kernel(HashSlot* __restrict__ slots, uint32_t mask, const int64_t* __restrict__ keys,
                                   const int32_t* __restrict__ corner_ids, int64_t n, int32_t node_base,
                                   int32_t* __restrict__ overflow) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const unsigned long long key = (unsigned long long)keys[i];
    const uint32_t h0 = hash_key(key) & mask;
    for (uint32_t it = 0; it <= mask; ++it) {
        const uint32_t h = probe_pos(h0, it, mask);
        const unsigned long long prev = atomicCAS(&slots[h].key, kEmptyKey, key);
        if (prev == kEmptyKey || prev == key) {
            slots[h].node = node_base + (int32_t)i;
            slots[h].key2 = key;
#pragma unroll
            for (int c = 0; c < 4; ++c) {
                slots[h].ids0[c] = corner_ids[i * 8 + 2 * c];
                slots[h].ids1[c] = corner_ids[i * 8 + 2 * c + 1];
            }
            note_displacement(slots, h0, it);
            return;
        }
    }
    if (overflow) atomicAdd(overflow, 1);   // table full: the key was NOT stored — the caller must grow the table
}

__global__ void points_to_morton_kernel(const float* __restrict__ coord, int64_t n, int level,
                                        int64_t* __restrict__ out) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    out[i] = (int64_t)morton_of(coord[3 * i], coord[3 * i + 1], coord[3 * i + 2], level);
}

// ------------------------------------------------------------------------------------------------------
// get_indices (model/feature_octree.py:199-218): one thread per (point, level)
// ------------------------------------------------------------------------------------------------------

__global__ void get_indices_kernel(const __grid_constant__ shine_octree oct, const float* __restrict__ coord,
                                   int64_t n, int64_t* __restrict__ out) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    const int lvl = blockIdx.y;
    if (i >= n) return;
    const shine_level& lv = oct.lv[lvl];
    const HashSlot* slots = reinterpret_cast<const HashSlot*>(lv.hash_slots);
    const unsigned long long key = morton_of(coord[3 * i], coord[3 * i + 1], coord[3 * i + 2], lv.level);
    const int s = probe_slot(slots, lv.hash_capacity - 1, key);
    longlong2* dst = reinterpret_cast<longlong2*>(out + ((int64_t)lvl * n + i) * 8);
    if (s < 0) {
#pragma unroll
        for (int c = 0; c < 4; ++c) dst[c] = make_longlong2(-1, -1);
    } else {
        const int4 a = ldg_i4(slots[s].ids0), b = ldg_i4(slots[s].ids1);   // a: even corners, b: odd corners
        dst[0] = make_longlong2(a.x, b.x); dst[1] = make_longlong2(a.y, b.y);
        dst[2] = make_longlong2(a.z, b.z); dst[3] = make_longlong2(a.w, b.w);
    }
}

// ------------------------------------------------------------------------------------------------------
// query_feature forward / backward for any F = 4*LP (LP lanes share one point)
// ------------------------------------------------------------------------------------------------------

template <int LP>
__global__ void __launch_bounds__(256) query_fwd_kernel(const __grid_constant__ shine_octree oct,
                                                        const float* __restrict__ coord, int64_t n,
                                                        float* __restrict__ out) {
    constexpr int F = 4 * LP;
    const int64_t gtid = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    const int64_t p = gtid / LP;
    const int part = (int)(gtid % LP);
    if (p >= n) return;
    const float x = coord[3 * p], y = coord[3 * p + 1], z = coord[3 * p + 2];
    float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
    for (int i = 0; i < oct.num_levels; ++i) {
        const shine_level& lv = oct.lv[i];
        const HashSlot* slots = reinterpret_cast<const HashSlot*>(lv.hash_slots);
        const int s = probe_slot(slots, lv.hash_capacity - 1, morton_of(x, y, z, lv.level));
        if (s < 0) continue;
        const int4 ia = ldg_i4(slots[s].ids0), ib = ldg_i4(slots[s].ids1);
        const int ids[8] = {ia.x, ib.x, ia.y, ib.y, ia.z, ib.z, ia.w, ib.w};   // un-permute (z-bit-major storage)
        float4 v[8];
#pragma unroll
        for (int c = 0; c < 8; ++c) v[c] = ldg_f4(lv.features + (int64_t)ids[c] * F + 4 * part);
        Blend b; b.init(x, y, z, lv.level, oct.poly_interp != 0);
        float4 lsum = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
        for (int c = 0; c < 8; ++c) {
            const float w = b.w(c);
            lsum.x = fmaf(w, v[c].x, lsum.x); lsum.y = fmaf(w, v[c].y, lsum.y);
            lsum.z = fmaf(w, v[c].z, lsum.z); lsum.w = fmaf(w, v[c].w, lsum.w);
        }
        acc.x += lsum.x; acc.y += lsum.y; acc.z += lsum.z; acc.w += lsum.w;
    }
    *reinterpret_cast<float4*>(out + p * F + 4 * part) = acc;
}


// F = 8 specialisation of query_fwd: two adjacent lanes per point; lane `half` fetches the corners whose z bit is `half`
// as whole 32-byte rows (LDG.256; slot ids are stored z-bit-major), so the pair's two loads of one instruction hit
// z-neighbour rows = usually one 128-byte line; the partial blends are exchanged with one shfl per channel.
__global__ void __launch_bounds__(256) query_fwd8_kernel(const __grid_constant__ shine_octree oct,
                                                         const float* __restrict__ coord, int64_t n,
                                                         float* __restrict__ out) {
    const int64_t gtid = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    const int64_t p = gtid >> 1;
    const int half = (int)(gtid & 1);
    const bool valid = p < n;
    float x = 0.f, y = 0.f, z = 0.f;
    if (valid) { x = coord[3 * p]; y = coord[3 * p + 1]; z = coord[3 * p + 2]; }
    float acc[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
    for (int i = 0; i < oct.num_levels; ++i) {
        const shine_level& lv = oct.lv[i];
        const HashSlot* slots = reinterpret_cast<const HashSlot*>(lv.hash_slots);
        if (!valid) continue;
        const unsigned long long key = morton_of(x, y, z, lv.level);
        const uint32_t mask = lv.hash_capacity - 1;
        SlotSector sec = ldg_sector(slots, hash_key(key) & mask, half);
        if (!resolve_sector(slots, mask, key, half, sec)) continue;
        const int4 id4 = make_int4(sec.ids[0], sec.ids[1], sec.ids[2], sec.ids[3]);
        float r0[8], r1[8], r2[8], r3[8];
        ldg_row8(lv.features + (int64_t)id4.x * kF, r0);
        ldg_row8(lv.features + (int64_t)id4.y * kF, r1);
        ldg_row8(lv.features + (int64_t)id4.z * kF, r2);
        ldg_row8(lv.features + (int64_t)id4.w * kF, r3);
        Blend b; b.init(x, y, z, lv.level, oct.poly_interp != 0);
        const float wz = half ? b.tz : b.uz;
        const float w0 = __fmul_rn(__fmul_rn(b.ux, b.uy), wz), w1 = __fmul_rn(__fmul_rn(b.ux, b.ty), wz);
        const float w2 = __fmul_rn(__fmul_rn(b.tx, b.uy), wz), w3 = __fmul_rn(__fmul_rn(b.tx, b.ty), wz);
        blend4(acc, r0, r1, r2, r3, w0, w1, w2, w3);
    }
    float4 o;
    {
        float v[4];
#pragma unroll
        for (int q = 0; q < 4; ++q) {
            const float send = half ? acc[q] : acc[4 + q];
            const float recv = __shfl_xor_sync(kFull, send, 1);
            v[q] = (half ? acc[4 + q] : acc[q]) + recv;
        }
        o = make_float4(v[0], v[1], v[2], v[3]);
    }
    if (valid) *reinterpret_cast<float4*>(out + p * kF + 4 * half) = o;
}

template <int LP>
__global__ void __launch_bounds__(256) query_bwd_kernel(const __grid_constant__ shine_octree oct,
                                                        const float* __restrict__ coord, int64_t n,
                                                        const float* __restrict__ dfeat) {
    constexpr int F = 4 * LP;
    const int64_t gtid = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    const int64_t p = gtid / LP;
    const int part = (int)(gtid % LP);
    if (p >= n) return;
    const float x = coord[3 * p], y = coord[3 * p + 1], z = coord[3 * p + 2];
    const float4 d = ldg_f4(dfeat + p * F + 4 * part);
    for (int i = 0; i < oct.num_levels; ++i) {
        const shine_level& lv = oct.lv[i];
        const HashSlot* slots = reinterpret_cast<const HashSlot*>(lv.hash_slots);
        const int s = probe_slot(slots, lv.hash_capacity - 1, morton_of(x, y, z, lv.level));
        if (s < 0) continue;
        const int4 ia = ldg_i4(slots[s].ids0), ib = ldg_i4(slots[s].ids1);
        const int ids[8] = {ia.x, ib.x, ia.y, ib.y, ia.z, ib.z, ia.w, ib.w};   // un-permute (z-bit-major storage)
        Blend b; b.init(x, y, z, lv.level, oct.poly_interp != 0);
        float* gb = grad_base(lv, (uint32_t)(gtid >> 5), F) + 4 * part;
#pragma unroll
        for (int c = 0; c < 8; ++c) {
            const float w = b.w(c);
            red_add_f4(gb + (int64_t)ids[c] * F, w * d.x, w * d.y, w * d.z, w * d.w);
        }
    }
}


// ------------------------------------------------------------------------------------------------------
// coordinate derivatives of query_feature (eikonal / normal terms; reference utils/tools.py:175-185)
// ------------------------------------------------------------------------------------------------------

// MODE 0: coord_grad   1: tangent_fwd   2: tangent_bwd
template <int LP, int MODE>
__global__ void __launch_bounds__(256) query_tangent_kernel(const __grid_constant__ shine_octree oct,
                                                            const float* __restrict__ coord, int64_t n,
                                                            const float* __restrict__ vin,      // dfeat (0,2)
                                                            const float* __restrict__ tangent,  // [n,3] (1,2)
                                                            float* __restrict__ out) {
    constexpr int F = 4 * LP;
    const int64_t gtid = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    const int64_t p = gtid / LP;
    const int part = (int)(gtid % LP);
    const bool valid = p < n;
    float x = 0.f, y = 0.f, z = 0.f;
    float4 d = make_float4(0.f, 0.f, 0.f, 0.f);
    float tg[3] = {0.f, 0.f, 0.f};
    if (valid) {
        x = coord[3 * p]; y = coord[3 * p + 1]; z = coord[3 * p + 2];
        if (MODE != 1) d = ldg_f4(vin + p * F + 4 * part);
        if (MODE != 0) { tg[0] = tangent[3 * p]; tg[1] = tangent[3 * p + 1]; tg[2] = tangent[3 * p + 2]; }
    }
    float g3[3] = {0.f, 0.f, 0.f};
    float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
    for (int i = 0; i < oct.num_levels; ++i) {
        const shine_level& lv = oct.lv[i];
        const HashSlot* slots = reinterpret_cast<const HashSlot*>(lv.hash_slots);
        const int s = valid ? probe_slot(slots, lv.hash_capacity - 1, morton_of(x, y, z, lv.level)) : -1;
        if (s < 0) continue;
        const int4 ia = ldg_i4(slots[s].ids0), ib = ldg_i4(slots[s].ids1);
        const int ids[8] = {ia.x, ib.x, ia.y, ib.y, ia.z, ib.z, ia.w, ib.w};   // un-permute (z-bit-major storage)
        BlendD b; b.init(x, y, z, lv.level, oct.poly_interp != 0);
#pragma unroll
        for (int c = 0; c < 8; ++c) {
            float g[3]; b.dw(c, g);
            if (MODE == 0) {
                const float4 v = ldg_f4(lv.features + (int64_t)ids[c] * F + 4 * part);
                const float q = v.x * d.x + v.y * d.y + v.z * d.z + v.w * d.w;
                g3[0] = fmaf(g[0], q, g3[0]); g3[1] = fmaf(g[1], q, g3[1]); g3[2] = fmaf(g[2], q, g3[2]);
            } else {
                const float w = tg[0] * g[0] + tg[1] * g[1] + tg[2] * g[2];
                if (MODE == 1) {
                    const float4 v = ldg_f4(lv.features + (int64_t)ids[c] * F + 4 * part);
                    acc.x = fmaf(w, v.x, acc.x); acc.y = fmaf(w, v.y, acc.y); acc.z = fmaf(w, v.z, acc.z); acc.w = fmaf(w, v.w, acc.w);
                } else {
                    red_add_f4(lv.feature_grads + (int64_t)ids[c] * F + 4 * part, w * d.x, w * d.y, w * d.z, w * d.w);
                }
            }
        }
    }
    if (MODE == 0) {
#pragma unroll
        for (int o = 1; o < LP; o <<= 1) {   // the LP lanes of a point are adjacent
            g3[0] += __shfl_xor_sync(kFull, g3[0], o); g3[1] += __shfl_xor_sync(kFull, g3[1], o); g3[2] += __shfl_xor_sync(kFull, g3[2], o);
        }
        if (valid && part == 0) { out[3 * p] = g3[0]; out[3 * p + 1] = g3[1]; out[3 * p + 2] = g3[2]; }
    } else if (MODE == 1) {
        if (valid) *reinterpret_cast<float4*>(out + p * F + 4 * part) = acc;
    }
}

// row-half layout (this lane: 4 channels of its own point) -> A fragment of the 16x8 tile.
// k-slot t <-> channel 2t, k-slot t+4 <-> channel 2t+1 (the B fragments use the same permutation).
__device__ __forceinline__ void to_afrag(const float (&v)[4], int odd, float (&a)[4]) {
    const float s0 = odd ? v[0] : v[2], s1 = odd ? v[1] : v[3];
    const float r0 = __shfl_xor_sync(kFull, s0, 1), r1 = __shfl_xor_sync(kFull, s1, 1);
    if (!odd) { a[0] = v[0]; a[2] = v[1]; a[1] = r0; a[3] = r1; }
    else      { a[0] = r0;   a[2] = r1;   a[1] = v[2]; a[3] = v[3]; }
}
// C fragment of a 16x8 tile (rows g,g+8; cols 2t,2t+1) -> row-half layout
__device__ __forceinline__ void from_cfrag(const float (&c)[4], int odd, float (&v)[4]) {
    const float s0 = odd ? c[0] : c[2], s1 = odd ? c[1] : c[3];
    const float r0 = __shfl_xor_sync(kFull, s0, 1), r1 = __shfl_xor_sync(kFull, s1, 1);
    if (!odd) { v[0] = c[0]; v[1] = c[1]; v[2] = r0; v[3] = r1; }
    else      { v[0] = r0;   v[1] = r1;   v[2] = c[2]; v[3] = c[3]; }
}

// decoder-gradient accumulators of a lane in the per-point kernels (mma.sync C fragments): dW2[2][4][4], dW1[2][4], and the
// per-column partial sums of db2, db1, dw3 ([4][2]: columns 8j + 2t + q)
#define SHINE_ACC_DECL float dW2[2][4][4], dW1[2][4], db2p[4][2], db1p[4][2], dw3p[4][2]

// Sums 8 per-lane values over the 8 lanes of equal t and leaves lane (g, t) the sum of slot g (7 shuffles)
__device__ __forceinline__ float reduce_scatter_g8(const float (&v)[8], int lane) {
    float a[4], b[2];
    const bool b4 = (lane & 16) != 0, b3 = (lane & 8) != 0, b2 = (lane & 4) != 0;
#pragma unroll
    for (int i = 0; i < 4; ++i) a[i] = (b4 ? v[4 + i] : v[i]) + __shfl_xor_sync(kFull, b4 ? v[i] : v[4 + i], 16);
#pragma unroll
    for (int i = 0; i < 2; ++i) b[i] = (b3 ? a[2 + i] : a[i]) + __shfl_xor_sync(kFull, b3 ? a[i] : a[2 + i], 8);
    return (b2 ? b[1] : b[0]) + __shfl_xor_sync(kFull, b2 ? b[0] : b[1], 4);
}

// Decoder-weight-gradient operands are staged in mma fragment order: a consumer lane builds an A fragment with one LDS.128
// and a B fragment with one LDS.64.  The contraction runs over a tile's 16 points in an order of our choosing (A and B
// agree on it): points g and g + 8 are k-step g >> 2, k-slots (g & 3) and (g & 3) + 4, so that the producer lane of a
// C-fragment row pair (rows g, g + 8) holds both k-slots of a fragment register pair.  The 32 lane chunks of a fragment
// are stored at frag_chunk(lane), a permutation inside each group of 8 lanes: a consumer's 8 (LDS.128) or 16 (LDS.64)
// consecutive lanes still read whole 128-byte lines, and the producers' stores, where lane (g, t) writes the chunk of
// consumer lane 8t + 4q + (g & 3), land on distinct banks because the XOR with 2t separates the four values of t.
// Bank conflicts stay at zero by this layout, without padding.
__device__ __forceinline__ int frag_chunk(int lane) { return lane ^ ((lane >> 2) & 6); }
// A fragment ([32][4] block) / B fragment ([32][2] block) of chunk c, split for 3xTF32
template <int NTF>
__device__ __forceinline__ void load_afrag(const float* blk, int c, AFrag<NTF>& a) {
    const float4 v = *reinterpret_cast<const float4*>(blk + 4 * c);
    a.set_packed(v.x, v.y, v.z, v.w);
}
__device__ __forceinline__ void load_bfrag(const float* blk, int c, uint2& bh, uint2& bl) {
    const float2 v = *reinterpret_cast<const float2*>(blk + 2 * c);
    split_fast2(v.x, v.y, bh.x, bh.y, bl.x, bl.y);
}
// C fragments of a [16 points][32] tile (rows g, g + 8) -> the A fragments [m-tile 2][32][4] of this lane's k-step:
// column pairs 8j + 2t + q and 8j + 8 + 2t + q of both rows are one chunk
__device__ __forceinline__ void stage_afrags(float* blk, const int (&sq)[2], const float (&c)[4][4]) {
#pragma unroll
    for (int mt = 0; mt < 2; ++mt)
#pragma unroll
        for (int q = 0; q < 2; ++q)
            *reinterpret_cast<float4*>(blk + 128 * mt + 4 * sq[q]) = make_float4(c[2 * mt][q], c[2 * mt + 1][q], c[2 * mt][2 + q], c[2 * mt + 1][2 + q]);
}
// feat fragments [k-step 2][32][2]: each lane stores single elements, so k-step 1 also flips chunk bit 3 (16 banks) to
// keep the two k-steps' stores apart
__device__ __forceinline__ int xfrag_word(int ks, int c) { return 64 * ks + 2 * (c ^ (8 * ks)); }
__device__ __forceinline__ void load_xfrag(const float* sx, int ks, int c, uint2& bh, uint2& bl) {
    const float2 v = *reinterpret_cast<const float2*>(sx + xfrag_word(ks, c));
    split_fast2(v.x, v.y, bh.x, bh.y, bl.x, bl.y);
}

// ------------------------------------------------------------------------------------------------------
// the fused kernel: hash walk + gather + blend + MLP (+ BCE loss) (+ full backward with scatter-add)
// ------------------------------------------------------------------------------------------------------

constexpr int kGatherGroup = SHINE_GATHER_GROUP;

using shine_internal::StepParams;

// shared-memory plan (floats).  Weight matrices are pre-split into tf32 hi / lo words.
struct SmemPlan {
    static constexpr int W1 = 0;                       // [32][8]   W1[n][k]
    static constexpr int W1T = W1 + 2 * kH * kF;       // [8][kWS]  W1T[k][n]
    static constexpr int W2 = W1T + 2 * kF * kWS;      // [32][kWS] W2[n][k]
    static constexpr int W3W2T = W2 + 2 * kH * kWS;    // [32][kWS] w3[n] * W2[n][k] at [k][n] (layer-2 dgrad through the mask)
    static constexpr int B1 = W3W2T + 2 * kH * kWS;    // [32]
    static constexpr int B2 = B1 + kH;
    static constexpr int W3 = B2 + kH;
    static constexpr int B3 = W3 + kH;                 // [1]
    static constexpr int GSCALE = B3 + 1;              // [1] (+2 pad) dL/dpred scale: read per tile, not held in a register
    static constexpr int kDecGradFloats = kH * kF + kH + kH * kH + kH + kH + 1;   // 1377 (a warp's partial goes to its staging area)
    static constexpr int ZSUM = B3 + 4;                // [8] the warps' dL/dpred sums of their zero tiles (zero-tile shortcut)
    static constexpr int H1Z = ZSUM + 8;               // [32] h1(0) = relu(b1)     } the gradient g0 of Decoder.sdf(0) per unit
    static constexpr int H2Z = H1Z + kH;               // [32] h2(0)                } dL/dpred, in fp32 (zero_tile_gradient)
    static constexpr int D2Z = H2Z + kH;               // [32] db2 = w3 * [a2(0) > 0]
    static constexpr int DB1Z = D2Z + kH;              // [32] db1 = (W2^T db2) * [b1 > 0]
    static constexpr int kZsumFloats = 8 * 5 * kTile;  // more than the sums and g0 need: the offsets below and the block's
                                                       // shared-memory footprint were timed with this size
    static_assert(DB1Z + kH <= ZSUM + kZsumFloats, "g0 fits the zero-tile corner");
    static constexpr int STAGE = ZSUM + kZsumFloats;   // per-warp staging of one tile, in mma fragment order (below)
    static constexpr int SB2 = 0;                      // h1:  B fragments of dW2, [k-step 2][n-tile 4][32 lanes][2]
    static constexpr int SU = SB2;                     // GROUPED: h1 as A fragments of T = (dp h1)^T M2 (rows = layer-1
                                                       // units, k = points), [k-step 2][m-tile 2][32 lanes][4]
    static constexpr int SA1 = SB2 + kTile * kH;       // dh1: A fragments of dW1, [k-step 2][m-tile 2][32 lanes][4]
    static constexpr int SX = SA1 + kTile * kH;        // feat: B fragments of dW1, [k-step 2][32 lanes][2]
    static constexpr int SA2 = SX + kTile * kF;        // per-point kernels: dh2, A fragments of dW2, [k-step 2][m-tile 2][32 lanes][4]
    static constexpr int SDP = SA2;                    // GROUPED: [16 points] {dL/dpred, ReLU mask of h2 (bit n)}: the
                                                       // scale of u = dp h1 and the B operand M2 of T
    static constexpr int kStagePerWarp = SA2 + kTile * kH;
    static constexpr int kStageGrouped = SDP + 2 * kTile;
    __host__ __device__ static constexpr int stage_per_warp(bool grouped) { return grouped ? kStageGrouped : kStagePerWarp; }
    // GROUPED only, after the staging area: per warp and level [tx | ty | tz | node slot] x 16 points, and (frozen decoder:
    // no staging area to borrow from) the [16][8] dL/dfeature tile
    static constexpr int kGroupPerLevel = 4 * kTile;
    // GROUPED with decoder gradients, after the level tables: per warp its dW2 partial as the image of the C fragments
    // [m-tile 2][n-tile 4][32 lanes][4]
    static constexpr int kW2Part = kH * kH;
};

// The zero-tile shortcut's closed form (sdf_fused_kernel).  A point with features 0 has h1 = relu(b1) and a2 = W2 h1 + b2,
// so the gradient of Decoder.sdf(0) is  dW1 = 0, db1 = (W2^T db2) * [b1 > 0], dW2 = db2 h1^T, db2 = w3 * [a2 > 0],
// dw3 = relu(a2), db3 = 1.  One warp (lane = unit) writes its vectors to SmemPlan::H1Z .. DB1Z in plain fp32.
__device__ __forceinline__ void zero_tile_gradient(float* smem, const float* __restrict__ w2, int lane) {
    const float h1 = fmaxf(smem[SmemPlan::B1 + lane], 0.f);
    float a2 = smem[SmemPlan::B2 + lane];
#pragma unroll
    for (int k = 0; k < kH; ++k) a2 = fmaf(__ldg(w2 + lane * kH + k), __shfl_sync(kFull, h1, k), a2);
    const float d2 = a2 > 0.f ? smem[SmemPlan::W3 + lane] : 0.f;
    float db1 = 0.f;
#pragma unroll
    for (int n = 0; n < kH; ++n) db1 = fmaf(__ldg(w2 + n * kH + lane), __shfl_sync(kFull, d2, n), db1);
    smem[SmemPlan::H1Z + lane] = h1;
    smem[SmemPlan::H2Z + lane] = fmaxf(a2, 0.f);
    smem[SmemPlan::D2Z + lane] = d2;
    smem[SmemPlan::DB1Z + lane] = h1 > 0.f ? db1 : 0.f;
}
// The block's dL/dpred sum over its zero tiles (the warps' sums are in SmemPlan::ZSUM, after a block barrier).  A block
// with zero tiles then also gets g0 (one more barrier); a block without any leaves g0 unwritten and must not read it.
__device__ __forceinline__ float zero_tile_sum_and_gradient(float* smem, const float* __restrict__ w2, int warp, int lane) {
    float s = 0.f;
#pragma unroll
    for (int w = 0; w < 8; ++w) s += smem[SmemPlan::ZSUM + w];
    if (s != 0.f) {                 // block-uniform
        if (warp == 0) zero_tile_gradient(smem, w2, lane);
        __syncthreads();
    }
    return s;
}

// ---- voxel-grouped scatter (GROUPED kernels: batches in Morton order) ---------------------------------------------
// In a Morton-ordered batch the 16 points of a tile fall into a few groups of equal node per level.  The per-group gradient
// of the node's 8 corner rows is a small contraction over the group's points,
//     G[corner][channel] = sum_p w_corner(p) * dL/dfeature(p)[channel]          (8 x npts) x (npts x 8),
// so it runs on the tensor cores (m16n8k8, 3xTF32, rows 0-7 = corners of one group, rows 8-15 = corners of the next) and
// each group issues ONE 8-byte red per lane (8 rows x 32 B per instruction) instead of one 16-byte red per point and corner:
// the same-address atomics that serialise in L2 when neighbouring points share a voxel disappear.  Correct for any order
// (a level with more than kMaxGroupedRuns groups in a tile takes the per-point path).
constexpr int kMaxGroupedRuns = 6;

__device__ __forceinline__ void red_add_f2(float* p, float a, float b) {
    asm volatile("red.global.add.v2.f32 [%0], {%1,%2};" ::"l"(p), "f"(a), "f"(b) : "memory");
}
// permuted point index of the per-level tables: points t, t+4, t+8, t+12 are contiguous (one LDS.128 per field)
__device__ __forceinline__ int group_slot(int p) { return 4 * (p & 3) + (p >> 2); }

template <int LMAX>
__device__ __forceinline__ void grouped_scatter(const StepParams& P, int L, int tile, const float* __restrict__ pt,
                                                float* __restrict__ dtile, const float (&dxc)[4], int lane) {
    const int g = lane >> 2, t = lane & 3;
    // dL/dfeature tile: C fragment (rows = points g, g+8; cols = channels 2t, 2t+1) -> [point][channel]
    *reinterpret_cast<float2*>(dtile + g * kF + 2 * t) = make_float2(dxc[0], dxc[1]);
    *reinterpret_cast<float2*>(dtile + (g + 8) * kF + 2 * t) = make_float2(dxc[2], dxc[3]);
    __syncwarp();
    // B fragments (k = point, n = channel g): chunk c covers points 8c .. 8c+7
    uint2 bh[2], bl[2];
#pragma unroll
    for (int c = 0; c < 2; ++c)
        split_fast2(dtile[(8 * c + t) * kF + g], dtile[(8 * c + t + 4) * kF + g], bh[c].x, bh[c].y, bl[c].x, bl[c].y);
    // this lane's row of the A operand is corner g = (x bit 2, y bit 1, z bit 0): X = bit ? t : 1 - t as one FMA
    const float sx = (g & 4) ? 1.f : -1.f, ox = (g & 4) ? 0.f : 1.f;
    const float sy = (g & 2) ? 1.f : -1.f, oy = (g & 2) ? 0.f : 1.f;
    const float sz = (g & 1) ? 1.f : -1.f, oz = (g & 1) ? 0.f : 1.f;
    const int id_off = 8 * (g & 1) + 4 + (g >> 1);            // word of corner g's row index inside a 16-word HashSlot
    const int own = group_slot(lane & 15);
#pragma unroll
    for (int i = 0; i < LMAX; ++i) {
        if (i >= L) break;
        const float* lt = pt + i * SmemPlan::kGroupPerLevel;
        // groups of the level: the points of the tile that fall into the same node (lanes 0..15 <-> points; the upper half
        // of the warp mirrors them).  The lowest lane of a group leads it; a point's group index is its leader's rank
        // among the leaders.  Misses belong to no group.
        const int v_own = __float_as_int(lt[48 + own]);
        const uint32_t same = __match_any_sync(kFull, v_own);
        const int lead = __ffs(same) - 1;
        const uint32_t bmask = __ballot_sync(kFull, v_own >= 0 && lead == lane);      // leaders (all in lanes 0..15)
        if (bmask == 0) continue;
        const int rid_own = v_own >= 0 ? __popc(bmask & ((1u << lead) - 1u)) : 255;
        const shine_level& lv = P.oct.lv[i];
        const int32_t* slot_words = reinterpret_cast<const int32_t*>(lv.hash_slots);
        float* gb = grad_base(lv, (uint32_t)tile, kF);
        const int nruns = __popc(bmask);
        if (nruns > kMaxGroupedRuns) {
            // scattered tile (batch not in Morton order): per-point reds, this lane = channels 4*half.. of point g + 8*odd
            const int odd = t & 1, half = t >> 1, mp = group_slot(g + 8 * odd);
            const int v = __float_as_int(lt[48 + mp]);
            if (v >= 0) {
                const float tx = lt[mp], ty = lt[16 + mp], tz = lt[32 + mp];
                const float ux = __fsub_rn(1.0f, tx), uy = __fsub_rn(1.0f, ty), uz = __fsub_rn(1.0f, tz);
                const int4 e = ldg_i4(slot_words + 16 * (int64_t)v + 4), o = ldg_i4(slot_words + 16 * (int64_t)v + 12);
                const int ids[8] = {e.x, o.x, e.y, o.y, e.z, o.z, e.w, o.w};
                const float4 d = *reinterpret_cast<const float4*>(dtile + (g + 8 * odd) * kF + 4 * half);
                const float xy[4] = {__fmul_rn(ux, uy), __fmul_rn(ux, ty), __fmul_rn(tx, uy), __fmul_rn(tx, ty)};
                const f2_t zz = f2_pack(uz, tz), d01 = f2_pack(d.x, d.y), d23 = f2_pack(d.z, d.w);
#pragma unroll
                for (int c = 0; c < 8; c += 2) {
                    float w[2];
                    f2_unpack(f2_mul(f2_pack(xy[c >> 1], xy[c >> 1]), zz), w[0], w[1]);
#pragma unroll
                    for (int k = 0; k < 2; ++k) {
                        const f2_t wk = f2_pack(w[k], w[k]);
                        float g0, g1, g2, g3;
                        f2_unpack(f2_mul(wk, d01), g0, g1); f2_unpack(f2_mul(wk, d23), g2, g3);
                        red_add_f4(gb + (int64_t)ids[c + k] * kF + 4 * half, g0, g1, g2, g3);
                    }
                }
            }
            continue;
        }
        // weights of corner g for points t, t+4, t+8, t+12 (reference association (X*Y)*Z)
        const float4 tx4 = *reinterpret_cast<const float4*>(lt + 4 * t);
        const float4 ty4 = *reinterpret_cast<const float4*>(lt + 16 + 4 * t);
        const float4 tz4 = *reinterpret_cast<const float4*>(lt + 32 + 4 * t);
        float w[4];
        {
            const f2_t s_x = f2_pack(sx, sx), o_x = f2_pack(ox, ox), s_y = f2_pack(sy, sy), o_y = f2_pack(oy, oy);
            const f2_t s_z = f2_pack(sz, sz), o_z = f2_pack(oz, oz);
            const f2_t X01 = f2_fma(f2_pack(tx4.x, tx4.y), s_x, o_x), X23 = f2_fma(f2_pack(tx4.z, tx4.w), s_x, o_x);
            const f2_t Y01 = f2_fma(f2_pack(ty4.x, ty4.y), s_y, o_y), Y23 = f2_fma(f2_pack(ty4.z, ty4.w), s_y, o_y);
            const f2_t Z01 = f2_fma(f2_pack(tz4.x, tz4.y), s_z, o_z), Z23 = f2_fma(f2_pack(tz4.z, tz4.w), s_z, o_z);
            f2_unpack(f2_mul(f2_mul(X01, Y01), Z01), w[0], w[1]);
            f2_unpack(f2_mul(f2_mul(X23, Y23), Z23), w[2], w[3]);
        }
        // group index of those four points
        int rid[4];
#pragma unroll
        for (int q = 0; q < 4; ++q) rid[q] = __shfl_sync(kFull, rid_own, t + 4 * q);
        uint32_t rem = bmask;
        for (int r = 0; r < nruns; r += 2) {
            const int p1 = __ffs(rem) - 1; rem &= rem - 1;
            const int p2 = rem ? __ffs(rem) - 1 : p1; rem &= rem - 1;     // odd run count: the last pass has one run only
            const int v1 = __shfl_sync(kFull, v_own, p1);
            const int v2 = (r + 1 < nruns) ? __shfl_sync(kFull, v_own, p2) : -1;
            AFrag<3> a0, a1;     // rows g: run r, rows g + 8: run r + 1; k = points of chunk 0 / chunk 1
            a0.set(rid[0] == r ? w[0] : 0.f, rid[0] == r + 1 ? w[0] : 0.f, rid[1] == r ? w[1] : 0.f, rid[1] == r + 1 ? w[1] : 0.f);
            a1.set(rid[2] == r ? w[2] : 0.f, rid[2] == r + 1 ? w[2] : 0.f, rid[3] == r ? w[3] : 0.f, rid[3] == r + 1 ? w[3] : 0.f);
            float c0[4] = {0.f, 0.f, 0.f, 0.f}, c1[4] = {0.f, 0.f, 0.f, 0.f};
            mma3x2<3>(c0, c1, a0, a1, bh[0], bl[0], bh[1], bl[1]);
            if (v1 >= 0) {
                const int row = __ldg(slot_words + 16 * (int64_t)v1 + id_off);
                red_add_f2(gb + (int64_t)row * kF + 2 * t, c0[0] + c1[0], c0[1] + c1[1]);
            }
            if (v2 >= 0) {
                const int row = __ldg(slot_words + 16 * (int64_t)v2 + id_off);
                red_add_f2(gb + (int64_t)row * kF + 2 * t, c0[2] + c1[2], c0[3] + c1[3]);
            }
        }
    }
    __syncwarp();
}

// Where a point's coordinates come from, and the sign its prediction is stored with.
struct BatchCoords {        // P.coord [n, 3]
    __device__ __forceinline__ void load(const StepParams& P, int64_t p, float& x, float& y, float& z) const {
        x = __ldg(P.coord + 3 * p); y = __ldg(P.coord + 3 * p + 1); z = __ldg(P.coord + 3 * p + 2);
    }
    __device__ __forceinline__ float out(float v) const { return v; }
};
struct GridCoords {         // the points of a shine_internal::BrickGrid, generated from brick id and index
    shine_internal::BrickGrid g;
    __device__ __forceinline__ void load(const StepParams&, int64_t p, float& x, float& y, float& z) const {
        const int n1 = g.n + 1, per = n1 * n1 * n1;
        const int64_t b = p / per;
        const int r = (int)(p - b * per);
        const int i = r / (n1 * n1), j = (r / n1) % n1, k = r % n1;
        x = __fadd_rn(g.origin[0], __fmul_rn(g.spacing, (float)(__ldg(g.bricks + 3 * b) * g.n + i)));
        y = __fadd_rn(g.origin[1], __fmul_rn(g.spacing, (float)(__ldg(g.bricks + 3 * b + 1) * g.n + j)));
        z = __fadd_rn(g.origin[2], __fmul_rn(g.spacing, (float)(__ldg(g.bricks + 3 * b + 2) * g.n + k)));
    }
    __device__ __forceinline__ float out(float v) const { return -v; }
};

// Minimum resident blocks/SM of the inference kernels.  The mesher's grid points are generated in the kernel (brick id and
// index from a 64-bit division, the brick origin) and that extra live state spills at SHINE_INFER_MINB's 80-register cap:
// its instantiations take 2 blocks/SM (128 registers) and do not spill.
template <class Src>
constexpr int infer_min_blocks() { return std::is_same<Src, BatchCoords>::value ? SHINE_INFER_MINB : 2; }

template <int NTF, bool TRAIN, bool DEC_GRAD, int LMAX, bool GROUPED = false, class Src = BatchCoords, int LOSS = kLossBce>
__global__ void __launch_bounds__(256, !TRAIN ? infer_min_blocks<Src>() : (DEC_GRAD && !GROUPED) ? SHINE_TRAIN_DECGRAD_MINB : SHINE_TRAIN_MINB)
sdf_fused_kernel(const __grid_constant__ StepParams P, const __grid_constant__ Src src) {
    static_assert(std::is_same<Src, BatchCoords>::value || !TRAIN, "generated coordinates are for inference only");
    static_assert(!GROUPED || TRAIN, "the grouped scatter belongs to the training kernels");
    static_assert(!DEC_GRAD || TRAIN, "decoder gradients belong to the training kernels");
    static_assert(LOSS == kLossBce || std::is_same<Src, BatchCoords>::value, "the loss belongs to labelled batches");
    static_assert(SmemPlan::kStagePerWarp >= SmemPlan::kDecGradFloats, "a warp's staging area holds its partial decoder gradient");
    static_assert(SmemPlan::kStageGrouped >= kH * kF + 3 * kH + 1, "a grouped warp's staging area holds its partial bias / dW1 gradients");
    static_assert(!(GROUPED && DEC_GRAD) ||
                      (SmemPlan::STAGE + 8 * (SmemPlan::kStageGrouped + LMAX * SmemPlan::kGroupPerLevel + SmemPlan::kW2Part)) * 4 + 1024 <=
                          227 * 1024 / SHINE_TRAIN_MINB,
                  "the grouped kernel's shared memory fits SHINE_TRAIN_MINB blocks/SM");
    extern __shared__ __align__(16) float smem[];
    uint32_t* smu = reinterpret_cast<uint32_t*>(smem);
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int g = lane >> 2, t = lane & 3, odd = t & 1, half = t >> 1;
    constexpr int kWarps = 8;

    // ---- stage decoder weights (hi/lo split) into shared memory --------------------------------------
    for (int i = tid; i < kH * kF; i += blockDim.x) {
        const int nrow = i / kF, k = i % kF;
        uint32_t hi, lo; split_tf32(P.dec.w1[i], hi, lo);
        smu[SmemPlan::W1 + i] = hi; smu[SmemPlan::W1 + kH * kF + i] = lo;
        smu[SmemPlan::W1T + k * kWS + nrow] = hi; smu[SmemPlan::W1T + kF * kWS + k * kWS + nrow] = lo;
    }
    for (int i = tid; i < kH * kH; i += blockDim.x) {
        const int nrow = i / kH, k = i % kH;
        const float w = P.dec.w2[i];
        uint32_t hi, lo; split_tf32(w, hi, lo);
        smu[SmemPlan::W2 + nrow * kWS + k] = hi; smu[SmemPlan::W2 + kH * kWS + nrow * kWS + k] = lo;
        split_tf32(__fmul_rn(P.dec.w3[nrow], w), hi, lo);
        smu[SmemPlan::W3W2T + k * kWS + nrow] = hi; smu[SmemPlan::W3W2T + kH * kWS + k * kWS + nrow] = lo;
    }
    if (tid < kH) {
        smem[SmemPlan::B1 + tid] = P.dec.b1 ? P.dec.b1[tid] : 0.f;
        smem[SmemPlan::B2 + tid] = P.dec.b2 ? P.dec.b2[tid] : 0.f;
        smem[SmemPlan::W3 + tid] = P.dec.w3[tid];
    }
    if (tid == 0) {
        smem[SmemPlan::B3] = P.dec.b3 ? P.dec.b3[0] : 0.f;
        smem[SmemPlan::GSCALE] = P.loss_scale * ((TRAIN && P.d_loss) ? __ldg(P.d_loss) : 1.0f);
    }
    constexpr int kPark = LMAX <= 4 ? 16 : 32;                           // blend factors of every level, per lane
    constexpr int kIdPark = 4 * LMAX;                                    // this lane's 4 corner rows of every level
    __syncthreads();
    // Decoder gradients, per-point kernels: every warp accumulates the whole gradient over its own tiles (SHINE_ACC_DECL).
    SHINE_ACC_DECL;
#pragma unroll
    for (int a = 0; a < 2; ++a) {
#pragma unroll
        for (int b = 0; b < 4; ++b) { dW2[a][b][0] = dW2[a][b][1] = dW2[a][b][2] = dW2[a][b][3] = 0.f; }
        dW1[a][0] = dW1[a][1] = dW1[a][2] = dW1[a][3] = 0.f;
    }
#pragma unroll
    for (int j = 0; j < 4; ++j) { db2p[j][0] = db2p[j][1] = db1p[j][0] = db1p[j][1] = dw3p[j][0] = dw3p[j][1] = 0.f; }
    // Grouped kernel: every warp contracts the tile it has just staged.  Only dW2 does not fit the registers at 2 blocks/SM:
    // it is a per-warp partial in shared memory (SmemPlan::kW2Part), read, updated and written back once per tile.
    //   dW1: dW1[2][4] as in the per-point kernels;
    //   db1: sums of the A fragments of dW1 (rows 16 mt + g, + 8), reduced over the lanes in the epilogue;
    //   db2 / w3: sums of dp over the B fragments of T (columns 8 nt + g), reduced over the lanes in the epilogue;
    //   dw3: reduced per tile to 1 column per lane (reduce_scatter_g8);  db3: lane sums.
    float dw3acc = 0.f, db2acc[4] = {0.f, 0.f, 0.f, 0.f}, db1acc[2][2] = {{0.f, 0.f}, {0.f, 0.f}};

    // hash walk: inference reads key + its 4 corner rows as one 32-byte sector per level (every lane probes every level);
    // training uses the level-split walk, because the grouped scatter needs the node slots it resolves
    constexpr bool kSectorProbe = !TRAIN;
    const bool poly = P.oct.poly_interp != 0;
    const int L = P.oct.num_levels;

    float db3p = 0.f;
    float loss_acc = 0.f;

    constexpr int kStage = SmemPlan::stage_per_warp(GROUPED);
    float* stage = smem + SmemPlan::STAGE + warp * kStage;   // only touched when DEC_GRAD
    float* stX = stage + SmemPlan::SX;
    // fragment-order staging (frag_chunk): this lane's points g, g + 8 are k-step kp, and its C-fragment columns 2t + q
    // are the chunks sq[q] of that k-step's fragments; the consumer side reads chunk fc
    const int kp = g >> 2, fc = frag_chunk(lane);
    const int sq[2] = {frag_chunk(8 * t + (g & 3)), frag_chunk(8 * t + 4 + (g & 3))};
    // GROUPED: per-warp level tables behind the staging area; the dL/dfeature tile borrows stX (dead after the wgrad section)
    float* gpt = smem + SmemPlan::STAGE + (DEC_GRAD ? 8 * kStage : 0) +
                 warp * (LMAX * SmemPlan::kGroupPerLevel + (DEC_GRAD ? 0 : kTile * kF));
    float* gdx = DEC_GRAD ? stX : gpt + LMAX * SmemPlan::kGroupPerLevel;
    // GROUPED with decoder gradients: this warp's dW2 partial behind the level tables; a lane only ever touches its own
    // float4 of each fragment, so no synchronisation guards it until the epilogue
    float* w2p = smem + SmemPlan::STAGE + 8 * kStage + 8 * LMAX * SmemPlan::kGroupPerLevel + warp * SmemPlan::kW2Part;
    if (DEC_GRAD && GROUPED) {
#pragma unroll
        for (int f = 0; f < 8; ++f) *reinterpret_cast<float4*>(w2p + 128 * f + 4 * lane) = make_float4(0.f, 0.f, 0.f, 0.f);
    }

    const int warp_global = blockIdx.x * kWarps + warp;
    const int warp_stride = gridDim.x * kWarps;

    // levels are normally consecutive (W, W-1, ...): then floor(2^l u) == floor(2^W u) >> (W - l) bit-exactly, so the
    // coarser Morton keys are shifts of the leaf key instead of fresh quantise + bit-interleave rounds
    bool consecutive = true;
#pragma unroll
    for (int i = 1; i < LMAX; ++i)
        if (i < L && P.oct.lv[i].level != P.oct.lv[0].level - i) consecutive = false;

    // software pipeline, depth 1: the next tile's coordinates / label are in flight (registers) while this tile computes
    float nx = 0.f, ny = 0.f, nz = 0.f, nlab = 0.f, nwgt = 1.f;
    bool nvalid = false;
    auto prefetch_inputs = [&](int tl) {
        const int64_t p = (int64_t)tl * kTile + g + 8 * odd;
        nvalid = tl < P.num_tiles && p < P.n;
        if (nvalid) {
            src.load(P, p, nx, ny, nz);
            if (P.label) nlab = __ldg(P.label + p);
            if (P.weighted) nwgt = fabsf(__ldg(P.weight + p));   // shine_batch.py:172 abs()
        }
    };
    prefetch_inputs(warp_global);

    // Zero-tile shortcut.  A point that misses every level has the feature vector 0, so every such point gets the
    // SAME prediction pred0 = Decoder.sdf(0), and its decoder gradients are dL/dpred times the gradient g0 of that one
    // forward: linear in dL/dpred.  In a Morton-ordered batch free-space samples fill whole tiles (35 % of the C2 tiles):
    // such a tile only walks the hash, evaluates its loss terms against pred0 and adds its dL/dpred to a sum.  Pass 0 of
    // the loop below is one virtual tile (no points: features 0) run through the forward to get pred0; the epilogue adds
    // the block's dL/dpred sum times g0 in closed form (zero_tile_gradient).
    int phase = 0;                          // 0: virtual forward, 1: this warp's tiles
    bool advance = false;
    // Inference kernels only: an exit flag that never becomes true (phase is never 2).  The loop had a third pass (a virtual backward tile, now
    // the closed form above) that ended it through this flag; without its test ptxas lays the inference loop out anew
    // and spills inside it (<3,0,0,4,BatchCoords>: 52 B).  With it their SASS is the one they had.  The training kernels
    // do better without it (the grouped kernel spills nothing).
    bool infer_exit = false;
    float pred0 = 0.f, zsum = 0.f;
    // one sample's loss term li (the caller weights it) and dL/dpred dp (weighted and scaled)
    auto loss_point = [&](float pv, float lb, float wg, float& li, float& dp) {
        if constexpr (LOSS == kLossBce) {
            // MUFU-based exp / log / reciprocal (~2 ulp): |d loss| <~ 1e-7, far inside the 2e-5 parity tolerance
            const float zt = __fdividef(1.0f, 1.0f + __expf(-__fdividef(lb, P.sigma)));   // sigmoid(label / sigma)
            const float e = __expf(-fabsf(pv));
            li = fmaxf(pv, 0.f) - pv * zt + __logf(1.0f + e);                               // log1p(e), e in (0, 1]
            dp = 0.f;
            if (TRAIN) {
                const float rs = __fdividef(1.0f, 1.0f + e);
                const float sg = pv >= 0.f ? rs : e * rs;                                   // sigmoid(pred)
                dp = (sg - zt) * wg * smem[SmemPlan::GSCALE];
            }
        } else {
            float dli;
            diff_point<LOSS>(pv, lb, P.scale, li, dli);
            dp = TRAIN ? dli * wg * smem[SmemPlan::GSCALE] : 0.f;
        }
    };
    for (int seq = warp_global;; seq = advance ? seq + warp_stride : seq) {
        if (!TRAIN && infer_exit) break;
        const int tile = seq;
        if (phase == 1 && seq >= P.num_tiles) break;
        const bool virt = phase != 1;
        if (!TRAIN) infer_exit = phase == 2;
        advance = !virt;
        const int64_t base = (int64_t)tile * kTile;
        const int64_t myp = base + g + 8 * odd;
        const bool valid = virt ? false : nvalid;
        const float x = nx, y = ny, z = nz, lab = nlab, wgt = nwgt;
        if (!virt) prefetch_inputs(seq + warp_stride);

        float feat[4];
        float pk[kPark];      // [3i..3i+2] = tx,ty,tz of level i (kept over the MLP phase for the scatter)
        float idp[kIdPark];   // [4i..4i+3] = rows of this lane's corners (z bit == half) of level i, -1 on a miss
        uint32_t hitmask = 0;
        if constexpr (kSectorProbe) {
        // ---- hash walk + 8-corner gather + blend, summed over levels (model/feature_octree.py:199-234).
        //      The two lanes of a point split the CORNERS by z bit: lane `half` reads sector `half` of the first-probe
        //      slot of EVERY level with one 256-bit load (key + its 4 corner rows; all levels in flight together), then
        //      fetches those rows whole (one LDG.256 each; the pair's two loads of one instruction hit z-neighbours =
        //      consecutive table rows, usually one 128-byte line) and blends all 8 channels.  The partial sums are
        //      exchanged so that each lane ends with the 4 channels of its row-half. ----
        {
            float acc[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
#pragma unroll
            for (int i = 0; i < kPark; ++i) pk[i] = 0.f;
            const unsigned long long key0 = valid ? morton_of(x, y, z, P.oct.lv[0].level) : 0ull;
#pragma unroll
            for (int g0 = 0; g0 < LMAX; g0 += kGatherGroup) {
                SlotSector sec[kGatherGroup];
#pragma unroll
                for (int j = 0; j < kGatherGroup; ++j) {
                    const int i = g0 + j;
                    if (i < L && valid) {
                        const shine_level& lv = P.oct.lv[i];
                        const unsigned long long kq = consecutive ? (key0 >> (3 * i)) : morton_of(x, y, z, lv.level);
                        sec[j] = ldg_sector(reinterpret_cast<const HashSlot*>(lv.hash_slots),
                                            hash_key(kq) & (lv.hash_capacity - 1), half);
                    }
                }
#pragma unroll
                for (int j = 0; j < kGatherGroup; ++j) {
                    const int i = g0 + j;
                    bool hit = false;
                    if (i < L && valid) {
                        const shine_level& lv = P.oct.lv[i];
                        const unsigned long long kq = consecutive ? (key0 >> (3 * i)) : morton_of(x, y, z, lv.level);
                        hit = resolve_sector(reinterpret_cast<const HashSlot*>(lv.hash_slots), lv.hash_capacity - 1, kq, half,
                                             sec[j]);
                    }
                    idp[4 * i] = __int_as_float(hit ? sec[j].ids[0] : -1); idp[4 * i + 1] = __int_as_float(hit ? sec[j].ids[1] : -1);
                    idp[4 * i + 2] = __int_as_float(hit ? sec[j].ids[2] : -1); idp[4 * i + 3] = __int_as_float(hit ? sec[j].ids[3] : -1);
                    if (hit) {
                        const shine_level& lv = P.oct.lv[i];
                        hitmask |= 1u << i;
                        float r0[8], r1[8], r2[8], r3[8];
                        ldg_row8(lv.features + (int64_t)sec[j].ids[0] * kF, r0);
                        ldg_row8(lv.features + (int64_t)sec[j].ids[1] * kF, r1);
                        ldg_row8(lv.features + (int64_t)sec[j].ids[2] * kF, r2);
                        ldg_row8(lv.features + (int64_t)sec[j].ids[3] * kF, r3);
                        Blend b; b.init(x, y, z, lv.level, poly);
                        pk[3 * i] = b.tx; pk[3 * i + 1] = b.ty; pk[3 * i + 2] = b.tz;
                        const float wz = half ? b.tz : b.uz;
                        const float w0 = __fmul_rn(__fmul_rn(b.ux, b.uy), wz), w1 = __fmul_rn(__fmul_rn(b.ux, b.ty), wz);
                        const float w2 = __fmul_rn(__fmul_rn(b.tx, b.uy), wz), w3 = __fmul_rn(__fmul_rn(b.tx, b.ty), wz);
                        blend4(acc, r0, r1, r2, r3, w0, w1, w2, w3);
                    }
                }
            }
#pragma unroll
            for (int q = 0; q < 4; ++q) {
                const float send = half ? acc[q] : acc[4 + q];
                const float recv = __shfl_xor_sync(kFull, send, 2);
                feat[q] = (half ? acc[4 + q] : acc[q]) + recv;
            }
        }
        } else {
        // ---- hash walk (model/feature_octree.py:199-218).  The two lanes of a point split the LEVELS: lane `half`
        //      probes levels half, half+2, ... (first-probe keys of all its levels in flight together), then the
        //      pair exchanges slot indices.  Serial dependent probes per lane: 1 instead of L. ----
        int slot[LMAX];
        {
            constexpr int LH = LMAX / 2;
            const unsigned long long key0 = valid ? morton_of(x, y, z, P.oct.lv[0].level) : 0ull;
            unsigned long long kq[LH];
            uint4 kf[LH];          // home slot: {key lo, key hi, node, maxdisp}
            int mine[LH];
#pragma unroll
            for (int j = 0; j < LH; ++j) {
                const int i = 2 * j + half;
                mine[j] = -1;
                if (i < L && valid) {
                    const shine_level& lv = P.oct.lv[i];
                    const HashSlot* slots = reinterpret_cast<const HashSlot*>(lv.hash_slots);
                    kq[j] = consecutive ? (key0 >> (3 * i)) : morton_of(x, y, z, lv.level);
                    mine[j] = (int)(hash_key(kq[j]) & (lv.hash_capacity - 1));
                    kf[j] = __ldg(reinterpret_cast<const uint4*>(slots + mine[j]));
                }
            }
#pragma unroll
            for (int j = 0; j < LH; ++j) {
                const int i = 2 * j + half;
                if (i < L && valid) {
                    const unsigned long long k0 = ((unsigned long long)kf[j].y << 32) | kf[j].x;
                    if (k0 != kq[j]) {
                        // not in its home slot: a miss unless the home slot says one of its keys was displaced (rare)
                        if (k0 == kEmptyKey || (int)kf[j].w <= 0) {
                            mine[j] = -1;
                        } else {
                            const shine_level& lv = P.oct.lv[i];
                            mine[j] = probe_slot_from(reinterpret_cast<const HashSlot*>(lv.hash_slots),
                                                      lv.hash_capacity - 1, kq[j], (uint32_t)mine[j], (int)kf[j].w);
                        }
                    }
                }
            }
            __syncwarp();
#pragma unroll
            for (int j = 0; j < LH; ++j) {
                const int other = __shfl_xor_sync(kFull, mine[j], 2);
                slot[2 * j] = half ? other : mine[j];
                slot[2 * j + 1] = half ? mine[j] : other;
            }
        }

        // ---- 8-corner gather + blend, summed over levels (model/feature_octree.py:222-234).  The pair splits the
        //      CORNERS: lane `half` fetches the corners with z bit == half as whole 32-byte rows (one LDG.256 each) and
        //      blends all 8 channels; the two partial sums are then exchanged so that each lane ends with the 4
        //      channels of its row-half. ----
        {
            float acc[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
#pragma unroll
            for (int i = 0; i < kPark; ++i) pk[i] = 0.f;
#pragma unroll
            for (int i = 0; i < kIdPark; ++i) idp[i] = __int_as_float(-1);
#pragma unroll
            for (int i = 0; i < LMAX; ++i) {
                if (GROUPED && i < L && half) gpt[i * SmemPlan::kGroupPerLevel + 48 + group_slot(g + 8 * odd)] = __int_as_float(slot[i]);
                if (i < L && slot[i] >= 0) {
                    const shine_level& lv = P.oct.lv[i];
                    const HashSlot* slots = reinterpret_cast<const HashSlot*>(lv.hash_slots);
                    hitmask |= 1u << i;
                    const int4 id4 = ldg_i4(slot_ids(slots, slot[i], half));
                    idp[4 * i] = __int_as_float(id4.x); idp[4 * i + 1] = __int_as_float(id4.y);
                    idp[4 * i + 2] = __int_as_float(id4.z); idp[4 * i + 3] = __int_as_float(id4.w);
                    float r0[8], r1[8], r2[8], r3[8];
                    ldg_row8(lv.features + (int64_t)id4.x * kF, r0);
                    ldg_row8(lv.features + (int64_t)id4.y * kF, r1);
                    ldg_row8(lv.features + (int64_t)id4.z * kF, r2);
                    ldg_row8(lv.features + (int64_t)id4.w * kF, r3);
                    Blend b; b.init(x, y, z, lv.level, poly);
                    pk[3 * i] = b.tx; pk[3 * i + 1] = b.ty; pk[3 * i + 2] = b.tz;
                    if (GROUPED) {
                        float* lt = gpt + i * SmemPlan::kGroupPerLevel + group_slot(g + 8 * odd);
                        if (half) lt[32] = b.tz; else { lt[0] = b.tx; lt[16] = b.ty; }
                    }
                    const float wz = half ? b.tz : b.uz;
                    const float w0 = __fmul_rn(__fmul_rn(b.ux, b.uy), wz), w1 = __fmul_rn(__fmul_rn(b.ux, b.ty), wz);
                    const float w2 = __fmul_rn(__fmul_rn(b.tx, b.uy), wz), w3 = __fmul_rn(__fmul_rn(b.tx, b.ty), wz);
                    blend4(acc, r0, r1, r2, r3, w0, w1, w2, w3);
                }
            }
#pragma unroll
            for (int q = 0; q < 4; ++q) {
                const float send = half ? acc[q] : acc[4 + q];
                const float recv = __shfl_xor_sync(kFull, send, 2);
                feat[q] = (half ? acc[4 + q] : acc[q]) + recv;
            }
        }
        }
        if (phase == 1 && __ballot_sync(kFull, hitmask != 0u) == 0u) {
            // no point of this tile sees a node on any level: features 0, prediction pred0, no table gradient; the decoder
            // gradients follow by linearity from the sum of dL/dpred (g0 in the epilogue)
            if (!TRAIN && P.mask && half == 0 && valid) P.mask[myp] = 0;
            if (P.pred && half == 0 && valid) P.pred[myp] = src.out(pred0);
            if (P.label != nullptr && valid) {
                float li, dpz;
                loss_point(pred0, lab, wgt, li, dpz);
                if (half == 0) { loss_acc += wgt * li; zsum += dpz; }
            }
            continue;
        }
        if (!TRAIN && P.mask) {
            bool present = false;
#pragma unroll
            for (int i = 0; i < LMAX; ++i) present = (i == P.mask_level) ? (((hitmask >> i) & 1u) != 0) : present;
            if (half == 0 && valid) P.mask[myp] = (uint8_t)present;
        }

        // ---- Decoder.sdf forward (model/decoder.py:49-63) on tensor cores -----------------------------
        AFrag<NTF> ax;
        {
            float a[4]; to_afrag(feat, odd, a);
            ax.set(a[0], a[1], a[2], a[3]);
        }
        // operands of the weight-gradient contraction go to this warp's shared-memory staging (fragment order) the moment
        // they are produced (feat -> SX, h1 -> SB2 or, grouped, SU, dh2 -> SA2, dh1 -> SA1) so that they do not pin registers.
        // feat (row-half layout): point g + 8 odd is k-slot odd of chunk (4 half + q) * 4 + (g & 3) of k-step kp.
        if (DEC_GRAD) {
#pragma unroll
            for (int q = 0; q < 4; ++q) stX[xfrag_word(kp, frag_chunk(16 * half + 4 * q + (g & 3))) + odd] = feat[q];
        }
        float h1[4][4];
        uint32_t m1 = 0;   // ReLU mask of h1: bit 4j+r
        {
            uint2 bh[4], bl[4];
#pragma unroll
            for (int j = 0; j < 4; ++j) {
                const float bA = smem[SmemPlan::B1 + 8 * j + 2 * t], bB = smem[SmemPlan::B1 + 8 * j + 2 * t + 1];
                h1[j][0] = bA; h1[j][1] = bB; h1[j][2] = bA; h1[j][3] = bB;
                const int off = (8 * j + g) * kF + 2 * t;
                bh[j] = *reinterpret_cast<const uint2*>(smu + SmemPlan::W1 + off);
                bl[j] = *reinterpret_cast<const uint2*>(smu + SmemPlan::W1 + kH * kF + off);
            }
            mma3x4<NTF>(h1, ax, bh, bl);
#pragma unroll
            for (int j = 0; j < 4; ++j) {
#pragma unroll
                for (int r = 0; r < 4; ++r) {
                    if (TRAIN && h1[j][r] > 0.f) m1 |= 1u << (4 * j + r);
                    h1[j][r] = fmaxf(h1[j][r], 0.f);
                }
                if (DEC_GRAD && !GROUPED) {
#pragma unroll
                    for (int q = 0; q < 2; ++q)
                        *reinterpret_cast<float2*>(stage + SmemPlan::SB2 + (4 * kp + j) * 64 + 2 * sq[q]) = make_float2(h1[j][q], h1[j][2 + q]);
                }
            }
            if (DEC_GRAD && GROUPED) stage_afrags(stage + SmemPlan::SU + 256 * kp, sq, h1);
        }
        float h2[4][4];
        {
#pragma unroll
            for (int j = 0; j < 4; ++j) {
                const float bA = smem[SmemPlan::B2 + 8 * j + 2 * t], bB = smem[SmemPlan::B2 + 8 * j + 2 * t + 1];
                h2[j][0] = bA; h2[j][1] = bB; h2[j][2] = bA; h2[j][3] = bB;
            }
#pragma unroll
            for (int kk = 0; kk < 4; ++kk) {
                AFrag<NTF> a; a.set(h1[kk][0], h1[kk][2], h1[kk][1], h1[kk][3]);
                uint2 bh[4], bl[4];
#pragma unroll
                for (int j = 0; j < 4; ++j) {
                    const int off = (8 * j + g) * kWS + 8 * kk + 2 * t;
                    bh[j] = *reinterpret_cast<const uint2*>(smu + SmemPlan::W2 + off);
                    bl[j] = *reinterpret_cast<const uint2*>(smu + SmemPlan::W2 + kH * kWS + off);
                }
                mma3x4<NTF>(h2, a, bh, bl);
            }
#pragma unroll
            for (int j = 0; j < 4; ++j) {
#pragma unroll
                for (int r = 0; r < 4; ++r) h2[j][r] = fmaxf(h2[j][r], 0.f);
            }
        }
        float w3a[4], w3b[4];
#pragma unroll
        for (int j = 0; j < 4; ++j) { w3a[j] = smem[SmemPlan::W3 + 8 * j + 2 * t]; w3b[j] = smem[SmemPlan::W3 + 8 * j + 2 * t + 1]; }
        float p0 = 0.f, p8 = 0.f;   // rows g and g+8
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            p0 = fmaf(h2[j][0], w3a[j], p0); p0 = fmaf(h2[j][1], w3b[j], p0);
            p8 = fmaf(h2[j][2], w3a[j], p8); p8 = fmaf(h2[j][3], w3b[j], p8);
        }
        p0 += __shfl_xor_sync(kFull, p0, 1); p0 += __shfl_xor_sync(kFull, p0, 2);
        p8 += __shfl_xor_sync(kFull, p8, 1); p8 += __shfl_xor_sync(kFull, p8, 2);
        const float b3 = smem[SmemPlan::B3];
        p0 += b3; p8 += b3;
        const float pown = odd ? p8 : p0;
        if (phase == 0) { pred0 = pown; phase = 1; continue; }     // the virtual forward: every row is Decoder.sdf(0)
        if (P.pred && half == 0 && valid) P.pred[myp] = src.out(pown);

        if (P.label == nullptr) continue;   // pure inference

        // ---- sdf_bce_loss (utils/loss.py:17-24) or sdf_diff_loss (:6-14) + dL/dpred -------------------------
        float dpo = 0.f;
        if (valid) {
            float li;
            loss_point(pown, lab, wgt, li, dpo);
            if (half == 0) loss_acc += wgt * li;
        }
        if (!TRAIN) continue;

        // ---- backward: MLP dgrad on tensor cores ------------------------------------------------------
        const float dpx = __shfl_xor_sync(kFull, dpo, 1);
        const float dp0 = odd ? dpx : dpo, dp8 = odd ? dpo : dpx;
        float db1t[4][2], dw3t[4][2];   // this tile's partials (rows g, g+8)
        if (DEC_GRAD) {
#pragma unroll
            for (int j = 0; j < 4; ++j) { dw3t[j][0] = dp0 * h2[j][0] + dp8 * h2[j][2];  dw3t[j][1] = dp0 * h2[j][1] + dp8 * h2[j][3]; }
        }
        if (DEC_GRAD && !GROUPED) {
            // dh2 = dL/dpred * w3 where h2 > 0, the A operand of this kernel's dW2 contraction
            float dh2[4][4];
#pragma unroll
            for (int j = 0; j < 4; ++j) {
                dh2[j][0] = h2[j][0] > 0.f ? dp0 * w3a[j] : 0.f; dh2[j][1] = h2[j][1] > 0.f ? dp0 * w3b[j] : 0.f;
                dh2[j][2] = h2[j][2] > 0.f ? dp8 * w3a[j] : 0.f; dh2[j][3] = h2[j][3] > 0.f ? dp8 * w3b[j] : 0.f;
                db2p[j][0] += dh2[j][0] + dh2[j][2]; db2p[j][1] += dh2[j][1] + dh2[j][3];
            }
            stage_afrags(stage + SmemPlan::SA2 + 256 * kp, sq, dh2);
        }
        if (DEC_GRAD && GROUPED) {
            // per point its dL/dpred and the 32-bit ReLU mask of its h2 row are staged instead of the 512 values of dh2
            // (the four lanes of equal g hold 8 columns each of rows g and g + 8)
            uint32_t mg = 0, mg8 = 0;
#pragma unroll
            for (int j = 0; j < 4; ++j)
#pragma unroll
                for (int q = 0; q < 2; ++q) {
                    mg |= (h2[j][q] > 0.f ? 1u : 0u) << (8 * j + 2 * t + q);
                    mg8 |= (h2[j][2 + q] > 0.f ? 1u : 0u) << (8 * j + 2 * t + q);
                }
            mg |= __shfl_xor_sync(kFull, mg, 1); mg8 |= __shfl_xor_sync(kFull, mg8, 1);
            mg |= __shfl_xor_sync(kFull, mg, 2); mg8 |= __shfl_xor_sync(kFull, mg8, 2);
            if (t == 0) {
                *reinterpret_cast<float2*>(stage + SmemPlan::SDP + 2 * g) = make_float2(dp0, __uint_as_float(mg));
                *reinterpret_cast<float2*>(stage + SmemPlan::SDP + 2 * (g + 8)) = make_float2(dp8, __uint_as_float(mg8));
            }
        }
        if (DEC_GRAD && t == 0) db3p += dp0 + dp8;

        // dh1 = dp * (M2 W2') with M2 = [h2 > 0] and W2' = diag(w3) W2 (SmemPlan::W3W2T): M2 is exact in tf32, so 3xTF32
        // takes two products, and each row is scaled by its dL/dpred afterwards
        float dh1[4][4];
        {
#pragma unroll
            for (int j = 0; j < 4; ++j) { dh1[j][0] = dh1[j][1] = dh1[j][2] = dh1[j][3] = 0.f; }
#pragma unroll
            for (int kk = 0; kk < 4; ++kk) {
                const uint32_t a[4] = {h2[kk][0] > 0.f ? kTf32One : 0u, h2[kk][2] > 0.f ? kTf32One : 0u,
                                       h2[kk][1] > 0.f ? kTf32One : 0u, h2[kk][3] > 0.f ? kTf32One : 0u};
                uint2 bh[4], bl[4];
#pragma unroll
                for (int j = 0; j < 4; ++j) {
                    const int off = (8 * j + g) * kWS + 8 * kk + 2 * t;
                    bh[j] = *reinterpret_cast<const uint2*>(smu + SmemPlan::W3W2T + off);
                    bl[j] = *reinterpret_cast<const uint2*>(smu + SmemPlan::W3W2T + kH * kWS + off);
                }
                mma2x4_exact_a<NTF>(dh1, a, bh, bl);
            }
#pragma unroll
            for (int j = 0; j < 4; ++j) {
                dh1[j][0] *= dp0; dh1[j][1] *= dp0; dh1[j][2] *= dp8; dh1[j][3] *= dp8;
#pragma unroll
                for (int r = 0; r < 4; ++r) dh1[j][r] = ((m1 >> (4 * j + r)) & 1u) ? dh1[j][r] : 0.f;
                if (DEC_GRAD) { db1t[j][0] = dh1[j][0] + dh1[j][2]; db1t[j][1] = dh1[j][1] + dh1[j][3]; }
            }
            if (DEC_GRAD) stage_afrags(stage + SmemPlan::SA1 + 256 * kp, sq, dh1);
        }
        float dxc[4] = {0.f, 0.f, 0.f, 0.f};
        {
            float dxo[4] = {0.f, 0.f, 0.f, 0.f};   // odd k-chunks: two interleaved accumulation chains instead of one
#pragma unroll
            for (int kk = 0; kk < 4; kk += 2) {
                AFrag<NTF> a0, a1;
                a0.set(dh1[kk][0], dh1[kk][2], dh1[kk][1], dh1[kk][3]);
                a1.set(dh1[kk + 1][0], dh1[kk + 1][2], dh1[kk + 1][1], dh1[kk + 1][3]);
                const int off = g * kWS + 8 * kk + 2 * t;
                const uint2 bh0 = *reinterpret_cast<const uint2*>(smu + SmemPlan::W1T + off);
                const uint2 bl0 = *reinterpret_cast<const uint2*>(smu + SmemPlan::W1T + kF * kWS + off);
                const uint2 bh1 = *reinterpret_cast<const uint2*>(smu + SmemPlan::W1T + off + 8);
                const uint2 bl1 = *reinterpret_cast<const uint2*>(smu + SmemPlan::W1T + kF * kWS + off + 8);
                mma3x2<NTF>(dxc, dxo, a0, a1, bh0, bl0, bh1, bl1);
            }
#pragma unroll
            for (int r = 0; r < 4; ++r) dxc[r] += dxo[r];
        }

        // ---- backward: decoder weight grads ------------------------------------------------------------------------
        if (DEC_GRAD && !GROUPED) {       // contraction over the tile's 16 points
#pragma unroll
            for (int j = 0; j < 4; ++j) {
                db1p[j][0] += db1t[j][0]; db1p[j][1] += db1t[j][1];
                dw3p[j][0] += dw3t[j][0]; dw3p[j][1] += dw3t[j][1];
            }
            __syncwarp();
            // dW2[n2][k1] += sum_rows dh2[row][n2] * h1[row][k1]
#pragma unroll
            for (int ks = 0; ks < 2; ++ks) {
                uint2 bh[4], bl[4];
#pragma unroll
                for (int nt = 0; nt < 4; ++nt) load_bfrag(stage + SmemPlan::SB2 + (4 * ks + nt) * 64, fc, bh[nt], bl[nt]);
#pragma unroll
                for (int mt = 0; mt < 2; ++mt) {
                    AFrag<NTF> a;
                    load_afrag(stage + SmemPlan::SA2 + (2 * ks + mt) * 128, fc, a);
                    mma3x4<NTF>(dW2[mt], a, bh, bl);
                }
            }
            // dW1[n1][ch] += sum_rows dh1[row][n1] * feat[row][ch]
#pragma unroll
            for (int ks = 0; ks < 2; ++ks) {
                uint2 bh, bl;
                load_xfrag(stX, ks, fc, bh, bl);
                AFrag<NTF> a0, a1;
                load_afrag(stage + SmemPlan::SA1 + (2 * ks) * 128, fc, a0);
                load_afrag(stage + SmemPlan::SA1 + (2 * ks + 1) * 128, fc, a1);
                mma3x2<NTF>(dW1[0], dW1[1], a0, a1, bh, bl, bh, bl);
            }
            __syncwarp();
        }
        if (DEC_GRAD && GROUPED) {        // the same contraction, dW2 accumulated into this warp's shared-memory partial
            float cols[8];   // slot 2j + q: column 8j + 2t + q of dw3
#pragma unroll
            for (int j = 0; j < 4; ++j) { cols[2 * j] = dw3t[j][0]; cols[2 * j + 1] = dw3t[j][1]; }
            dw3acc += reduce_scatter_g8(cols, lane);    // column 8 (g >> 1) + 2t + (g & 1)
            __syncwarp();
            // dW2[n2][k1] = w3[n2] T[k1][n2] with T[k1][n2] = sum_rows u[row][k1] M2[row][n2], u = dp h1, M2 = [h2 > 0];
            // w3 is applied in the epilogue.  T runs one m-tile at a time (16 accumulators).  A (rows k1 = 16 mt + g, + 8;
            // k-slots = points 4 ks + t, + 8) is the forward's h1, scaled by the two points' dp as it is loaded; B (same
            // k-slots, n2 = 8 nt + g) is the 0/1 mask, exact in tf32, so 3xTF32 takes two products
            float dpk[2][2];
            uint32_t mk[2][2];   // the points' masks, shifted to column g
#pragma unroll
            for (int ks = 0; ks < 2; ++ks) {
                const float2 e0 = *reinterpret_cast<const float2*>(stage + SmemPlan::SDP + 2 * (4 * ks + t));
                const float2 e8 = *reinterpret_cast<const float2*>(stage + SmemPlan::SDP + 2 * (4 * ks + t + 8));
                dpk[ks][0] = e0.x; dpk[ks][1] = e8.x;
                mk[ks][0] = __float_as_uint(e0.y) >> g; mk[ks][1] = __float_as_uint(e8.y) >> g;
#pragma unroll
                for (int nt = 0; nt < 4; ++nt)   // db2[n2] / w3[n2]: the mask's column sums weighted by dp
                    db2acc[nt] += ((mk[ks][0] >> (8 * nt)) & 1u ? dpk[ks][0] : 0.f) + ((mk[ks][1] >> (8 * nt)) & 1u ? dpk[ks][1] : 0.f);
            }
#pragma unroll
            for (int mt = 0; mt < 2; ++mt) {
                float acc[4][4];
#pragma unroll
                for (int nt = 0; nt < 4; ++nt) {
                    const float4 v = *reinterpret_cast<const float4*>(w2p + 128 * (4 * mt + nt) + 4 * lane);
                    acc[nt][0] = v.x; acc[nt][1] = v.y; acc[nt][2] = v.z; acc[nt][3] = v.w;
                }
#pragma unroll
                for (int ks = 0; ks < 2; ++ks) {
                    uint2 b[4];
#pragma unroll
                    for (int nt = 0; nt < 4; ++nt) {
                        b[nt].x = (mk[ks][0] >> (8 * nt)) & 1u ? kTf32One : 0u;
                        b[nt].y = (mk[ks][1] >> (8 * nt)) & 1u ? kTf32One : 0u;
                    }
                    const float4 v = *reinterpret_cast<const float4*>(stage + SmemPlan::SU + (2 * ks + mt) * 128 + 4 * fc);
                    AFrag<NTF> af;
                    af.set_packed(v.x * dpk[ks][0], v.y * dpk[ks][0], v.z * dpk[ks][1], v.w * dpk[ks][1]);
                    mma2x4_exact_b<NTF>(acc, af, b);
                }
#pragma unroll
                for (int nt = 0; nt < 4; ++nt)
                    *reinterpret_cast<float4*>(w2p + 128 * (4 * mt + nt) + 4 * lane) = make_float4(acc[nt][0], acc[nt][1], acc[nt][2], acc[nt][3]);
            }
            // dW1[n1][ch] += sum_rows dh1[row][n1] * feat[row][ch]
#pragma unroll
            for (int ks = 0; ks < 2; ++ks) {
                uint2 bh, bl;
                load_xfrag(stX, ks, fc, bh, bl);
                AFrag<NTF> a[2];
#pragma unroll
                for (int mt = 0; mt < 2; ++mt) {
                    const float4 av = *reinterpret_cast<const float4*>(stage + SmemPlan::SA1 + (2 * ks + mt) * 128 + 4 * fc);
                    db1acc[mt][0] += av.x + av.z; db1acc[mt][1] += av.y + av.w;
                    a[mt].set_packed(av.x, av.y, av.z, av.w);
                }
                mma3x2<NTF>(dW1[0], dW1[1], a[0], a[1], bh, bl, bh, bl);
            }
            __syncwarp();
        }

        // ---- backward: scatter-add into the corner-feature tables (index_put_ accumulate) -------------
        if constexpr (GROUPED) {
            grouped_scatter<LMAX>(P, L, tile, gpt, gdx, dxc, lane);
            continue;
        }
        float dx[4];
        from_cfrag(dxc, odd, dx);
        const float (&qk)[kPark] = pk;
        const float (&qid)[kIdPark] = idp;
#pragma unroll
        for (int i = 0; i < LMAX; ++i) {
            // the 8 corner rows: this lane kept the 4 with z bit == half, its partner (lane ^ 2) the other 4
            int ids[8];
#pragma unroll
            for (int k = 0; k < 4; ++k) {
                const int mine = __float_as_int(qid[4 * i + k]);
                const int other = __shfl_xor_sync(kFull, mine, 2);
                ids[2 * k] = half ? other : mine;
                ids[2 * k + 1] = half ? mine : other;
            }
            if (i < L && ids[0] >= 0) {      // a miss parked -1 for all of its rows
                const shine_level& lv = P.oct.lv[i];
                Blend b;
                b.tx = qk[3 * i]; b.ty = qk[3 * i + 1]; b.tz = qk[3 * i + 2];
                b.ux = __fsub_rn(1.0f, b.tx); b.uy = __fsub_rn(1.0f, b.ty); b.uz = __fsub_rn(1.0f, b.tz);
                float* gb = grad_base(lv, (uint32_t)tile, kF) + 4 * half;
                // w_c = (X * Y) * Z in the reference's association; the four X*Y products are shared by the z pair
                const float xy[4] = {__fmul_rn(b.ux, b.uy), __fmul_rn(b.ux, b.ty), __fmul_rn(b.tx, b.uy), __fmul_rn(b.tx, b.ty)};
                const f2_t zz = f2_pack(b.uz, b.tz), dx01 = f2_pack(dx[0], dx[1]), dx23 = f2_pack(dx[2], dx[3]);
#pragma unroll
                for (int c = 0; c < 8; c += 2) {
                    float w[2];
                    f2_unpack(f2_mul(f2_pack(xy[c >> 1], xy[c >> 1]), zz), w[0], w[1]);    // (X*Y)*uz, (X*Y)*tz
#pragma unroll
                    for (int k = 0; k < 2; ++k) {
                        const f2_t wk = f2_pack(w[k], w[k]);
                        float g0, g1, g2, g3;
                        f2_unpack(f2_mul(wk, dx01), g0, g1); f2_unpack(f2_mul(wk, dx23), g2, g3);
                        red_add_f4(gb + (int64_t)ids[c + k] * kF, g0, g1, g2, g3);
                    }
                }
            }
        }
    }

    // ---- epilogue: loss and decoder-gradient reductions --------------------------------------------------
    if (P.loss && P.label) {
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) loss_acc += __shfl_xor_sync(kFull, loss_acc, o);
        if (lane == 0 && loss_acc != 0.f) atomicAdd(P.loss, loss_acc * P.loss_scale);
    }
    if (DEC_GRAD) {       // this warp's dL/dpred sum over its zero tiles: the block adds their sum times g0 below
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) zsum += __shfl_xor_sync(kFull, zsum, o);
        if (lane == 0) smem[SmemPlan::ZSUM + warp] = zsum;
    }
    if (DEC_GRAD && GROUPED) {
        // per-warp partials [gw1 256 | gb1 32 | gb2 32 | gw3 32 | gb3 1] in the staging area (each element has exactly one
        // owner lane) and dW2 in its C-fragment image; the block sums the eight partials of each element and issues one
        // global atomic per non-zero element
        float* part = stage;
        constexpr int oB1 = 256, oB2 = 288, oW3 = 320, oB3 = 352, kVec = 353;
#pragma unroll
        for (int mt = 0; mt < 2; ++mt) {
            *reinterpret_cast<float2*>(part + (16 * mt + g) * kF + 2 * t) = make_float2(dW1[mt][0], dW1[mt][1]);
            *reinterpret_cast<float2*>(part + (16 * mt + g + 8) * kF + 2 * t) = make_float2(dW1[mt][2], dW1[mt][3]);
#pragma unroll
            for (int r = 0; r < 2; ++r) {   // db1 rows 16 mt + g + 8 r / db2 columns 8 (2 mt + r) + g: sums over this lane's
                float d1 = db1acc[mt][r], d2 = db2acc[2 * mt + r];   // k-slots, then over the 4 lanes of equal g
#pragma unroll
                for (int o = 1; o < 4; o <<= 1) { d1 += __shfl_xor_sync(kFull, d1, o); d2 += __shfl_xor_sync(kFull, d2, o); }
                if (t == 0) { part[oB1 + 16 * mt + g + 8 * r] = d1; part[oB2 + 8 * (2 * mt + r) + g] = d2; }
            }
        }
        part[oW3 + 8 * (g >> 1) + 2 * t + (g & 1)] = dw3acc;
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) db3p += __shfl_xor_sync(kFull, db3p, o);
        if (lane == 0) part[oB3] = db3p;
        __syncthreads();
        const float zs = zero_tile_sum_and_gradient(smem, P.dec.w2, warp, lane);
        for (int i = tid; i < kVec + kH * kH; i += blockDim.x) {
            float v = 0.f, g0 = 0.f;   // g0: this element's gradient of Decoder.sdf(0) (dW1: 0)
            float* dst;
            if (i < kVec) {
#pragma unroll
                for (int w = 0; w < kWarps; ++w) v += smem[SmemPlan::STAGE + w * kStage + i];
                if (i < oB1) dst = P.dec.gw1 + i;
                else if (i < oB2) { g0 = smem[SmemPlan::DB1Z + (i - oB1)]; dst = P.dec.gb1 ? P.dec.gb1 + (i - oB1) : nullptr; }
                else if (i < oW3) {
                    v *= smem[SmemPlan::W3 + (i - oB2)]; g0 = smem[SmemPlan::D2Z + (i - oB2)];
                    dst = P.dec.gb2 ? P.dec.gb2 + (i - oB2) : nullptr;
                } else if (i < oB3) { g0 = smem[SmemPlan::H2Z + (i - oW3)]; dst = P.dec.gw3 + (i - oW3); }
                else { g0 = 1.f; dst = P.dec.gb3; }
            } else {   // dW2[r][c] = w3[r] T[c][r]: fragment (c >> 4, r >> 3), lane 4 (c & 7) + ((r & 7) >> 1), register
                       // 2 ((c >> 3) & 1) + (r & 1)
                const int e = i - kVec, r = e / kH, c = e % kH;
                const int f = 128 * (4 * (c >> 4) + (r >> 3)) + 4 * (4 * (c & 7) + ((r & 7) >> 1)) + 2 * ((c >> 3) & 1) + (r & 1);
#pragma unroll
                for (int w = 0; w < kWarps; ++w) v += w2p[(w - warp) * SmemPlan::kW2Part + f];
                v *= smem[SmemPlan::W3 + r];
                if (zs != 0.f) g0 = smem[SmemPlan::D2Z + r] * smem[SmemPlan::H1Z + c];
                dst = P.dec.gw2 + e;
            }
            if (zs != 0.f) v = fmaf(zs, g0, v);
            if (v != 0.f && dst) atomicAdd(dst, v);
        }
    }
    if (DEC_GRAD && !GROUPED) {
        // every warp writes its complete partial gradient vector [gw1 256 | gb1 32 | gw2 1024 | gb2 32 | gw3 32 | gb3 1]
        // into its own staging area (each element has exactly one owner lane: plain stores, no shared-memory atomics),
        // then the block sums the eight vectors and issues one global atomic per non-zero element
        float* part = stage;
        constexpr int oW1 = 0, oB1 = 256, oW2 = 288, oB2 = 1312, oW3 = 1344, oB3 = 1376;
        __syncwarp();
#pragma unroll
        for (int mt = 0; mt < 2; ++mt) {
#pragma unroll
            for (int nt = 0; nt < 4; ++nt) {
                *reinterpret_cast<float2*>(part + oW2 + (16 * mt + g) * kH + 8 * nt + 2 * t) = make_float2(dW2[mt][nt][0], dW2[mt][nt][1]);
                *reinterpret_cast<float2*>(part + oW2 + (16 * mt + g + 8) * kH + 8 * nt + 2 * t) = make_float2(dW2[mt][nt][2], dW2[mt][nt][3]);
            }
            *reinterpret_cast<float2*>(part + oW1 + (16 * mt + g) * kF + 2 * t) = make_float2(dW1[mt][0], dW1[mt][1]);
            *reinterpret_cast<float2*>(part + oW1 + (16 * mt + g + 8) * kF + 2 * t) = make_float2(dW1[mt][2], dW1[mt][3]);
        }
#pragma unroll
        for (int j = 0; j < 4; ++j) {
#pragma unroll
            for (int q = 0; q < 2; ++q) {
                float a = db1p[j][q], b = db2p[j][q], c = dw3p[j][q];
#pragma unroll
                for (int o = 4; o < 32; o <<= 1) {
                    a += __shfl_xor_sync(kFull, a, o); b += __shfl_xor_sync(kFull, b, o); c += __shfl_xor_sync(kFull, c, o);
                }
                if (g == 0) {
                    part[oB1 + 8 * j + 2 * t + q] = a;
                    part[oB2 + 8 * j + 2 * t + q] = b;
                    part[oW3 + 8 * j + 2 * t + q] = c;
                }
            }
        }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) db3p += __shfl_xor_sync(kFull, db3p, o);
        if (lane == 0) part[oB3] = db3p;
        __syncthreads();
        const float zs = zero_tile_sum_and_gradient(smem, P.dec.w2, warp, lane);
        for (int i = tid; i < SmemPlan::kDecGradFloats; i += blockDim.x) {
            float v = 0.f;
#pragma unroll
            for (int w = 0; w < kWarps; ++w) v += smem[SmemPlan::STAGE + w * kStage + i];
            if (zs != 0.f && i >= oB1) {   // dW1 of a zero tile is 0
                float g0;
                if (i < oW2) g0 = smem[SmemPlan::DB1Z + (i - oB1)];
                else if (i < oB2) g0 = smem[SmemPlan::D2Z + (i - oW2) / kH] * smem[SmemPlan::H1Z + (i - oW2) % kH];
                else if (i < oW3) g0 = smem[SmemPlan::D2Z + (i - oB2)];
                else if (i < oB3) g0 = smem[SmemPlan::H2Z + (i - oW3)];
                else g0 = 1.f;
                v = fmaf(zs, g0, v);
            }
            if (v == 0.f) continue;
            float* dst;
            if (i < oB1) dst = P.dec.gw1 + i;
            else if (i < oW2) dst = P.dec.gb1 ? P.dec.gb1 + (i - oB1) : nullptr;
            else if (i < oB2) dst = P.dec.gw2 + (i - oW2);
            else if (i < oW3) dst = P.dec.gb2 ? P.dec.gb2 + (i - oB2) : nullptr;
            else if (i < oB3) dst = P.dec.gw3 + (i - oW3);
            else dst = P.dec.gb3;
            if (dst) atomicAdd(dst, v);
        }
    }
}

// ------------------------------------------------------------------------------------------------------
// fold the gradient replicas back: grads[l] += sum_r replicas[l][r]; replicas[l] = 0
// ------------------------------------------------------------------------------------------------------

__global__ void __launch_bounds__(256) reduce_replicas_kernel(const __grid_constant__ shine_octree oct) {
    const shine_level& lv = oct.lv[blockIdx.y];
    if (lv.num_replicas <= 1 || !lv.grad_replicas || !lv.feature_grads) return;
    const int64_t n4 = (int64_t)lv.rows * oct.feature_dim / 4;
    float4* main4 = reinterpret_cast<float4*>(lv.feature_grads);
    float4* rep4 = reinterpret_cast<float4*>(lv.grad_replicas);
    const float4 zero = make_float4(0.f, 0.f, 0.f, 0.f);
    const int nrep = lv.num_replicas - 1;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n4; i += (int64_t)gridDim.x * blockDim.x) {
        float4 acc = main4[i];
        int r = 0;
        for (; r + 8 <= nrep; r += 8) {          // 8 independent loads in flight per thread
            float4 v[8];
#pragma unroll
            for (int u = 0; u < 8; ++u) v[u] = rep4[(int64_t)(r + u) * n4 + i];
#pragma unroll
            for (int u = 0; u < 8; ++u) {
                acc.x += v[u].x; acc.y += v[u].y; acc.z += v[u].z; acc.w += v[u].w;
                rep4[(int64_t)(r + u) * n4 + i] = zero;
            }
        }
        for (; r < nrep; ++r) {
            const float4 v = rep4[(int64_t)r * n4 + i];
            acc.x += v.x; acc.y += v.y; acc.z += v.z; acc.w += v.w;
            rep4[(int64_t)r * n4 + i] = zero;
        }
        main4[i] = acc;
    }
}

// ------------------------------------------------------------------------------------------------------
// dense Adam over several tensors (utils/tools.py:78-79)
// ------------------------------------------------------------------------------------------------------

struct AdamParams {
    shine_adam_tensor t[SHINE_ADAM_MAX_TENSORS];
    int32_t count;
    float beta1, beta2, omb1, omb2, eps, bc1, bc2_sqrt;
    int32_t zero_grad;
    const float* bc_dev;   // optional {bc1, bc2_sqrt} on the device (graph replay); overrides bc1 / bc2_sqrt
};

struct AdamDevState { int32_t step; float bc1, bc2_sqrt; };

__global__ void adam_bump_kernel(AdamDevState* st, float beta1, float beta2) {
    const int step = st->step + 1;
    st->step = step;
    st->bc1 = (float)(1.0 - pow((double)beta1, (double)step));
    st->bc2_sqrt = (float)sqrt(1.0 - pow((double)beta2, (double)step));
}

__global__ void __launch_bounds__(256) adam_kernel(const __grid_constant__ AdamParams A) {
    const shine_adam_tensor& T = A.t[blockIdx.y];
    const int64_t n4 = T.numel >> 2;
    const float bc1 = A.bc_dev ? A.bc_dev[0] : A.bc1;
    const float bc2_sqrt = A.bc_dev ? A.bc_dev[1] : A.bc2_sqrt;
    const float step_size = T.lr / bc1;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n4; i += (int64_t)gridDim.x * blockDim.x) {
        float4 p = reinterpret_cast<float4*>(T.param)[i];
        float4 gr = reinterpret_cast<float4*>(T.grad)[i];
        float4 m = reinterpret_cast<float4*>(T.exp_avg)[i];
        float4 v = reinterpret_cast<float4*>(T.exp_avg_sq)[i];
        float* pp = &p.x; float* gg = &gr.x; float* mm = &m.x; float* vv = &v.x;
#pragma unroll
        for (int k = 0; k < 4; ++k) {
            float gk = gg[k];
            if (T.weight_decay != 0.f) gk = fmaf(T.weight_decay, pp[k], gk);
            mm[k] = mm[k] + (gk - mm[k]) * A.omb1;                          // torch lerp_
            vv[k] = A.beta2 * vv[k] + A.omb2 * gk * gk;
            const float denom = sqrtf(vv[k]) / bc2_sqrt + A.eps;
            pp[k] -= step_size * (mm[k] / denom);
        }
        reinterpret_cast<float4*>(T.param)[i] = p;
        reinterpret_cast<float4*>(T.exp_avg)[i] = m;
        reinterpret_cast<float4*>(T.exp_avg_sq)[i] = v;
        if (A.zero_grad) reinterpret_cast<float4*>(T.grad)[i] = make_float4(0.f, 0.f, 0.f, 0.f);
    }
    // tail (numel % 4) handled by the first block
    if (blockIdx.x == 0) {
        for (int64_t i = (n4 << 2) + threadIdx.x; i < T.numel; i += blockDim.x) {
            float gk = T.grad[i];
            if (T.weight_decay != 0.f) gk = fmaf(T.weight_decay, T.param[i], gk);
            const float m = T.exp_avg[i] + (gk - T.exp_avg[i]) * A.omb1;
            const float v = A.beta2 * T.exp_avg_sq[i] + A.omb2 * gk * gk;
            T.exp_avg[i] = m; T.exp_avg_sq[i] = v;
            T.param[i] -= step_size * (m / (sqrtf(v) / bc2_sqrt + A.eps));
            if (A.zero_grad) T.grad[i] = 0.f;
        }
    }
}

// ------------------------------------------------------------------------------------------------------
// host side
// ------------------------------------------------------------------------------------------------------

template <int NTF, bool TRAIN, bool DEC_GRAD, int LMAX, bool GROUPED = false, class Src = BatchCoords, int LOSS = kLossBce>
int launch_fused_t(const StepParams& P, cudaStream_t st, const Src& src = Src()) {
    auto kern = sdf_fused_kernel<NTF, TRAIN, DEC_GRAD, LMAX, GROUPED, Src, LOSS>;
    const int smem_floats = SmemPlan::STAGE + (DEC_GRAD ? 8 * SmemPlan::stage_per_warp(GROUPED) : 0) +
                            (GROUPED ? 8 * (LMAX * SmemPlan::kGroupPerLevel + (DEC_GRAD ? SmemPlan::kW2Part : kTile * kF)) : 0);
    const size_t smem_bytes = (size_t)smem_floats * sizeof(float);
    static int per_sm_by_dev[kMaxDevices] = {0};   // per template instantiation AND per device: the >48 KB dynamic
    int& per_sm_cached = per_sm_by_dev[current_device()];   // shared-memory opt-in is a per-device function attribute
    cudaError_t e;
    if (per_sm_cached == 0) {
        e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_bytes);
        if (e != cudaSuccess) return (int)e;
        e = cudaFuncSetAttribute(kern, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared);
        if (e != cudaSuccess) return (int)e;
        int q = 1;
        e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&q, kern, 256, smem_bytes);
        if (e != cudaSuccess) return (int)e;
        // the API is conservative about the shared-memory carve-out; the tile loop is grid-size agnostic, so size the
        // grid from the hardware limits directly (64K registers, 227 KB usable shared memory + 1 KB/block reserved)
        cudaFuncAttributes fa;
        e = cudaFuncGetAttributes(&fa, kern);
        if (e != cudaSuccess) return (int)e;
        const int by_regs = fa.numRegs > 0 ? 65536 / (fa.numRegs * 256) : 1;
        const int by_smem = (int)((227 * 1024) / (smem_bytes + 1024));
        int own = by_regs < by_smem ? by_regs : by_smem;
        if (own > 8) own = 8;
        if (own > q) q = own;
        per_sm_cached = q < 1 ? 1 : q;
    }
    const int per_sm = per_sm_cached;
    const int blocks_needed = (P.num_tiles + 7) / 8;
    int grid = sm_count() * per_sm;
    if (grid > blocks_needed) grid = blocks_needed;
    if (grid < 1) grid = 1;
    kern<<<grid, 256, smem_bytes, st>>>(P, src);
    return (int)cudaGetLastError();
}

template <bool TRAIN, bool DEC_GRAD, class Src = BatchCoords, int LOSS = kLossBce>
int launch_fused(const StepParams& P, uint32_t flags, cudaStream_t st, const Src& src = Src()) {
    const bool x1 = (flags & SHINE_FLAG_TF32X1) != 0;
    const bool small = P.oct.num_levels <= 4;
    if constexpr (TRAIN) {      // Morton-ordered batches: voxel-grouped scatter (3xTF32, up to 4 levels; else the general kernel)
        if ((flags & SHINE_FLAG_MORTON_ORDERED) && !x1 && small)
            return launch_fused_t<3, TRAIN, DEC_GRAD, 4, true, Src, LOSS>(P, st);
    }
    if (x1) return small ? launch_fused_t<1, TRAIN, DEC_GRAD, 4, false, Src, LOSS>(P, st, src)
                         : launch_fused_t<1, TRAIN, DEC_GRAD, 8, false, Src, LOSS>(P, st, src);
    return small ? launch_fused_t<3, TRAIN, DEC_GRAD, 4, false, Src, LOSS>(P, st, src)
                 : launch_fused_t<3, TRAIN, DEC_GRAD, 8, false, Src, LOSS>(P, st, src);
}

// the flag bits of shine_sdf_infer and of the sdf_bce loss: any other bit is SHINE_ERR_UNSUPPORTED, never silently ignored
constexpr uint32_t kSdfFlags = SHINE_FLAG_REDUCTION_SUM | SHINE_FLAG_WEIGHTED | SHINE_FLAG_TF32X1 | SHINE_FLAG_MORTON_ORDERED;

int fill_params(StepParams& P, const shine_octree* oct, const shine_decoder* dec, const float* coord, int64_t n) {
    if (n < 0 || (n > 0 && !coord)) return SHINE_ERR_INVALID_ARG;
    if (n > (int64_t)INT32_MAX * 8) return SHINE_ERR_UNSUPPORTED;
    P.oct = *oct; P.dec = *dec; P.coord = coord; P.n = n;
    P.num_tiles = (int32_t)((n + kTile - 1) / kTile);
    P.label = nullptr; P.weight = nullptr; P.d_loss = nullptr; P.pred = nullptr; P.loss = nullptr; P.mask = nullptr;
    P.mask_level = 0; P.sigma = 1.f; P.loss_scale = 1.f; P.weighted = 0; P.scale = 1.f;
    return SHINE_OK;
}

template <bool TRAIN, bool DEC_GRAD>
int launch_loss(const StepParams& P, int loss, uint32_t flags, cudaStream_t st) {
    if (loss == kLossL1) return launch_fused<TRAIN, DEC_GRAD, BatchCoords, kLossL1>(P, flags, st);
    if (loss == kLossL2) return launch_fused<TRAIN, DEC_GRAD, BatchCoords, kLossL2>(P, flags, st);
    return launch_fused<TRAIN, DEC_GRAD>(P, flags, st);
}

// shine_sdf_fwd (train false) and shine_sdf_step: the checks of the loss the flags pick, then one launch
int sdf_loss_call(bool train, const shine_octree* oct, const shine_decoder* dec, const float* coord, const float* label,
                  const float* weight, int64_t n, float sigma, float scale, float loss_scale, const float* d_loss,
                  float* out_pred, float* out_loss, uint32_t flags, cudaStream_t st) {
    // sdf_diff_loss has no reduction or weighting flag: it always weighs by |weight| and divides by the count
    const int loss = sdf_loss_of(flags, kSdfFlags, SHINE_FLAG_TF32X1 | (train ? SHINE_FLAG_MORTON_ORDERED : 0u));
    if (loss < 0) return SHINE_ERR_UNSUPPORTED;
    int rc = check_octree(oct, train);
    if (rc) return rc;
    bool dec_grad = false;
    rc = check_decoder(dec, oct, train ? &dec_grad : nullptr);
    if (rc) return rc;
    if (n > 0 && !label) return SHINE_ERR_INVALID_ARG;
    if (loss == kLossBce ? ((flags & SHINE_FLAG_WEIGHTED) && !weight) || !(sigma > 0.f) : !weight || !valid_scale(scale))
        return SHINE_ERR_INVALID_ARG;
    StepParams P;
    rc = fill_params(P, oct, dec, coord, n);
    if (rc) return rc;
    if (n == 0) return SHINE_OK;
    if ((rc = check_same_device(oct, coord))) return rc;
    DeviceGuard guard(oct->lv[0].features);
    P.label = label; P.weight = weight; P.d_loss = d_loss; P.pred = out_pred; P.loss = out_loss;
    P.sigma = sigma; P.scale = scale; P.loss_scale = loss_scale;
    P.weighted = (loss != kLossBce || (flags & SHINE_FLAG_WEIGHTED)) ? 1 : 0;   // sdf_l1 / sdf_l2: shine_batch.py:172 |weight|
    if (!train) return launch_loss<false, false>(P, loss, flags, st);
    return dec_grad ? launch_loss<true, true>(P, loss, flags, st) : launch_loss<true, false>(P, loss, flags, st);
}

template <int LP>
int launch_query(bool bwd, const shine_octree* oct, const float* coord, int64_t n, float* fwd_out, const float* dfeat,
                 cudaStream_t st) {
    const int64_t threads = n * LP;
    const int64_t blocks = (threads + 255) / 256;
    if (blocks > INT32_MAX) return SHINE_ERR_UNSUPPORTED;
    if (bwd) query_bwd_kernel<LP><<<(unsigned)blocks, 256, 0, st>>>(*oct, coord, n, dfeat);
    else if (LP == 2) query_fwd8_kernel<<<(unsigned)blocks, 256, 0, st>>>(*oct, coord, n, fwd_out);
    else query_fwd_kernel<LP><<<(unsigned)blocks, 256, 0, st>>>(*oct, coord, n, fwd_out);
    return (int)cudaGetLastError();
}

int dispatch_query(bool bwd, const shine_octree* oct, const float* coord, int64_t n, float* fwd_out, const float* dfeat,
                   cudaStream_t st) {
    switch (oct->feature_dim) {
        case 4: return launch_query<1>(bwd, oct, coord, n, fwd_out, dfeat, st);
        case 8: return launch_query<2>(bwd, oct, coord, n, fwd_out, dfeat, st);
        case 16: return launch_query<4>(bwd, oct, coord, n, fwd_out, dfeat, st);
        case 32: return launch_query<8>(bwd, oct, coord, n, fwd_out, dfeat, st);
        default: return SHINE_ERR_UNSUPPORTED;
    }
}

template <int MODE>
int dispatch_tangent(const shine_octree* oct, const float* coord, int64_t n, const float* vin, const float* tangent,
                     float* out, cudaStream_t st) {
    const int lp = oct->feature_dim / 4;
    const int64_t blocks = (n * lp + 255) / 256;
    if (blocks > INT32_MAX) return SHINE_ERR_UNSUPPORTED;
    switch (lp) {
        case 1: query_tangent_kernel<1, MODE><<<(unsigned)blocks, 256, 0, st>>>(*oct, coord, n, vin, tangent, out); break;
        case 2: query_tangent_kernel<2, MODE><<<(unsigned)blocks, 256, 0, st>>>(*oct, coord, n, vin, tangent, out); break;
        case 4: query_tangent_kernel<4, MODE><<<(unsigned)blocks, 256, 0, st>>>(*oct, coord, n, vin, tangent, out); break;
        case 8: query_tangent_kernel<8, MODE><<<(unsigned)blocks, 256, 0, st>>>(*oct, coord, n, vin, tangent, out); break;
        default: return SHINE_ERR_UNSUPPORTED;
    }
    return (int)cudaGetLastError();
}

}  // namespace

int shine_internal::launch_sdf_grid(const StepParams& P, const BrickGrid& grid, uint32_t flags, cudaStream_t st) {
    if (flags & ~kSdfFlags) return SHINE_ERR_UNSUPPORTED;
    const int rc = check_decoder(&P.dec, &P.oct);
    if (rc) return rc;
    return launch_fused<false, false, GridCoords>(P, flags, st, GridCoords{grid});
}

// ------------------------------------------------------------------------------------------------------
// C ABI
// ------------------------------------------------------------------------------------------------------

extern "C" {

int shine_abi_version(void) { return SHINE_ABI_VERSION; }

const char* shine_error_string(int code) {
    if (code == SHINE_OK) return "ok";
    if (code == SHINE_ERR_INVALID_ARG) return "shine_b200: invalid argument";
    if (code == SHINE_ERR_UNSUPPORTED) return "shine_b200: unsupported configuration for the sm_90a kernels";
    if (code == SHINE_ERR_CAPACITY) return "shine_b200: output buffer too small";
    if (code > 0) return cudaGetErrorString((cudaError_t)code);
    return "shine_b200: unknown error";
}

int shine_hash_insert(void* slots, uint32_t capacity, const int64_t* keys, const int32_t* corner_ids, int64_t n,
                      int32_t node_base, int32_t* overflow_count, void* stream) {
    if (!slots || !is_pow2(capacity) || n < 0 || (n > 0 && (!keys || !corner_ids))) return SHINE_ERR_INVALID_ARG;
    if (n == 0) return SHINE_OK;
    DeviceGuard guard(slots);
    const int64_t blocks = (n + 255) / 256;
    hash_insert_kernel<<<(unsigned)blocks, 256, 0, (cudaStream_t)stream>>>(reinterpret_cast<HashSlot*>(slots),
                                                                          capacity - 1, keys, corner_ids, n, node_base,
                                                                          overflow_count);
    return (int)cudaGetLastError();
}

int shine_points_to_morton(const float* coord, int64_t n, int32_t level, int64_t* morton, void* stream) {
    if (n < 0 || level < 1 || level > 16 || (n > 0 && (!coord || !morton))) return SHINE_ERR_INVALID_ARG;
    if (n == 0) return SHINE_OK;
    DeviceGuard guard(morton);
    points_to_morton_kernel<<<(unsigned)((n + 255) / 256), 256, 0, (cudaStream_t)stream>>>(coord, n, level, morton);
    return (int)cudaGetLastError();
}

int shine_get_indices(const shine_octree* oct, const float* coord, int64_t n, int64_t* out_idx, void* stream) {
    int rc = check_octree(oct, false);
    if (rc) return rc;
    if (n < 0 || (n > 0 && (!coord || !out_idx))) return SHINE_ERR_INVALID_ARG;
    if (n == 0) return SHINE_OK;
    if ((rc = check_same_device(oct, coord))) return rc;
    DeviceGuard guard(oct->lv[0].features);
    dim3 grid((unsigned)((n + 255) / 256), (unsigned)oct->num_levels);
    get_indices_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>(*oct, coord, n, out_idx);
    return (int)cudaGetLastError();
}

int shine_query_fwd(const shine_octree* oct, const float* coord, int64_t n, float* out_feat, void* stream) {
    int rc = check_octree(oct, false);
    if (rc) return rc;
    if (n < 0 || (n > 0 && (!coord || !out_feat))) return SHINE_ERR_INVALID_ARG;
    if (n == 0) return SHINE_OK;
    if ((rc = check_same_device(oct, coord))) return rc;
    DeviceGuard guard(oct->lv[0].features);
    return dispatch_query(false, oct, coord, n, out_feat, nullptr, (cudaStream_t)stream);
}

int shine_query_bwd(const shine_octree* oct, const float* coord, int64_t n, const float* dfeat, void* stream) {
    int rc = check_octree(oct, true);
    if (rc) return rc;
    if (n < 0 || (n > 0 && (!coord || !dfeat))) return SHINE_ERR_INVALID_ARG;
    if (n == 0) return SHINE_OK;
    if ((rc = check_same_device(oct, coord))) return rc;
    DeviceGuard guard(oct->lv[0].features);
    return dispatch_query(true, oct, coord, n, nullptr, dfeat, (cudaStream_t)stream);
}

int shine_query_coord_grad(const shine_octree* oct, const float* coord, int64_t n, const float* dfeat, float* out_dcoord,
                           void* stream) {
    int rc = check_octree(oct, false);
    if (rc) return rc;
    if (n < 0 || (n > 0 && (!coord || !dfeat || !out_dcoord))) return SHINE_ERR_INVALID_ARG;
    if (n == 0) return SHINE_OK;
    if ((rc = check_same_device(oct, coord))) return rc;
    DeviceGuard guard(oct->lv[0].features);
    return dispatch_tangent<0>(oct, coord, n, dfeat, nullptr, out_dcoord, (cudaStream_t)stream);
}

int shine_query_tangent_fwd(const shine_octree* oct, const float* coord, int64_t n, const float* tangent, float* out_feat,
                            void* stream) {
    int rc = check_octree(oct, false);
    if (rc) return rc;
    if (n < 0 || (n > 0 && (!coord || !tangent || !out_feat))) return SHINE_ERR_INVALID_ARG;
    if (n == 0) return SHINE_OK;
    if ((rc = check_same_device(oct, coord))) return rc;
    DeviceGuard guard(oct->lv[0].features);
    return dispatch_tangent<1>(oct, coord, n, nullptr, tangent, out_feat, (cudaStream_t)stream);
}

int shine_query_tangent_bwd(const shine_octree* oct, const float* coord, int64_t n, const float* tangent,
                            const float* dfeat, void* stream) {
    int rc = check_octree(oct, true);
    if (rc) return rc;
    if (n < 0 || (n > 0 && (!coord || !tangent || !dfeat))) return SHINE_ERR_INVALID_ARG;
    if (n == 0) return SHINE_OK;
    if ((rc = check_same_device(oct, coord))) return rc;
    DeviceGuard guard(oct->lv[0].features);
    return dispatch_tangent<2>(oct, coord, n, dfeat, tangent, nullptr, (cudaStream_t)stream);
}

int shine_sdf_infer(const shine_octree* oct, const shine_decoder* dec, const float* coord, int64_t n, float* out_pred,
                    uint8_t* out_mask, int32_t mask_level, uint32_t flags, void* stream) {
    if (flags & ~kSdfFlags) return SHINE_ERR_UNSUPPORTED;
    int rc = check_octree(oct, false);
    if (rc) return rc;
    rc = check_decoder(dec, oct);
    if (rc) return rc;
    if (n > 0 && !out_pred) return SHINE_ERR_INVALID_ARG;
    if (out_mask && (mask_level < 0 || mask_level >= oct->num_levels)) return SHINE_ERR_INVALID_ARG;
    StepParams P;
    rc = fill_params(P, oct, dec, coord, n);
    if (rc) return rc;
    if (n == 0) return SHINE_OK;
    if ((rc = check_same_device(oct, coord))) return rc;
    DeviceGuard guard(oct->lv[0].features);
    P.pred = out_pred; P.mask = out_mask; P.mask_level = mask_level;
    return launch_fused<false, false>(P, flags, (cudaStream_t)stream);
}

int shine_sdf_fwd(const shine_octree* oct, const shine_decoder* dec, const float* coord, const float* label,
                  const float* weight, int64_t n, float sigma, float scale, float loss_scale, float* out_pred,
                  float* out_loss, uint32_t flags, void* stream) {
    return sdf_loss_call(false, oct, dec, coord, label, weight, n, sigma, scale, loss_scale, nullptr, out_pred, out_loss,
                         flags, (cudaStream_t)stream);
}

int shine_sdf_step(const shine_octree* oct, const shine_decoder* dec, const float* coord, const float* label,
                   const float* weight, int64_t n, float sigma, float scale, float loss_scale, const float* d_loss,
                   float* out_pred, float* out_loss, uint32_t flags, void* stream) {
    return sdf_loss_call(true, oct, dec, coord, label, weight, n, sigma, scale, loss_scale, d_loss, out_pred, out_loss,
                         flags, (cudaStream_t)stream);
}

int shine_sdf_bce_fwd(const shine_octree* oct, const shine_decoder* dec, const float* coord, const float* label,
                      const float* weight, int64_t n, float sigma, float loss_scale, float* out_pred, float* out_loss,
                      uint32_t flags, void* stream) {
    if (flags & (SHINE_FLAG_LOSS_L1 | SHINE_FLAG_LOSS_L2)) return SHINE_ERR_UNSUPPORTED;
    return shine_sdf_fwd(oct, dec, coord, label, weight, n, sigma, 1.f, loss_scale, out_pred, out_loss, flags, stream);
}

int shine_reduce_grad_replicas(const shine_octree* oct, void* stream) {
    int rc = check_octree(oct, false);
    if (rc) return rc;
    int64_t max_n4 = 0;
    for (int i = 0; i < oct->num_levels; ++i)
        if (oct->lv[i].num_replicas > 1 && oct->lv[i].feature_grads) {
            const int64_t n4 = (int64_t)oct->lv[i].rows * oct->feature_dim / 4;
            if (n4 > max_n4) max_n4 = n4;
        }
    if (max_n4 == 0) return SHINE_OK;
    DeviceGuard guard(oct->lv[0].features);
    int64_t blocks = (max_n4 + 255) / 256;
    const int64_t cap = (int64_t)sm_count() * 8;
    if (blocks > cap) blocks = cap;
    dim3 grid((unsigned)blocks, (unsigned)oct->num_levels);
    reduce_replicas_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>(*oct);
    return (int)cudaGetLastError();
}

// every argument is checked before anything is launched: a rejected shine_adam_step_dev leaves its step counter alone
static int adam_check(const shine_adam_tensor* tensors, int32_t count) {
    if (!tensors || count < 1 || count > SHINE_ADAM_MAX_TENSORS) return SHINE_ERR_INVALID_ARG;
    for (int i = 0; i < count; ++i) {
        const shine_adam_tensor& t = tensors[i];
        if (!t.param || !t.grad || !t.exp_avg || !t.exp_avg_sq || t.numel < 0) return SHINE_ERR_INVALID_ARG;
        if ((((uintptr_t)t.param | (uintptr_t)t.grad | (uintptr_t)t.exp_avg | (uintptr_t)t.exp_avg_sq) & 15) != 0)
            return SHINE_ERR_INVALID_ARG;
    }
    return SHINE_OK;
}

static int adam_launch(const shine_adam_tensor* tensors, int32_t count, float beta1, float beta2, float eps, int32_t step,
                       const float* bc_dev, int32_t zero_grad, cudaStream_t st) {
    AdamParams A;
    DeviceGuard guard(tensors[0].param);
    int64_t max_n = 0;
    for (int i = 0; i < count; ++i) {
        const shine_adam_tensor& t = tensors[i];
        A.t[i] = t;
        if (t.numel > max_n) max_n = t.numel;
    }
    A.count = count; A.beta1 = beta1; A.beta2 = beta2; A.eps = eps; A.zero_grad = zero_grad; A.bc_dev = bc_dev;
    A.omb1 = (float)(1.0 - (double)beta1); A.omb2 = (float)(1.0 - (double)beta2);
    A.bc1 = (float)(1.0 - pow((double)beta1, (double)step));
    A.bc2_sqrt = (float)sqrt(1.0 - pow((double)beta2, (double)step));
    int64_t blocks = (max_n / 4 + 255) / 256;
    const int64_t cap = (int64_t)sm_count() * 8;
    if (blocks > cap) blocks = cap;
    if (blocks < 1) blocks = 1;
    dim3 grid((unsigned)blocks, (unsigned)count);
    adam_kernel<<<grid, 256, 0, st>>>(A);
    return (int)cudaGetLastError();
}

int shine_adam_step(const shine_adam_tensor* tensors, int32_t count, float beta1, float beta2, float eps, int32_t step,
                    int32_t zero_grad, void* stream) {
    if (step < 1) return SHINE_ERR_INVALID_ARG;
    if (int rc = adam_check(tensors, count)) return rc;
    return adam_launch(tensors, count, beta1, beta2, eps, step, nullptr, zero_grad, (cudaStream_t)stream);
}

int shine_adam_step_dev(const shine_adam_tensor* tensors, int32_t count, float beta1, float beta2, float eps,
                        void* state, int32_t zero_grad, void* stream) {
    if (!state) return SHINE_ERR_INVALID_ARG;
    if (int rc = adam_check(tensors, count)) return rc;
    AdamDevState* st = reinterpret_cast<AdamDevState*>(state);
    DeviceGuard guard(state);
    adam_bump_kernel<<<1, 1, 0, (cudaStream_t)stream>>>(st, beta1, beta2);
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) return (int)e;
    return adam_launch(tensors, count, beta1, beta2, eps, 1, &st->bc1, zero_grad, (cudaStream_t)stream);
}

}  // extern "C"
