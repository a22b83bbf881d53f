// shine_train_tc.cu — the training step with the decoder on the warpgroup tensor-core instructions (wgmma, sm_90a),
// warp-specialised.  Same contract as sdf_fused_kernel<TRAIN> (reference shine_batch.py:123-209); selected with
// SHINE_FLAG_TCGEN05 on shine_sdf_bce_step.
//
// Why: in the mma.sync kernel every warp re-reads the decoder weights and stages the weight-gradient operands through
// the LSU for each 16-point tile.  Here the 2 lanes-per-point gather / scatter warps do nothing but gather and scatter,
// and the decoder runs as 128-point wgmma tiles whose operands the tensor core reads from shared memory itself.
//
// One CTA per SM, 20 warps:
//   warps 0-15  gather/scatter (GS), two groups of 8.  Group g owns the rounds r = g, g+2, ... of this CTA; a round is a
//               tile of 128 points, warp w of the group owns rows 16w..16w+15 (lane layout of the mma.sync kernel:
//               2 lanes per point, z-split corners, 32-byte rows).  Per round: hash walk + gather + blend -> X rows
//               (hi/lo tf32) into the round's operand buffer, arrive on x_full; later wait dx_full, read dL/dfeature
//               rows, walk the hash again (the slots are L2-resident by then) and scatter-add (red.v4) into the tables.
//   warps 16-19 decoder epilogue (EP), one warpgroup; it issues the MMAs (two m64 halves per 128-row tile) and after
//               each one stages the accumulators through shared memory so that thread i works on row i of the tile:
//               D1 = X W1^T            -> +b1, ReLU (mask kept), H1 hi/lo -> smem
//               D2 = H1 W2^T           -> +b2, ReLU, pred, BCE loss, dL/dpred, dH2 hi/lo -> smem, dW3/db3 in registers
//               D3 = dH2 W2            -> ReLU mask, dH1 hi/lo -> smem
//               D4 = dH1 W1 (wgmma, in flight)  ||  dW2 += dH2^T H1, dW1 += dH1^T X, bias sums: mma.sync by the four
//                                                   warps, fragments read straight from the operand tiles (tf32 wgmma
//                                                   operands must be K-major)
//               D4 -> dX rows -> smem, arrive dx_full.
//   The gather warps run one round ahead per group (4 X / dX slots), so they only wait for the decoder when it is the
//   bottleneck.  All contractions are 3xTF32 (hi*hi + lo*hi + hi*lo, fp32 accumulate).
//
// Shared-memory operand layout (no swizzle): an activation matrix [128 points][C columns] is stored as core matrices of
// 8 points x 16 bytes (4 columns): offset(pt, c) = (pt>>3)*S_pt + (c>>2)*128 + (pt&7)*16 + (c&3)*4 — the canonical
// K-major layout of the forward / dgrad MMAs (M = points, K = columns; LBO = 128, SBO = S_pt).
#include "shine_device.cuh"

using shine_internal::StepParams;

namespace {

constexpr int kGSWarps = 16, kEPWarps = 4;
constexpr int kTcThreads = 32 * (kGSWarps + kEPWarps);     // 640
constexpr int kRound = 128;                                 // points per round (MMA M)
constexpr int kGSRegs = 80, kEPRegs = 160;                  // setmaxnreg: 512 x 80 + 128 x 160 = 640 x 96
constexpr int kRowStride = 36;                              // floats per row of the accumulator staging tile

struct TP {                                               // byte offsets in dynamic shared memory
    static constexpr int X_PT = 2 * 128;                  // X tile [128][8]: 2 chunks per 8-point group
    static constexpr int X_BYTES = 16 * X_PT;             // 4 096 per hi / lo
    static constexpr int X = 0;                           // [slot 4][hi/lo 2]                        32 768
    static constexpr int H1_PT = 8 * 128;                 // H1 [128][32]
    static constexpr int H1_BYTES = 16 * H1_PT;           // 16 384
    static constexpr int H1 = X + 8 * X_BYTES;            // [hi/lo 2]                                32 768
    static constexpr int DH_PT = 16 * 128;                // [dH2 32 | dH1 32]
    static constexpr int DH_BYTES = 16 * DH_PT;           // 32 768
    static constexpr int DH = H1 + 2 * H1_BYTES;          // [hi/lo 2]                                65 536
    static constexpr int W1H = DH + 2 * DH_BYTES;         // W1  [N 32][K 8]   K-major: 4 groups x 2 chunks x 128 B
    static constexpr int W1L = W1H + 1024;
    static constexpr int W2H = W1L + 1024;                // W2  [N 32][K 32]  (forward layer 2: B[n2][k1])
    static constexpr int W2L = W2H + 4096;
    static constexpr int W2TH = W2L + 4096;               // W2^T [N = k1][K = n2]  (dgrad layer 2)
    static constexpr int W2TL = W2TH + 4096;
    static constexpr int W1TH = W2TL + 4096;              // W1^T [N = 16 (8 used)][K = n1 32]  (dgrad layer 1)
    static constexpr int W1TL = W1TH + 2048;
    static constexpr int VEC = W1TL + 2048;               // b1[32] b2[32] w3[32] b3 + pad            400 B
    static constexpr int DX = VEC + 400;                  // [slot 4][128][8] fp32                    16 384 B
    static constexpr int RED = DX + 16384;                // decoder-gradient block accumulator [1380] 5 520 B
    static constexpr int ACC = RED + 5520;                // accumulator staging [128][kRowStride] fp32          18 432 B
    static constexpr int BAR = ACC + 128 * kRowStride * 4; // x_full[4], dx_full[4] : 8 x 8 B
    static constexpr int BYTES = BAR + 64;
};
static_assert(TP::DX % 16 == 0 && TP::BAR % 8 == 0 && TP::RED % 16 == 0 && TP::ACC % 16 == 0, "alignment");

__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint32_t bar) {
    asm volatile("{\n\t.reg .b64 st;\n\tmbarrier.arrive.shared::cta.b64 st, [%0];\n\t}" ::"r"(bar) : "memory");
}
__device__ __forceinline__ void ep_bar() { asm volatile("bar.sync 1, 128;" ::: "memory"); }

// 3xTF32 product D = A B of the 128-row tile over KS K = 8 steps (each step = 2 chunks = 256 B further in both
// operands), as two m64 halves (A advanced by 8 row groups = a_half bytes); the descriptors are built once and only
// their address field is advanced.  The MMAs are committed, not waited for.
template <int KS, int NR>
__device__ __forceinline__ void mma3x_issue(float (&d)[2][NR], uint64_t ah, uint64_t al, uint64_t bh, uint64_t bl,
                                            uint32_t a_half) {
    wgmma_fence();
#pragma unroll
    for (int h = 0; h < 2; ++h) {
        const uint64_t ho = (uint64_t)((h * a_half) >> 4);
#pragma unroll
        for (int k = 0; k < KS; ++k) {
            const uint64_t ko = (uint64_t)(16 * k);      // 256 B >> 4 in the start-address field
            if constexpr (NR == 16) {
                wgmma_n32(d[h], al + ho + ko, bh + ko, k > 0 ? 1u : 0u);
                wgmma_n32(d[h], ah + ho + ko, bl + ko, 1u);
                wgmma_n32(d[h], ah + ho + ko, bh + ko, 1u);
            } else {
                wgmma_n8(d[h], al + ho + ko, bh + ko, k > 0 ? 1u : 0u);
                wgmma_n8(d[h], ah + ho + ko, bl + ko, 1u);
                wgmma_n8(d[h], ah + ho + ko, bh + ko, 1u);
            }
        }
    }
    wgmma_commit();
}

// accumulator fragments of the EP warpgroup -> staging tile [row][kRowStride] (columns 8j + 2t, +1 of rows g, g + 8 of
// every 16-row slice); the caller synchronises the warpgroup before reading rows back
template <int NR>
__device__ __forceinline__ void stage_acc(float* acc, const float (&d)[2][NR], int eq, int lane) {
    const int g = lane >> 2, t = lane & 3;
#pragma unroll
    for (int h = 0; h < 2; ++h) {
#pragma unroll
        for (int j = 0; j < NR / 4; ++j) {
#pragma unroll
            for (int rr = 0; rr < 2; ++rr) {
                const int row = 64 * h + 16 * eq + g + 8 * rr;
                *reinterpret_cast<float2*>(acc + row * kRowStride + 8 * j + 2 * t) = make_float2(d[h][4 * j + 2 * rr], d[h][4 * j + 2 * rr + 1]);
            }
        }
    }
}

template <bool DEC_GRAD>
__global__ void __launch_bounds__(kTcThreads, 1) sdf_train_tc_kernel(const __grid_constant__ StepParams P) {
    extern __shared__ __align__(1024) unsigned char sm[];
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const uint32_t sbase = (uint32_t)__cvta_generic_to_shared(sm);
    float* vec = reinterpret_cast<float*>(sm + TP::VEC);
    const uint32_t bar_x = sbase + TP::BAR, bar_dx = sbase + TP::BAR + 32;
    float* accs = reinterpret_cast<float*>(sm + TP::ACC);

    // ---- prologue: weights in the K-major operand layouts (hi/lo), barriers ------------------------------------------
    for (int i = tid; i < 2048 / 4; i += kTcThreads) {             // W1^T rows 8..15 must be zero
        reinterpret_cast<uint32_t*>(sm + TP::W1TH)[i] = 0u; reinterpret_cast<uint32_t*>(sm + TP::W1TL)[i] = 0u;
    }
    for (int i = tid; i < 1380; i += kTcThreads) reinterpret_cast<float*>(sm + TP::RED)[i] = 0.f;
    __syncthreads();
    for (int i = tid; i < kH * kF; i += kTcThreads) {
        const int n = i / kF, k = i % kF;
        uint32_t hi, lo; split_tf32(P.dec.w1[i], hi, lo);
        const int off = (n >> 3) * 256 + (k >> 2) * 128 + (n & 7) * 16 + (k & 3) * 4;               // W1 [n][k]
        *reinterpret_cast<uint32_t*>(sm + TP::W1H + off) = hi; *reinterpret_cast<uint32_t*>(sm + TP::W1L + off) = lo;
        const int offt = (k >> 3) * 1024 + (n >> 2) * 128 + (k & 7) * 16 + (n & 3) * 4;              // W1^T [k][n]
        *reinterpret_cast<uint32_t*>(sm + TP::W1TH + offt) = hi; *reinterpret_cast<uint32_t*>(sm + TP::W1TL + offt) = lo;
    }
    for (int i = tid; i < kH * kH; i += kTcThreads) {
        const int n = i / kH, k = i % kH;
        uint32_t hi, lo; split_tf32(P.dec.w2[i], hi, lo);
        const int off = (n >> 3) * 1024 + (k >> 2) * 128 + (n & 7) * 16 + (k & 3) * 4;              // W2 [n2][k1]
        *reinterpret_cast<uint32_t*>(sm + TP::W2H + off) = hi; *reinterpret_cast<uint32_t*>(sm + TP::W2L + off) = lo;
        const int offt = (k >> 3) * 1024 + (n >> 2) * 128 + (k & 7) * 16 + (n & 3) * 4;             // W2^T [k1][n2]
        *reinterpret_cast<uint32_t*>(sm + TP::W2TH + offt) = hi; *reinterpret_cast<uint32_t*>(sm + TP::W2TL + offt) = lo;
    }
    if (tid < kH) {
        vec[tid] = P.dec.b1 ? P.dec.b1[tid] : 0.f;
        vec[32 + tid] = P.dec.b2 ? P.dec.b2[tid] : 0.f;
        vec[64 + tid] = P.dec.w3[tid];
    }
    if (tid == 0) {
        vec[96] = P.dec.b3 ? P.dec.b3[0] : 0.f;
        for (int s = 0; s < 4; ++s) { mbar_init(bar_x + 8 * s, 8); mbar_init(bar_dx + 8 * s, 1); }
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
    __syncthreads();

    const int64_t tiles_total = (P.n + kRound - 1) / kRound;
    const int rounds = (int)((tiles_total > blockIdx.x) ? (tiles_total - blockIdx.x + gridDim.x - 1) / gridDim.x : 0);
    const float up = P.d_loss ? __ldg(P.d_loss) : 1.0f;
    const float gscale = P.loss_scale * up;

    if (warp < kGSWarps) {
        // ============================== gather / scatter warps =====================================================
        asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(kGSRegs));
        const int grp = warp >> 3, wg = warp & 7;
        const int g = lane >> 2, t = lane & 3, odd = t & 1, half = t >> 1;
        const int row = 16 * wg + g + 8 * odd;                                   // this lane pair's row of the tile
        const bool poly = P.oct.poly_interp != 0;
        const int L = P.oct.num_levels;
        bool consecutive = true;
#pragma unroll
        for (int i = 1; i < 4; ++i)
            if (i < L && P.oct.lv[i].level != P.oct.lv[0].level - i) consecutive = false;
        const int xoff = (row >> 3) * TP::X_PT + half * 128 + (row & 7) * 16;

        // this lane pair's point of round r and its node slot on every level (-1: miss)
        auto locate = [&](int r, float& x, float& y, float& z, int (&slotl)[4]) {
            const int64_t myp = ((int64_t)blockIdx.x + (int64_t)r * gridDim.x) * kRound + row;
            const bool valid = myp < P.n;
            x = 0.f; y = 0.f; z = 0.f;
            if (valid) { x = __ldg(P.coord + 3 * myp); y = __ldg(P.coord + 3 * myp + 1); z = __ldg(P.coord + 3 * myp + 2); }
            // hash walk (model/feature_octree.py:199-218): the pair splits the LEVELS for the first probe
            {
                const unsigned long long key0 = valid ? morton_of(x, y, z, P.oct.lv[0].level) : 0ull;
                unsigned long long kq[2];
                uint4 kf[2];
                int mine[2];
#pragma unroll
                for (int j = 0; j < 2; ++j) {
                    const int i = 2 * j + half;
                    mine[j] = -1;
                    if (i < L && valid) {
                        const shine_level& lv = P.oct.lv[i];
                        kq[j] = consecutive ? (key0 >> (3 * i)) : morton_of(x, y, z, lv.level);
                        mine[j] = (int)(hash_key(kq[j]) & (lv.hash_capacity - 1));
                        kf[j] = __ldg(reinterpret_cast<const uint4*>(reinterpret_cast<const HashSlot*>(lv.hash_slots) + mine[j]));
                    }
                }
#pragma unroll
                for (int j = 0; j < 2; ++j) {
                    const int i = 2 * j + half;
                    if (i < L && valid) {
                        const unsigned long long k0 = ((unsigned long long)kf[j].y << 32) | kf[j].x;
                        if (k0 != kq[j]) {
                            if (k0 == kEmptyKey || (int)kf[j].w <= 0) mine[j] = -1;
                            else {
                                const shine_level& lv = P.oct.lv[i];
                                mine[j] = probe_slot_from(reinterpret_cast<const HashSlot*>(lv.hash_slots), lv.hash_capacity - 1,
                                                          kq[j], (uint32_t)mine[j], (int)kf[j].w);
                            }
                        }
                    }
                }
                __syncwarp();
#pragma unroll
                for (int j = 0; j < 2; ++j) {
                    const int other = __shfl_xor_sync(kFull, mine[j], 2);
                    slotl[2 * j] = half ? other : mine[j];
                    slotl[2 * j + 1] = half ? mine[j] : other;
                }
            }
        };

        // gather of one round: hash walk, 8-corner blend, X rows -> slot
        auto gather = [&](int r, int slot) {
            float x, y, z;
            int slotl[4];
            locate(r, x, y, z, slotl);
            // 8-corner gather + blend (model/feature_octree.py:222-234): the pair splits the CORNERS by z bit
            float acc[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
#pragma unroll
            for (int i = 0; i < 4; ++i) {
                if (i < L && slotl[i] >= 0) {
                    const shine_level& lv = P.oct.lv[i];
                    const int4 id4 = ldg_i4(slot_ids(reinterpret_cast<const HashSlot*>(lv.hash_slots), slotl[i], half));
                    float r0[8], r1[8], r2[8], r3[8];
                    ldg_row8(lv.features + (int64_t)id4.x * kF, r0);
                    ldg_row8(lv.features + (int64_t)id4.y * kF, r1);
                    ldg_row8(lv.features + (int64_t)id4.z * kF, r2);
                    ldg_row8(lv.features + (int64_t)id4.w * kF, r3);
                    Blend b; b.init(x, y, z, lv.level, poly);
                    const float wz = half ? b.tz : b.uz;
                    const float w0 = __fmul_rn(__fmul_rn(b.ux, b.uy), wz), w1 = __fmul_rn(__fmul_rn(b.ux, b.ty), wz);
                    const float w2 = __fmul_rn(__fmul_rn(b.tx, b.uy), wz), w3 = __fmul_rn(__fmul_rn(b.tx, b.ty), wz);
                    blend4(acc, r0, r1, r2, r3, w0, w1, w2, w3);
                }
            }
            // X rows (this lane: the 4 channels of its half = one 16-byte K chunk), hi / lo
            uint32_t h4[4], l4[4];
#pragma unroll
            for (int q = 0; q < 4; ++q) {
                const float send = half ? acc[q] : acc[4 + q];
                const float recv = __shfl_xor_sync(kFull, send, 2);
                split_fast((half ? acc[4 + q] : acc[q]) + recv, h4[q], l4[q]);
            }
            unsigned char* xs = sm + TP::X + (2 * slot) * TP::X_BYTES;
            *reinterpret_cast<uint4*>(xs + xoff) = make_uint4(h4[0], h4[1], h4[2], h4[3]);
            *reinterpret_cast<uint4*>(xs + TP::X_BYTES + xoff) = make_uint4(l4[0], l4[1], l4[2], l4[3]);
            asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
            __syncwarp();
            if (lane == 0) mbar_arrive(bar_x + 8 * slot);
        };

        // software pipeline, depth 2 per group: the gather of local round k+1 is issued before waiting for the decoder of k
        if (grp < rounds) gather(grp, grp);
        for (int r = grp, k = 0; r < rounds; r += 2, ++k) {
            const int slot = 2 * (k & 1) + grp;
            if (r + 2 < rounds) gather(r + 2, 2 * ((k + 1) & 1) + grp);
            // ---- dL/dfeature of round r, then scatter-add (index_put_ accumulate) ------------------------------------------
            mbar_wait(bar_dx + 8 * slot, (uint32_t)((k >> 1) & 1));
            const float4 dxv = *reinterpret_cast<const float4*>(sm + TP::DX + slot * 4096 + row * 32 + 16 * half);
            const float dx[4] = {dxv.x, dxv.y, dxv.z, dxv.w};
            float x, y, z;
            int slotl[4];
            locate(r, x, y, z, slotl);
#pragma unroll
            for (int i = 0; i < 4; ++i) {
                int4 id4 = make_int4(-1, -1, -1, -1);
                if (i < L && slotl[i] >= 0)
                    id4 = ldg_i4(slot_ids(reinterpret_cast<const HashSlot*>(P.oct.lv[i].hash_slots), slotl[i], half));
                const int qid[4] = {id4.x, id4.y, id4.z, id4.w};
                int ids[8];
#pragma unroll
                for (int c = 0; c < 4; ++c) {
                    const int mine = qid[c];
                    const int other = __shfl_xor_sync(kFull, mine, 2);
                    ids[2 * c] = half ? other : mine;
                    ids[2 * c + 1] = half ? mine : other;
                }
                if (i < L && ids[0] >= 0) {
                    const shine_level& lv = P.oct.lv[i];
                    Blend b; b.init(x, y, z, lv.level, poly);
                    float* gb = grad_base(lv, (uint32_t)(blockIdx.x * kGSWarps + warp + r), kF) + 4 * half;
                    // w_c = (X * Y) * Z in the reference's association; the four X*Y products are shared by the z pair
                    const float xy[4] = {__fmul_rn(b.ux, b.uy), __fmul_rn(b.ux, b.ty), __fmul_rn(b.tx, b.uy), __fmul_rn(b.tx, b.ty)};
#pragma unroll
                    for (int c = 0; c < 8; ++c) {
                        const float w = __fmul_rn(xy[c >> 1], (c & 1) ? b.tz : b.uz);
                        red_add_f4(gb + (int64_t)ids[c] * kF, w * dx[0], w * dx[1], w * dx[2], w * dx[3]);
                    }
                }
            }
            __syncwarp();
        }
    } else {
        // ============================== decoder epilogue warps (+ MMA issue by thread 0) ==============================
        asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(kEPRegs));
        const int et = tid - 32 * kGSWarps;                     // row of the tile owned by this thread
        const int eq = et >> 5;                                 // warp of the warpgroup: rows 16eq.. of each m64 half
        const int g = lane >> 2, t = lane & 3;
        const float* arow = accs + et * kRowStride;             // this thread's row of the staged accumulators
        // K-major descriptors (LBO = 128 between the two K chunks of a step, SBO = stride of an 8-row group)
        const uint64_t dH1h = wgmma_desc(sbase + TP::H1, 128, TP::H1_PT), dH1l = wgmma_desc(sbase + TP::H1 + TP::H1_BYTES, 128, TP::H1_PT);
        const uint64_t dDHh = wgmma_desc(sbase + TP::DH, 128, TP::DH_PT), dDHl = wgmma_desc(sbase + TP::DH + TP::DH_BYTES, 128, TP::DH_PT);
        const uint64_t dW1h = wgmma_desc(sbase + TP::W1H, 128, 256), dW1l = wgmma_desc(sbase + TP::W1L, 128, 256);
        const uint64_t dW2h = wgmma_desc(sbase + TP::W2H, 128, 1024), dW2l = wgmma_desc(sbase + TP::W2L, 128, 1024);
        const uint64_t dW2Th = wgmma_desc(sbase + TP::W2TH, 128, 1024), dW2Tl = wgmma_desc(sbase + TP::W2TL, 128, 1024);
        const uint64_t dW1Th = wgmma_desc(sbase + TP::W1TH, 128, 1024), dW1Tl = wgmma_desc(sbase + TP::W1TL, 128, 1024);
        const uint64_t dX0h = wgmma_desc(sbase + TP::X, 128, TP::X_PT);
        float dw3acc[32];
#pragma unroll
        for (int j = 0; j < 32; ++j) dw3acc[j] = 0.f;
        float db3acc = 0.f, loss_acc = 0.f;
        // weight-gradient accumulators of this warp (mma.sync fragments): dW2[n2][k1], dW1[n1][k], bias sums in column 0
        float aW2[2][4][4], aW1[2][4], aB2[2][4], aB1[2][4];
#pragma unroll
        for (int a = 0; a < 2; ++a) {
#pragma unroll
            for (int b = 0; b < 4; ++b) { aW2[a][b][0] = aW2[a][b][1] = aW2[a][b][2] = aW2[a][b][3] = 0.f; aW1[a][b] = aB2[a][b] = aB1[a][b] = 0.f; }
        }
        const int hoff = (et >> 3) * TP::H1_PT + (et & 7) * 16;           // + chunk * 128
        const int doff = (et >> 3) * TP::DH_PT + (et & 7) * 16;
        const uint32_t* h1h = reinterpret_cast<const uint32_t*>(sm + TP::H1);
        const uint32_t* h1l = reinterpret_cast<const uint32_t*>(sm + TP::H1 + TP::H1_BYTES);
        const uint32_t* dhh = reinterpret_cast<const uint32_t*>(sm + TP::DH);
        const uint32_t* dhl = reinterpret_cast<const uint32_t*>(sm + TP::DH + TP::DH_BYTES);

        for (int r = 0; r < rounds; ++r) {
            const int grp = r & 1, k = r >> 1, slot = 2 * (k & 1) + grp;
            const int64_t p = ((int64_t)blockIdx.x + (int64_t)r * gridDim.x) * kRound + et;
            const bool valid = p < P.n;
            float lab = 0.f, wgt = 1.f;
            if (valid) {
                lab = __ldg(P.label + p);
                if (P.weighted) wgt = fabsf(__ldg(P.weight + p));                 // shine_batch.py:172 abs()
            }
            const uint64_t dXh = dX0h + (uint64_t)((2 * slot) * (TP::X_BYTES >> 4));
            const uint64_t dXl = dXh + (uint64_t)(TP::X_BYTES >> 4);

            // ---- layer 1: D1 = X W1^T --------------------------------------------------------------------------------
            mbar_wait(bar_x + 8 * slot, (uint32_t)((k >> 1) & 1));
            float d[2][16];
            float hv[32];
            auto rows_of = [&]() {                              // stage d, read back this thread's row
                stage_acc(accs, d, eq, lane);
                ep_bar();
#pragma unroll
                for (int c = 0; c < 8; ++c) {
                    const float4 v = *reinterpret_cast<const float4*>(arow + 4 * c);
                    hv[4 * c] = v.x; hv[4 * c + 1] = v.y; hv[4 * c + 2] = v.z; hv[4 * c + 3] = v.w;
                }
            };
            mma3x_issue<1>(d, dXh, dXl, dW1h, dW1l, 8 * TP::X_PT);
            wgmma_wait_all();
            rows_of();
            uint32_t m1 = 0;
#pragma unroll
            for (int c = 0; c < 8; ++c) {
                const float4 bb = *reinterpret_cast<const float4*>(vec + 4 * c);
                const float v0 = hv[4 * c] + bb.x, v1 = hv[4 * c + 1] + bb.y, v2 = hv[4 * c + 2] + bb.z, v3 = hv[4 * c + 3] + bb.w;
                m1 |= (v0 > 0.f ? 1u : 0u) << (4 * c) | (v1 > 0.f ? 1u : 0u) << (4 * c + 1) | (v2 > 0.f ? 1u : 0u) << (4 * c + 2) |
                      (v3 > 0.f ? 1u : 0u) << (4 * c + 3);
                uint32_t h0, h1, h2, h3, l0, l1, l2, l3;
                split_fast(fmaxf(v0, 0.f), h0, l0); split_fast(fmaxf(v1, 0.f), h1, l1);
                split_fast(fmaxf(v2, 0.f), h2, l2); split_fast(fmaxf(v3, 0.f), h3, l3);
                *reinterpret_cast<uint4*>(sm + TP::H1 + hoff + 128 * c) = make_uint4(h0, h1, h2, h3);
                *reinterpret_cast<uint4*>(sm + TP::H1 + TP::H1_BYTES + hoff + 128 * c) = make_uint4(l0, l1, l2, l3);
            }
            asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
            ep_bar();

            // ---- layer 2: D2 = H1 W2^T, output layer, loss, dL/dpred ------------------------------------------------------
            mma3x_issue<4>(d, dH1h, dH1l, dW2h, dW2l, 8 * TP::H1_PT);
            wgmma_wait_all();
            rows_of();
            float pr = vec[96];
            uint32_t m2 = 0;
#pragma unroll
            for (int j = 0; j < 32; ++j) {
                const float v = hv[j] + vec[32 + j];
                m2 |= (v > 0.f ? 1u : 0u) << j;
                hv[j] = fmaxf(v, 0.f);
                pr = fmaf(hv[j], vec[64 + j], pr);
            }
            if (P.pred && valid) P.pred[p] = pr;
            float dp = 0.f;
            if (valid) {      // sdf_bce_loss (utils/loss.py:17-24), MUFU-based like the mma.sync kernel
                const float zt = __fdividef(1.0f, 1.0f + __expf(-__fdividef(lab, P.sigma)));
                const float e = __expf(-fabsf(pr));
                loss_acc += wgt * (fmaxf(pr, 0.f) - pr * zt + __logf(1.0f + e));
                const float rs = __fdividef(1.0f, 1.0f + e);
                dp = ((pr >= 0.f ? rs : e * rs) - zt) * wgt * gscale;
            }
            db3acc += dp;
#pragma unroll
            for (int c = 0; c < 8; ++c) {
                float d[4];
#pragma unroll
                for (int q = 0; q < 4; ++q) {
                    const int j = 4 * c + q;
                    if (DEC_GRAD) dw3acc[j] = fmaf(dp, hv[j], dw3acc[j]);
                    d[q] = ((m2 >> j) & 1u) ? dp * vec[64 + j] : 0.f;
                }
                uint32_t h0, h1, h2, h3, l0, l1, l2, l3;
                split_fast(d[0], h0, l0); split_fast(d[1], h1, l1); split_fast(d[2], h2, l2); split_fast(d[3], h3, l3);
                *reinterpret_cast<uint4*>(sm + TP::DH + doff + 128 * c) = make_uint4(h0, h1, h2, h3);
                *reinterpret_cast<uint4*>(sm + TP::DH + TP::DH_BYTES + doff + 128 * c) = make_uint4(l0, l1, l2, l3);
            }
            asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
            ep_bar();

            // ---- dgrad layer 2: D3 = dH2 W2 ------------------------------------------------------------------------------
            mma3x_issue<4>(d, dDHh, dDHl, dW2Th, dW2Tl, 8 * TP::DH_PT);
            wgmma_wait_all();
            rows_of();
#pragma unroll
            for (int c = 0; c < 8; ++c) {
                uint32_t h0, h1, h2, h3, l0, l1, l2, l3;
                split_fast(((m1 >> (4 * c)) & 1u) ? hv[4 * c] : 0.f, h0, l0);
                split_fast(((m1 >> (4 * c + 1)) & 1u) ? hv[4 * c + 1] : 0.f, h1, l1);
                split_fast(((m1 >> (4 * c + 2)) & 1u) ? hv[4 * c + 2] : 0.f, h2, l2);
                split_fast(((m1 >> (4 * c + 3)) & 1u) ? hv[4 * c + 3] : 0.f, h3, l3);
                *reinterpret_cast<uint4*>(sm + TP::DH + doff + 128 * (8 + c)) = make_uint4(h0, h1, h2, h3);
                *reinterpret_cast<uint4*>(sm + TP::DH + TP::DH_BYTES + doff + 128 * (8 + c)) = make_uint4(l0, l1, l2, l3);
            }
            asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
            ep_bar();

            // ---- dgrad layer 1 on the tensor core: D4 = dH1 W1 (N = 8) ... ------------------------------------------------------
            float d4[2][4];
            mma3x_issue<4>(d4, dDHh + 64, dDHl + 64, dW1Th, dW1Tl, 8 * TP::DH_PT);      // + 8 chunks (1024 B >> 4)
            // ---- ... while the four warps contract the weight gradients of this round over its 128 points with mma.sync,
            //      straight from the operand tiles (tf32 wgmma operands must be K-major, these are MN-major):
            //      dW2 += dH2^T H1, dW1 += dH1^T X, db2 / db1 = column sums (an all-ones B column).  Warp q: points 32q..32q+31
            if (DEC_GRAD) {
                const uint32_t* xh = reinterpret_cast<const uint32_t*>(sm + TP::X + (2 * slot) * TP::X_BYTES);
                const uint32_t* xl = xh + TP::X_BYTES / 4;
                const uint2 ones_h = make_uint2(g == 0 ? __float_as_uint(1.0f) : 0u, g == 0 ? __float_as_uint(1.0f) : 0u);
                const uint2 zero2 = make_uint2(0u, 0u);
#pragma unroll 1
                for (int ks = 4 * eq; ks < 4 * eq + 4; ++ks) {
                    // element (pt, c) of a tile with S_pt bytes per 8-point group: word (pt>>3)*S_pt/4 + (c>>2)*32 + (pt&7)*4 + (c&3)
                    const int pa = ks * (TP::DH_PT / 4) + t * 4, pb = pa + 16;                    // points 8ks+t and 8ks+t+4
                    const int ha = ks * (TP::H1_PT / 4) + t * 4, hb = ha + 16;
                    const int xa = ks * (TP::X_PT / 4) + t * 4, xb = xa + 16;
                    uint2 bh[4], bl[4];
#pragma unroll
                    for (int nt = 0; nt < 4; ++nt) {       // B[k = point][n = k1 = 8nt + g] = H1
                        const int cw = ((8 * nt + g) >> 2) * 32 + ((8 * nt + g) & 3);
                        bh[nt] = make_uint2(h1h[ha + cw], h1h[hb + cw]); bl[nt] = make_uint2(h1l[ha + cw], h1l[hb + cw]);
                    }
                    const int cx = (g >> 2) * 32 + (g & 3);
                    const uint2 vh = make_uint2(xh[xa + cx], xh[xb + cx]), vl = make_uint2(xl[xa + cx], xl[xb + cx]);
#pragma unroll
                    for (int mt = 0; mt < 2; ++mt) {
                        const int c0 = 16 * mt + g, c1 = c0 + 8;
                        const int w0 = (c0 >> 2) * 32 + (c0 & 3), w1 = (c1 >> 2) * 32 + (c1 & 3);
                        AFrag<3> a2, a1;      // A[m = column][k = point]: dH2 columns 0..31, dH1 columns 32..63 (+ 8 chunks = 256 words)
                        a2.hi[0] = dhh[pa + w0]; a2.hi[1] = dhh[pa + w1]; a2.hi[2] = dhh[pb + w0]; a2.hi[3] = dhh[pb + w1];
                        a2.lo[0] = dhl[pa + w0]; a2.lo[1] = dhl[pa + w1]; a2.lo[2] = dhl[pb + w0]; a2.lo[3] = dhl[pb + w1];
                        a1.hi[0] = dhh[pa + 256 + w0]; a1.hi[1] = dhh[pa + 256 + w1]; a1.hi[2] = dhh[pb + 256 + w0]; a1.hi[3] = dhh[pb + 256 + w1];
                        a1.lo[0] = dhl[pa + 256 + w0]; a1.lo[1] = dhl[pa + 256 + w1]; a1.lo[2] = dhl[pb + 256 + w0]; a1.lo[3] = dhl[pb + 256 + w1];
#pragma unroll
                        for (int nt = 0; nt < 4; ++nt) mma3<3>(aW2[mt][nt], a2, bh[nt], bl[nt]);
                        mma3<3>(aB2[mt], a2, ones_h, zero2);
                        mma3<3>(aW1[mt], a1, vh, vl);
                        mma3<3>(aB1[mt], a1, ones_h, zero2);
                    }
                }
            }
            wgmma_wait_all();
            stage_acc(accs, d4, eq, lane);
            ep_bar();
            float dxr[8];
            {
                const float4 v0 = *reinterpret_cast<const float4*>(arow), v1 = *reinterpret_cast<const float4*>(arow + 4);
                dxr[0] = v0.x; dxr[1] = v0.y; dxr[2] = v0.z; dxr[3] = v0.w; dxr[4] = v1.x; dxr[5] = v1.y; dxr[6] = v1.z; dxr[7] = v1.w;
            }
            float* dxo = reinterpret_cast<float*>(sm + TP::DX + slot * 4096) + et * 8;
            *reinterpret_cast<float4*>(dxo) = make_float4(dxr[0], dxr[1], dxr[2], dxr[3]);
            *reinterpret_cast<float4*>(dxo + 4) = make_float4(dxr[4], dxr[5], dxr[6], dxr[7]);
            if (P.debug_dx && valid) {
#pragma unroll
                for (int q = 0; q < 8; ++q) P.debug_dx[p * 8 + q] = dxr[q];
            }
            ep_bar();
            if (et == 0) mbar_arrive(bar_dx + 8 * slot);
        }

        // ---- epilogue: loss, decoder gradients ---------------------------------------------------------------------------
        if (P.loss) {
#pragma unroll
            for (int o = 16; o > 0; o >>= 1) loss_acc += __shfl_xor_sync(kFull, loss_acc, o);
            if (lane == 0 && loss_acc != 0.f) atomicAdd(P.loss, loss_acc * P.loss_scale);
        }
        if (DEC_GRAD && rounds > 0) {
            float* red = reinterpret_cast<float*>(sm + TP::RED);   // [gw1 256 | gb1 32 | gw2 1024 | gb2 32 | gw3 32 | gb3 1]
            constexpr int oW1 = 0, oB1 = 256, oW2 = 288, oB2 = 1312, oW3 = 1344, oB3 = 1376;
            float mine = 0.f;
#pragma unroll
            for (int j = 0; j < 32; ++j) {
                float s = dw3acc[j];
#pragma unroll
                for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(kFull, s, o);
                if (lane == j) mine = s;
            }
            atomicAdd(red + oW3 + lane, mine);
#pragma unroll
            for (int o = 16; o > 0; o >>= 1) db3acc += __shfl_xor_sync(kFull, db3acc, o);
            if (lane == 0) atomicAdd(red + oB3, db3acc);
#pragma unroll
            for (int mt = 0; mt < 2; ++mt) {
#pragma unroll
                for (int nt = 0; nt < 4; ++nt) {
                    atomicAdd(red + oW2 + (16 * mt + g) * kH + 8 * nt + 2 * t, aW2[mt][nt][0]);
                    atomicAdd(red + oW2 + (16 * mt + g) * kH + 8 * nt + 2 * t + 1, aW2[mt][nt][1]);
                    atomicAdd(red + oW2 + (16 * mt + g + 8) * kH + 8 * nt + 2 * t, aW2[mt][nt][2]);
                    atomicAdd(red + oW2 + (16 * mt + g + 8) * kH + 8 * nt + 2 * t + 1, aW2[mt][nt][3]);
                }
                atomicAdd(red + oW1 + (16 * mt + g) * kF + 2 * t, aW1[mt][0]);
                atomicAdd(red + oW1 + (16 * mt + g) * kF + 2 * t + 1, aW1[mt][1]);
                atomicAdd(red + oW1 + (16 * mt + g + 8) * kF + 2 * t, aW1[mt][2]);
                atomicAdd(red + oW1 + (16 * mt + g + 8) * kF + 2 * t + 1, aW1[mt][3]);
                if (t == 0) {      // column 0 of the all-ones B tile
                    atomicAdd(red + oB2 + 16 * mt + g, aB2[mt][0]); atomicAdd(red + oB2 + 16 * mt + g + 8, aB2[mt][2]);
                    atomicAdd(red + oB1 + 16 * mt + g, aB1[mt][0]); atomicAdd(red + oB1 + 16 * mt + g + 8, aB1[mt][2]);
                }
            }
            ep_bar();
            for (int i = et; i < 1377; i += 128) {
                const float v = red[i];
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

}

}  // namespace

namespace shine_internal {

static float* g_debug_dx = nullptr;
extern "C" void shine_debug_set_dx(float* p) { g_debug_dx = p; }

int launch_train_tc(const StepParams& P, bool dec_grad, cudaStream_t st) {
    if (P.oct.num_levels > 4 || P.oct.feature_dim != kF) return SHINE_ERR_UNSUPPORTED;
    auto kern = dec_grad ? sdf_train_tc_kernel<true> : sdf_train_tc_kernel<false>;
    static int ready[2][kMaxDevices] = {{0}};
    int& done = ready[dec_grad ? 1 : 0][current_device()];
    if (!done) {
        cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, TP::BYTES);
        if (e != cudaSuccess) return (int)e;
        done = 1;
    }
    const int64_t tiles = (P.n + kRound - 1) / kRound;
    int64_t grid = sm_count();
    if (grid > tiles) grid = tiles;
    if (grid < 1) grid = 1;
    StepParams Q = P;
    Q.debug_dx = g_debug_dx;
    kern<<<(unsigned)grid, kTcThreads, TP::BYTES, st>>>(Q);
    return (int)cudaGetLastError();
}

}  // namespace shine_internal
