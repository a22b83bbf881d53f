// shine_eikonal.cu — the training step with `ekional_loss_on` (config/kitti/kitti_batch.yaml:46) as ONE kernel.
//
// Reference (shine_batch.py:119-142,172-185,208-209 + utils/tools.py:175-185):
//     coord.requires_grad_(True); feature = octree.query_feature(coord); pred = mlp.sdf(feature)
//     g = autograd.grad(pred, coord, ones, create_graph=True)[0] * sigma_sigmoid
//     loss = sdf_bce_loss(pred, label, ...) + weight_e * ((1 - |g[surface]|)^2).mean();  loss.backward()
// i.e. a double backward through gather, MLP and loss (~10 autograd kernels + cuBLAS).  Written out per point:
//     f = sum_c w_c F_c            J = df/dx = sum_c F_c (x) grad w_c                     (one gather, primal + tangent)
//     h1 = relu(W1 f + b1), h2 = relu(W2 h1 + b2), p = w3.h2 + b3        (masks D1, D2)
//     a2 = D2 w3, a1 = D1 W2^T a2, q = W1^T a1 = dp/df;   g = sigma J^T q
//     E = (1 - |g|)^2 on surface samples;   gamma = dL/dg = 2 weight_e / N_surf * (|g| - 1) g / |g|
//     r = dL/dq = sigma J gamma;   s1 = W1 r, t1 = D1 s1, s2 = W2 t1       (ReLU'' = 0: q depends on f only via masks)
// and with dp = dL_bce/dp the gradients of BOTH terms collapse into rank-1 forms that share a1 / a2:
//     dW3 = dp h2 + D2 s2      db3 = dp      dW2 = a2 (x) (dp h1 + t1)   db2 = dp a2
//     dW1 = a1 (x) (dp f + r)  db1 = dp a1   dF_c += (dp w_c + sigma gamma.grad w_c) q
// One thread owns one point (fp32 FFMA, weights broadcast from shared memory); the two rank-1 sums over the 32 points
// of a warp are contracted on the tensor cores (3xTF32 mma.sync, operands staged in the warp's shared-memory tiles).
#include "shine_device.cuh"

namespace {

constexpr int kEW = 4;                 // warps per block
constexpr int kET = 32 * kEW;

struct EikParams {
    shine_octree oct;
    shine_decoder dec;
    const float* coord;
    const float* label;
    const float* weight;       // sign: surface (+) / free space (-); magnitude used only with SHINE_FLAG_WEIGHTED
    const int32_t* n_surface;  // device scalar: number of samples with weight > 0
    float* pred;               // nullable
    float* grad_out;           // nullable [n,3]: g
    float* loss;               // += BCE (or sdf_diff_loss) part
    float* eikonal;            // += sum_surface (1-|g|)^2 / N_surf
    int64_t n;
    float sigma, loss_scale, weight_e;
    int32_t weighted;
    float scale;               // sdf_diff_loss: config.scale
};

constexpr int kTS = 36;     // row stride (floats) of the per-warp [component][point] tiles: conflict-free for the
                            // per-lane column writes AND for the mma fragment reads (bank = 4g + t)

struct EikSmem {
    static constexpr int W1 = 0;                 // [32][8]
    static constexpr int W2 = W1 + kH * kF;      // [32][32]   W2[j][n]
    static constexpr int W2T = W2 + kH * kH;     // [32][32]   W2T[n][j]
    static constexpr int B1 = W2T + kH * kH;
    static constexpr int B2 = B1 + kH;
    static constexpr int W3 = B2 + kH;
    static constexpr int B3 = W3 + kH;           // [1] + 3 pad
    static constexpr int RED = B3 + 4;           // [1380] block accumulator of decoder gradients
    static constexpr int TILES = RED + 1380;     // per warp: tA1 | tA2 | tU (= h1 scratch) | tH2 : [32][kTS], tV: [8][kTS]
    static constexpr int kPerWarp = (4 * 32 + 8) * kTS;
    static constexpr int FLOATS = TILES + kEW * kPerWarp;
};

template <bool DEC_GRAD, int LOSS = kLossBce>
__global__ void __launch_bounds__(kET, 2) sdf_eikonal_kernel(const __grid_constant__ EikParams P) {
    extern __shared__ __align__(16) float sm[];
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int g = lane >> 2, t = lane & 3;
    for (int i = tid; i < kH * kF; i += kET) sm[EikSmem::W1 + i] = P.dec.w1[i];
    for (int i = tid; i < kH * kH; i += kET) {
        const float w = P.dec.w2[i];
        sm[EikSmem::W2 + i] = w;
        sm[EikSmem::W2T + (i % kH) * kH + i / kH] = w;
    }
    if (tid < kH) {
        sm[EikSmem::B1 + tid] = P.dec.b1 ? P.dec.b1[tid] : 0.f;
        sm[EikSmem::B2 + tid] = P.dec.b2 ? P.dec.b2[tid] : 0.f;
        sm[EikSmem::W3 + tid] = P.dec.w3[tid];
    }
    if (tid == 0) sm[EikSmem::B3] = P.dec.b3 ? P.dec.b3[0] : 0.f;
    for (int i = tid; i < 1380; i += kET) sm[EikSmem::RED + i] = 0.f;
    __syncthreads();

    const float* W1 = sm + EikSmem::W1;
    const float* W2 = sm + EikSmem::W2;
    const float* W2T = sm + EikSmem::W2T;
    const float* w3 = sm + EikSmem::W3;
    // per-warp tiles, [component][point]: element (c, this lane) lives at tile[c * kTS + lane]
    float* tA1 = sm + EikSmem::TILES + warp * EikSmem::kPerWarp;     // a1
    float* tA2 = tA1 + 32 * kTS;                                        // a2 = D2 w3
    float* tU = tA2 + 32 * kTS;                                         // h1, later u = dp h1 + t1
    float* tH2 = tU + 32 * kTS;                                         // h2
    float* tV = tH2 + 32 * kTS;                                         // v = dp f + r   [8][kTS]
    float* red = sm + EikSmem::RED;
    constexpr int oW1 = 0, oB1 = 256, oW2 = 288, oB2 = 1312, oW3 = 1344, oB3 = 1376;

    const bool poly = P.oct.poly_interp != 0;
    const int L = P.oct.num_levels;
    const int nsurf = P.n_surface ? *P.n_surface : 0;
    const float ce = nsurf > 0 ? 2.0f * P.weight_e / (float)nsurf : 0.f;
    const float inv_ns = nsurf > 0 ? 1.0f / (float)nsurf : 0.f;

    float dW2[2][4][4], dW1[2][4], db2x[2][4], db1x[2][4];
#pragma unroll
    for (int a = 0; a < 2; ++a) {
#pragma unroll
        for (int b = 0; b < 4; ++b) { dW2[a][b][0] = dW2[a][b][1] = dW2[a][b][2] = dW2[a][b][3] = 0.f; }
#pragma unroll
        for (int b = 0; b < 4; ++b) { dW1[a][b] = db2x[a][b] = db1x[a][b] = 0.f; }
    }
    float loss_acc = 0.f, eik_acc = 0.f;

    const int64_t num_tiles = (P.n + 31) / 32;
    for (int64_t tile = (int64_t)blockIdx.x * kEW + warp; tile < num_tiles; tile += (int64_t)gridDim.x * kEW) {
        const int64_t p = tile * 32 + lane;
        const bool valid = p < P.n;
        float x = 0.f, y = 0.f, z = 0.f, lab = 0.f, wraw = 0.f;
        if (valid) {
            x = __ldg(P.coord + 3 * p); y = __ldg(P.coord + 3 * p + 1); z = __ldg(P.coord + 3 * p + 2);
            lab = __ldg(P.label + p);
            wraw = __ldg(P.weight + p);
        }
        const bool surface = valid && wraw > 0.f;                      // shine_batch.py:137
        const float wgt = P.weighted ? fabsf(wraw) : 1.0f;              // shine_batch.py:172 + utils/loss.py:18-21

        // ---- gather: primal feature f and tangent J = df/dx in one pass over the 8 x L corner rows ---------------
        float f[8], J[8][3];
#pragma unroll
        for (int k = 0; k < 8; ++k) { f[k] = 0.f; J[k][0] = J[k][1] = J[k][2] = 0.f; }
#pragma unroll 1
        for (int i = 0; i < L; ++i) {
            const shine_level& lv = P.oct.lv[i];
            const HashSlot* slots = reinterpret_cast<const HashSlot*>(lv.hash_slots);
            const int s = valid ? probe_slot(slots, lv.hash_capacity - 1, morton_of(x, y, z, lv.level)) : -1;
            if (s < 0) continue;
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

        // ---- Decoder.sdf forward (model/decoder.py:49-63), fp32: outputs go to the warp's column tiles ---------------------
        uint32_t m1 = 0, m2 = 0;
#pragma unroll 1
        for (int n = 0; n < 32; ++n) {
            const float4 wa = *reinterpret_cast<const float4*>(W1 + n * 8), wb = *reinterpret_cast<const float4*>(W1 + n * 8 + 4);
            float a = sm[EikSmem::B1 + n];
            a = fmaf(wa.x, f[0], a); a = fmaf(wa.y, f[1], a); a = fmaf(wa.z, f[2], a); a = fmaf(wa.w, f[3], a);
            a = fmaf(wb.x, f[4], a); a = fmaf(wb.y, f[5], a); a = fmaf(wb.z, f[6], a); a = fmaf(wb.w, f[7], a);
            m1 |= (a > 0.f ? 1u : 0u) << n;
            tU[n * kTS + lane] = fmaxf(a, 0.f);
        }
        float h1[32];
#pragma unroll
        for (int n = 0; n < 32; ++n) h1[n] = tU[n * kTS + lane];
        float pr = sm[EikSmem::B3];
#pragma unroll 1
        for (int j = 0; j < 32; ++j) {
            float a = sm[EikSmem::B2 + j];
#pragma unroll
            for (int n = 0; n < 32; n += 4) {
                const float4 w = *reinterpret_cast<const float4*>(W2 + j * 32 + n);
                a = fmaf(w.x, h1[n], a); a = fmaf(w.y, h1[n + 1], a); a = fmaf(w.z, h1[n + 2], a); a = fmaf(w.w, h1[n + 3], a);
            }
            const bool on = a > 0.f;
            m2 |= (on ? 1u : 0u) << j;
            const float hj = fmaxf(a, 0.f);
            tH2[j * kTS + lane] = hj;
            tA2[j * kTS + lane] = on ? w3[j] : 0.f;               // a2 = D2 w3
            pr = fmaf(hj, w3[j], pr);
        }
        if (P.pred && valid) P.pred[p] = pr;

        // ---- sdf_bce_loss (utils/loss.py:17-24) or sdf_diff_loss (:6-14) and its dL/dpred --------------------------------
        float dp = 0.f;
        if (valid) {
            if constexpr (LOSS == kLossBce) {
                const float zt = __fdividef(1.0f, 1.0f + __expf(-__fdividef(lab, P.sigma)));
                const float e = __expf(-fabsf(pr));
                loss_acc += wgt * (fmaxf(pr, 0.f) - pr * zt + __logf(1.0f + e));
                const float rs = __fdividef(1.0f, 1.0f + e);
                dp = ((pr >= 0.f ? rs : e * rs) - zt) * wgt * P.loss_scale;
            } else {
                float li, dli;
                diff_point<LOSS>(pr, lab, P.scale, li, dli);
                loss_acc += wgt * li;
                dp = dli * wgt * P.loss_scale;
            }
        }

        // ---- a1 = D1 W2^T a2,  q = W1^T a1 = dpred/dfeature -----------------------------------------------------------------
        float q[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
        {
            float a2[32];
#pragma unroll
            for (int j = 0; j < 32; ++j) a2[j] = ((m2 >> j) & 1u) ? w3[j] : 0.f;
#pragma unroll 1
            for (int n = 0; n < 32; ++n) {
                float a = 0.f;
#pragma unroll
                for (int j = 0; j < 32; j += 4) {
                    const float4 w = *reinterpret_cast<const float4*>(W2T + n * 32 + j);
                    a = fmaf(w.x, a2[j], a); a = fmaf(w.y, a2[j + 1], a); a = fmaf(w.z, a2[j + 2], a); a = fmaf(w.w, a2[j + 3], a);
                }
                a = ((m1 >> n) & 1u) ? a : 0.f;
                tA1[n * kTS + lane] = a;
                const float4 wa = *reinterpret_cast<const float4*>(W1 + n * 8), wb = *reinterpret_cast<const float4*>(W1 + n * 8 + 4);
                q[0] = fmaf(a, wa.x, q[0]); q[1] = fmaf(a, wa.y, q[1]); q[2] = fmaf(a, wa.z, q[2]); q[3] = fmaf(a, wa.w, q[3]);
                q[4] = fmaf(a, wb.x, q[4]); q[5] = fmaf(a, wb.y, q[5]); q[6] = fmaf(a, wb.z, q[6]); q[7] = fmaf(a, wb.w, q[7]);
            }
        }

        // ---- g = sigma J^T q; eikonal term and gamma = dL/dg (shine_batch.py:141-142,183-185) -------------------------
        float gv[3];
#pragma unroll
        for (int a = 0; a < 3; ++a) {
            float acc = 0.f;
#pragma unroll
            for (int k = 0; k < 8; ++k) acc = fmaf(J[k][a], q[k], acc);
            gv[a] = P.sigma * acc;
        }
        if (P.grad_out && valid) { P.grad_out[3 * p] = gv[0]; P.grad_out[3 * p + 1] = gv[1]; P.grad_out[3 * p + 2] = gv[2]; }
        float gam[3] = {0.f, 0.f, 0.f};
        if (surface) {
            const float nrm = sqrtf(gv[0] * gv[0] + gv[1] * gv[1] + gv[2] * gv[2]);
            eik_acc += (1.0f - nrm) * (1.0f - nrm);
            const float coef = nrm > 0.f ? ce * (nrm - 1.0f) / nrm : 0.f;      // torch: d|g|/dg = 0 at g = 0
            gam[0] = coef * gv[0]; gam[1] = coef * gv[1]; gam[2] = coef * gv[2];
        }
        // r = dL/dq = sigma J gamma;  v = dp f + r
        float r[8];
#pragma unroll
        for (int k = 0; k < 8; ++k) {
            r[k] = P.sigma * (J[k][0] * gam[0] + J[k][1] * gam[1] + J[k][2] * gam[2]);
            tV[k * kTS + lane] = fmaf(dp, f[k], r[k]);
        }
        // t1 = D1 W1 r;  u = dp h1 + t1
        float t1[32];
#pragma unroll
        for (int n = 0; n < 32; ++n) {
            const float4 wa = *reinterpret_cast<const float4*>(W1 + n * 8), wb = *reinterpret_cast<const float4*>(W1 + n * 8 + 4);
            float a = wa.x * r[0];
            a = fmaf(wa.y, r[1], a); a = fmaf(wa.z, r[2], a); a = fmaf(wa.w, r[3], a);
            a = fmaf(wb.x, r[4], a); a = fmaf(wb.y, r[5], a); a = fmaf(wb.z, r[6], a); a = fmaf(wb.w, r[7], a);
            t1[n] = ((m1 >> n) & 1u) ? a : 0.f;
            tU[n * kTS + lane] = fmaf(dp, h1[n], t1[n]);
        }
        // c3 = dp h2 + D2 W2 t1: this point's share of dW3, summed over the warp right away
        float mine = 0.f;
#pragma unroll 1
        for (int j = 0; j < 32; ++j) {
            float a = 0.f;
#pragma unroll
            for (int n = 0; n < 32; n += 4) {
                const float4 w = *reinterpret_cast<const float4*>(W2 + j * 32 + n);
                a = fmaf(w.x, t1[n], a); a = fmaf(w.y, t1[n + 1], a); a = fmaf(w.z, t1[n + 2], a); a = fmaf(w.w, t1[n + 3], a);
            }
            float c3 = fmaf(dp, tH2[j * kTS + lane], ((m2 >> j) & 1u) ? a : 0.f);
            if (DEC_GRAD) {
#pragma unroll
                for (int o = 16; o > 0; o >>= 1) c3 += __shfl_xor_sync(kFull, c3, o);
                if (lane == j) mine = c3;
            }
        }

        // ---- decoder gradients: the rank-1 sums over the warp's 32 points on the tensor cores -------------------------
        if (DEC_GRAD) {
            atomicAdd(red + oW3 + lane, mine);
            float sdp = dp;
#pragma unroll
            for (int o = 16; o > 0; o >>= 1) sdp += __shfl_xor_sync(kFull, sdp, o);
            if (lane == 0) atomicAdd(red + oB3, sdp);
            __syncwarp();
#pragma unroll
            for (int ks = 0; ks < 4; ++ks) {
                // dp of points 8ks+t / 8ks+t+4 as an extra B column (n = 0): the bias gradients ride on the same MMAs
                const float d0 = __shfl_sync(kFull, dp, 8 * ks + t), d1 = __shfl_sync(kFull, dp, 8 * ks + t + 4);
                uint2 bdh, bdl;
                split_fast2(g == 0 ? d0 : 0.f, g == 0 ? d1 : 0.f, bdh.x, bdh.y, bdl.x, bdl.y);
                uint2 bh[4], bl[4];
#pragma unroll
                for (int nt = 0; nt < 4; ++nt) {       // B[k = point][n = k1] = u
                    split_fast2(tU[(8 * nt + g) * kTS + 8 * ks + t], tU[(8 * nt + g) * kTS + 8 * ks + t + 4], bh[nt].x, bh[nt].y,
                                bl[nt].x, bl[nt].y);
                }
                uint2 vh, vl;
                split_fast2(tV[g * kTS + 8 * ks + t], tV[g * kTS + 8 * ks + t + 4], vh.x, vh.y, vl.x, vl.y);
#pragma unroll
                for (int mt = 0; mt < 2; ++mt) {
                    AFrag<3> a;       // a2^T: rows = n2, cols = points
                    a.set_packed(tA2[(16 * mt + g) * kTS + 8 * ks + t], tA2[(16 * mt + g + 8) * kTS + 8 * ks + t],
                                 tA2[(16 * mt + g) * kTS + 8 * ks + t + 4], tA2[(16 * mt + g + 8) * kTS + 8 * ks + t + 4]);
                    AFrag<3> c;       // a1^T: rows = n1, cols = points
                    c.set_packed(tA1[(16 * mt + g) * kTS + 8 * ks + t], tA1[(16 * mt + g + 8) * kTS + 8 * ks + t],
                                 tA1[(16 * mt + g) * kTS + 8 * ks + t + 4], tA1[(16 * mt + g + 8) * kTS + 8 * ks + t + 4]);
                    mma3x4<3>(dW2[mt], a, bh, bl);                       // term-major: no back-to-back dependent HMMAs
                    mma3x2<3>(db2x[mt], dW1[mt], a, c, bdh, bdl, vh, vl);
                    mma3<3>(db1x[mt], c, bdh, bdl);
                }
            }
            __syncwarp();
        }

        // ---- scatter: dF_c += (dp w_c + sigma gamma . grad w_c) q   (both loss terms, one pass) ------------------------
#pragma unroll 1
        for (int i = 0; i < L; ++i) {
            const shine_level& lv = P.oct.lv[i];
            const HashSlot* slots = reinterpret_cast<const HashSlot*>(lv.hash_slots);
            const int s = valid ? probe_slot(slots, lv.hash_capacity - 1, morton_of(x, y, z, lv.level)) : -1;
            if (s < 0) continue;
            const int4 ia = ldg_i4(slots[s].ids0), ib = ldg_i4(slots[s].ids1);
            const int ids[8] = {ia.x, ib.x, ia.y, ib.y, ia.z, ib.z, ia.w, ib.w};
            BlendD b; b.init(x, y, z, lv.level, poly);
#pragma unroll
            for (int c = 0; c < 8; ++c) {
                const float X = (c & 4) ? b.t[0] : b.u[0], Y = (c & 2) ? b.t[1] : b.u[1], Z = (c & 1) ? b.t[2] : b.u[2];
                const float w = __fmul_rn(__fmul_rn(X, Y), Z);
                float dw[3]; b.dw(c, dw);
                const float sc = fmaf(dp, w, P.sigma * (gam[0] * dw[0] + gam[1] * dw[1] + gam[2] * dw[2]));
                float* dst = lv.feature_grads + (int64_t)ids[c] * kF;
                red_add_f4(dst, sc * q[0], sc * q[1], sc * q[2], sc * q[3]);
                red_add_f4(dst + 4, sc * q[4], sc * q[5], sc * q[6], sc * q[7]);
            }
        }
    }

    // ---- epilogue: loss terms and the block's decoder gradients -------------------------------------------------------------
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        loss_acc += __shfl_xor_sync(kFull, loss_acc, o);
        eik_acc += __shfl_xor_sync(kFull, eik_acc, o);
    }
    if (lane == 0) {
        if (P.loss && loss_acc != 0.f) atomicAdd(P.loss, loss_acc * P.loss_scale);
        if (P.eikonal && eik_acc != 0.f) atomicAdd(P.eikonal, eik_acc * inv_ns);
    }
    if (DEC_GRAD) {
#pragma unroll
        for (int mt = 0; mt < 2; ++mt) {
#pragma unroll
            for (int nt = 0; nt < 4; ++nt) {
                atomicAdd(red + oW2 + (16 * mt + g) * kH + 8 * nt + 2 * t, dW2[mt][nt][0]);
                atomicAdd(red + oW2 + (16 * mt + g) * kH + 8 * nt + 2 * t + 1, dW2[mt][nt][1]);
                atomicAdd(red + oW2 + (16 * mt + g + 8) * kH + 8 * nt + 2 * t, dW2[mt][nt][2]);
                atomicAdd(red + oW2 + (16 * mt + g + 8) * kH + 8 * nt + 2 * t + 1, dW2[mt][nt][3]);
            }
            atomicAdd(red + oW1 + (16 * mt + g) * kF + 2 * t, dW1[mt][0]);
            atomicAdd(red + oW1 + (16 * mt + g) * kF + 2 * t + 1, dW1[mt][1]);
            atomicAdd(red + oW1 + (16 * mt + g + 8) * kF + 2 * t, dW1[mt][2]);
            atomicAdd(red + oW1 + (16 * mt + g + 8) * kF + 2 * t + 1, dW1[mt][3]);
            if (t == 0) {      // column 0 of the extra B tile carried dp
                atomicAdd(red + oB2 + 16 * mt + g, db2x[mt][0]); atomicAdd(red + oB2 + 16 * mt + g + 8, db2x[mt][2]);
                atomicAdd(red + oB1 + 16 * mt + g, db1x[mt][0]); atomicAdd(red + oB1 + 16 * mt + g + 8, db1x[mt][2]);
            }
        }
        __syncthreads();
        for (int i = tid; i < 1377; i += kET) {
            const float val = red[i];
            if (val == 0.f) continue;
            float* dst;
            if (i < oB1) dst = P.dec.gw1 + i;
            else if (i < oW2) dst = P.dec.gb1 ? P.dec.gb1 + (i - oB1) : nullptr;
            else if (i < oB2) dst = P.dec.gw2 + (i - oW2);
            else if (i < oW3) dst = P.dec.gb2 ? P.dec.gb2 + (i - oB2) : nullptr;
            else if (i < oB3) dst = P.dec.gw3 + (i - oW3);
            else dst = P.dec.gb3;
            if (dst) atomicAdd(dst, val);
        }
    }
}

__global__ void count_positive_kernel(const float* __restrict__ w, int64_t n, int32_t* __restrict__ out) {
    int local = 0;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x)
        local += w[i] > 0.f ? 1 : 0;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) local += __shfl_xor_sync(kFull, local, o);
    if ((threadIdx.x & 31) == 0 && local) atomicAdd(out, local);
}

template <bool DEC_GRAD, int LOSS = kLossBce>
int launch_eikonal(const EikParams& P, cudaStream_t st) {
    auto kern = sdf_eikonal_kernel<DEC_GRAD, LOSS>;
    const size_t bytes = (size_t)EikSmem::FLOATS * sizeof(float);
    static int ready[kMaxDevices] = {0};
    int& done = ready[current_device()];
    if (!done) {
        cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bytes);
        if (e != cudaSuccess) return (int)e;
        done = 1;
    }
    const int64_t tiles = (P.n + 31) / 32;
    int64_t grid = (tiles + kEW - 1) / kEW;
    const int64_t cap = (int64_t)sm_count() * 2;
    if (grid > cap) grid = cap;
    kern<<<(unsigned)grid, kET, bytes, st>>>(P);
    return (int)cudaGetLastError();
}

}  // namespace

extern "C" {

int shine_count_positive(const float* values, int64_t n, int32_t* out_count, void* stream) {
    if (n < 0 || !out_count || (n > 0 && !values)) return SHINE_ERR_INVALID_ARG;
    if (n == 0) return SHINE_OK;
    DeviceGuard guard(out_count);
    int64_t blocks = (n + 1023) / 1024;
    if (blocks > 1024) blocks = 1024;
    count_positive_kernel<<<(unsigned)blocks, 256, 0, (cudaStream_t)stream>>>(values, n, out_count);
    return (int)cudaGetLastError();
}

int shine_sdf_bce_eikonal_step(const shine_octree* oct, const shine_decoder* dec, const float* coord, const float* label,
                               const float* weight, int64_t n, float sigma, float loss_scale, float weight_e,
                               const int32_t* n_surface, float* out_pred, float* out_grad, float* out_loss,
                               float* out_eikonal, uint32_t flags, void* stream) {
    int rc = check_octree(oct, true);
    if (rc) return rc;
    if (!dec) return SHINE_ERR_INVALID_ARG;
    if (dec->in_dim != kF || dec->hidden != kH || dec->mlp_level != 2 || oct->feature_dim != kF) return SHINE_ERR_UNSUPPORTED;
    if (!dec->w1 || !dec->w2 || !dec->w3) return SHINE_ERR_INVALID_ARG;
    if (n < 0 || (n > 0 && (!coord || !label || !weight || !n_surface))) return SHINE_ERR_INVALID_ARG;
    if (!(sigma > 0.f)) return SHINE_ERR_INVALID_ARG;
    const bool dec_grad = dec->gw1 || dec->gw2 || dec->gw3;
    if (dec_grad && !(dec->gw1 && dec->gw2 && dec->gw3)) return SHINE_ERR_INVALID_ARG;
    if (n == 0) return SHINE_OK;
    if ((rc = check_same_device(oct, coord))) return rc;
    DeviceGuard guard(oct->lv[0].features);
    EikParams P;
    P.oct = *oct; P.dec = *dec; P.coord = coord; P.label = label; P.weight = weight; P.n_surface = n_surface;
    P.pred = out_pred; P.grad_out = out_grad; P.loss = out_loss; P.eikonal = out_eikonal; P.n = n;
    P.sigma = sigma; P.loss_scale = loss_scale; P.weight_e = weight_e;
    P.weighted = (flags & SHINE_FLAG_WEIGHTED) ? 1 : 0;
    return dec_grad ? launch_eikonal<true>(P, (cudaStream_t)stream) : launch_eikonal<false>(P, (cudaStream_t)stream);
}

int shine_sdf_diff_eikonal_step(const shine_octree* oct, const shine_decoder* dec, const float* coord, const float* label,
                                const float* weight, int64_t n, float scale, float sigma, float loss_scale, float weight_e,
                                const int32_t* n_surface, float* out_pred, float* out_grad, float* out_loss,
                                float* out_eikonal, uint32_t flags, void* stream) {
    if (flags & ~(SHINE_FLAG_TF32X1 | SHINE_FLAG_LOSS_L2)) return SHINE_ERR_UNSUPPORTED;
    int rc = check_octree(oct, true);
    if (rc) return rc;
    if (!dec) return SHINE_ERR_INVALID_ARG;
    if (dec->in_dim != kF || dec->hidden != kH || dec->mlp_level != 2 || oct->feature_dim != kF) return SHINE_ERR_UNSUPPORTED;
    if (!dec->w1 || !dec->w2 || !dec->w3) return SHINE_ERR_INVALID_ARG;
    if (!weight || n < 0 || (n > 0 && (!coord || !label || !n_surface))) return SHINE_ERR_INVALID_ARG;
    if (!(sigma > 0.f) || !valid_scale(scale)) return SHINE_ERR_INVALID_ARG;
    const bool dec_grad = dec->gw1 || dec->gw2 || dec->gw3;
    if (dec_grad && !(dec->gw1 && dec->gw2 && dec->gw3)) return SHINE_ERR_INVALID_ARG;
    if (n == 0) return SHINE_OK;
    if ((rc = check_same_device(oct, coord))) return rc;
    DeviceGuard guard(oct->lv[0].features);
    EikParams P;
    P.oct = *oct; P.dec = *dec; P.coord = coord; P.label = label; P.weight = weight; P.n_surface = n_surface;
    P.pred = out_pred; P.grad_out = out_grad; P.loss = out_loss; P.eikonal = out_eikonal; P.n = n;
    P.sigma = sigma; P.loss_scale = loss_scale; P.weight_e = weight_e;
    P.weighted = 1;                                       // shine_batch.py:172 |weight|, always applied
    P.scale = scale;
    const cudaStream_t st = (cudaStream_t)stream;
    if (flags & SHINE_FLAG_LOSS_L2)
        return dec_grad ? launch_eikonal<true, kLossL2>(P, st) : launch_eikonal<false, kLossL2>(P, st);
    return dec_grad ? launch_eikonal<true, kLossL1>(P, st) : launch_eikonal<false, kLossL1>(P, st);
}

}  // extern "C"
