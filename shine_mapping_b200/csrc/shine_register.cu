// shine_register.cu — the normal equations of scan-to-map registration against the SDF map (odometry.py).
//
// For a scan p_i (sensor frame, scaled) and a pose T = (R, t), per point, one thread each:
//     q = R p + t (fp32, every operation rounded on its own)
//     f = sum_c w_c F_c,  J = df/dq = sum_c F_c (x) grad w_c         (one gather over the 8 x L corner rows)
//     pred = Decoder.sdf(f) (fp32 FMA chains, weights in shared memory), masks D1, D2 of the two ReLUs
//     a1 = D1 W2^T (D2 w3),  dq = W1^T a1 = dpred/df,  g = sigma J^T dq    (the input gradient of shine_eikonal.cu)
//     r = sigma pred (the SDF in scaled units), valid = q's voxel exists at lv[0]
// and then in fp64 from those fp32 values: the Jacobian of a left-multiplied twist (rho, phi), Jr = [g, q x g], the
// Geman-McClure weight w = (k^2 / (k^2 + r^2))^2 and the point's share of H = sum w Jr^T Jr (upper triangle, row-major),
// b = sum w Jr^T r, sum w r^2 and the valid count.  Each thread sums its points in fp64, warps by a fixed shuffle tree,
// blocks by warp order into one row of the scratch; a second kernel adds the rows in a fixed order into out[29].  No
// floating-point atomics: two launches on the same inputs give the same bits.
#include "shine_device.cuh"

namespace {

constexpr int kRT = 256;                       // threads per block
constexpr int kRW = kRT / 32;
constexpr int kOut = SHINE_REGISTER_OUT;       // 21 (H) + 6 (b) + cost + count
constexpr int kMaxBlocks = SHINE_REGISTER_MAX_BLOCKS;

struct RegParams {
    shine_octree oct;
    shine_decoder dec;
    const float* points;
    double* partials;          // [blocks, kOut]
    int64_t n;
    float R[9], t[3];
    float sigma;
    double kappa2;
};

struct RegSmem {
    float W1[kH * kF];         // [32][8]
    float W2[kH * kH];         // W2[j][n]
    float W2T[kH * kH];        // W2T[n][j]
    float b1[kH], b2[kH], w3[kH];
    float b3;
    double warp_sum[kRW][kOut];
};

__global__ void __launch_bounds__(kRT) register_normal_eq_kernel(const __grid_constant__ RegParams P) {
    __shared__ __align__(16) RegSmem sm;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    for (int i = tid; i < kH * kF; i += kRT) sm.W1[i] = P.dec.w1[i];
    for (int i = tid; i < kH * kH; i += kRT) {
        const float w = P.dec.w2[i];
        sm.W2[i] = w;
        sm.W2T[(i % kH) * kH + i / kH] = w;
    }
    if (tid < kH) {
        sm.b1[tid] = P.dec.b1 ? P.dec.b1[tid] : 0.f;
        sm.b2[tid] = P.dec.b2 ? P.dec.b2[tid] : 0.f;
        sm.w3[tid] = P.dec.w3[tid];
    }
    if (tid == 0) sm.b3 = P.dec.b3 ? P.dec.b3[0] : 0.f;
    __syncthreads();

    const bool poly = P.oct.poly_interp != 0;
    const int L = P.oct.num_levels;
    double acc[kOut];
#pragma unroll
    for (int k = 0; k < kOut; ++k) acc[k] = 0.0;

    for (int64_t p = (int64_t)blockIdx.x * kRT + tid; p < P.n; p += (int64_t)gridDim.x * kRT) {
        const float px = __ldg(P.points + 3 * p), py = __ldg(P.points + 3 * p + 1), pz = __ldg(P.points + 3 * p + 2);
        float qv[3];
#pragma unroll
        for (int a = 0; a < 3; ++a)
            qv[a] = __fadd_rn(__fadd_rn(__fadd_rn(__fmul_rn(P.R[3 * a], px), __fmul_rn(P.R[3 * a + 1], py)),
                                        __fmul_rn(P.R[3 * a + 2], pz)), P.t[a]);
        const float x = qv[0], y = qv[1], z = qv[2];

        // ---- gather: f and J = df/dq over the 8 x L corner rows; valid = a hit at lv[0] ---------------------------------
        float f[8], J[8][3];
#pragma unroll
        for (int k = 0; k < 8; ++k) { f[k] = 0.f; J[k][0] = J[k][1] = J[k][2] = 0.f; }
        bool valid = false;
#pragma unroll 1
        for (int i = 0; i < L; ++i) {
            const shine_level& lv = P.oct.lv[i];
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
        if (!valid) continue;                // masked: contributes nothing (also to the count)

        // ---- Decoder.sdf forward (model/decoder.py:49-63), fp32 FMA chains ---------------------------------------------------
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

        // ---- dq = W1^T D1 W2^T D2 w3 = dpred/df, g = sigma J^T dq ------------------------------------------------------------
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
        float gv[3];
#pragma unroll
        for (int a = 0; a < 3; ++a) {
            float s = 0.f;
#pragma unroll
            for (int k = 0; k < 8; ++k) s = fmaf(J[k][a], dq[k], s);
            gv[a] = P.sigma * s;
        }
        const float r = P.sigma * pr;

        // ---- fp64 from here: Jr = [g, q x g], Geman-McClure weight, the point's share --------------------------------------
        const double g0 = gv[0], g1 = gv[1], g2 = gv[2], q0 = x, q1 = y, q2 = z, rd = r;
        const double Jr[6] = {g0, g1, g2, q1 * g2 - q2 * g1, q2 * g0 - q0 * g2, q0 * g1 - q1 * g0};
        const double den = P.kappa2 + rd * rd;
        const double wk = P.kappa2 / den;
        const double w = wk * wk;
        int k = 0;
#pragma unroll
        for (int i = 0; i < 6; ++i) {
            const double wi = w * Jr[i];
#pragma unroll
            for (int j = i; j < 6; ++j) acc[k++] += wi * Jr[j];
        }
#pragma unroll
        for (int i = 0; i < 6; ++i) acc[21 + i] += w * Jr[i] * rd;
        acc[27] += w * rd * rd;
        acc[28] += 1.0;
    }

    // ---- block partial: shuffle tree per warp, warps in order ---------------------------------------------------------
#pragma unroll
    for (int k = 0; k < kOut; ++k) {
        double v = acc[k];
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(kFull, v, o);
        if (lane == 0) sm.warp_sum[warp][k] = v;
    }
    __syncthreads();
    if (tid < kOut) {
        double v = 0.0;
#pragma unroll
        for (int wi = 0; wi < kRW; ++wi) v += sm.warp_sum[wi][tid];
        P.partials[(int64_t)blockIdx.x * kOut + tid] = v;
    }
}

// out[k] = sum over the block partials of column k: warp k sums blocks lane, lane + 32, ... then a shuffle tree
__global__ void __launch_bounds__(32 * kOut) register_fold_kernel(const double* __restrict__ partials, int blocks,
                                                                 double* __restrict__ out) {
    const int k = threadIdx.x >> 5, lane = threadIdx.x & 31;
    double v = 0.0;
    for (int b = lane; b < blocks; b += 32) v += partials[(int64_t)b * kOut + k];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(kFull, v, o);
    if (lane == 0) out[k] = v;
}

__global__ void register_zero_kernel(double* __restrict__ out) {
    if (threadIdx.x < kOut) out[threadIdx.x] = 0.0;
}

inline bool is_finite(double v) { return v == v && v - v == 0.0; }

}  // namespace

extern "C" {

int shine_register_normal_eq(const shine_octree* oct, const shine_decoder* dec, const float* points, int64_t n,
                             const double* pose, float sigma, double kappa, double* out, void* scratch,
                             int64_t scratch_bytes, void* stream) {
    if (!oct || !dec || !pose || !out || n < 0 || (n > 0 && !points)) return SHINE_ERR_INVALID_ARG;
    int rc = check_octree(oct, false);
    if (rc) return rc;
    if ((rc = check_decoder(dec, oct))) return rc;
    if (!(sigma > 0.f) || !is_finite(sigma) || !(kappa > 0.0) || !is_finite(kappa)) return SHINE_ERR_INVALID_ARG;
    for (int i = 0; i < 12; ++i)
        if (!is_finite(pose[i])) return SHINE_ERR_INVALID_ARG;
    if (!scratch || scratch_bytes < (int64_t)SHINE_REGISTER_SCRATCH_BYTES || ((uintptr_t)scratch & 7)) return SHINE_ERR_INVALID_ARG;
    if ((rc = check_same_device(oct, points))) return rc;
    DeviceGuard guard(oct->lv[0].features);
    const cudaStream_t st = (cudaStream_t)stream;
    if (n == 0) {
        register_zero_kernel<<<1, 32, 0, st>>>(out);
        return (int)cudaGetLastError();
    }
    RegParams P;
    P.oct = *oct; P.dec = *dec; P.points = points; P.partials = static_cast<double*>(scratch); P.n = n;
    for (int a = 0; a < 3; ++a) {
        for (int b = 0; b < 3; ++b) P.R[3 * a + b] = (float)pose[4 * a + b];
        P.t[a] = (float)pose[4 * a + 3];
    }
    P.sigma = sigma;
    P.kappa2 = kappa * kappa;
    int64_t blocks = (n + kRT - 1) / kRT;
    if (blocks > kMaxBlocks) blocks = kMaxBlocks;
    register_normal_eq_kernel<<<(unsigned)blocks, kRT, 0, st>>>(P);
    register_fold_kernel<<<1, 32 * kOut, 0, st>>>(P.partials, (int)blocks, out);
    return (int)cudaGetLastError();
}

}  // extern "C"
