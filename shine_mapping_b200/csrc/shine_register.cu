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
//
// shine_register_normal_eq_poses evaluates K poses of the same scan: the grid's second dimension is the pose, so row k of
// its [K, 29] output comes from exactly the per-point work, the block count and the fold order that
// shine_register_normal_eq (the K = 1 case of the same code) runs at pose k.  The poses travel in the kernel parameters:
// one pose per launch for K = 1 (a Gauss-Newton iteration keeps the small parameter block it had), up to kPosesPerLaunch
// per launch otherwise.
#include "shine_device.cuh"

namespace {

constexpr int kRT = 256;                       // threads per block
constexpr int kRW = kRT / 32;
constexpr int kOut = SHINE_REGISTER_OUT;       // 21 (H) + 6 (b) + cost + count
constexpr int kMaxBlocks = SHINE_REGISTER_MAX_BLOCKS;
// poses per launch: 48 bytes each in the parameter block, which may hold up to 32 764 bytes on sm_70 and newer
constexpr int kPosesPerLaunch = 512;

struct RegPose {
    float R[9], t[3];          // rounded from the caller's fp64 pose
};

template <int Cap>
struct RegParams {
    shine_octree oct;
    shine_decoder dec;
    const float* points;
    double* partials;          // [poses of this launch, blocks, kOut]
    int64_t n;
    float sigma;
    double kappa2;
    RegPose pose[Cap];         // blockIdx.y selects one
};
static_assert(sizeof(RegParams<kPosesPerLaunch>) <= 32764, "kernel parameters are limited to 32 764 bytes");

struct RegSmem {
    float W1[kH * kF];         // [32][8]
    float W2[kH * kH];         // W2[j][n]
    float W2T[kH * kH];        // W2T[n][j]
    float b1[kH], b2[kH], w3[kH];
    float b3;
    double warp_sum[kRW][kOut];
};

template <int Cap>
__global__ void __launch_bounds__(kRT) register_normal_eq_kernel(const __grid_constant__ RegParams<Cap> P) {
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

    const RegPose& T = P.pose[blockIdx.y];
    double acc[kOut];
#pragma unroll
    for (int k = 0; k < kOut; ++k) acc[k] = 0.0;

    for (int64_t p = (int64_t)blockIdx.x * kRT + tid; p < P.n; p += (int64_t)gridDim.x * kRT) {
        const float px = __ldg(P.points + 3 * p), py = __ldg(P.points + 3 * p + 1), pz = __ldg(P.points + 3 * p + 2);
        float qv[3];
#pragma unroll
        for (int a = 0; a < 3; ++a)
            qv[a] = __fadd_rn(__fadd_rn(__fadd_rn(__fmul_rn(T.R[3 * a], px), __fmul_rn(T.R[3 * a + 1], py)),
                                        __fmul_rn(T.R[3 * a + 2], pz)), T.t[a]);
        const float x = qv[0], y = qv[1], z = qv[2];

        // ---- pred and dpred/dq (shine_device.cuh sdf_grad_at); a q outside lv[0] contributes nothing (also to the count)
        float pr, gs[3];
        if (!sdf_grad_at<true>(P.oct, sm, x, y, z, pr, gs)) continue;
        float gv[3];
#pragma unroll
        for (int a = 0; a < 3; ++a) gv[a] = P.sigma * gs[a];
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
        P.partials[((int64_t)blockIdx.y * gridDim.x + blockIdx.x) * kOut + tid] = v;
    }
}

// out[pose][k] = sum over the pose's block partials of column k: warp k sums blocks lane, lane + 32, ... then a shuffle
// tree; one block per pose
__global__ void __launch_bounds__(32 * kOut) register_fold_kernel(const double* __restrict__ partials, int blocks,
                                                                 double* __restrict__ out) {
    const int k = threadIdx.x >> 5, lane = threadIdx.x & 31;
    partials += (int64_t)blockIdx.x * blocks * kOut;
    double v = 0.0;
    for (int b = lane; b < blocks; b += 32) v += partials[(int64_t)b * kOut + k];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(kFull, v, o);
    if (lane == 0) out[(int64_t)blockIdx.x * kOut + k] = v;
}

__global__ void register_zero_kernel(double* __restrict__ out, int64_t count) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < count) out[i] = 0.0;
}

inline bool is_finite(double v) { return v == v && v - v == 0.0; }

inline int64_t register_blocks(int64_t n) {
    const int64_t blocks = (n + kRT - 1) / kRT;
    return blocks > kMaxBlocks ? kMaxBlocks : blocks;
}

// checks shared by both entries (the scratch is checked by each); none touches the device
int check_register_args(const shine_octree* oct, const shine_decoder* dec, const float* points, int64_t n,
                        const double* poses, int64_t K, float sigma, double kappa, const double* out) {
    if (!oct || !dec || !poses || !out || n < 0 || (n > 0 && !points) || K <= 0 || K > INT32_MAX)
        return SHINE_ERR_INVALID_ARG;
    int rc = check_octree(oct, false);
    if (rc) return rc;
    if ((rc = check_decoder(dec, oct))) return rc;
    if (!(sigma > 0.f) || !is_finite(sigma) || !(kappa > 0.0) || !is_finite(kappa)) return SHINE_ERR_INVALID_ARG;
    for (int64_t k = 0; k < K; ++k)
        for (int i = 0; i < 12; ++i)
            if (!is_finite(poses[16 * k + i])) return SHINE_ERR_INVALID_ARG;
    return SHINE_OK;
}

// the K poses after the checks: chunks of Cap poses, each one normal-equations launch (grid blocks x chunk) and one
// fold launch (one block per pose)
template <int Cap>
int register_chunks(const shine_octree* oct, const shine_decoder* dec, const float* points, int64_t n,
                    const double* poses, int64_t K, float sigma, double kappa, double* out, void* scratch,
                    cudaStream_t st) {
    int rc;
    const int64_t blocks = register_blocks(n);
    const int kPosesPerLaunch = Cap;
    RegParams<Cap> P;
    P.oct = *oct; P.dec = *dec; P.points = points; P.n = n;
    P.sigma = sigma;
    P.kappa2 = kappa * kappa;
    for (int64_t k0 = 0; k0 < K; k0 += kPosesPerLaunch) {
        const int kc = (int)(K - k0 < kPosesPerLaunch ? K - k0 : kPosesPerLaunch);
        for (int k = 0; k < kc; ++k) {
            const double* pose = poses + 16 * (k0 + k);
            for (int a = 0; a < 3; ++a) {
                for (int b = 0; b < 3; ++b) P.pose[k].R[3 * a + b] = (float)pose[4 * a + b];
                P.pose[k].t[a] = (float)pose[4 * a + 3];
            }
        }
        P.partials = static_cast<double*>(scratch) + k0 * blocks * kOut;
        register_normal_eq_kernel<Cap><<<dim3((unsigned)blocks, (unsigned)kc), kRT, 0, st>>>(P);
        register_fold_kernel<<<(unsigned)kc, 32 * kOut, 0, st>>>(P.partials, (int)blocks, out + k0 * kOut);
        if ((rc = (int)cudaGetLastError())) return rc;
    }
    return SHINE_OK;
}

int register_launch(const shine_octree* oct, const shine_decoder* dec, const float* points, int64_t n,
                    const double* poses, int64_t K, float sigma, double kappa, double* out, void* scratch,
                    void* stream) {
    int rc = check_same_device(oct, points);
    if (rc) return rc;
    DeviceGuard guard(oct->lv[0].features);
    const cudaStream_t st = (cudaStream_t)stream;
    if (n == 0) {
        const int64_t count = K * kOut;
        register_zero_kernel<<<(unsigned)((count + 255) / 256), 256, 0, st>>>(out, count);
        return (int)cudaGetLastError();
    }
    if (K == 1) return register_chunks<1>(oct, dec, points, n, poses, K, sigma, kappa, out, scratch, st);
    return register_chunks<kPosesPerLaunch>(oct, dec, points, n, poses, K, sigma, kappa, out, scratch, st);
}

}  // namespace

extern "C" {

int shine_register_normal_eq(const shine_octree* oct, const shine_decoder* dec, const float* points, int64_t n,
                             const double* pose, float sigma, double kappa, double* out, void* scratch,
                             int64_t scratch_bytes, void* stream) {
    int rc = check_register_args(oct, dec, points, n, pose, 1, sigma, kappa, out);
    if (rc) return rc;
    if (!scratch || scratch_bytes < (int64_t)SHINE_REGISTER_SCRATCH_BYTES || ((uintptr_t)scratch & 7)) return SHINE_ERR_INVALID_ARG;
    return register_launch(oct, dec, points, n, pose, 1, sigma, kappa, out, scratch, stream);
}

int64_t shine_register_scratch_bytes(int64_t n, int64_t num_poses) {
    if (n < 0 || num_poses <= 0 || num_poses > INT32_MAX) return -1;
    return register_blocks(n) * num_poses * kOut * (int64_t)sizeof(double);
}

int shine_register_normal_eq_poses(const shine_octree* oct, const shine_decoder* dec, const float* points, int64_t n,
                                   const double* poses, int64_t num_poses, float sigma, double kappa, double* out,
                                   void* scratch, int64_t scratch_bytes, void* stream) {
    int rc = check_register_args(oct, dec, points, n, poses, num_poses, sigma, kappa, out);
    if (rc) return rc;
    if (!scratch || scratch_bytes < shine_register_scratch_bytes(n, num_poses) || ((uintptr_t)scratch & 7))
        return SHINE_ERR_INVALID_ARG;
    return register_launch(oct, dec, points, n, poses, num_poses, sigma, kappa, out, scratch, stream);
}

}  // extern "C"
