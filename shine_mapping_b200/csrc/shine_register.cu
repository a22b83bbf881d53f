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
//
// shine_register_normal_eq_scans generalises that to items, each a pose and its own segment (begin, n) of one
// concatenated points array: item k runs G_k = min(ceil(n_k / 256), 1024) blocks with a grid-stride of G_k blocks, its
// partials sit at its own prefix offset of the scratch and its fold adds its G_k rows in block order, so row k equals
// shine_register_normal_eq(points + 3 begin_k, n_k, pose_k) bit for bit.  A launch's grid is as wide as its widest item;
// the blocks of an item at or past its G_k return before they touch anything.  Both entries instantiate one kernel
// template: its Item is a bare pose (one segment shared by every pose, n in the parameters) or a pose with its segment.
#include <type_traits>

#include "shine_device.cuh"

namespace {

constexpr int kRT = 256;                       // threads per block
constexpr int kRW = kRT / 32;
constexpr int kOut = SHINE_REGISTER_OUT;       // 21 (H) + 6 (b) + cost + count
constexpr int kMaxBlocks = SHINE_REGISTER_MAX_BLOCKS;
// items per launch: the parameter block may hold up to 32 764 bytes on sm_70 and newer.  A bare pose takes 48 bytes, so
// 512 fit; a pose with its segment takes 72, so the scans entry launches at most 384 items at a time (the segment table
// stays in the parameters rather than in device memory: nothing to copy or allocate per call)
constexpr int kPosesPerLaunch = 512;
constexpr int kItemsPerLaunch = SHINE_REGISTER_ITEMS_PER_LAUNCH;

struct RegPose {
    float R[9], t[3];          // rounded from the caller's fp64 pose
};

struct RegItem {
    RegPose pose;
    int64_t begin, n;          // the item's points: points[begin .. begin + n)
    int32_t block0, blocks;    // its partials: rows block0 .. block0 + blocks of the launch's scratch, blocks = G_k
};

template <int Cap, class Item>
struct RegParams {
    shine_octree oct;
    shine_decoder dec;
    const float* points;
    double* partials;          // [blocks of this launch's items, kOut]
    int64_t n;                 // the shared segment of RegPose items: points[0 .. n)
    float sigma;
    double kappa2;
    Item item[Cap];            // blockIdx.y selects one
};
static_assert(sizeof(RegParams<kPosesPerLaunch, RegPose>) <= 32764, "kernel parameters are limited to 32 764 bytes");
static_assert(sizeof(RegParams<kItemsPerLaunch, RegItem>) <= 32764, "kernel parameters are limited to 32 764 bytes");
static_assert(sizeof(RegParams<kItemsPerLaunch + 64, RegItem>) > 32764, "the item cap is near the parameter limit");

__host__ __device__ inline int64_t register_blocks(int64_t n) {
    const int64_t blocks = (n + kRT - 1) / kRT;
    return blocks > kMaxBlocks ? kMaxBlocks : blocks;
}

// item k's points and partial rows.  RegPose items share points[0 .. n) and run g = register_blocks(n) blocks each, which
// the normal-equations kernel reads as gridDim.x (its launch is exactly that wide)
struct RegSegment {
    int64_t begin, n, block0, blocks;
};

template <int Cap>
__device__ inline RegSegment segment_of(const RegParams<Cap, RegPose>& P, unsigned k, unsigned g) {
    return {0, P.n, (int64_t)k * g, (int64_t)g};
}

template <int Cap>
__device__ inline RegSegment segment_of(const RegParams<Cap, RegItem>& P, unsigned k, unsigned) {
    const RegItem& it = P.item[k];
    return {it.begin, it.n, it.block0, it.blocks};
}

__device__ inline const RegPose& pose_of(const RegPose& p) { return p; }
__device__ inline const RegPose& pose_of(const RegItem& it) { return it.pose; }

struct RegSmem {
    float W1[kH * kF];         // [32][8]
    float W2[kH * kH];         // W2[j][n]
    float W2T[kH * kH];        // W2T[n][j]
    float b1[kH], b2[kH], w3[kH];
    float b3;
    double warp_sum[kRW][kOut];
};

template <int Cap, class Item>
__global__ void __launch_bounds__(kRT) register_normal_eq_kernel(const __grid_constant__ RegParams<Cap, Item> P) {
    __shared__ __align__(16) RegSmem sm;
    const RegSegment seg = segment_of(P, blockIdx.y, gridDim.x);
    if constexpr (std::is_same_v<Item, RegItem>)
        if (blockIdx.x >= seg.blocks) return;      // past this item's G_k blocks: the whole block writes nothing
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

    const RegPose& T = pose_of(P.item[blockIdx.y]);
    const float* points = P.points + 3 * seg.begin;
    double acc[kOut];
#pragma unroll
    for (int k = 0; k < kOut; ++k) acc[k] = 0.0;

    for (int64_t p = (int64_t)blockIdx.x * kRT + tid; p < seg.n; p += seg.blocks * kRT) {
        const float px = __ldg(points + 3 * p), py = __ldg(points + 3 * p + 1), pz = __ldg(points + 3 * p + 2);
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
        P.partials[(seg.block0 + blockIdx.x) * kOut + tid] = v;
    }
}

// out[item][k] = sum over the item's block partials of column k: warp k sums blocks lane, lane + 32, ... then a shuffle
// tree; one block per item of the launch.  An item of no blocks (n = 0) gets a row of zeros.
template <int Cap, class Item>
__global__ void __launch_bounds__(32 * kOut) register_fold_kernel(const __grid_constant__ RegParams<Cap, Item> P,
                                                                 double* __restrict__ out) {
    const int k = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const RegSegment seg = segment_of(P, blockIdx.x, (unsigned)register_blocks(P.n));
    const double* partials = P.partials + (int64_t)seg.block0 * kOut;
    double v = 0.0;
    for (int b = lane; b < seg.blocks; b += 32) v += partials[(int64_t)b * kOut + k];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(kFull, v, o);
    if (lane == 0) out[(int64_t)blockIdx.x * kOut + k] = v;
}

__global__ void register_zero_kernel(double* __restrict__ out, int64_t count) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < count) out[i] = 0.0;
}

inline bool is_finite(double v) { return v == v && v - v == 0.0; }

// checks shared by every entry (the scratch and the segments are checked by each); none touches the device
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

// the scratch of the scans entry: each item's G_k rows; -1 for a bad table
int64_t scans_scratch_bytes(const int64_t* seg_n, int64_t K) {
    if (!seg_n || K <= 0 || K > INT32_MAX) return -1;
    int64_t rows = 0;
    for (int64_t k = 0; k < K; ++k) {
        if (seg_n[k] < 0) return -1;
        rows += register_blocks(seg_n[k]);
    }
    return rows * kOut * (int64_t)sizeof(double);
}

inline void set_pose(RegPose& T, const double* pose) {
    for (int a = 0; a < 3; ++a) {
        for (int b = 0; b < 3; ++b) T.R[3 * a + b] = (float)pose[4 * a + b];
        T.t[a] = (float)pose[4 * a + 3];
    }
}

// the K items after the checks: chunks of Cap items, each one normal-equations launch (grid: the chunk's widest item x
// the chunk) and one fold launch (one block per item).  RegPose items share points[0 .. n); RegItem items have their own
// segments (seg_begin, seg_n).  Each chunk's partials follow the previous chunk's in the scratch.
template <int Cap, class Item>
int register_chunks(const shine_octree* oct, const shine_decoder* dec, const float* points, int64_t n,
                    const int64_t* seg_begin, const int64_t* seg_n, const double* poses, int64_t K, float sigma,
                    double kappa, double* out, void* scratch, cudaStream_t st) {
    int rc;
    RegParams<Cap, Item> P;
    P.oct = *oct; P.dec = *dec; P.points = points; P.n = n;
    P.sigma = sigma;
    P.kappa2 = kappa * kappa;
    P.partials = static_cast<double*>(scratch);
    for (int64_t k0 = 0; k0 < K; k0 += Cap) {
        const int kc = (int)(K - k0 < Cap ? K - k0 : Cap);
        int64_t rows = 0, widest = 0;
        for (int k = 0; k < kc; ++k) {
            int64_t blocks;
            if constexpr (std::is_same_v<Item, RegItem>) {
                RegItem& it = P.item[k];
                set_pose(it.pose, poses + 16 * (k0 + k));
                it.begin = seg_begin[k0 + k];
                it.n = seg_n[k0 + k];
                blocks = register_blocks(it.n);
                it.block0 = (int32_t)rows;
                it.blocks = (int32_t)blocks;
            } else {
                set_pose(P.item[k], poses + 16 * (k0 + k));
                blocks = register_blocks(n);
            }
            rows += blocks;
            widest = blocks > widest ? blocks : widest;
        }
        if (widest > 0)                       // a chunk of empty segments only has nothing to sum; its fold writes zeros
            register_normal_eq_kernel<Cap, Item><<<dim3((unsigned)widest, (unsigned)kc), kRT, 0, st>>>(P);
        register_fold_kernel<Cap, Item><<<(unsigned)kc, 32 * kOut, 0, st>>>(P, out + k0 * kOut);
        if ((rc = (int)cudaGetLastError())) return rc;
        P.partials += rows * kOut;
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
    if (K == 1)
        return register_chunks<1, RegPose>(oct, dec, points, n, nullptr, nullptr, poses, K, sigma, kappa, out, scratch, st);
    return register_chunks<kPosesPerLaunch, RegPose>(oct, dec, points, n, nullptr, nullptr, poses, K, sigma, kappa, out,
                                                     scratch, st);
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

int64_t shine_register_scans_scratch_bytes(const int64_t* seg_n, int64_t num_items) {
    return scans_scratch_bytes(seg_n, num_items);
}

int shine_register_normal_eq_scans(const shine_octree* oct, const shine_decoder* dec, const float* points,
                                   int64_t num_points, const int64_t* seg_begin, const int64_t* seg_n,
                                   const double* poses, int64_t num_items, float sigma, double kappa, double* out,
                                   void* scratch, int64_t scratch_bytes, void* stream) {
    int rc = check_register_args(oct, dec, points, num_points, poses, num_items, sigma, kappa, out);
    if (rc) return rc;
    if (!seg_begin || !seg_n) return SHINE_ERR_INVALID_ARG;
    for (int64_t k = 0; k < num_items; ++k)
        if (seg_n[k] < 0 || seg_begin[k] < 0 || seg_begin[k] > num_points - seg_n[k]) return SHINE_ERR_INVALID_ARG;
    const int64_t need = scans_scratch_bytes(seg_n, num_items);
    if (!scratch || scratch_bytes < need || ((uintptr_t)scratch & 7)) return SHINE_ERR_INVALID_ARG;
    if ((rc = check_same_device(oct, points))) return rc;
    DeviceGuard guard(oct->lv[0].features);
    return register_chunks<kItemsPerLaunch, RegItem>(oct, dec, points, num_points, seg_begin, seg_n, poses, num_items,
                                                     sigma, kappa, out, scratch, (cudaStream_t)stream);
}

}  // extern "C"
