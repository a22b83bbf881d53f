// shine_raycast.cu — rays cast through the SDF map: where a ray from the sensor origin first meets the zero level set
// (evaluate.py eval_scans: the range errors of held-out scans).
//
// One thread per ray.  For ray i from the origin o towards the point p_i (fp32, every operation rounded on its own):
//     v = p_i - o,  r = sqrt((vx vx + vy vy) + vz vz),  d = v / r
//     K = min(floor((min(r + beyond, t_max) - t_min) / h), 2^24 - 1)          (no sample when K < 0, r = 0 or not finite)
//     t_k = t_min + k h,  x_k = o + t_k d                                       (k = 0 .. K, k as an exact fp32)
//     m_k = x_k's voxel exists at lv[mask_level],  s_k = -Decoder.sdf(f(x_k))  (f: fp32 FMA blend over every level, the
//                                                                               decoder as fp32 FMA chains, weights in
//                                                                               shared memory, as in shine_register.cu)
// The hit is the first k >= 1 with m_{k-1}, m_k, s_{k-1} > 0 and s_k <= 0.  Bisection of the bracket, refine_iters steps
// at most: t_mid = 0.5 (t_a + t_b), stopping when t_mid is not strictly inside or x(t_mid) is masked; then the zero of
// the linear interpolation, t_a + (t_b - t_a) (s_a / (s_a - s_b)).
//
// Empty-space skipping.  A sample whose node at the coarsest featured level lv[L-1] is absent is masked, and so is every
// later sample in the same cell of that level.  Each axis's cell index is a non-decreasing or non-increasing function of
// k (t_k, t_k d, o + t_k d and the quantisation are all monotone roundings), so if sample j lies in sample k's cell, so
// does every sample between them.  The march estimates the last sample j before the cell's exit, halves j - k until
// sample j's cell is k's (checked on the quantised indices, not on fp32 geometry), and resumes at j + 1.  It therefore
// visits the same unmasked samples, and returns the same bits, as a march without skipping.
//
// shine_render (render.py) runs the same march, `march` below, for the rays of one camera view, one thread per pixel,
// with K = floor((t_max - t_min) / h) for every ray, and takes each hit's normal from sdf_grad_at (shine_device.cuh).
#include "shine_device.cuh"

namespace {

constexpr int kCT = 128;                   // threads (rays) per block
constexpr float kMaxK = 16777215.f;        // 2^24 - 1: larger lattice indices are not exact in fp32

struct CastParams {
    shine_octree oct;
    shine_decoder dec;
    const float* points;
    float* out_t;
    uint8_t* out_status;
    int64_t n;
    float o[3];
    float h, t_min, beyond, t_max;
    int32_t refine_iters, mask_level;
};

struct CastSmem {
    float W1[kH * kF];     // [32][8]
    float W2[kH * kH];     // W2[j][n]
    float b1[kH], b2[kH], w3[kH];
    float b3;
};

__device__ __forceinline__ void cell_of(const float (&x)[3], float res, uint32_t (&c)[3]) {
#pragma unroll
    for (int a = 0; a < 3; ++a) c[a] = quantize1(x[a], res);
}

struct Ray {
    float o[3], d[3];
    __device__ __forceinline__ void at(float t, float (&x)[3]) const {
#pragma unroll
        for (int a = 0; a < 3; ++a) x[a] = __fadd_rn(o[a], __fmul_rn(t, d[a]));
    }
};

template <class Params>
__device__ __forceinline__ float lattice_t(const Params& P, int k) {
    return __fadd_rn(P.t_min, __fmul_rn((float)k, P.h));
}

// m and s at x; s is only formed when m holds
template <class Params, class Smem>
__device__ bool field_at(const Params& P, const Smem& sm, const float (&x)[3], float& s) {
    const int L = P.oct.num_levels;
    {
        const shine_level& lv = P.oct.lv[P.mask_level];
        if (probe_slot(reinterpret_cast<const HashSlot*>(lv.hash_slots), lv.hash_capacity - 1,
                       morton_of(x[0], x[1], x[2], lv.level)) < 0)
            return false;
    }
    const bool poly = P.oct.poly_interp != 0;
    float f[8];
#pragma unroll
    for (int k = 0; k < 8; ++k) f[k] = 0.f;
#pragma unroll 1
    for (int i = 0; i < L; ++i) {
        const shine_level& lv = P.oct.lv[i];
        const HashSlot* slots = reinterpret_cast<const HashSlot*>(lv.hash_slots);
        const int sl = probe_slot(slots, lv.hash_capacity - 1, morton_of(x[0], x[1], x[2], lv.level));
        if (sl < 0) continue;
        const int4 ia = ldg_i4(slots[sl].ids0), ib = ldg_i4(slots[sl].ids1);
        const int ids[8] = {ia.x, ib.x, ia.y, ib.y, ia.z, ib.z, ia.w, ib.w};
        Blend b; b.init(x[0], x[1], x[2], lv.level, poly);
#pragma unroll
        for (int c = 0; c < 8; ++c) {
            float row[8];
            ldg_row8(lv.features + (int64_t)ids[c] * kF, row);
            const float w = b.w(c);
#pragma unroll
            for (int k = 0; k < 8; ++k) f[k] = fmaf(w, row[k], f[k]);
        }
    }
    // Decoder.sdf (model/decoder.py:49-63), fp32 FMA chains
    float h1[32];
#pragma unroll
    for (int n = 0; n < 32; ++n) {
        const float4 wa = *reinterpret_cast<const float4*>(sm.W1 + n * 8), wb = *reinterpret_cast<const float4*>(sm.W1 + n * 8 + 4);
        float a = sm.b1[n];
        a = fmaf(wa.x, f[0], a); a = fmaf(wa.y, f[1], a); a = fmaf(wa.z, f[2], a); a = fmaf(wa.w, f[3], a);
        a = fmaf(wb.x, f[4], a); a = fmaf(wb.y, f[5], a); a = fmaf(wb.z, f[6], a); a = fmaf(wb.w, f[7], a);
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
        pr = fmaf(fmaxf(a, 0.f), sm.w3[j], pr);
    }
    s = -pr;
    return true;
}

// The march of one ray over lattice samples k = 0 .. K (the header's shine_raycast definition, after the ray and K):
// true and the refined hit distance in t_hit, or false (t_hit untouched).  Params: oct, h, t_min, refine_iters and
// mask_level as in CastParams.
template <class Params, class Smem>
__device__ __forceinline__ bool march(const Params& P, const Smem& sm, const Ray& ray, int K, float& t_hit) {
    const shine_level& top = P.oct.lv[P.oct.num_levels - 1];
    const HashSlot* top_slots = reinterpret_cast<const HashSlot*>(top.hash_slots);
    const float top_res = (float)(1u << top.level);
    bool prev = false;          // m_{k-1} && s_{k-1} > 0
    float prev_s = 0.f;
    int k = 0;
    while (k <= K) {
        const float t = lattice_t(P, k);
        float x[3];
        ray.at(t, x);
        if (probe_slot(top_slots, top.hash_capacity - 1, morton_of(x[0], x[1], x[2], top.level)) < 0) {
            // absent at the coarsest level: skip to the sample after the last one in this cell
            uint32_t c0[3];
            cell_of(x, top_res, c0);
            float t_exit = __int_as_float(0x7f800000);
#pragma unroll
            for (int a = 0; a < 3; ++a) {
                // the cell's faces are exact in fp32: -1 + 2 c / res; the boundary cells extend without end (clamp)
                if (ray.d[a] > 0.f && c0[a] + 1u < (uint32_t)top_res)
                    t_exit = fminf(t_exit, (-1.f + 2.f * (float)(c0[a] + 1u) / top_res - ray.o[a]) / ray.d[a]);
                else if (ray.d[a] < 0.f && c0[a] > 0u)
                    t_exit = fminf(t_exit, (-1.f + 2.f * (float)c0[a] / top_res - ray.o[a]) / ray.d[a]);
            }
            const float je = floorf((t_exit - P.t_min) / P.h);
            int j = je >= (float)K ? K : (je <= (float)k ? k : (int)je);
            while (j > k) {
                float xj[3];
                uint32_t cj[3];
                ray.at(lattice_t(P, j), xj);
                cell_of(xj, top_res, cj);
                if (cj[0] == c0[0] && cj[1] == c0[1] && cj[2] == c0[2]) break;
                j = k + (j - k) / 2;
            }
            prev = false;
            k = j + 1;
            continue;
        }
        float s;
        const bool m = field_at(P, sm, x, s);
        if (m && prev && s <= 0.f) {
            // bracket [t_{k-1}, t_k]: bisection while the midpoint is inside and unmasked, then linear interpolation
            float ta = lattice_t(P, k - 1), tb = t, sa = prev_s, sb = s;
            for (int it = 0; it < P.refine_iters; ++it) {
                const float tm = __fmul_rn(0.5f, __fadd_rn(ta, tb));
                if (!(tm > ta && tm < tb)) break;
                float xm[3], sm_;
                ray.at(tm, xm);
                if (!field_at(P, sm, xm, sm_)) break;
                if (sm_ > 0.f) { ta = tm; sa = sm_; } else { tb = tm; sb = sm_; }
            }
            t_hit = __fadd_rn(ta, __fmul_rn(__fsub_rn(tb, ta), __fdiv_rn(sa, __fsub_rn(sa, sb))));
            return true;
        }
        prev = m && s > 0.f;
        prev_s = s;
        ++k;
    }
    return false;
}

// the decoder's weights into shared memory
template <int kThreads, class Smem>
__device__ __forceinline__ void load_decoder(const shine_decoder& dec, Smem& sm) {
    const int tid = threadIdx.x;
    for (int i = tid; i < kH * kF; i += kThreads) sm.W1[i] = dec.w1[i];
    for (int i = tid; i < kH * kH; i += kThreads) sm.W2[i] = dec.w2[i];
    if (tid < kH) {
        sm.b1[tid] = dec.b1 ? dec.b1[tid] : 0.f;
        sm.b2[tid] = dec.b2 ? dec.b2[tid] : 0.f;
        sm.w3[tid] = dec.w3[tid];
    }
    if (tid == 0) sm.b3 = dec.b3 ? dec.b3[0] : 0.f;
}

__global__ void __launch_bounds__(kCT) raycast_kernel(const __grid_constant__ CastParams P) {
    __shared__ __align__(16) CastSmem sm;
    const int tid = threadIdx.x;
    load_decoder<kCT>(P.dec, sm);
    __syncthreads();

    const int64_t i = (int64_t)blockIdx.x * kCT + tid;
    if (i >= P.n) return;
    Ray ray;
    float v[3];
#pragma unroll
    for (int a = 0; a < 3; ++a) {
        ray.o[a] = P.o[a];
        v[a] = __fsub_rn(__ldg(P.points + 3 * i + a), P.o[a]);
    }
    const float r = __fsqrt_rn(__fadd_rn(__fadd_rn(__fmul_rn(v[0], v[0]), __fmul_rn(v[1], v[1])), __fmul_rn(v[2], v[2])));
#pragma unroll
    for (int a = 0; a < 3; ++a) ray.d[a] = __fdiv_rn(v[a], r);
    const float kf = floorf(__fdiv_rn(__fsub_rn(fminf(__fadd_rn(r, P.beyond), P.t_max), P.t_min), P.h));
    float out_t = __int_as_float(0x7fc00000);
    uint8_t status = 0;
    if (r > 0.f && r <= 3.402823466e38f && kf >= 0.f && march(P, sm, ray, (int)fminf(kf, kMaxK), out_t)) status = 1;
    P.out_t[i] = out_t;
    P.out_status[i] = status;
}

// ---- shine_render: one camera view, one thread per pixel ---------------------------------------------------------------

struct RenderParams {
    shine_octree oct;
    shine_decoder dec;
    float* out_range;
    float* out_depth;
    float* out_normal;
    uint8_t* out_status;
    int32_t width, height, model, K;
    float c[4];                // pinhole: fx fy cx cy; range image: el0 del az0 daz (radians)
    float R[9], o[3];          // camera-to-map rotation (row-major) and origin
    float h, t_min;
    int32_t refine_iters, mask_level;
};

struct RenderSmem {
    float W1[kH * kF];
    float W2[kH * kH];
    float W2T[kH * kH];
    float b1[kH], b2[kH], w3[kH];
    float b3;
};

__global__ void __launch_bounds__(kCT) render_kernel(const __grid_constant__ RenderParams P) {
    __shared__ __align__(16) RenderSmem sm;
    const int tid = threadIdx.x;
    load_decoder<kCT>(P.dec, sm);
    for (int i = tid; i < kH * kH; i += kCT) sm.W2T[(i % kH) * kH + i / kH] = P.dec.w2[i];
    __syncthreads();

    const int64_t i = (int64_t)blockIdx.x * kCT + tid;
    if (i >= (int64_t)P.width * P.height) return;
    const int u = (int)(i % P.width), v = (int)(i / P.width);
    // the camera-frame unit direction c and its z (depth = t cz)
    float c[3], cz;
    if (P.model == SHINE_CAMERA_PINHOLE) {
        const float a = __fdiv_rn(__fsub_rn((float)u, P.c[2]), P.c[0]), b = __fdiv_rn(__fsub_rn((float)v, P.c[3]), P.c[1]);
        const float n = __fsqrt_rn(__fadd_rn(__fadd_rn(__fmul_rn(a, a), __fmul_rn(b, b)), 1.f));
        c[0] = __fdiv_rn(a, n); c[1] = __fdiv_rn(b, n); c[2] = __fdiv_rn(1.f, n);
        cz = c[2];
    } else {
        const double el = (double)__fsub_rn(P.c[0], __fmul_rn((float)v, P.c[1]));
        const double az = (double)__fsub_rn(P.c[2], __fmul_rn((float)u, P.c[3]));
        const float ce = (float)cos(el), se = (float)sin(el), ca = (float)cos(az), sa = (float)sin(az);
        c[0] = __fmul_rn(ce, ca); c[1] = __fmul_rn(ce, sa); c[2] = se;
        cz = 1.f;
    }
    Ray ray;
#pragma unroll
    for (int a = 0; a < 3; ++a) {
        ray.o[a] = P.o[a];
        ray.d[a] = __fadd_rn(__fadd_rn(__fmul_rn(P.R[3 * a], c[0]), __fmul_rn(P.R[3 * a + 1], c[1])),
                             __fmul_rn(P.R[3 * a + 2], c[2]));
    }
    const float nan = __int_as_float(0x7fc00000);
    float t = nan, nrm[3] = {nan, nan, nan};
    const bool hit = march(P, sm, ray, P.K, t);
    if (hit) {
        if (P.out_normal) {
            float x[3], pr, g[3];
            ray.at(t, x);
            sdf_grad_at<false>(P.oct, sm, x[0], x[1], x[2], pr, g);
            const float len = __fsqrt_rn(__fadd_rn(__fadd_rn(__fmul_rn(g[0], g[0]), __fmul_rn(g[1], g[1])), __fmul_rn(g[2], g[2])));
#pragma unroll
            for (int a = 0; a < 3; ++a) nrm[a] = -__fdiv_rn(g[a], len);
        }
    }
    if (P.out_range) P.out_range[i] = t;
    if (P.out_depth) P.out_depth[i] = __fmul_rn(t, cz);
    if (P.out_normal) {
#pragma unroll
        for (int a = 0; a < 3; ++a) P.out_normal[3 * i + a] = nrm[a];
    }
    if (P.out_status) P.out_status[i] = hit ? 1 : 0;
}

inline bool finite_f(float v) { return v == v && v - v == 0.f; }

// the checks shine_raycast and shine_render share: pointers, octree, decoder, h, t_min, t_max, refine_iters, mask_level
int check_march_args(const shine_octree* oct, const shine_decoder* dec, float h, float t_min, float t_max,
                     int32_t refine_iters, int32_t mask_level) {
    if (!oct || !dec) return SHINE_ERR_INVALID_ARG;
    int rc = check_octree(oct, false);
    if (rc) return rc;
    if ((rc = check_decoder(dec, oct))) return rc;
    if (!finite_f(h) || !(h > 0.f) || !finite_f(t_min) || !(t_max > t_min)) return SHINE_ERR_INVALID_ARG;
    if (refine_iters < 0 || refine_iters > SHINE_RAYCAST_MAX_REFINE) return SHINE_ERR_INVALID_ARG;
    if (mask_level < 0 || mask_level >= oct->num_levels) return SHINE_ERR_INVALID_ARG;
    return SHINE_OK;
}

}  // namespace

extern "C" {

int shine_raycast(const shine_octree* oct, const shine_decoder* dec, const float* origin, const float* points, int64_t n,
                  float h, float t_min, float beyond, float t_max, int32_t refine_iters, int32_t mask_level,
                  float* out_t, uint8_t* out_status, void* stream) {
    if (!oct || !dec || !origin || n < 0 || (n > 0 && (!points || !out_t || !out_status))) return SHINE_ERR_INVALID_ARG;
    int rc = check_march_args(oct, dec, h, t_min, t_max, refine_iters, mask_level);
    if (rc) return rc;
    if (!(beyond >= 0.f) || !finite_f(beyond)) return SHINE_ERR_INVALID_ARG;
    for (int a = 0; a < 3; ++a)
        if (!finite_f(origin[a])) return SHINE_ERR_INVALID_ARG;
    if (n == 0) return SHINE_OK;
    if ((rc = check_same_device(oct, points))) return rc;
    DeviceGuard guard(oct->lv[0].features);
    CastParams P;
    P.oct = *oct; P.dec = *dec; P.points = points; P.out_t = out_t; P.out_status = out_status; P.n = n;
    for (int a = 0; a < 3; ++a) P.o[a] = origin[a];
    P.h = h; P.t_min = t_min; P.beyond = beyond; P.t_max = t_max;
    P.refine_iters = refine_iters; P.mask_level = mask_level;
    const int64_t blocks = (n + kCT - 1) / kCT;
    if (blocks > INT32_MAX) return SHINE_ERR_UNSUPPORTED;
    raycast_kernel<<<(unsigned)blocks, kCT, 0, (cudaStream_t)stream>>>(P);
    return (int)cudaGetLastError();
}

int shine_render(const shine_octree* oct, const shine_decoder* dec, const shine_camera* cam, const float* pose, float h,
                 float t_min, float t_max, int32_t refine_iters, int32_t mask_level, float* out_range, float* out_depth,
                 float* out_normal, uint8_t* out_status, void* stream) {
    if (!cam || !pose) return SHINE_ERR_INVALID_ARG;
    int rc = check_march_args(oct, dec, h, t_min, t_max, refine_iters, mask_level);
    if (rc) return rc;
    if (!finite_f(t_max)) return SHINE_ERR_INVALID_ARG;
    if (cam->width <= 0 || cam->height <= 0 || (int64_t)cam->width * cam->height > ((int64_t)1 << 31))
        return SHINE_ERR_INVALID_ARG;
    for (int i = 0; i < 12; ++i)
        if (!finite_f(pose[i])) return SHINE_ERR_INVALID_ARG;
    RenderParams P;
    if (cam->model == SHINE_CAMERA_PINHOLE) {
        if (!finite_f(cam->fx) || !finite_f(cam->fy) || !finite_f(cam->cx) || !finite_f(cam->cy) || !(cam->fx > 0.f) ||
            !(cam->fy > 0.f))
            return SHINE_ERR_INVALID_ARG;
        P.c[0] = cam->fx; P.c[1] = cam->fy; P.c[2] = cam->cx; P.c[3] = cam->cy;
    } else if (cam->model == SHINE_CAMERA_RANGE_IMAGE) {
        if (!finite_f(cam->fov_up) || !finite_f(cam->fov_down) || !(cam->fov_up > cam->fov_down))
            return SHINE_ERR_INVALID_ARG;
        const double deg = 3.14159265358979323846 / 180.0;
        P.c[0] = (float)((double)cam->fov_up * deg);
        P.c[1] = cam->height > 1 ? (float)(((double)cam->fov_up - (double)cam->fov_down) * deg / (cam->height - 1)) : 0.f;
        P.c[2] = (float)3.14159265358979323846;
        P.c[3] = (float)(2.0 * 3.14159265358979323846 / cam->width);
    } else {
        return SHINE_ERR_INVALID_ARG;
    }
    const float* outs[3] = {out_range, out_depth, out_normal};
    for (const float* p : outs)
        if ((rc = check_same_device(oct, p))) return rc;
    if ((rc = check_same_device(oct, out_status))) return rc;
    if (!out_range && !out_depth && !out_normal && !out_status) return SHINE_OK;
    DeviceGuard guard(oct->lv[0].features);
    P.oct = *oct; P.dec = *dec;
    P.out_range = out_range; P.out_depth = out_depth; P.out_normal = out_normal; P.out_status = out_status;
    P.width = cam->width; P.height = cam->height; P.model = cam->model;
    P.K = (int)fminf(floorf((t_max - t_min) / h), kMaxK);
    for (int a = 0; a < 3; ++a) {
        for (int b = 0; b < 3; ++b) P.R[3 * a + b] = pose[4 * a + b];
        P.o[a] = pose[4 * a + 3];
    }
    P.h = h; P.t_min = t_min;
    P.refine_iters = refine_iters; P.mask_level = mask_level;
    const int64_t blocks = ((int64_t)cam->width * cam->height + kCT - 1) / kCT;
    render_kernel<<<(unsigned)blocks, kCT, 0, (cudaStream_t)stream>>>(P);
    return (int)cudaGetLastError();
}

}  // extern "C"
