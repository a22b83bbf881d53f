// shine_rgbd.cu — one depth image to camera points on the GPU.
// Reference: dataset/rgbd_to_kitti_format.py (open3d's RGBDImage.create_from_color_and_depth with
// convert_rgb_to_intensity=False and PointCloud.create_from_rgbd_image), which writes the frames that
// dataset/lidar_dataset.py then reads as point clouds.
//
//   shine_rgbd_backproject   per pixel: d = (float)raw / (float)depth_scale, 0 when d >= depth_trunc (fp64 compare);
//                            a pixel with d > 0 becomes camera_pose · (x, y, z, 1) in fp64, x = ((j - cx) * z) / fx,
//                            y = ((i - cy) * z) / fy, z = d; any other pixel becomes (NaN, NaN, NaN)
//
// The output keeps every pixel in row-major order, so the scan pipeline (csrc/shine_scan.cu) takes it as 24-byte fp64
// records: its filter drops the NaN records and the voxel average sees the valid points in the converter's order.
#include "shine_device.cuh"

namespace {

constexpr int kRgbdThreads = 256;

struct BackprojectParams {
    const uint16_t* depth;
    const uint8_t* rgb_in;
    double* xyz;
    uint8_t* rgb_out;
    int64_t n;                 // H * W
    int32_t W, pitch;
    double fx, fy, cx, cy, trunc;
    float scale;
    double m[12];              // rows 0..2 of the row-major 4x4 camera pose
};

// Every operation is rounded on its own (no contraction), in the order of the contract above: the products of a row
// are summed in k order, ((m0 x + m1 y) + m2 z) + m3 · 1.
__global__ void __launch_bounds__(kRgbdThreads) rgbd_backproject_kernel(const BackprojectParams a) {
    for (int64_t p = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; p < a.n; p += (int64_t)gridDim.x * blockDim.x) {
        const int i = (int)(p / a.W), j = (int)(p - (int64_t)i * a.W);
        const int64_t src = (int64_t)i * a.pitch + j;
        const float d = __fdiv_rn((float)a.depth[src], a.scale);
        double q[3];
        if (d > 0.0f && !((double)d >= a.trunc)) {
            const double z = (double)d;
            const double x = __ddiv_rn(__dmul_rn(__dsub_rn((double)j, a.cx), z), a.fx);
            const double y = __ddiv_rn(__dmul_rn(__dsub_rn((double)i, a.cy), z), a.fy);
#pragma unroll
            for (int r = 0; r < 3; ++r) {
                const double* m = a.m + 4 * r;
                q[r] = __dadd_rn(__dadd_rn(__dadd_rn(__dmul_rn(m[0], x), __dmul_rn(m[1], y)), __dmul_rn(m[2], z)),
                                 __dmul_rn(m[3], 1.0));
            }
        } else {
            q[0] = q[1] = q[2] = __longlong_as_double(0x7ff8000000000000ll);
        }
        a.xyz[3 * p] = q[0];
        a.xyz[3 * p + 1] = q[1];
        a.xyz[3 * p + 2] = q[2];
        if (a.rgb_out) {
            a.rgb_out[3 * p] = a.rgb_in[3 * src];
            a.rgb_out[3 * p + 1] = a.rgb_in[3 * src + 1];
            a.rgb_out[3 * p + 2] = a.rgb_in[3 * src + 2];
        }
    }
}

}  // namespace

extern "C" {

int shine_rgbd_backproject(const uint16_t* depth, int32_t height, int32_t width, int32_t row_pitch, double fx,
                           double fy, double cx, double cy, double depth_scale, double depth_trunc,
                           const double* camera_pose, double* xyz_out, uint8_t* rgb_out, const uint8_t* rgb_in,
                           void* stream) {
    if (!depth || !camera_pose || !xyz_out || (!rgb_out) != (!rgb_in)) return SHINE_ERR_INVALID_ARG;
    if (height <= 0 || width <= 0 || row_pitch < width) return SHINE_ERR_INVALID_ARG;
    if ((uintptr_t)depth % 2 || (uintptr_t)xyz_out % 8) return SHINE_ERR_INVALID_ARG;
    const float scale = (float)depth_scale;
    if (!(depth_scale > 0.0) || !(scale > 0.0f) || !isfinite(scale)) return SHINE_ERR_INVALID_ARG;
    // the scan pipeline counts records in int32 (CUB); the input is addressed up to height * row_pitch
    if ((int64_t)height * row_pitch > 0x7fffffffLL) return SHINE_ERR_UNSUPPORTED;
    BackprojectParams a;
    a.depth = depth; a.rgb_in = rgb_in; a.xyz = xyz_out; a.rgb_out = rgb_out;
    a.n = (int64_t)height * width; a.W = width; a.pitch = row_pitch;
    a.fx = fx; a.fy = fy; a.cx = cx; a.cy = cy; a.trunc = depth_trunc; a.scale = scale;
    for (int k = 0; k < 12; ++k) a.m[k] = camera_pose[k];
    DeviceGuard guard(xyz_out);
    int64_t blocks = (a.n + kRgbdThreads - 1) / kRgbdThreads;
    const int64_t cap = (int64_t)sm_count() * 8;
    if (blocks > cap) blocks = cap;
    rgbd_backproject_kernel<<<(unsigned)blocks, kRgbdThreads, 0, (cudaStream_t)stream>>>(a);
    return (int)cudaGetLastError();
}

}  // extern "C"
