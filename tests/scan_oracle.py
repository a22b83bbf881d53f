"""numpy restatement of one frame of the reference's `LiDARDataset.process_frame` (dataset/lidar_dataset.py:115-218), the
yardstick of csrc/shine_scan.cu.  open3d is not a dependency, so its crop, voxel down-sampling, transform and scale are
restated from their published semantics (open3d geometry/PointCloud.cpp, AxisAlignedBoundingBox), like the kaolin
pieces of oracle/kaolin_shim.

Where the order of operations may differ from open3d's: the transform's row sums are taken as ((m0*x + m1*y) + m2*z) + m3
here and in the kernel; Eigen's 4x4 · 4-vector product may associate differently, which can change a coordinate by one
fp64 ulp and reaches the fp32 points only at a rounding tie.  The voxel order is ascending key here and in the kernel;
open3d's is the iteration order of an unordered_map, which is unspecified."""
from __future__ import annotations

import numpy as np

AXIS_BITS = 21


def preprocess(points: np.ndarray, min_z: float, min_range: float) -> np.ndarray:
    """preprocess_kitti (:334-339)."""
    z = points[:, 2]
    points = points[z > min_z]
    return points[np.linalg.norm(points, axis=1) >= min_range]


def crop(points: np.ndarray, pc_radius: float, min_z: float, max_z: float) -> np.ndarray:
    """AxisAlignedBoundingBox([-r, -r, min_z], [r, r, max_z]) crop (:139-142), bounds inclusive."""
    lo = np.array([-pc_radius, -pc_radius, min_z])
    hi = np.array([pc_radius, pc_radius, max_z])
    return points[np.all((points >= lo) & (points <= hi), axis=1)]


def voxel_keys(points: np.ndarray, voxel: float) -> np.ndarray:
    vmin = points.min(0) - voxel * 0.5
    idx = np.floor((points - vmin) / voxel).astype(np.int64)
    return (idx[:, 0] << (2 * AXIS_BITS)) | (idx[:, 1] << AXIS_BITS) | idx[:, 2]


def voxel_down(points: np.ndarray, voxel: float) -> np.ndarray:
    """VoxelDownSample (:158): per voxel the fp64 sum of its points in input order / count, voxels in ascending key."""
    if points.shape[0] == 0:
        return np.zeros((0, 3))
    keys = voxel_keys(points, voxel)
    order = np.argsort(keys, kind="stable")
    k = keys[order]
    heads = np.flatnonzero(np.r_[True, k[1:] != k[:-1]])
    ends = np.r_[heads[1:], k.shape[0]]
    out = np.empty((heads.shape[0], 3))
    for v, (b, e) in enumerate(zip(heads, ends)):
        s = np.zeros(3)
        for j in order[b:e]:
            s = s + points[j]
        out[v] = s / float(e - b)
    return out


def transform_scale(points: np.ndarray, pose: np.ndarray, scale: float) -> np.ndarray:
    """TransformPoints (:179), ScalePoints about the origin (:189), then torch.tensor(..., dtype=float32) (:191)."""
    m = pose
    q = [((m[r, 0] * points[:, 0] + m[r, 1] * points[:, 1]) + m[r, 2] * points[:, 2]) + m[r, 3] for r in range(4)]
    p = np.stack(q[:3], 1) / q[3][:, None]
    return ((p - 0.0) * scale + 0.0).astype(np.float32)


def frame_points(points64: np.ndarray, pose: np.ndarray, cfg, voxels: bool = False):
    """Stages 1-3 -> fp32 scaled points (and the fp64 voxel averages)."""
    p = crop(preprocess(points64, cfg.min_z, cfg.min_range), cfg.pc_radius, cfg.min_z, cfg.max_z)
    v = voxel_down(p, cfg.vox_down_m)
    pts = transform_scale(v, pose, cfg.scale)
    return (pts, v) if voxels else pts


def sample(points: np.ndarray, origin: np.ndarray, u_surface: np.ndarray, u_free: np.ndarray, cfg):
    """dataSampler.sample (utils/data_sampler.py:18-139) in fp32, one numpy operation per torch operation.
    u_surface [R*ns] and u_free [R*nf] are the reference's torch.rand draws (sample-major).  -> coord, label, weight."""
    f32 = np.float32
    ns, nf = cfg.surface_sample_n, cfg.free_sample_n
    R = points.shape[0]
    rng, end = f32(cfg.surface_sample_range_m * cfg.scale), f32(cfg.free_sample_end_dist_m * cfg.scale)
    begin = f32(cfg.free_sample_begin_ratio)
    shift = (points.astype(f32) - origin.astype(f32)).astype(f32)
    d = np.sqrt((shift[:, 0] * shift[:, 0] + shift[:, 1] * shift[:, 1]) + shift[:, 2] * shift[:, 2]).reshape(R, 1)
    us = u_surface.astype(f32).reshape(ns, R, 1)
    uf = u_free.astype(f32).reshape(nf, R, 1)
    surf_disp = ((us - f32(0.5)) * f32(2.0)) * rng
    surf_ratio = surf_disp / d + f32(1.0)
    free_max = (f32(1.0) / d) * end + f32(1.0)
    free_ratio = uf * (free_max - begin) + begin
    free_disp = (free_ratio - f32(1.0)) * d
    ratio = np.concatenate((surf_ratio, free_ratio), 0)            # [ns+nf, R, 1]
    disp = np.concatenate((surf_disp, free_disp), 0)
    coord = shift[None] * ratio + origin.astype(f32)
    weight = np.concatenate((np.ones((ns, R), f32), -np.ones((nf, R), f32)), 0)
    return (coord.transpose(1, 0, 2).reshape(-1, 3), disp[..., 0].T.reshape(-1), weight.T.reshape(-1))
