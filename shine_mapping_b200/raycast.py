"""Judge a map by the scans it was not built from: cast each held-out scan's rays through the SDF on the GPU and compare
where they meet the zero level set with the measured ranges.

* `cast_rays`          — `shine_raycast` (csrc/shine_raycast.cu) over one scan, in calls of at most MAX_RAYS_PER_CALL
                         rays -> the hit range in metres and a hit flag per ray.
* `scan_frames`        — frames of a `scans.LiDARDataset` / `rgbd.RGBDDataset`, read and preprocessed as mapping does
                         (filter, crop, voxel down-sampling, transform, scale: `ScanProcessor.points`), in the map frame.
* `eval_scans`         — per-frame and total metrics over all rays (`ray_metrics`).
* `held_out_frames`, `parse_frames` — the frame selection of `python -m shine_mapping_b200.evaluate scans`.

The field and mask along a ray are those the mesher meshes (`shine_mesh_grid`): -Decoder.sdf, positive in free space,
and the voxel mask at the mesher's mask level.  DESIGN.md §13 states the definition and how it is tested.
"""
from __future__ import annotations

import ctypes as C
import math
import os

import numpy as np
import torch

from . import _abi

MAX_RAYS_PER_CALL = 1 << 22     # rays per shine_raycast call (a few million-point scans at most split once or twice)
REFINE_ITERS = 8                # bisection steps: a hit is bracketed to step / 256 before the final interpolation
METRIC_COLUMNS = ["rays", "hits", "hit_ratio", "mean_abs_err_m", "median_abs_err_m", "rmse_m", "bias_m",
                  "within_threshold"]


def mask_level(config, octree) -> int:
    """The mesher's mask level (utils/mesher.py:47, `Mesher._mask_level`), bottom-up from the leaf."""
    return min(octree.featured_level_num, config.mc_vis_level) - 1


def cast_rays(config, octree, decoder, origin_scaled, points_scaled: torch.Tensor, step_m: float, beyond_m: float,
              refine_iters: int = REFINE_ITERS, t_min_m: float = 0.0, t_max_m: float = math.inf):
    """Rays from origin_scaled (3 values, scaled map coordinates) towards points_scaled (CUDA fp32 [n,3], scaled, map
    frame), sampled every step_m from t_min_m to min(|p - o| + beyond_m, t_max_m).
    -> (range_m fp64 [n]: the hit distance in metres, NaN on a miss; hit bool [n])."""
    pts = points_scaled.reshape(-1, 3)
    _abi.require_cuda(pts, "cast_rays points")
    pts = pts.to(torch.float32).contiguous()
    n = pts.shape[0]
    dev = pts.device
    scale = float(config.scale)
    out_t = torch.empty(n, dtype=torch.float32, device=dev)
    status = torch.empty(n, dtype=torch.uint8, device=dev)
    o = (C.c_float * 3)(*np.asarray(origin_scaled, dtype=np.float32).reshape(3).tolist())
    args = [float(np.float32(v * scale)) for v in (step_m, t_min_m, beyond_m)] + [float(t_max_m) * scale]
    od, dd = octree._descriptor(None, None), decoder.c_descriptor(None)
    lib, st = _abi.lib(), _abi.stream_ptr(dev)
    level = mask_level(config, octree)
    for s in range(0, max(n, 1), MAX_RAYS_PER_CALL):
        m = min(MAX_RAYS_PER_CALL, n - s)
        _abi.check(lib.shine_raycast(C.byref(od), C.byref(dd), o, _abi.ptr(pts[s:]) if m else None, m, args[0], args[1],
                                     args[2], args[3], int(refine_iters), level, _abi.ptr(out_t[s:]) if m else None,
                                     _abi.ptr(status[s:]) if m else None, st), "shine_raycast")
    return out_t.double() / scale, status.bool()


# ---- metrics -----------------------------------------------------------------------------------------------------------

def ray_metrics(range_m, hit, measured_m, threshold_m: float) -> dict:
    """Metrics of one set of rays from their hit ranges, hit flags and measured ranges (metres): the ray and hit counts,
    the hit ratio, mean, median and RMSE of |range - measured| over the hits, the mean signed error (bias; positive: the
    map's surface lies behind the measurement) and the fraction of ALL rays that hit within threshold_m of the measured
    range (a miss counts as outside).  Statistics of an empty set are NaN."""
    r = np.asarray(torch.as_tensor(range_m).detach().cpu(), dtype=np.float64).reshape(-1)
    h = np.asarray(torch.as_tensor(hit).detach().cpu(), dtype=bool).reshape(-1)
    meas = np.asarray(torch.as_tensor(measured_m).detach().cpu(), dtype=np.float64).reshape(-1)
    if not (r.shape == h.shape == meas.shape):
        raise ValueError(f"ray_metrics: {r.shape[0]} ranges, {h.shape[0]} hit flags, {meas.shape[0]} measured ranges")
    n = r.shape[0]
    err = r[h] - meas[h]
    a = np.abs(err)
    nan = float("nan")
    return {"rays": int(n), "hits": int(h.sum()),
            "hit_ratio": float(h.sum()) / n if n else nan,
            "mean_abs_err_m": float(a.mean()) if a.size else nan,
            "median_abs_err_m": float(np.median(a)) if a.size else nan,
            "rmse_m": float(np.sqrt(np.mean(err * err))) if a.size else nan,
            "bias_m": float(err.mean()) if a.size else nan,
            "within_threshold": float((a <= threshold_m).sum()) / n if n else nan}


# ---- frames ------------------------------------------------------------------------------------------------------------

def held_out_frames(config, total_frames: int) -> list:
    """The frame ids in [begin_frame, end_frame] (and below total_frames) that mapping skips (`scans.used_frame`)."""
    from .scans import used_frame
    last = min(int(config.end_frame), int(total_frames) - 1)
    return [f for f in range(max(0, int(config.begin_frame)), last + 1) if not used_frame(config, f)]


def parse_frames(text: str) -> range:
    """'START:STOP[:STEP]' -> range(START, STOP, STEP), Python's half-open convention; raises ValueError."""
    parts = text.split(":")
    if len(parts) not in (2, 3) or not all(p.strip().lstrip("-").isdigit() for p in parts):
        raise ValueError(f"--frames {text!r}: expected START:STOP or START:STOP:STEP with integers")
    start, stop, step = (int(p) for p in parts) if len(parts) == 3 else (int(parts[0]), int(parts[1]), 1)
    if start < 0 or stop <= start or step < 1:
        raise ValueError(f"--frames {text!r}: need 0 <= START < STOP and STEP >= 1")
    return range(start, stop, step)


def map_pose(dataset, frame_id: int) -> np.ndarray:
    """A frame's pose in the map frame, begin_pose_inv @ world pose.  `poses_ref` holds that for the frames mapping uses
    and the world pose for the others (dataset/lidar_dataset.py:84-91)."""
    pose = np.asarray(dataset.poses_ref[frame_id], dtype=np.float64)
    if frame_id in set(dataset.used_frames):
        return pose
    return np.asarray(dataset.begin_pose_inv, dtype=np.float64) @ pose


def scan_frames(dataset, frame_ids):
    """-> (frame id, origin_scaled fp64 [3], points fp32 [m,3] scaled map coordinates on the device) per frame: the scan
    read and preprocessed exactly as mapping preprocesses it (`ScanProcessor.points`), at its map-frame pose."""
    for f in frame_ids:
        if not 0 <= f < dataset.total_pc_count:
            raise ValueError(f"frame {f}: the sequence has frames 0 .. {dataset.total_pc_count - 1}")
        pose = map_pose(dataset, f)
        pts = dataset.processor.points(dataset.read_frame(f), pose)
        yield f, pose[:3, 3] * dataset.config.scale, pts


def eval_scans(config, octree, decoder, frames, threshold_m: float, step_m: float | None = None, beyond_m: float = 1.0,
               refine_iters: int = REFINE_ITERS, points_dir: str | None = None, to_world=None) -> dict:
    """frames: (name, origin_scaled, points_scaled) per frame (`scan_frames`).  step_m defaults to mc_res_m, the
    resolution the mesh is made at.  points_dir: write each frame's hit points as points_dir/{name}.ply, metres, through
    to_world (a 4x4, e.g. inv(begin_pose_inv); default identity).
    -> {"frames": [{"frame": name, **ray_metrics}], "total": ray_metrics over every ray of every frame}."""
    step = float(config.mc_res_m if step_m is None else step_m)
    scale = float(config.scale)
    T = np.eye(4) if to_world is None else np.asarray(to_world, dtype=np.float64)
    rows, all_r, all_h, all_m = [], [], [], []
    for name, origin, pts in frames:
        rng, hit = cast_rays(config, octree, decoder, origin, pts, step, beyond_m, refine_iters)
        o64 = torch.as_tensor(np.asarray(origin, dtype=np.float32).astype(np.float64), device=pts.device)
        v = pts.double() - o64
        dist = v.norm(dim=1)
        measured = dist / scale
        rows.append({"frame": name, **ray_metrics(rng, hit, measured, threshold_m)})
        if points_dir is not None:
            d = v[hit] / dist[hit, None]
            p = o64 / scale + d * rng[hit, None]
            p = p @ torch.as_tensor(T[:3, :3].T, device=p.device) + torch.as_tensor(T[:3, 3], device=p.device)
            from .evaluate import write_point_ply
            write_point_ply(os.path.join(points_dir, f"{name}.ply"), p)
        all_r.append(rng.cpu()); all_h.append(hit.cpu()); all_m.append(measured.cpu())
    cat = (lambda xs, dt: torch.cat(xs) if xs else torch.zeros(0, dtype=dt))
    total = ray_metrics(cat(all_r, torch.float64), cat(all_h, torch.bool), cat(all_m, torch.float64), threshold_m)
    return {"frames": rows, "total": total}
