"""Cost and accuracy of pose-free mapping (odometry.py) on a synthetic drive.

    python tools/odometry_bench.py [--frames 20] [--azimuth 1024] [--iters 150] [--reps 200] [--out FILE]

1. Writes `synth.write_drive` (the analytic street, --frames scans 1.5 m apart) to a temporary directory and maps it
   with `OdometryScans` in the incremental loop (replay mode): per frame, the registration (host clock around
   `estimate_pose`, which ends in the host read of the last normal equations) against the frame's training (host clock
   around the rest of the frame, synchronised), and the ATE of the estimated poses against the written ones.  Each frame
   prints one line: its error against the written pose (translation m, rotation deg), the registration's info and the
   error of the pose after each stage of `register` (the constant-velocity prediction, the best coarse candidate, each
   Gauss-Newton run and the weak-direction search).  The drive runs twice, alternately:
   with `launch_items` forced through one `launch` per pose ("per_pose", the registration before the batched entries:
   the same poses, bit for bit) and as built ("batched").
2. `shine_register_normal_eq` alone at the scans' point counts on the final map: CUDA events around --reps launches
   (one Gauss-Newton iteration each, without its 29-double read; the interval includes the host's launch cost when the
   host is the slower side), and the two kernels' own durations from a torch.profiler run of the same launches.
3. The coarse grid's 1105 poses at the last scan: `shine_register_normal_eq_poses` in one call against 1105 single
   launches, kernel durations from the profiler and the host clock around each (synchronised).

Prints one JSON object with the card name and power limit read in the same run.  Needs a GPU.
"""
from __future__ import annotations

import argparse
import json
import math
import os
import subprocess
import sys
import tempfile
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return {"name": torch.cuda.get_device_name(0), "nvidia_smi": q.stdout.strip().splitlines()[:1]}


def main(argv=None):
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--frames", type=int, default=20)
    ap.add_argument("--azimuth", type=int, default=1024)
    ap.add_argument("--iters", type=int, default=150)
    ap.add_argument("--reps", type=int, default=200)
    ap.add_argument("--out", default=None)
    args = ap.parse_args(argv)
    if not torch.cuda.is_available():
        raise SystemExit("odometry_bench needs a GPU")
    from shine_mapping_b200 import Decoder, FeatureOctree, odometry, synth
    from shine_mapping_b200.config import SHINEConfig
    from shine_mapping_b200.incre_loop import run_shine_mapping_incremental

    cfg = SHINEConfig(tree_level_world=12, tree_level_feat=3, leaf_vox_size=0.2, feature_dim=8, device="cuda:0",
                      surface_sample_range_m=0.3, surface_sample_n=3, free_sample_begin_ratio=0.3,
                      free_sample_end_dist_m=0.8, free_sample_n=3, min_range=2.75, pc_radius=25.0, min_z=-10.0,
                      vox_down_m=0.1, rand_downsample=False, continual_learning_reg=False, window_replay_on=False,
                      bs=4096, lr=0.01, end_frame=10 ** 6, seed=7)
    class Traced(odometry.ScanToMapRegistration):
        """`register` as built, keeping (stage, pose) after each of its stages in `stages`."""

        def register(self, points, init):
            self.stages = [("prediction", np.array(init))]
            return super().register(points, init)

        def coarse_scans(self, points, segments, poses):
            r = super().coarse_scans(points, segments, poses)
            self.stages.append(("coarse", r[0]))
            return r

        def gauss_newton_scans(self, points, segments, poses):
            r = super().gauss_newton_scans(points, segments, poses)
            if r:
                self.stages.append(("gauss_newton", r[0][0]))
            return r

        def search_scans(self, points, segments, poses):
            r = super().search_scans(points, segments, poses)
            if r:
                self.stages.append(("weak_direction", r[0][0]))
            return r

    class PerPose(Traced):
        def launch_items(self, points, segments, poses_scaled, kappa_scaled, out):
            for k, T in enumerate(np.asarray(poses_scaled).reshape(-1, 4, 4)):
                b, n = (int(v) for v in np.asarray(segments).reshape(-1, 2)[k])
                self.launch(points[b:b + n], T, kappa_scaled, out[k])

    def err(E, W):
        D = np.linalg.inv(W) @ E
        return [round(float(np.linalg.norm(D[:3, 3])), 4), round(math.degrees(float(np.linalg.norm(odometry.se3_log(D)[3:]))), 3)]

    def drive_run(drive, per_pose):
        torch.manual_seed(cfg.seed)
        octree, decoder = FeatureOctree(cfg), Decoder(cfg)
        ds = odometry.OdometryScans(cfg, octree, decoder)
        ds.registration = (PerPose if per_pose else Traced)(cfg, octree, decoder)
        reg_s, train_s, points = [], [], []
        truth = drive["poses"]

        def frames():
            for f in ds.used_frames:
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                ds.estimate_pose(f)
                reg_s.append(time.perf_counter() - t0)
                if not per_pose:
                    rec = {"frame": f, "error": err(ds.poses_ref[f], truth[f]), "info": ds.reg_info[f]}
                    if f:
                        rec["stages"] = [(name, err(T, truth[f])) for name, T in ds.registration.stages]
                    print(json.dumps(rec), flush=True)
                sample = ds.frame_samples(f)
                points.append(int(sample[4].shape[0]))
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                yield sample[:4]                   # the loop trains the frame before it asks for the next one
                torch.cuda.synchronize()
                train_s.append(time.perf_counter() - t0)

        run_shine_mapping_incremental(cfg, octree, decoder, frames(), iters=args.iters, pool=synth.ReplayPool(ds.device))
        return ds, reg_s, train_s, points

    with tempfile.TemporaryDirectory() as tmp:
        drive = synth.write_drive(tmp, n_frames=args.frames, n_azimuth=args.azimuth)
        cfg.pc_path = drive["pc_path"]
        runs = {}
        for name in ("per_pose", "batched", "per_pose", "batched"):
            ds, reg_s, train_s, points = drive_run(drive, name == "per_pose")
            runs.setdefault(name, []).append(1e3 * float(np.median(reg_s[1:])))
        truth = drive["poses"]
        t_err, r_err = [], []
        for f in ds.used_frames:
            D = np.linalg.inv(truth[f]) @ ds.poses_ref[f]
            t_err.append(float(np.linalg.norm(D[:3, 3])))
            r_err.append(math.degrees(float(np.linalg.norm(odometry.se3_log(D)[3:]))))
        iters = [ds.reg_info[f]["iters"] for f in ds.used_frames[1:]]

        # the kernel alone, at the scans' point counts, on the final map
        reg = ds.registration
        rec = ds.read_frame(ds.used_frames[-1])
        local = ds.processor.points(rec, np.eye(4))
        pose = ds.poses_ref[ds.used_frames[-1]].copy()
        pose[:3, 3] *= cfg.scale
        kernel = {}
        for n in sorted({min(points), int(np.median(points)), max(points), 10 ** 6}):
            pts = local[torch.arange(n, device=local.device) % local.shape[0]].contiguous()
            for _ in range(10):
                reg.launch(pts, pose, 0.1 * cfg.scale)
            start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            start.record()
            for _ in range(args.reps):
                reg.launch(pts, pose, 0.1 * cfg.scale)
            end.record()
            end.synchronize()
            kernel[str(n)] = {"events_ms_per_launch": start.elapsed_time(end) / args.reps}
            # the kernels' own durations (the events interval also holds the host's launch cost when that is longer)
            with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
                for _ in range(args.reps):
                    reg.launch(pts, pose, 0.1 * cfg.scale)
                torch.cuda.synchronize()
            for e in prof.key_averages():
                if "register_normal_eq_kernel" in e.key or "register_fold_kernel" in e.key:
                    us = getattr(e, "device_time_total", None) or getattr(e, "cuda_time_total", 0.0)
                    kernel[str(n)]["fold_ms" if "fold" in e.key else "kernel_ms"] = us / 1e3 / args.reps
        # the coarse grid's poses at the last scan: one batched call against one launch per pose
        P = []
        for yaw in reg.GRID_YAW:
            Rz = np.array([[math.cos(yaw), -math.sin(yaw), 0.0], [math.sin(yaw), math.cos(yaw), 0.0], [0.0, 0.0, 1.0]])
            for dx in reg.GRID_X:
                for dy in reg.GRID_Y:
                    T = pose.copy()
                    T[:3, :3] = Rz @ pose[:3, :3]
                    T[:3, 3] += np.array([dx, dy, 0.0]) * cfg.scale
                    P.append(T)
        P = np.stack(P)
        outs = torch.empty(len(P), 29, dtype=torch.float64, device=local.device)
        grid = {"K": len(P), "points": int(local.shape[0])}
        for name, fn in (("batched", lambda: reg.launch_poses(local, P, 0.2 * cfg.scale, outs)),
                         ("single", lambda: [reg.launch(local, T, 0.2 * cfg.scale, outs[k]) for k, T in enumerate(P)])):
            for _ in range(3):
                fn()
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            for _ in range(5):
                fn()
            torch.cuda.synchronize()
            grid[f"{name}_host_ms"] = 1e3 * (time.perf_counter() - t0) / 5
            with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
                for _ in range(5):
                    fn()
                torch.cuda.synchronize()
            total = 0.0
            for e in prof.key_averages():
                if "register_normal_eq_kernel" in e.key or "register_fold_kernel" in e.key:
                    total += getattr(e, "device_time_total", None) or getattr(e, "cuda_time_total", 0.0)
            grid[f"{name}_kernel_ms"] = total / 1e3 / 5
    res = {
        "card": card(), "frames": args.frames, "azimuth": args.azimuth, "train_iters_per_frame": args.iters,
        "scan_points": {"min": min(points), "median": int(np.median(points)), "max": max(points)},
        "kernel_ms_per_gauss_newton_iteration": kernel,
        "gauss_newton_iterations": {"mean": float(np.mean(iters)), "max": int(max(iters))},
        "converged_frames": sum(bool(ds.reg_info[f]["converged"]) for f in ds.used_frames),
        "registration_ms_per_frame": {"median": 1e3 * float(np.median(reg_s[1:])), "max": 1e3 * float(max(reg_s[1:])),
                                      "median_per_drive": runs},
        "coarse_grid": grid,
        "training_ms_per_frame": {"median": 1e3 * float(np.median(train_s)), "max": 1e3 * float(max(train_s))},
        "ate_rmse_m": float(np.sqrt(np.mean(np.square(t_err)))), "max_translation_error_m": float(max(t_err)),
        "max_rotation_error_deg": float(max(r_err)),
    }
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as fh:
            fh.write(line + "\n")
    return res


if __name__ == "__main__":
    main()
