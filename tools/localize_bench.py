"""Cost of localizing scans in a saved map (odometry.register_scans) against one `register` per scan.

    python tools/localize_bench.py [--frames 20] [--azimuth 1024] [--iters 150] [--reps 3] [--out FILE]

The workload of tools/odometry_bench.py: `synth.write_drive` (the analytic street, --frames scans 1.5 m apart, --azimuth
steps per revolution).  The even frames are mapped on their true poses by the incremental loop (replay mode, --iters
per frame); the odd frames are then localized in that map from a fixed pattern of starts, 0.5 m along or across the
street, 5 degrees of yaw, or combinations (those of test_registration_recovers_perturbed_pose).

In one process, --reps times each and alternating:
* "lock_step": `register_scans` over all odd frames at once;
* "per_scan":  `register` of each frame in turn.
Both start from a synchronised device and end in a synchronise; the host clock around them gives ms per scan.  Both
must return the same poses and info bit for bit.  A separate torch.profiler run of each gives the register kernels'
own time, the number of register kernel launches and the device-to-host copies, per scan.  The preprocessed scans are
made once, before the timed runs.  Prints one JSON object with the card's name and power limit, read in the same run.
Needs a GPU.
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

STARTS = [(0.5, 0.0, 0.0), (0.0, 0.5, 0.0), (0.3, -0.3, 5.0), (-0.35, 0.35, -5.0), (0.0, 0.0, 5.0)]


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return {"name": torch.cuda.get_device_name(0), "nvidia_smi": q.stdout.strip().splitlines()[:1]}


def perturbed(pose, dx, dy, dyaw_deg):
    out = pose.copy()
    out[:3, 3] += (dx, dy, 0.0)
    c, s = math.cos(math.radians(dyaw_deg)), math.sin(math.radians(dyaw_deg))
    out[:3, :3] = np.array([[c, -s, 0], [s, c, 0], [0, 0, 1]]) @ out[:3, :3]
    return out


def same(a, b) -> bool:
    for (pa, ia), (pb, ib) in zip(a, b):
        if not np.array_equal(pa.view(np.int64), pb.view(np.int64)) or ia.keys() != ib.keys():
            return False
        if not all(ia[k] == ib[k] or (ia[k] != ia[k] and ib[k] != ib[k]) for k in ia):
            return False
    return len(a) == len(b)


def profile(fn, n_scans):
    """The register kernels' device time, their launch count and the device-to-host copies, per scan."""
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    kernel_us, launches, d2h = 0.0, 0, 0
    for e in prof.key_averages():
        if "register_normal_eq_kernel" in e.key or "register_fold_kernel" in e.key:
            kernel_us += getattr(e, "device_time_total", None) or getattr(e, "cuda_time_total", 0.0)
            launches += e.count
        elif "Memcpy DtoH" in e.key:
            d2h += e.count
    return {"kernel_ms_per_scan": kernel_us / 1e3 / n_scans, "register_launches_per_scan": launches / n_scans,
            "d2h_copies_per_scan": d2h / n_scans}


def main(argv=None):
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--frames", type=int, default=20)
    ap.add_argument("--azimuth", type=int, default=1024)
    ap.add_argument("--iters", type=int, default=150)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--out", default=None)
    args = ap.parse_args(argv)
    if not torch.cuda.is_available():
        raise SystemExit("localize_bench needs a GPU")
    from shine_mapping_b200 import Decoder, FeatureOctree, odometry, synth
    from shine_mapping_b200.config import SHINEConfig
    from shine_mapping_b200.incre_loop import run_shine_mapping_incremental
    from shine_mapping_b200.localize import pose_errors
    from shine_mapping_b200.raycast import map_pose
    from shine_mapping_b200.scans import LiDARDataset

    with tempfile.TemporaryDirectory() as tmp:
        drive = synth.write_drive(tmp, n_frames=args.frames, n_azimuth=args.azimuth)
        cfg = SHINEConfig(tree_level_world=12, tree_level_feat=3, leaf_vox_size=0.2, feature_dim=8, device="cuda:0",
                          surface_sample_range_m=0.3, surface_sample_n=3, free_sample_begin_ratio=0.3,
                          free_sample_end_dist_m=0.8, free_sample_n=3, min_range=2.75, pc_radius=25.0, min_z=-10.0,
                          vox_down_m=0.1, rand_downsample=False, continual_learning_reg=False, window_replay_on=False,
                          bs=4096, lr=0.01, begin_frame=0, end_frame=10 ** 6, every_frame=2, seed=7,
                          pc_path=drive["pc_path"], pose_path=drive["pose_path"], calib_path="")
        torch.manual_seed(cfg.seed)
        octree, decoder = FeatureOctree(cfg), Decoder(cfg)
        ds = LiDARDataset(cfg)
        run_shine_mapping_incremental(cfg, octree, decoder, ds.frames(), iters=args.iters, pool=synth.ReplayPool(ds.device))
        frames = [f for f in range(args.frames) if f % 2]
        truth = [map_pose(ds, f) for f in frames]
        local = [ds.processor.points(ds.read_frame(f), np.eye(4)) for f in frames]
        starts = [perturbed(T, *STARTS[i % len(STARTS)]) for i, T in enumerate(truth)]
        reg = odometry.ScanToMapRegistration(cfg, octree, decoder)
        torch.cuda.synchronize()

        runs = {"lock_step": lambda: reg.register_scans(local, starts),
                "per_scan": lambda: [reg.register(p, s) for p, s in zip(local, starts)]}
        results = {name: fn() for name, fn in runs.items()}          # warm-up: every shape of the timed runs
        identical = same(results["lock_step"], results["per_scan"])
        host_ms = {name: [] for name in runs}
        for _ in range(args.reps):
            for name, fn in runs.items():
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                out = fn()
                torch.cuda.synchronize()
                host_ms[name].append(1e3 * (time.perf_counter() - t0) / len(frames))
                identical = identical and same(out, results["lock_step"])
        prof = {name: profile(fn, len(frames)) for name, fn in runs.items()}

    errs = [pose_errors(p, T) for (p, _), T in zip(results["lock_step"], truth)]
    infos = [i for _, i in results["lock_step"]]
    res = {
        "card": card(), "frames": args.frames, "azimuth": args.azimuth, "train_iters_per_frame": args.iters,
        "localized_frames": frames, "scan_points": [int(p.shape[0]) for p in local],
        "identical_poses_and_info": identical,
        "ms_per_scan": {name: {"median": float(np.median(v)), "min": float(min(v)), "max": float(max(v))}
                        for name, v in host_ms.items()},
        "profile": prof,
        "ok": sum(bool(i["ok"]) for i in infos), "converged": sum(bool(i["converged"]) for i in infos),
        "iters": [int(i["iters"]) for i in infos],
        "max_translation_error_m": max(e[0] for e in errs), "max_rotation_error_deg": max(e[1] for e in errs),
    }
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as fh:
            fh.write(line + "\n")
    if not identical:
        raise SystemExit("lock-step and per-scan registration returned different poses or info")
    return res


if __name__ == "__main__":
    main()
