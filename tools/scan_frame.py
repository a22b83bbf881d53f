"""Time `LiDARDataset.process_frame` on one synthetic HDL-64 scan (about 130 k points, KITTI .bin) stage by stage with
CUDA events, and the numpy oracle of the same frame (tests/scan_oracle.py) on the host.

    python tools/scan_frame.py [--repeat 20] [--out OUT.json]
"""
from __future__ import annotations

import argparse
import ctypes as C
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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--repeat", type=int, default=20)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("tools/scan_frame.py measures on the GPU; none is visible")
    from shine_mapping_b200 import FeatureOctree, _abi, scans, synth
    from shine_mapping_b200.config import SHINEConfig
    from tests import scan_oracle
    dev = "cuda:0"
    tmp = tempfile.mkdtemp()
    dirs = synth.lidar_directions(2048).double()
    hits = synth.raycast_scene(torch.zeros(3), dirs.float(), synth.default_boxes(), min_range=1.0, max_range=80.0)
    pts = hits.numpy().astype(np.float32)
    pts += np.random.default_rng(0).normal(scale=0.01, size=pts.shape).astype(np.float32)
    np.concatenate((pts, np.ones((len(pts), 1), np.float32)), 1).tofile(os.path.join(tmp, "0.bin"))
    cfg = SHINEConfig(device=dev, rand_downsample=False, vox_down_m=0.05, pc_radius=50.0, min_range=2.75,
                      tree_level_world=12, leaf_vox_size=0.2, tree_level_feat=3, surface_sample_n=3, free_sample_n=3,
                      continual_learning_reg=False, window_replay_on=False)
    path = os.path.join(tmp, "0.bin")
    pose = np.eye(4)
    proc = scans.ScanProcessor(cfg, dev)
    lib, st = _abi.lib(), _abi.stream_ptr(dev)
    stages = ["read_h2d", "filter_keys", "sort", "average_transform", "sample", "octree_update", "pool_append"]
    times = {k: [] for k in stages}
    for r in range(args.repeat + 3):
        octree, pool = FeatureOctree(cfg), synth.SamplePool(dev)
        ev = [torch.cuda.Event(enable_timing=True) for _ in range(len(stages) + 1)]
        torch.cuda.synchronize()
        ev[0].record()
        rec = scans.read_scan(path)
        data = rec.data.to(dev, non_blocking=True)
        ev[1].record()
        inp = _abi.ShineScanInput(data.data_ptr(), rec.n, rec.stride, 0)
        scratch = proc._scratch_for(rec.n)
        _abi.check(lib.shine_scan_filter_keys(C.byref(inp), cfg.min_z, cfg.max_z, cfg.min_range, cfg.pc_radius,
                                              cfg.vox_down_m, _abi.ptr(scratch), scratch.numel(), st), "filter")
        ev[2].record()
        _abi.check(lib.shine_scan_sort_voxels(rec.n, _abi.ptr(proc.count), _abi.ptr(scratch), scratch.numel(), st), "sort")
        ev[3].record()
        m = int(proc.count.item())
        p = torch.empty(m, 3, device=dev)
        T = (C.c_double * 16)(*pose.reshape(16).tolist())
        _abi.check(lib.shine_scan_average_transform(C.byref(inp), T, cfg.scale, m, None, _abi.ptr(p), _abi.ptr(scratch),
                                                    scratch.numel(), st), "average")
        ev[4].record()
        coord, label, weight = proc.sample(p, np.zeros(3, np.float32))
        ev[5].record()
        octree.update(coord.view(-1, 6, 3)[:, :3].reshape(-1, 3))
        ev[6].record()
        pool.append(coord, label, weight)
        ev[7].record()
        torch.cuda.synchronize()
        if r >= 3:
            for k, name in enumerate(stages):
                times[name].append(ev[k].elapsed_time(ev[k + 1]))
    t0 = time.perf_counter()
    reps = 3
    for _ in range(reps):
        scan_oracle.frame_points(scans.read_scan(path, pinned=False).points(), pose, cfg)
    oracle_ms = (time.perf_counter() - t0) / reps * 1e3
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                         text=True).stdout.strip().splitlines()[0]
    med = {k: float(np.median(v)) for k, v in times.items()}
    line = {"points": int(rec.n), "voxels": m, "samples": int(coord.shape[0]), "gpu": smi,
            "median_ms": {k: round(v, 3) for k, v in med.items()}, "process_frame_ms": round(sum(med.values()), 3),
            "numpy_oracle_stages_1_3_ms": round(oracle_ms, 1)}
    print(json.dumps(line))
    if args.out:
        os.makedirs(os.path.dirname(args.out), exist_ok=True)
        with open(args.out, "w") as fh:
            json.dump(line, fh)


if __name__ == "__main__":
    main()
