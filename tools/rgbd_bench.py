"""Time one 640x480 RGB-D frame on the direct path: PNG decode on the host, the H2D copy, the back-projection kernel and
the existing scan pipeline (filter, voxel grid, transform, sampling), with CUDA events; and a numpy restatement of the
back-projection on the CPU for comparison.

    python tools/rgbd_bench.py [--reps 50]

The frame is the synthetic sequence's camera (tests/test_gpu_rgbd.py) at 640x480, focal 400 px, with
config/rgbd/rgbd_batch.yaml's settings.  Medians over --reps after one warm-up; one JSON line with the card's name and
power limit read in the same run.  Writes only to a temporary directory.
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import sys
import tempfile
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--reps", type=int, default=50)
    args = ap.parse_args()
    import __graft_entry__ as ge
    ge.build()
    from bench import device_info
    from shine_mapping_b200 import rgbd, scans
    from tests import test_gpu_rgbd as t
    from tests.test_rgbd_host import write_png

    raw = t.render_depth(t.camera_to_world(0), 480, 640, 400.0)
    cam = rgbd.RGBDCamera(640, 480, 400.0, 400.0, 319.5, 239.5, 1000.0, t.FLIP)
    cfg = t._rgbd_cfg()
    proc = scans.ScanProcessor(cfg, "cuda:0")
    pose = np.eye(4)
    with tempfile.TemporaryDirectory() as tmp:
        path = os.path.join(tmp, "depth.png")
        write_png(path, raw)
        times = {k: [] for k in ("decode_ms", "h2d_ms", "kernel_ms", "scan_pipeline_ms", "numpy_backproject_ms")}
        for rep in range(args.reps + 1):
            t0 = time.perf_counter()
            depth = rgbd.read_depth(path)
            t1 = time.perf_counter()
            ev = [torch.cuda.Event(enable_timing=True) for _ in range(4)]
            ev[0].record()
            d = depth.view(torch.uint8).to("cuda:0", non_blocking=True)
            ev[1].record()
            xyz = rgbd.backproject(d.view(torch.uint16), cam, 5.0, "cuda:0")
            ev[2].record()
            rec = scans.ScanRecords(xyz.view(torch.uint8).reshape(-1), xyz.shape[0], 24, True)
            pts = proc.points(rec, pose)
            proc.sample(pts, np.zeros(3, np.float32))
            ev[3].record()
            torch.cuda.synchronize()
            t2 = time.perf_counter()
            t.oracle(raw, cam.fx, cam.fy, cam.cx, cam.cy, 1000.0, 5.0, cam.camera_pose)
            t3 = time.perf_counter()
            if rep == 0:
                continue
            times["decode_ms"].append((t1 - t0) * 1e3)
            times["h2d_ms"].append(ev[0].elapsed_time(ev[1]))
            times["kernel_ms"].append(ev[1].elapsed_time(ev[2]))
            times["scan_pipeline_ms"].append(ev[2].elapsed_time(ev[3]))
            times["numpy_backproject_ms"].append((t3 - t2) * 1e3)
        # the kernel alone, back to back
        ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        ev0.record()
        for _ in range(200):
            rgbd.backproject(d.view(torch.uint16), cam, 5.0, "cuda:0")
        ev1.record()
        torch.cuda.synchronize()
    out = {k: round(statistics.median(v), 4) for k, v in times.items()}
    out["kernel_ms_back_to_back"] = round(ev0.elapsed_time(ev1) / 200, 4)
    out.update(frame="640x480", valid_pixels=int(((raw > 0) & (raw < 5000)).sum()), points=int(pts.shape[0]), reps=args.reps,
               stat="median", device=device_info(0))
    print(json.dumps(out))


if __name__ == "__main__":
    main()
