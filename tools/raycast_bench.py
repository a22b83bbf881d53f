"""Cost of casting held-out scans through a map (`shine_raycast`, raycast.py) on the synthetic drive.

    python tools/raycast_bench.py [--frames 20] [--iters 1000] [--reps 50] [--subset 64]

1. Writes `synth.write_drive` (the analytic street, --frames scans 1.5 m apart) to a temporary directory, maps every
   other frame with the batch loop (`--scans`, every_frame 2, --iters iterations) and loads the saved checkpoint.
2. Each held-out scan at its real ray count (preprocessed as `evaluate scans` does), with the command's defaults (step
   mc_res_m = 0.1 m, 1 m past each point, 8 bisection steps): CUDA events around --reps launches after 5 warm-up
   launches, ms per launch and rays per second; and one batch of 10^6 rays from the first held-out frame's origin
   towards its points repeated, same settings.
3. From the oracle's cell walk (tests/raycast_oracle.py `skip_samples`) on --subset rays of every held-out frame: the
   lattice samples a ray probes with empty-space skipping against the samples of the whole lattice (a count, not a time).

Prints one JSON object with the card's name and power limit read in the same run.  Writes nothing outside a temporary
directory.  Needs a GPU.
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
import types

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True, check=False)
    return {"name": torch.cuda.get_device_name(0), "nvidia_smi": q.stdout.strip().splitlines()[:1]}


def main(argv=None):
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--frames", type=int, default=20)
    ap.add_argument("--iters", type=int, default=1000)
    ap.add_argument("--reps", type=int, default=50)
    ap.add_argument("--subset", type=int, default=64)
    args = ap.parse_args(argv)
    if not torch.cuda.is_available():
        raise SystemExit("raycast_bench times sm_90a kernels: no CUDA device")
    import yaml
    from shine_mapping_b200 import _abi, batch_loop, synth
    from shine_mapping_b200.checkpoint import load_checkpoint
    from shine_mapping_b200.config import SHINEConfig
    from shine_mapping_b200.decoder import Decoder
    from shine_mapping_b200.raycast import REFINE_ITERS, held_out_frames, mask_level, scan_frames
    from shine_mapping_b200.scans import LiDARDataset
    from tests.raycast_oracle import skip_samples
    dev = "cuda:0"
    report = {"card": card()}
    with tempfile.TemporaryDirectory() as tmp:
        paths = synth.write_drive(os.path.join(tmp, "drive"), n_frames=args.frames)
        doc = {"setting": dict(pc_path=paths["pc_path"], pose_path=paths["pose_path"], calib_path="", begin_frame=0,
                               end_frame=100000, every_frame=2, first_frame_ref=True, device=dev),
               "process": {"min_range_m": 2.75, "pc_radius_m": 30.0, "min_z_m": -10.0, "rand_downsample": False,
                           "vox_down_m": 0.1},
               "sampler": {"surface_sample_range_m": 0.3, "surface_sample_n": 3, "free_sample_begin_ratio": 0.3,
                           "free_sample_end_dist_m": 0.8, "free_sample_n": 3},
               "octree": {"tree_level_world": 12, "tree_level_feat": 3, "leaf_vox_size": 0.2, "feature_dim": 8},
               "continual": {"continual_learning_reg": False, "window_replay_on": False},
               "optimizer": {"batch_size": 8192, "learning_rate": 0.01},
               "eval": {"save_freq_iters": args.iters, "vis_freq_iters": 10 ** 9, "mc_res_m": 0.1}}
        cfg_path = os.path.join(tmp, "cfg.yaml")
        with open(cfg_path, "w") as fh:
            yaml.safe_dump(doc, fh)
        run = os.path.join(tmp, "run")
        batch_loop.main([cfg_path, "--scans", "--iters", str(args.iters), "--run-path", run])
        config = SHINEConfig()
        config.load(cfg_path)
        state, octree = load_checkpoint(os.path.join(run, "model", f"model_iter_{args.iters}.pth"), config, dev)
        decoder = Decoder(config)
        decoder.load_state_dict(state)
        dataset = LiDARDataset(config)
        frames = list(scan_frames(dataset, held_out_frames(config, dataset.total_pc_count)))

    lib, st = _abi.lib(), _abi.stream_ptr(dev)
    od, dd = octree._descriptor(None, None), decoder.c_descriptor(None)
    scale = config.scale
    h, beyond = float(np.float32(config.mc_res_m * scale)), float(np.float32(1.0 * scale))
    level = mask_level(config, octree)

    def timed(origin, pts):
        n = pts.shape[0]
        out_t = torch.empty(n, device=dev)
        out_s = torch.empty(n, dtype=torch.uint8, device=dev)
        o = (C.c_float * 3)(*np.asarray(origin, dtype=np.float32).tolist())

        def launch():
            _abi.check(lib.shine_raycast(C.byref(od), C.byref(dd), o, _abi.ptr(pts), n, h, 0.0, beyond, math.inf,
                                         REFINE_ITERS, level, _abi.ptr(out_t), _abi.ptr(out_s), st), "shine_raycast")
        for _ in range(5):
            launch()
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize()
        a.record()
        for _ in range(args.reps):
            launch()
        b.record()
        torch.cuda.synchronize()
        ms = a.elapsed_time(b) / args.reps
        return {"rays": n, "hits": int(out_s.sum()), "ms": round(ms, 4), "rays_per_s": round(n / ms * 1e3)}

    report["frames"] = {str(f): timed(origin, pts) for f, origin, pts in frames}
    f0, o0, p0 = frames[0]
    big = p0.repeat(-(-10 ** 6 // p0.shape[0]), 1)[:10 ** 6].contiguous()
    report["batch_1e6"] = timed(o0, big)
    # sample counts from the oracle's cell walk on a subset of every frame's rays
    L = octree.featured_level_num
    top = octree.max_level - (L - 1)
    o = types.SimpleNamespace(featured_level_num=L, max_level=octree.max_level,
                              nodes_lookup_tables={top: set(octree._levels[top].node_keys.cpu().tolist())})
    skipped = full = 0
    rng = np.random.default_rng(0)
    for f, origin, pts in frames:
        p = pts.cpu().numpy()
        sel = p[rng.choice(p.shape[0], min(args.subset, p.shape[0]), replace=False)]
        s, a = skip_samples(o, origin, sel, np.float32(h), 0.0, np.float32(beyond), math.inf)
        skipped += int(s.sum()); full += int(a.sum())
    report["samples_per_ray"] = {"with_skipping": round(skipped / max(1, args.subset * len(frames)), 1),
                                 "without_skipping": round(full / max(1, args.subset * len(frames)), 1),
                                 "rays": args.subset * len(frames)}
    print(json.dumps(report))


if __name__ == "__main__":
    main()
