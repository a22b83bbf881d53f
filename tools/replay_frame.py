"""Per-frame cost of the replay sample pool on the GPU.

    python tools/replay_frame.py [--sizes 4000000 16000000 40000000] [--frame 800000] [--reps 10] [--out FILE]

1. `ReplayPool.add_frame` on pools of --sizes samples with a --frame-sample frame and a window that drops about 5 % of
   the pool: the `shine_pool_window_append` launch (CUDA events), the whole `add_frame` (host clock, size read-back
   included), and the reference's torch mask-and-cat (tests/replay_oracle.py) on the same data.  Achieved bandwidth is
   the algorithmic bytes N*12 (coordinates) + moved*(8 + 20) (label and weight read, sample written, for the kept
   samples that change place) + n_new*40 (frame read and written) over kernel time, against the 3.35 TB/s HBM3
   data-sheet figure of the H100 SXM.
2. One replay frame of a synthetic drive with kitti_incre_replay-like settings: octree.update / add_frame / trainer
   set-up / the iterations, split into get_batch, step and Adam (CUDA events; the phases that read back to the host
   include that wait).

Prints one JSON object with the card name and power limit read in the same run.  Needs a GPU.
"""
from __future__ import annotations

import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

HBM_PEAK = 3.35e12


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return {"name": torch.cuda.get_device_name(0), "nvidia_smi": q.stdout.strip().splitlines()[:1]}


def time_events(fn, reps, before=None):
    """median ms of fn() between two events, `before()` run (untimed) ahead of every call"""
    out = []
    for _ in range(reps):
        if before:
            before()
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        b.synchronize()
        out.append(a.elapsed_time(b))
    out.sort()
    return out[len(out) // 2]


def add_frame_costs(n, n_new, reps, dev):
    from shine_mapping_b200 import _abi, synth
    from tests.replay_oracle import replay_pool_update, window_mask
    gen = torch.Generator(device=dev).manual_seed(n)
    origin = (0.0371, -0.0113, 0.0042)
    o = torch.tensor(origin, device=dev)
    coord = (o + (torch.rand(n, 3, device=dev, generator=gen) - 0.5) * 0.2).contiguous()
    label = torch.randn(n, device=dev, generator=gen)
    weight = torch.where(torch.rand(n, device=dev, generator=gen) < 0.5, 1.0, -1.0)
    new = ((o + (torch.rand(n_new, 3, device=dev, generator=gen) - 0.5) * 0.2).contiguous(),
           torch.randn(n_new, device=dev, generator=gen), torch.ones(n_new, device=dev))
    r = float((coord[::97] - o).norm(dim=1).quantile(0.95))
    mask = window_mask(coord, origin, r)
    pos = torch.cumsum(mask, 0) - 1
    moved = int((mask & (pos != torch.arange(n, device=dev))).sum())
    algo_bytes = n * 12 + moved * (8 + 20) + n_new * 40

    pool = synth.ReplayPool(dev, capacity=n + n_new)

    def restore():
        pool._coord[:n] = coord
        pool._label[:n] = label
        pool._weight[:n] = weight
        pool._set_size(n)

    restore()
    pool.add_frame(*new, origin, r)              # sizes the scratch
    lib = _abi.lib()

    def launch():
        desc = _abi.ShineSamplePool(pool._coord.data_ptr(), pool._label.data_ptr(), pool._weight.data_ptr(), n,
                                    pool.capacity)
        _abi.check(lib.shine_pool_window_append(C.byref(desc), _abi.ptr(new[0]), _abi.ptr(new[1]), _abi.ptr(new[2]), n_new,
                                                origin[0], origin[1], origin[2], r, _abi.ptr(pool._size_out),
                                                _abi.ptr(pool._scratch), pool._scratch.numel(), _abi.stream_ptr(dev)),
                   "shine_pool_window_append")

    for _ in range(3):
        restore(); launch()
    kernel_ms = time_events(launch, reps, restore)

    walls = []
    for _ in range(reps):
        restore()
        torch.cuda.synchronize()
        t = time.perf_counter()
        pool.add_frame(*new, origin, r)
        walls.append((time.perf_counter() - t) * 1e3)
    walls.sort()
    want = replay_pool_update(coord, label, weight, *new, origin, r)
    same = torch.equal(pool.coord_pool, want[0]) and torch.equal(pool.sdf_label_pool, want[1]) and \
        torch.equal(pool.weight_pool, want[2])
    del want
    oracle_ms = time_events(lambda: replay_pool_update(coord, label, weight, *new, origin, r), reps)
    return {"pool": n, "frame": n_new, "kept_fraction": float(mask.float().mean()), "moved": moved,
            "kernel_ms": kernel_ms, "add_frame_ms": walls[len(walls) // 2], "oracle_torch_ms": oracle_ms,
            "algorithmic_bytes": algo_bytes, "achieved_TBps": algo_bytes / (kernel_ms * 1e-3) / 1e12,
            "of_hbm_peak": algo_bytes / (kernel_ms * 1e-3) / HBM_PEAK, "equals_oracle": same}


def frame_breakdown(dev, n_frames, azimuth, step_m):
    from shine_mapping_b200 import Decoder, FeatureOctree, SdfTrainer, synth
    from shine_mapping_b200.config import SHINEConfig
    from shine_mapping_b200.incre_loop import run_shine_mapping_incremental
    # config/kitti/kitti_incre_replay.yaml
    cfg = SHINEConfig(tree_level_world=12, tree_level_feat=3, leaf_vox_size=0.3, device=dev, min_range=3.0,
                      pc_radius=30.0, surface_sample_range_m=0.3, surface_sample_n=3, free_sample_begin_ratio=0.3,
                      free_sample_end_dist_m=1.0, free_sample_n=3, continual_learning_reg=False, lambda_forget=0.0,
                      window_replay_on=True, window_radius=50.0, ekional_loss_on=True, weight_e=0.1, iters=100, bs=8192,
                      lr=0.01, weight_decay=0.0, freeze_after_frame=20)
    scans = synth.generate_scans(cfg, azimuth, n_frames, step_m, seed=3, device=dev)
    frames = [(c, l, w, torch.tensor([f * step_m, 0.0, 0.0]) * cfg.scale) for f, (c, l, w, _) in enumerate(scans)]
    torch.manual_seed(1)
    octree, decoder = FeatureOctree(cfg), Decoder(cfg)
    pool = synth.ReplayPool(dev)
    run_shine_mapping_incremental(cfg, octree, decoder, frames[:-1], pool=pool)
    coord, label, weight, origin = frames[-1]
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(4)]
    torch.cuda.synchronize()
    ev[0].record()
    octree.update(coord[weight > 0, :], incremental_on=False)
    ev[1].record()
    pool.add_frame(coord, label, weight, origin, cfg.window_radius * cfg.scale)
    ev[2].record()
    trainer = SdfTrainer(cfg, octree, decoder)
    trainer.zero_grad()
    ev[3].record()
    marks = []
    for _ in range(cfg.iters):
        e = [torch.cuda.Event(enable_timing=True) for _ in range(4)]
        e[0].record()
        c, l, w = pool.get_batch(cfg.bs)
        e[1].record()
        trainer.forward_backward_eikonal(c, l, w)
        e[2].record()
        trainer.optimizer_step(zero_grad=True)
        e[3].record()
        marks.append(e)
    torch.cuda.synchronize()
    get_batch = sum(e[0].elapsed_time(e[1]) for e in marks)
    step = sum(e[1].elapsed_time(e[2]) for e in marks)
    adam = sum(e[2].elapsed_time(e[3]) for e in marks)
    return {"frames_before": n_frames - 1, "pool": len(pool), "frame_samples": int(coord.shape[0]),
            "rows": [int(p.shape[0]) for p in octree.hier_features], "iters": cfg.iters, "bs": cfg.bs,
            "octree_update_ms": ev[0].elapsed_time(ev[1]), "add_frame_ms": ev[1].elapsed_time(ev[2]),
            "trainer_setup_ms": ev[2].elapsed_time(ev[3]), "get_batch_ms": get_batch, "step_ms": step, "adam_ms": adam,
            "adam_numel": int(trainer.flat_grad.numel())}


def main(argv=None):
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--sizes", type=int, nargs="+", default=[4_000_000, 16_000_000, 40_000_000])
    ap.add_argument("--frame", type=int, default=800_000)
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--drive-frames", type=int, default=24)
    ap.add_argument("--azimuth", type=int, default=2048)
    ap.add_argument("--out", default=None)
    args = ap.parse_args(argv)
    if not torch.cuda.is_available():
        raise SystemExit("replay_frame.py measures on the GPU and there is none")
    import __graft_entry__
    __graft_entry__.build()
    dev = "cuda:0"
    result = {"card": card(), "add_frame": [add_frame_costs(n, args.frame, args.reps, dev) for n in args.sizes],
              "frame_breakdown": frame_breakdown(dev, args.drive_frames, args.azimuth, 5.0)}
    line = json.dumps(result)
    print(line)
    if args.out:
        with open(args.out, "w") as fh:
            fh.write(line + "\n")


if __name__ == "__main__":
    main()
