"""Time mesh evaluation on the GPU: surface sampling, both voxel down-samplings, both tree builds and both query
directions, with CUDA events, against scipy's cKDTree on the same point sets on the CPU.

    python tools/eval_bench.py [--iters 300] [--reps 5] [--samples 10000000]

Workload: the 20-frame synthetic street of tools/mesh_bench.py, trained for --iters iterations and meshed in bbx mode at
mc_res_m 0.1, against `synth.scene_surface_points` at 2 cm over the map's x range, with the reference's MaiCity settings
(eval/evaluator.py: 0.02 m voxels, 0.1 m threshold, truncation 0.2 m / 2.0 m, the ground truth's box as crop).  One
warm-up, then --reps timed runs; medians are reported.  Prints one JSON line for the GPU phases (with the metrics) and one
for the CPU reference, each with the card's name and power limit read in the same run.  Writes nothing.
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

SETTINGS = dict(down_sample_res=0.02, threshold=0.1, truncation_acc=0.2, truncation_com=2.0)


def time_eval(verts, faces, gt, samples_n, seed=42):
    """One evaluation with events around every phase -> (ms per phase, point counts, metrics)."""
    from shine_mapping_b200.evaluate import NearestNeighbours, assemble_metrics, sample_mesh, voxel_down
    s = SETTINGS
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(8)]
    ev[0].record()
    widen = torch.tensor([0.0, 0.0, s["down_sample_res"]], dtype=torch.float64, device=gt.device)
    box = torch.cat((gt.amin(0) - widen, gt.amax(0) + widen))
    samples = sample_mesh(verts, faces, samples_n, seed, box)
    ev[1].record()
    pred = voxel_down(samples, s["down_sample_res"])
    ev[2].record()
    gtd = voxel_down(gt, s["down_sample_res"])
    ev[3].record()
    tree_gt = NearestNeighbours(gtd)
    ev[4].record()
    dist_p, _ = tree_gt.query(pred, s["truncation_acc"])
    ev[5].record()
    tree_pred = NearestNeighbours(pred)
    ev[6].record()
    dist_r, _ = tree_pred.query(gtd, s["truncation_com"])
    ev[7].record()
    torch.cuda.synchronize()
    names = ["sample_ms", "down_pred_ms", "down_gt_ms", "build_gt_ms", "query_acc_ms", "build_pred_ms", "query_com_ms"]
    ms = {k: ev[i].elapsed_time(ev[i + 1]) for i, k in enumerate(names)}
    ms["total_ms"] = ev[0].elapsed_time(ev[7])
    counts = {"samples": int(samples.shape[0]), "pred_down": int(pred.shape[0]), "gt_down": int(gtd.shape[0])}
    metrics = assemble_metrics(dist_p, dist_r, s["down_sample_res"], s["threshold"], s["truncation_acc"],
                               s["truncation_com"])
    return ms, counts, metrics, (pred, gtd)


def main():
    from bench import device_info
    from mesh_bench import street_workload
    from shine_mapping_b200 import Mesher, synth
    from shine_mapping_b200.batch_loop import run_shine_mapping_batch
    from shine_mapping_b200.evaluate import load_mesh
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--iters", type=int, default=300)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--samples", type=int, default=10_000_000)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("eval_bench.py times the sm_90a kernels: it needs a GPU")
    dev = torch.device("cuda:0")
    card = device_info(0)
    cfg, octree, decoder, pool = street_workload(dev)
    cfg.mc_res_m = 0.1
    run_shine_mapping_batch(cfg, octree, decoder, pool, iters=args.iters)
    lo, hi = pool.map_bbx
    verts, faces, _ = Mesher(cfg, octree, decoder).recon_bbx_mesh(lo, hi, cfg.mc_res_m)
    verts, faces = load_mesh((verts, faces), dev)
    gt = synth.scene_surface_points(float(lo[0]), float(hi[0]), 0.02).to(dev)
    time_eval(verts, faces, gt, args.samples)                                     # warm-up
    runs = [time_eval(verts, faces, gt, args.samples) for _ in range(args.reps)]
    med = {k: statistics.median(r[0][k] for r in runs) for k in runs[0][0]}
    _, counts, metrics, (pred, gtd) = runs[-1]
    same = all(list(r[2].values()) == list(metrics.values()) for r in runs)
    print(json.dumps({"workload": "street_20_frames", "phase": "gpu", "train_iters": args.iters, "mc_res_m": cfg.mc_res_m,
                      "mesh_verts": int(verts.shape[0]), "mesh_tris": int(faces.shape[0]), "gt_points": int(gt.shape[0]),
                      **counts, **med, "reps": args.reps, "stat": "median of GPU event times",
                      "metrics_identical_across_reps": same, "metrics": metrics, "settings": SETTINGS, "device": card}))
    from scipy.spatial import cKDTree
    p, g = pred.cpu().numpy(), gtd.cpu().numpy()
    cpu = {}
    for name, ref, q in (("acc", g, p), ("com", p, g)):
        t0 = time.perf_counter()
        tree = cKDTree(ref)
        t1 = time.perf_counter()
        tree.query(q, k=1, workers=-1)
        t2 = time.perf_counter()
        cpu[f"build_{name}_ms"], cpu[f"query_{name}_ms"] = 1e3 * (t1 - t0), 1e3 * (t2 - t1)
    cpu["total_ms"] = sum(cpu.values())
    print(json.dumps({"workload": "street_20_frames", "phase": "cpu_ckdtree", **cpu, "threads": os.cpu_count(),
                      "pred_down": int(p.shape[0]), "gt_down": int(g.shape[0]), "stat": "one run, wall clock",
                      "device": card}))


if __name__ == "__main__":
    main()
