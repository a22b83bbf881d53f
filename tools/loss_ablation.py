"""The reference README's loss comparison (tip 1: sdf_bce against sdf_l1 / sdf_l2) on the synthetic street.

    python tools/loss_ablation.py [--iters 1000] [--bs 8192] [--repeats 3]

For each main_loss_type in (sdf_bce, sdf_l1, sdf_l2), without and with the eikonal term, `repeats` runs (seeds 0, 1, ...)
on the same map with the same iteration count: train with the batch loop, mesh the map with the `Mesher` over its
bounding box, evaluate the mesh with `evaluate.eval_mesh` against the street's ground-truth surface at the reference's
MaiCity settings.  The iteration time is measured after that, on the trained map: one loop iteration (batch draw + fused
step + Adam) captured as a CUDA graph and replayed 200 times between two CUDA events.  One JSON line per run, then one
line per configuration with the medians and the min / max of the runs.  Needs a GPU.
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from shine_mapping_b200 import Decoder, FeatureOctree, Mesher, synth  # noqa: E402
from shine_mapping_b200.batch_loop import _GraphedIteration, run_shine_mapping_batch  # noqa: E402
from shine_mapping_b200.config import SHINEConfig  # noqa: E402
from shine_mapping_b200.evaluate import eval_mesh  # noqa: E402
from shine_mapping_b200.trainer import SdfTrainer  # noqa: E402

# the reference's MaiCity evaluation (eval/evaluator.py): 10^7 mesh samples, 2 cm voxels, 10 cm threshold, 0.2 m / 2 m
MAICITY = dict(down_sample_res=0.02, threshold=0.1, truncation_acc=0.2, truncation_com=2.0, gt_bbx_mask_on=True,
               mesh_sample_point=10_000_000, seed=11)


def iteration_ms(cfg, octree, dec, pool, replays: int = 200) -> float:
    """Mean time of one graph-replayed loop iteration (batch draw + fused step + Adam), CUDA events around `replays`
    back-to-back replays after the capture."""
    step = _GraphedIteration(SdfTrainer(cfg, octree, dec), pool, cfg.bs)
    step.run()                                     # warm-up + capture
    for _ in range(5):
        step.run()
    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    start.record()
    for _ in range(replays):
        step.run()
    end.record()
    torch.cuda.synchronize()
    return start.elapsed_time(end) / replays


def run(loss_type: str, eikonal: bool, iters: int, bs: int, seed: int = 0) -> dict:
    dev = "cuda:0"
    cfg = SHINEConfig(tree_level_world=12, tree_level_feat=3, leaf_vox_size=0.3, device=dev, bs=bs, iters=iters,
                      mc_res_m=0.1, surface_sample_range_m=0.3, free_sample_end_dist_m=1.0, min_range=2.0, pc_radius=25.0,
                      main_loss_type=loss_type, ekional_loss_on=eikonal, weight_e=0.1)
    torch.manual_seed(seed)
    octree, dec = FeatureOctree(cfg), Decoder(cfg)
    pool = synth.build_scene_map(cfg, octree, 512, 10, frame_step_m=1.0, seed=3)
    out = run_shine_mapping_batch(cfg, octree, dec, pool, iters=iters)
    verts, faces, _ = Mesher(cfg, octree, dec).recon_bbx_mesh(pool.map_bbx[0], pool.map_bbx[1], cfg.mc_res_m)
    gt = synth.scene_surface_points(-10.0, 20.0, 0.1).to(dev)
    metrics = eval_mesh((verts, faces), gt, device=dev, **MAICITY)
    return {"main_loss_type": loss_type, "ekional_loss_on": eikonal, "seed": seed, "iters": iters, "bs": bs,
            "loss_first": out["loss_first"], "loss_last": out["loss_last"], "triangles": int(faces.shape[0]),
            **{k: round(float(v), 4) for k, v in metrics.items()}, "ms_per_iter": iteration_ms(cfg, octree, dec, pool)}


SUMMARY_KEYS = ("ms_per_iter", "F-score (%)", "Precision [Accuracy] (%)", "Recall [Completeness] (%)", "Chamfer_L1 (m)")


def main(argv=None) -> int:
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--iters", type=int, default=1000)
    ap.add_argument("--bs", type=int, default=8192)
    ap.add_argument("--repeats", type=int, default=3)
    args = ap.parse_args(argv)
    if not torch.cuda.is_available():
        sys.exit("loss_ablation needs a GPU")
    for eikonal in (False, True):
        for loss_type in ("sdf_bce", "sdf_l1", "sdf_l2"):
            runs = [run(loss_type, eikonal, args.iters, args.bs, seed) for seed in range(args.repeats)]
            for r in runs:
                print(json.dumps(r), flush=True)
            summary = {"summary": True, "main_loss_type": loss_type, "ekional_loss_on": eikonal, "runs": len(runs)}
            for k in SUMMARY_KEYS:
                v = [r[k] for r in runs]
                summary[k] = {"median": statistics.median(v), "min": min(v), "max": max(v)}
            print(json.dumps(summary), flush=True)
    return 0


if __name__ == "__main__":
    sys.exit(main())
