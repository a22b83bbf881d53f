"""Batch-mode mapping loop — the caller side of the hot path, after reference shine_batch.py:23-233.

    python -m shine_mapping_b200.batch_loop config.yaml [--synthetic-azimuth 2048 --frames 10]

Same sequence as the reference loop (T-points of shine_batch.py:107-212 kept as timing keys): build the octree
from all frames, set up the optimiser, then `iters` x { lr decay -> get_batch -> fwd+loss+bwd -> optimiser },
checkpoint in the reference's format.  What differs: the body of an iteration is TWO launches (the fused
`shine_sdf_step` kernel and the multi-tensor Adam kernel, which also re-zeroes the gradients) instead of
~300, and there is no host round trip inside the loop (loss is read back only when logging).
`main_loss_type` is the reference's point-wise menu (shine_batch.py:171-179): sdf_bce, or sdf_l1 / sdf_l2
(`sdf_diff_loss`), the loss bit of the same fused `shine_sdf_step`, each with or without the eikonal term.

Out of scope here (SURVEY.md §2): dataset I/O (open3d), meshing, visualiser, wandb.  `pool` is anything with the
`get_batch(bs)` contract of LiDARDataset (dataset/lidar_dataset.py:431-448); `synth.build_scene_map` provides one.
`ekional_loss_on` is one fused kernel (`shine_sdf_eikonal_step`; the class surface
supports the reference's autograd recipe too: query_feature is differentiable w.r.t. the coordinates, twice); normal /
consistency / semantic / ray losses are rejected explicitly.
"""
from __future__ import annotations

import os
import sys
import time

import numpy as np
import torch

from .config import SHINEConfig
from .decoder import Decoder
from .feature_octree import FeatureOctree
from .trainer import SdfTrainer


BATCH_LOSSES = ("sdf_bce", "sdf_l1", "sdf_l2")


def check_supported(config: SHINEConfig, main_losses=BATCH_LOSSES) -> None:
    """Raise NotImplementedError for a config this package cannot train.  main_losses: the main_loss_type values the
    calling loop trains (the batch loop: BATCH_LOSSES; the incremental loop only sdf_bce)."""
    unsupported = [k for k in ("normal_loss_on", "consistency_loss_on", "proj_correction_on",
                               "semantic_on", "time_conditioned", "ray_loss") if getattr(config, k)]
    if unsupported or config.main_loss_type not in main_losses:
        raise NotImplementedError(f"implemented: main_loss_type={'/'.join(main_losses)} (+ ekional_loss_on); "
                                  f"not {unsupported or config.main_loss_type}")
    if not config.opt_adam:
        raise NotImplementedError("only Adam (reference utils/tools.py:78-79) is implemented")


def step_lr_decay(trainer: SdfTrainer, base_lr: float, iteration: int, steps, ratio: float) -> None:
    """Step decay of reference utils/tools.py:135-155: lr = base * ratio^(number of milestones passed)."""
    passed = sum(1 for s in steps if iteration >= s)
    trainer.lr = base_lr * (ratio ** passed)


def save_checkpoint(octree, decoder, trainer, run_path, name, iters):
    """Same dict layout as reference utils/tools.py:200-213 (whole octree module pickled, decoder state_dict)."""
    os.makedirs(os.path.join(run_path, "model"), exist_ok=True)
    torch.save({"iters": iters, "feature_octree": octree, "geo_decoder": decoder.state_dict(),
                "optimizer": {"exp_avg": trainer.exp_avg, "exp_avg_sq": trainer.exp_avg_sq,
                              "step": trainer.step_count}},
               os.path.join(run_path, f"{name}.pth"))


def eikonal_iteration_fused(config: SHINEConfig, trainer: SdfTrainer, coord, sdf_label, weight, grad_out=None):
    """Loop body with ekional_loss_on (reference shine_batch.py:119-120,137-142,172-185,208-209) as one fused launch
    (`SdfTrainer.forward_backward_eikonal`).  -> (total loss, eikonal mean) device scalars."""
    bce, eik = trainer.forward_backward_eikonal(coord, sdf_label, weight, grad_out=grad_out)
    return bce + config.weight_e * eik, eik


def eikonal_iteration(config: SHINEConfig, octree: FeatureOctree, decoder: Decoder, trainer: SdfTrainer, coord, sdf_label,
                      weight):
    """The same loop body on the CLASS surface, call for call like the reference (kept as the drop-in path and as the
    cross-check of the fused kernel):
    `query_feature` is differentiable w.r.t. the coordinates (shine_query_coord_grad) and that gradient is itself
    differentiable (tangent kernels), so the reference's get_gradient(create_graph=True) recipe works as is.  Gradients
    accumulate into the trainer's flat buffer (param.grad are views of it)."""
    from .loss import sdf_bce_loss, sdf_diff_loss
    sigma = config.sigma_sigmoid
    coord = coord.detach().requires_grad_(True)
    feature = octree.query_feature(coord)
    pred = decoder.sdf(feature)
    g = torch.autograd.grad(pred, coord, torch.ones_like(pred), create_graph=True, retain_graph=True)[0] * sigma
    surface_mask = weight > 0
    if config.main_loss_type == "sdf_bce":
        loss = sdf_bce_loss(pred, sdf_label, sigma, torch.abs(weight), config.loss_weight_on, config.loss_reduction)
    else:                                                                         # shine_batch.py:176-179
        loss = sdf_diff_loss(pred, sdf_label, torch.abs(weight), config.scale, l2_loss=config.main_loss_type == "sdf_l2")
    eikonal = ((1.0 - g[surface_mask].norm(2, dim=-1)) ** 2).mean()
    total = loss + config.weight_e * eikonal
    total.backward()
    trainer.loss.copy_(total.detach())
    return total.detach(), eikonal.detach(), g.detach()


class _GraphedIteration:
    """One loop iteration {get_batch -> fused fwd+loss+bwd -> Adam(+zero grads)} captured as a CUDA graph: at
    bs=4096 the iteration is launch-latency bound (5 small kernels), replaying a graph removes the host from the
    loop.  Adam's step number lives on the device (`shine_adam_step_dev`); the graph is re-captured when the
    learning rate changes (lr is a kernel parameter)."""

    def __init__(self, trainer: SdfTrainer, pool, bs: int):
        self.trainer, self.pool, self.bs = trainer, pool, bs
        self.graph, self.lr = None, None

    def _body(self):
        # the eikonal kernel scatters per point: it wants the order drawn (Morton order = same-row atomics within a warp)
        eik = self.trainer.config.ekional_loss_on
        kw = {"ordered": False} if (eik and getattr(self.pool, "ordered", False)) else {}
        coord, sdf_label, weight = self.pool.get_batch(self.bs, **kw)
        if eik:
            self.trainer.forward_backward_eikonal(coord, sdf_label, weight)
        else:
            self.trainer.forward_backward(coord, sdf_label, weight, morton_ordered=getattr(self.pool, "ordered", False))
        self.trainer.optimizer_step(zero_grad=True, device_step=True)

    def run(self):
        tr = self.trainer
        if self.graph is None or self.lr != tr.lr:
            dev = tr.flat_grad.device
            side = torch.cuda.Stream(device=dev)
            side.wait_stream(torch.cuda.current_stream(dev))
            with torch.cuda.stream(side):     # warm-up outside capture (lazy inits, allocator)
                self._body()
            torch.cuda.current_stream(dev).wait_stream(side)
            torch.cuda.synchronize(dev)
            self.graph = torch.cuda.CUDAGraph()
            with torch.cuda.graph(self.graph):
                self._body()
            self.lr = tr.lr
            return        # the warm-up call above did this iteration's work; capturing does not execute anything
        tr._replay_with_adam(self.graph)


def run_shine_mapping_batch(config: SHINEConfig, octree: FeatureOctree, decoder: Decoder, pool, iters=None,
                            log_every: int = 0, run_path: str | None = None, process_group=None,
                            shard_mode: str = "replicated", use_cuda_graph: bool | None = None, map_bbx=None,
                            begin_pose_inv=None):
    """-> dict(loss_first, loss_last, points_per_s, timing, meshes).  `octree` must already hold the map of `pool`.
    With run_path, every vis_freq_iters iterations the map is meshed to run_path/mesh/mesh_iter_{it+1}.ply
    (shine_batch.py:236-245): octree or bbx mode (map_bbx, metres) as mc_with_octree selects, transformed by
    inv(begin_pose_inv), and with save_map the SDF map to run_path/map/sdf_map_iter_{it+1}.ply.  `meshes` lists the mesh
    files written."""
    check_supported(config)
    mesher = None
    if run_path:
        from .mesher import Mesher
        mesher = Mesher(config, octree, decoder)
        if begin_pose_inv is not None:
            mesher.global_transform = np.linalg.inv(begin_pose_inv)
    meshes = []
    dev = octree.hier_features[0].device
    trainer = SdfTrainer(config, octree, decoder, process_group=process_group, shard_mode=shard_mode)
    world = torch.distributed.get_world_size(process_group) if torch.distributed.is_initialized() else 1
    iters = config.iters if iters is None else iters
    if use_cuda_graph is None:
        use_cuda_graph = world == 1
    graphed = _GraphedIteration(trainer, pool, config.bs) if (use_cuda_graph and world == 1) else None
    trainer.zero_grad()
    losses = {}
    timing = {"load": 0.0, "step": 0.0}
    t_begin = None
    for it in range(iters):
        if it == min(3, iters - 1):       # skip warm-up iterations in the throughput figure
            torch.cuda.synchronize(dev); t_begin = time.perf_counter(); it_begin = it
        step_lr_decay(trainer, config.lr, it, config.lr_decay_step, config.lr_iters_reduce_ratio)
        if graphed is not None:
            graphed.run()
        elif config.ekional_loss_on:
            coord, sdf_label, weight = pool.get_batch(config.bs, **({"ordered": False} if getattr(pool, "ordered", False) else {}))
            trainer.forward_backward_eikonal(coord, sdf_label, weight, n_norm=config.bs * world)
            trainer.all_reduce_grads()
            trainer.optimizer_step(zero_grad=True)
        else:
            coord, sdf_label, weight = pool.get_batch(config.bs)                       # shine_batch.py:115
            trainer.forward_backward(coord, sdf_label, weight, n_norm=config.bs * world,   # :123-209
                                     morton_ordered=getattr(pool, "ordered", False))
            trainer.all_reduce_grads()
            trainer.optimizer_step(zero_grad=True)                                      # :208-210
        if it == 0 or it == iters - 1 or (log_every and it % log_every == 0):
            losses[it] = float(trainer.loss)          # the only host read-back
        if run_path and ((it + 1) % config.save_freq_iters == 0) and it > 0:
            save_checkpoint(octree, decoder, trainer, run_path, f"model/model_iter_{it + 1}", it)
        if mesher is not None and ((it + 1) % config.vis_freq_iters == 0) and it > 0:     # between graph replays
            from .mesher import reconstruct, sdf_map_path
            meshes.append(os.path.join(run_path, "mesh", f"mesh_iter_{it + 1}.ply"))
            reconstruct(config, mesher, meshes[-1], map_bbx, sdf_map_path(config, run_path, f"iter_{it + 1}"))
    torch.cuda.synchronize(dev)
    elapsed = time.perf_counter() - t_begin if t_begin is not None else float("nan")
    done = iters - it_begin if t_begin is not None else 0
    return {"loss_first": losses.get(0), "loss_last": losses.get(iters - 1), "losses": losses,
            "iters_per_s": done / elapsed if done else None,
            "points_per_s": done * config.bs * world / elapsed if done else None, "timing": timing,
            "meshes": meshes}


def main(argv=None):
    import argparse
    from . import rgbd, synth
    from .checkpoint import apply_load_model
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("config")
    ap.add_argument("--synthetic-azimuth", type=int, default=2048)
    ap.add_argument("--frames", type=int, default=10)
    ap.add_argument("--iters", type=int, default=None)
    ap.add_argument("--scans", action="store_true",
                    help="map the sequence of the config's pc_path / pose_path / calib_path instead of synthetic scans")
    ap.add_argument("--run-path", default=None, metavar="DIR",
                    help="write checkpoints (model/), meshes (mesh/mesh_iter_*.ply) and, with save_map, SDF maps "
                         "(map/sdf_map_iter_*.ply) under DIR")
    rgbd.add_loop_arguments(ap)
    args = ap.parse_args(argv)
    rgbd.check_loop_arguments(ap, args)
    config = SHINEConfig()
    config.load(args.config)
    torch.manual_seed(config.seed)
    octree, decoder = FeatureOctree(config), Decoder(config)
    octree = apply_load_model(config, octree, decoder)                             # shine_batch.py:45-55
    if args.scans or args.rgbd:
        from .scans import LiDARDataset
        print(f"Load, preprocess and sample data ({args.rgbd or config.pc_path})")
        if args.rgbd:
            dataset = rgbd.dataset_from_args(config, args, octree)
        else:
            dataset = LiDARDataset(config, octree)                                  # shine_batch.py:58-76
        for frame_id in dataset.used_frames:
            dataset.process_frame(frame_id)
        pool = dataset.pool
        map_bbx, begin_pose_inv = dataset.map_bbx, dataset.begin_pose_inv
    else:
        print("Load, preprocess and sample data (synthetic scans)")
        # more than pc_count_gpu_limit scans: the pool lives in pinned host memory (dataset/lidar_dataset.py:94-101)
        pool = synth.build_scene_map(config, octree, args.synthetic_azimuth, args.frames, seed=config.seed, pool="auto")
        map_bbx, begin_pose_inv = pool.map_bbx, None
    where = "pinned host memory" if isinstance(pool, synth.HostSamplePool) else "device memory"
    print(f"Sample pool: {type(pool).__name__} in {where}, {len(pool)} samples")
    octree.print_detail()
    print("Begin mapping")
    out = run_shine_mapping_batch(config, octree, decoder, pool, iters=args.iters, log_every=1000, run_path=args.run_path,
                                  map_bbx=map_bbx, begin_pose_inv=begin_pose_inv)
    print({k: v for k, v in out.items() if k != "losses"})


if __name__ == "__main__":
    sys.exit(main())
