"""Incremental mapping loop with the regularisation-based continual-learning term — the caller of the hot path for
BASELINE config 4, after reference shine_incre.py:86-194 and utils/incre_learning.py:8-40.

Per frame: the pool holds this frame's samples only, `octree.update(surface, incremental_on=True)` grows the map and
snapshots `features_last_frame` / extends `importance_weight`; the optimiser state is rebuilt (reference
shine_incre.py:108-109); `iters` x { get_batch -> fused fwd+loss(sum)+bwd -> + lambda_forget * d(reg)/d(features)
-> Adam }; then `cal_feature_importance` sweeps the frame's pool and accumulates |dL/dfeature| into the importance.
With `ekional_loss_on` (the reference's replay configs set it) the step is the fused BCE + eikonal launch instead
(shine_incre.py:159-165: + weight_e * mean over surface samples of (1 - |g|)^2).

The BCE part is the fused sm_90a step; the regulariser (model/feature_octree.py:246-255) and the importance update touch
only the rows the batch touched: `shine_mark_touched` collects them (bitmap + compact list, no unique()/sort) and
`shine_regularization_apply` / `shine_importance_accumulate` run over that list.

With `continual_learning_reg: False` the reference replays instead (the other half of its shipped incremental configs,
`*_incre_replay.yaml`): the pool keeps every earlier frame's samples, minus, with `window_replay_on`, those outside a
sliding window around the new sensor origin; pass a `synth.ReplayPool` as `pool`.

    python -m shine_mapping_b200.incre_loop config.yaml [--synthetic-azimuth N --frames F --frame-step-m S --iters I]

runs either mode, as the config selects it, on a synthetic drive along +x and prints the per-frame history.
"""
from __future__ import annotations

import ctypes as C
import os

import numpy as np
import torch

from . import _abi
from .config import SHINEConfig
from .decoder import Decoder
from .feature_octree import FeatureOctree
from .trainer import SdfTrainer


class TouchedRows:
    """Device scratch of the per-touched-row passes: one bitmap word per 32 rows and a compact row list per level
    (bottom-up like the C descriptors).  Rebuilt when `octree.update()` re-grows the tables."""

    def __init__(self, octree: FeatureOctree):
        dev = octree.hier_features[0].device
        L = octree.featured_level_num
        self.counts = torch.zeros(L, dtype=torch.int32, device=dev)
        self.bitmaps, self.rows = [], []
        self.desc = _abi.ShineTouched()
        self.rows_sig = tuple(int(p.shape[0]) for p in octree.hier_features)
        for i in range(L):
            k = L - i - 1
            n_rows = int(octree.hier_features[k].shape[0])
            bm = torch.zeros((n_rows + 31) // 32, dtype=torch.int32, device=dev)
            rl = torch.empty(n_rows, dtype=torch.int32, device=dev)
            self.bitmaps.append(bm); self.rows.append(rl)
            lv = self.desc.lv[i]
            lv.bitmap, lv.rows = bm.data_ptr(), rl.data_ptr()
            lv.count = self.counts.data_ptr() + 4 * i
            lv.capacity = n_rows

    @staticmethod
    def of(octree: FeatureOctree) -> "TouchedRows":
        t = getattr(octree, "_touched_rows", None)
        if t is None or t.rows_sig != tuple(int(p.shape[0]) for p in octree.hier_features) or \
                t.counts.device != octree.hier_features[0].device:
            t = TouchedRows(octree)
            octree._touched_rows = t
        return t


def _row_tables(octree: FeatureOctree, writable: bool) -> _abi.ShineRowTables:
    aux = _abi.ShineRowTables()
    L = octree.featured_level_num
    for i in range(L):
        k = L - i - 1
        aux.last[i] = octree.features_last_frame[k].data_ptr()
        aux.importance[i] = octree.importance_weight[k].data_ptr()
        aux.importance_rw[i] = octree.importance_weight[k].data_ptr() if writable else None
    return aux


def add_regularization(trainer: SdfTrainer, octree: FeatureOctree, lambda_forget: float, coord=None) -> torch.Tensor:
    """reg = cal_regularization() over the rows touched by the last batch (model/feature_octree.py:246-255) and
    grads += 2 lambda Omega (f - f_last) on those rows — two launches (mark, apply), no unique()/sort, nothing dense."""
    coord = octree._last_coord if coord is None else coord
    if coord is None:
        raise _abi.ShineB200Error("add_regularization needs the batch of the last step (octree._last_coord)")
    dev = trainer.flat_grad.device
    t = TouchedRows.of(octree)
    od = octree._descriptor(None, trainer.table_grads)
    reg = torch.zeros((), device=dev)
    t.counts.zero_()
    lib, st = _abi.lib(), _abi.stream_ptr(dev)
    _abi.check(lib.shine_mark_touched(C.byref(od), _abi.ptr(coord), coord.shape[0], C.byref(t.desc), st),
               "shine_mark_touched")
    aux = _row_tables(octree, writable=False)
    _abi.check(lib.shine_regularization_apply(C.byref(od), C.byref(t.desc), C.byref(aux), 2.0 * lambda_forget,
                                              _abi.ptr(reg), 1, st), "shine_regularization_apply")
    return reg


@torch.no_grad()
def cal_feature_importance(trainer: SdfTrainer, octree: FeatureOctree, coord_pool, label_pool, bs: int, down_rate: int = 1):
    """utils/incre_learning.py:8-40 on the fused kernel: per pool stride, one unweighted step, then
    importance[u] += |dL/dfeature[u]| over the rows that stride touched (which also re-zeroes their gradients)."""
    n = coord_pool.shape[0]
    interval = bs * down_rate
    dev = trainer.flat_grad.device
    t = TouchedRows.of(octree)
    aux = _row_tables(octree, writable=True)
    lib, st = _abi.lib(), _abi.stream_ptr(dev)
    trainer.zero_grad()
    for head in range(0, n, interval):
        c = coord_pool[head:min(head + interval, n):down_rate].contiguous()
        l = label_pool[head:min(head + interval, n):down_rate].contiguous()
        trainer.forward_backward(c, l, weighted=False)     # utils/incre_learning.py:33: weight=None
        od = octree._descriptor(None, trainer.table_grads)
        t.counts.zero_()
        _abi.check(lib.shine_mark_touched(C.byref(od), _abi.ptr(c), c.shape[0], C.byref(t.desc), st), "shine_mark_touched")
        _abi.check(lib.shine_importance_accumulate(C.byref(od), C.byref(t.desc), C.byref(aux), 1, 1, st),
                   "shine_importance_accumulate")
    trainer.zero_grad()          # decoder segment + loss accumulator


def run_shine_mapping_incremental(config: SHINEConfig, octree: FeatureOctree, decoder: Decoder, frames, iters=None,
                                  log=None, pool=None, run_path=None, begin_pose_inv=None, map_bbx=None):
    """frames: iterable of (coord, sdf_label, weight) sample sets, one per scan (what `process_frame` leaves in the
    pools).  Returns per-frame dicts with first/last loss (and first/last eikonal mean with ekional_loss_on).

    pool: a `synth.ReplayPool` (or anything with its `add_frame` / `get_batch` / `len`) selects the reference's replay mode
    (`continual_learning_reg: False`, dataset/lidar_dataset.py:235-271): frames are then (coord, sdf_label, weight,
    origin_scaled), the pool keeps the earlier frames' samples, dropping with `window_replay_on` those `window_radius`
    metres or more from the new frame's origin, and batches are drawn from the whole pool.  The history also records
    the pool size.

    run_path: mesh the map to run_path/mesh/mesh_frame_{frame+1}.ply after the first frame and every mesh_freq_frame
    frames (shine_incre.py:198-211), octree or bbx mode as mc_with_octree selects, transformed by inv(begin_pose_inv).
    At those frames the map is also saved to run_path/model/model_frame_{frame+1}.pth (batch_loop.save_checkpoint), from
    which `load_model` continues a run, and with save_map the SDF map goes to run_path/map/sdf_map_frame_{frame+1}.ply.
    map_bbx: a function returning the map's (min, max) metres so far (`lambda: dataset.map_bbx` for real scans, the box
    of the frames' points as in the reference); without it, the box of the surface samples so far; the history entry of such a frame records the file under "mesh"."""
    if pool is not None and config.continual_learning_reg:
        raise ValueError("continual_learning_reg keeps the current frame's samples only; a replay pool is the other "
                         "incremental mode (dataset/lidar_dataset.py:223 vs :235): pass pool=None or turn the "
                         "regularisation off")
    if config.continual_learning_reg:
        config.loss_reduction = "sum"          # reference shine_incre.py:77-78
    iters = config.iters if iters is None else iters
    window = config.window_radius * config.scale if config.window_replay_on else None    # lidar_dataset.py:237-239
    dev = None
    history = []
    mesher, samples_bbx = None, None
    if run_path:
        from .mesher import Mesher
        mesher = Mesher(config, octree, decoder)
        if begin_pose_inv is not None:
            mesher.global_transform = np.linalg.inv(begin_pose_inv)
    for fid, frame in enumerate(frames):
        coord, label, weight = frame[:3]
        if fid == config.freeze_after_frame:   # reference shine_incre.py:97-101
            for child in decoder.children():
                for p in child.parameters():
                    p.requires_grad = False
        surface = coord[weight > 0, :]
        octree.update(surface, incremental_on=config.continual_learning_reg)        # lidar_dataset.py:212-218
        if pool is not None:
            pool.add_frame(coord, label, weight, frame[3], window)                  # lidar_dataset.py:235-271
        trainer = SdfTrainer(config, octree, decoder)                               # fresh Adam state per frame
        dev = trainer.flat_grad.device
        trainer.zero_grad()
        first = last = None
        n = coord.shape[0]
        for it in range(iters):
            if pool is not None:
                c, l, w = pool.get_batch(config.bs)                                 # lidar_dataset.py:431-448
            else:
                index = torch.randint(0, n, (config.bs,), device=dev)
                c, l, w = coord[index], label[index], weight[index]
            if config.ekional_loss_on:                                              # shine_incre.py:159-165
                loss, eik = trainer.forward_backward_eikonal(c, l, w)
                total = loss + config.weight_e * eik
            else:
                loss, eik = trainer.forward_backward(c, l, w), None
                total = loss.clone()
            if config.continual_learning_reg:
                total = total + config.lambda_forget * add_regularization(trainer, octree, config.lambda_forget, c)
            trainer.optimizer_step(zero_grad=True)
            if it == 0:
                first, bce_first = float(total), float(loss)
                eik_first = float(eik) if eik is not None else None
        last, bce_last = float(total), float(loss)
        eik_last = float(eik) if eik is not None else None
        if config.continual_learning_reg:
            cal_feature_importance(trainer, octree, coord, label, config.bs, config.cal_importance_weight_down_rate)
        history.append({"frame": fid, "loss_first": first, "loss_last": last, "bce_first": bce_first, "bce_last": bce_last,
                        "rows": [int(p.shape[0]) for p in octree.hier_features]})
        if pool is not None:
            history[-1]["pool"] = len(pool)
        if config.ekional_loss_on:
            history[-1].update(eik_first=eik_first, eik_last=eik_last)
        if mesher is not None:
            from .batch_loop import save_checkpoint
            from .mesher import reconstruct, sdf_map_path, surface_bbx
            samples_bbx = surface_bbx(coord, weight, config.scale, samples_bbx)
            if fid == 0 or (fid + 1) % config.mesh_freq_frame == 0:
                history[-1]["mesh"] = os.path.join(run_path, "mesh", f"mesh_frame_{fid + 1}.ply")
                reconstruct(config, mesher, history[-1]["mesh"], map_bbx() if map_bbx is not None else samples_bbx,
                            sdf_map_path(config, run_path, f"frame_{fid + 1}"))
                save_checkpoint(octree, decoder, trainer, run_path, f"model/model_frame_{fid + 1}", fid)
        if log:
            log(history[-1])
    return history


def main(argv=None):
    import argparse
    from . import synth
    from .batch_loop import check_supported
    from .checkpoint import apply_load_model
    ap = argparse.ArgumentParser(description="Incremental mapping on a synthetic drive along +x (regularisation or replay, "
                                             "as the config selects)")
    ap.add_argument("config")
    ap.add_argument("--synthetic-azimuth", type=int, default=1024)
    ap.add_argument("--frames", type=int, default=10)
    ap.add_argument("--frame-step-m", type=float, default=2.0)
    ap.add_argument("--iters", type=int, default=None)
    ap.add_argument("--scans", action="store_true",
                    help="map the sequence of the config's pc_path / pose_path / calib_path instead of the synthetic drive")
    ap.add_argument("--run-path", default=None, metavar="DIR",
                    help="write meshes (mesh/mesh_frame_*.ply), checkpoints (model/model_frame_*.pth) and, with save_map, "
                         "SDF maps (map/sdf_map_frame_*.ply) under DIR")
    args = ap.parse_args(argv)
    config = SHINEConfig()
    config.load(args.config)
    check_supported(config)
    torch.manual_seed(config.seed)
    octree, decoder = FeatureOctree(config), Decoder(config)
    octree = apply_load_model(config, octree, decoder)                          # shine_incre.py:44-54
    if config.continual_learning_reg and not octree.is_empty() and not octree.importance_weight:
        # a map saved in batch mode carries no regularisation state: begin it as the map's first frame would
        octree.importance_weight = [torch.zeros_like(p.data) for p in octree.hier_features]
        octree.features_last_frame = [p.data.clone() for p in octree.hier_features]
    dev = config.device
    # shine_incre.py:106: the regularisation mode keeps the current frame's samples only, the other mode replays
    pool = None if config.continual_learning_reg else synth.ReplayPool(dev)
    begin_pose_inv = map_bbx = None
    if args.scans:
        from .scans import LiDARDataset
        dataset = LiDARDataset(config)
        frames, begin_pose_inv = dataset.frames(), dataset.begin_pose_inv   # read and sampled one frame at a time
        map_bbx = lambda: dataset.map_bbx
    else:
        scans = synth.generate_scans(config, args.synthetic_azimuth, args.frames, args.frame_step_m, seed=config.seed,
                                     device=dev)
        frames = [(coord, label, weight, torch.tensor([f * args.frame_step_m, 0.0, 0.0]) * config.scale)
                  for f, (coord, label, weight, _) in enumerate(scans)]
    print("Begin mapping:", "replay" + (f" (window {config.window_radius} m)" if config.window_replay_on else "")
          if pool is not None else "regularisation")
    history = run_shine_mapping_incremental(config, octree, decoder, frames, iters=args.iters, log=print, pool=pool,
                                            run_path=args.run_path, begin_pose_inv=begin_pose_inv, map_bbx=map_bbx)
    octree.print_detail()
    return history


if __name__ == "__main__":
    main()
