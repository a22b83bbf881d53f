"""Shared scaffolding of the spatial-partition tests: one global scene, its single-process reference step, and the
per-rank pieces (partition of the pool and of a fixed global batch, features copied from the global tables by corner
key so that duplicates start identical)."""
from __future__ import annotations

import numpy as np
import torch

from tests.parity_utils import DEC_KEYS, make_config, orc


def global_scene(levels=3, n_azimuth=96, n_frames=3, n_batch=6000, seed=3, frame_step_m=6.0):
    """CPU tensors: the whole pool (several scans), one global batch drawn from it, a decoder."""
    from shine_mapping_b200 import synth
    cfg = make_config(levels, device="cpu", pc_radius=30.0)
    frames = synth.generate_scans(cfg, n_azimuth, n_frames, frame_step_m, seed, "cpu")
    coord = torch.cat([f[0] for f in frames]); label = torch.cat([f[1] for f in frames])
    weight = torch.cat([f[2] for f in frames])
    gen = torch.Generator().manual_seed(seed)
    idx = torch.randint(0, coord.shape[0], (n_batch,), generator=gen)
    torch.manual_seed(seed)
    dec = orc.make_decoder_params(cfg.feature_dim, 32, 2, True)
    return cfg, (coord, label, weight), (coord[idx].contiguous(), label[idx].contiguous()), dec


def global_oracle_step(cfg, pool, batch, dec):
    """Single-process reference: oracle octree over ALL surface samples, mean-reduced step on the global batch.
    -> (oracle octree, key->row dicts per level (coarse->fine), result dict)."""
    coord, label, weight = pool
    o = orc.OracleOctree(cfg.tree_level_world, cfg.tree_level_feat, cfg.feature_dim, cfg.feature_std, cfg.poly_int_on)
    torch.manual_seed(11)
    o.update(coord[weight > 0])
    d = {k: v.detach().clone().requires_grad_(True) for k, v in dec.items()}
    res = orc.train_step(o, d, batch[0], batch[1], None, float(cfg.sigma_sigmoid), False, "mean")
    key_to_row = [o.corners_lookup_tables[o.free_level_num + k] for k in range(o.featured_level_num)]
    return o, key_to_row, res


def global_case(cfg, o, batch, dec):
    """The global batch as a case of tests/parity_utils (the oracle octree `o` reused, unweighted, mean), for the fp64
    reference `tests.test_gpu_replicas.Ref` and the bound of tests/boundary_oracle.py."""
    n = batch[0].shape[0]
    return {"cfg": dict(tree_level_world=cfg.tree_level_world, tree_level_feat=cfg.tree_level_feat,
                        feature_dim=cfg.feature_dim, poly_int_on=cfg.poly_int_on, leaf_vox_size=cfg.leaf_vox_size,
                        sigma=float(cfg.sigma_sigmoid), weighted=False, reduction="mean", bias=True),
            "frames": [], "oracle": o, "tables": [t.detach().numpy().copy() for t in o.hier_features],
            "dec": {k: v.detach().numpy().copy() for k, v in dec.items()},
            "coord": batch[0].numpy().copy(), "label": batch[1].numpy().copy(), "weight": np.ones(n, dtype=np.float32)}


def rows_in_global(corner_keys: torch.Tensor, key_to_row: dict) -> np.ndarray:
    return np.array([key_to_row[int(k)] for k in corner_keys.tolist()], dtype=np.int64)


def check_rank_against_global(local_grads, corner_keys_per_level, key_to_row, global_res, grad_rel=2e-4):
    """Every local row's gradient (after the boundary exchange) == the global gradient of the same corner."""
    worst = 0.0
    for lvl, (g_loc, keys) in enumerate(zip(local_grads, corner_keys_per_level)):
        g_glob = global_res["table_grads"][lvl].numpy()
        rows = rows_in_global(keys, key_to_row[lvl])
        want = g_glob[rows]
        got = np.asarray(g_loc)[:-1]
        scale = max(float(np.abs(g_glob).max()), 1e-30)
        err = float(np.abs(got - want).max()) / scale if got.size else 0.0
        worst = max(worst, err)
        assert err <= grad_rel, f"level {lvl}: local vs global table gradient rel err {err:.3e}"
    return worst
