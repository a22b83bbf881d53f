"""Mint tests/golden/ref_checkpoint_l3.pt / .npz: a checkpoint as the UNMODIFIED reference writes it.
*** TEST INFRASTRUCTURE ***

Same conventions as oracle/make_golden.py (whose `import_reference` / `reference_config` this uses): runs only where the
reference checkout is available, on the CPU, with oracle/kaolin_shim in place of kaolin.  The reference's own
`FeatureOctree` grows over two `update()` calls on a seeded cloud, and the dict of utils/tools.py:203-210 (the octree module,
both decoders' state dicts, an Adam state dict after one step) is written with `torch.save`: the file names the class
`model.feature_octree.FeatureOctree` and holds data only.  Beside it an .npz keeps, for 2 000 query points, the reference's
`hierarchical_indices`, `query_feature` and `Decoder.sdf`, and the keys of the lookup dicts in order.

    python oracle/make_checkpoint_golden.py
"""
from __future__ import annotations

import json
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from make_golden import REF, ROOT, import_reference, reference_config  # noqa: E402

NAME = "ref_checkpoint_l3"
FEAT_LEVELS, LEAF_VOX, SEED, N_QUERY = 3, 0.2, 47, 2000


def make(name=NAME):
    SHINEConfig, FeatureOctree, Decoder, _, sdf_bce_loss = import_reference()
    torch.manual_seed(SEED)
    cfg = reference_config(SHINEConfig, FEAT_LEVELS, LEAF_VOX, True, False, "mean")
    octree, geo, sem = FeatureOctree(cfg), Decoder(cfg), Decoder(cfg, is_geo_encoder=False)
    # two overlapping patches of a wavy surface, metres -> the [-1, 1] cube
    frames = []
    for f in range(2):
        xy = torch.rand(300, 2) * 4.0 + torch.tensor([2.0 * f - 3.0, -2.0])
        z = 0.4 * torch.sin(xy[:, :1]) + 0.3 * torch.cos(1.7 * xy[:, 1:])
        frames.append(torch.cat((xy, z), 1) * cfg.scale)
        octree.update(frames[-1], True)                    # incremental_on: importance / last-frame tables are saved too
    # utils/tools.py:57-79 (restated: utils/tools.py imports open3d), one step so that the state dict holds moments
    groups = [{"params": list(geo.parameters()), "lr": cfg.lr, "weight_decay": cfg.weight_decay}]
    groups += [{"params": octree.hier_features[cfg.tree_level_feat - i - 1], "lr": cfg.lr} for i in range(cfg.tree_level_feat)]
    opt = torch.optim.Adam(groups, betas=(0.9, 0.99), eps=cfg.adam_eps)
    surface = torch.cat(frames)
    coord = surface[torch.randint(0, surface.shape[0], (N_QUERY,))] + 0.15 * LEAF_VOX * cfg.scale * torch.randn(N_QUERY, 3)
    coord[-50:] = torch.rand(50, 3) * 2.0 - 1.0            # misses
    sigma = cfg.logistic_gaussian_ratio * cfg.sigma_sigmoid_m * cfg.scale
    loss = sdf_bce_loss(geo.sdf(octree.query_feature(coord)), torch.zeros(N_QUERY), sigma, None, False, "mean")
    loss.backward()
    opt.step()
    opt.zero_grad(set_to_none=True)
    octree.set_zero()
    with torch.no_grad():
        feature = octree.query_feature(coord)
        pred = geo.sdf(feature)
    indices = [i.numpy().astype(np.int32) for i in octree.hierarchical_indices]
    octree.hierarchical_indices = []                       # temporaries of the last batch (clear_temp keeps the rest)
    gold = os.path.join(ROOT, "tests", "golden")
    # utils/tools.py:203-210
    torch.save({"iters": 1, "feature_octree": octree, "geo_decoder": geo.state_dict(), "sem_decoder": sem.state_dict(),
                "optimizer": opt.state_dict()}, os.path.join(gold, name + ".pt"))
    out = {"cfg_json": np.array(json.dumps(dict(tree_level_world=cfg.tree_level_world, tree_level_feat=FEAT_LEVELS,
                                                 feature_dim=cfg.feature_dim, poly_int_on=True, leaf_vox_size=LEAF_VOX))),
           "coord": coord.numpy(), "exp_feature": feature.numpy(), "exp_pred": pred.numpy()}
    for i, idx in enumerate(indices):
        out[f"exp_indices_{i}"] = idx
    for lvl in range(cfg.tree_level_world + 1):
        if octree.nodes_lookup_tables[lvl]:
            out[f"node_keys_{lvl}"] = np.array(list(octree.nodes_lookup_tables[lvl].keys()), dtype=np.int64)
            out[f"node_ids_{lvl}"] = np.array(list(octree.nodes_lookup_tables[lvl].values()), dtype=np.int32)
            out[f"corner_keys_{lvl}"] = np.array(list(octree.corners_lookup_tables[lvl].keys()), dtype=np.int64)
            out[f"corner_rows_{lvl}"] = np.array(list(octree.corners_lookup_tables[lvl].values()), dtype=np.int64)
    for k, p in enumerate(octree.hier_features):
        out[f"table_{k}"] = p.detach().numpy()
    np.savez_compressed(os.path.join(gold, name + ".npz"), **out)
    sizes = {e: os.path.getsize(os.path.join(gold, name + e)) for e in (".pt", ".npz")}
    print(f"{name}: rows={[p.shape[0] for p in octree.hier_features]} misses={int((indices[0][:, 0] < 0).sum())} "
          f"loss={float(loss.detach()):.6f} -> {sizes}")


if __name__ == "__main__":
    if not os.path.isdir(REF):
        sys.exit(f"{REF} not found: goldens can only be minted where the reference is mounted")
    make()
