"""Freeze the reference's own `dataSampler.sample` (utils/data_sampler.py:18-139) into tests/golden/ref_sampler.npz.

    python tools/make_sampler_golden.py /path/to/SHINE_mapping

Runs the reference sampler on the CPU (kaolin through oracle/kaolin_shim), records the torch.rand draws it makes and
stores its inputs, those draws and its outputs.  The tests replay the draws through tests/scan_oracle.py and through the
sampling kernel."""
from __future__ import annotations

import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def main(ref: str) -> None:
    sys.path.insert(0, os.path.join(ROOT, "oracle", "kaolin_shim"))
    sys.path.insert(0, ref)
    from utils.config import SHINEConfig
    from utils.data_sampler import dataSampler
    cfg = SHINEConfig()
    cfg.device = "cpu"
    cfg.leaf_vox_size, cfg.tree_level_world = 0.2, 12
    cfg.surface_sample_n, cfg.free_sample_n = 3, 3
    cfg.scale = 1.0 / (cfg.leaf_vox_size * 2 ** (cfg.tree_level_world - 1))
    g = torch.Generator().manual_seed(5)
    R = 1000
    rng_dir = torch.randn(R, 3, generator=g)
    dist_m = torch.rand(R, 1, generator=g) * 45.0 + 2.0
    origin_m = torch.tensor([3.25, -1.5, 0.75], dtype=torch.float64)
    points = ((rng_dir / rng_dir.norm(dim=1, keepdim=True)) * dist_m).double() + origin_m
    points_s = torch.tensor((points * cfg.scale).numpy(), dtype=torch.float32)
    origin_s = torch.tensor((origin_m * cfg.scale).numpy(), dtype=torch.float32)
    draws = []
    real_rand = torch.rand

    def recording_rand(*args, **kw):
        out = real_rand(*args, **kw)
        draws.append(out.clone())
        return out

    torch.manual_seed(11)
    torch.rand = recording_rand
    try:
        coord, label, _, _, weight, _, _ = dataSampler(cfg).sample(points_s, origin_s, None, None)
    finally:
        torch.rand = real_rand
    assert [tuple(d.shape) for d in draws] == [(R * 3, 1), (0, 1), (R * 3, 1)]
    out = os.path.join(ROOT, "tests", "golden", "ref_sampler.npz")
    np.savez_compressed(out, points=points_s.numpy(), origin=origin_s.numpy(), u_surface=draws[0].numpy().reshape(-1),
                        u_free=draws[2].numpy().reshape(-1), coord=coord.numpy(), label=label.numpy(),
                        weight=weight.numpy(), scale=cfg.scale, surface_sample_n=3, free_sample_n=3,
                        surface_sample_range_m=cfg.surface_sample_range_m,
                        free_sample_end_dist_m=cfg.free_sample_end_dist_m,
                        free_sample_begin_ratio=cfg.free_sample_begin_ratio)
    print("wrote", out, coord.shape)


if __name__ == "__main__":
    main(sys.argv[1])
