"""Oracle of the replay sample pool (TEST INFRASTRUCTURE): the reference's window filter and concatenation,
dataset/lidar_dataset.py:235-271, restated in torch for the sdf path (coord, sdf_label and weight; the origin / time /
ray pools are not read by the sdf_bce step).  Runs on whatever device its inputs live on, so that the large-pool tests
can run it on the GPU."""
from __future__ import annotations

import torch


def window_mask(coord_pool, origin, radius):
    """lidar_dataset.py:238-239 `(coord_pool - frame_origin).norm(2, dim=-1) < window_radius * scale`, with the norm
    written out as separate fp32 operations in one fixed order, (dx*dx + dy*dy) + dz*dz then sqrt: each torch op rounds
    once, so the result is the same on every device.  torch's own norm may sum in another order; it differs from this
    only for distances within an ulp or two of the radius.  The Python scalar `radius` is compared as fp32, as torch does."""
    o = torch.as_tensor(origin, dtype=torch.float32).to(coord_pool.device).reshape(1, 3)
    d = coord_pool - o
    dist = ((d[:, 0] * d[:, 0] + d[:, 1] * d[:, 1]) + d[:, 2] * d[:, 2]).sqrt()
    return dist < radius


def replay_pool_update(coord_pool, label_pool, weight_pool, coord, label, weight, origin, radius_or_none):
    """One frame of `process_frame` with `incremental_on=False`: with a radius (window_replay_on, :237) the masked
    gathers of :244-251, then the `torch.cat`s of :263-270.  -> (coord_pool, label_pool, weight_pool)."""
    if radius_or_none is not None:
        mask = window_mask(coord_pool, origin, radius_or_none)
        coord_pool, weight_pool, label_pool = coord_pool[mask], weight_pool[mask], label_pool[mask]
    dev = coord_pool.device
    return (torch.cat((coord_pool, coord.to(dev)), 0), torch.cat((label_pool, label.to(dev)), 0),
            torch.cat((weight_pool, weight.to(dev)), 0))


class OraclePool:
    """The same interface as `synth.ReplayPool` (add_frame / get_batch / len) over `replay_pool_update`: the loop run with
    it is the reference's pool upkeep, call for call."""

    def __init__(self, device):
        from shine_mapping_b200.synth import SamplePool
        self._pool = SamplePool(device)
        self.device = device
        self.ordered = False

    def add_frame(self, coord, label, weight, origin_scaled=None, window_radius_scaled=None):
        p = self._pool
        p.coord_pool, p.sdf_label_pool, p.weight_pool = replay_pool_update(
            p.coord_pool, p.sdf_label_pool, p.weight_pool, coord, label, weight, origin_scaled, window_radius_scaled)
        return self

    def get_batch(self, bs, generator=None):
        return self._pool.get_batch(bs, generator)

    def __len__(self):
        return len(self._pool)
