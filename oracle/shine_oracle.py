"""CPU oracle for SHINE's per-point SDF training step.  *** TEST INFRASTRUCTURE — NOT A PRODUCT PATH ***

Only `tests/`, `__graft_entry__.smoke()` and `bench.py`'s `cpu_baseline` / `--impl reference` legs may import
this module.  `shine_mapping_b200/` never does: the product path is CUDA-only and raises when its extension
is missing.

What this is: a plain numpy (integer work) + torch-CPU (float work, autograd for the backward) restatement of
the reference algorithm, written from the reference's behaviour, every function citing the reference
`file:line` it follows (paths relative to PRBonn/SHINE_mapping @ 0fbaf8a).  The integer arithmetic of the
path lives in a third-party dependency that is NOT vendored in the reference: NVIDIA kaolin, pinned v0.13.0
by the reference `Dockerfile:33`; its five ops are restated here from kaolin's published semantics and
cross-pinned by the reference's own consumers (corner order by `model/feature_octree.py:186-195,229`).

Parity pin: the reference ships no tests / golden vectors for this path ("parity unpinned" upstream).  This
oracle is pinned instead against the outputs of the *unmodified reference classes* run in the build
container (imported from /root/reference with `oracle/kaolin_shim`), frozen as `tests/golden/*.npz` by
`oracle/make_golden.py`; `tests/test_oracle_golden.py` checks oracle == golden (indices bit-exact).

Like the reference, the lookup is a Python `dict.get` per point (`model/feature_octree.py:209`) — that is
the reference's CPU algorithm and is what `cpu_baseline` times.
"""
from __future__ import annotations

import numpy as np
import torch

# --------------------------------------------------------------------------------------------------
# kaolin SPC integer ops (call sites model/feature_octree.py:88-89,97,116,123,131,134,162-164,203-204)
# --------------------------------------------------------------------------------------------------


def quantize_points(x: np.ndarray, level: int) -> np.ndarray:
    """kal.ops.spc.quantize_points (call site model/feature_octree.py:203): fp32
    floor(clamp(2^level * (x + 1) / 2, 0, 2^level - 1)) -> int16 xyz."""
    x = np.asarray(x, dtype=np.float32)
    res = np.float32(2 ** level)
    v = res * (x + np.float32(1.0)) / np.float32(2.0)
    v = np.minimum(np.maximum(v, np.float32(0.0)), res - np.float32(1.0))
    return np.floor(v).astype(np.int16)


def _part1by2(v: np.ndarray) -> np.ndarray:
    """Spread the low 16 bits of v so bit i lands at bit 3i."""
    v = v.astype(np.uint64) & np.uint64(0xFFFF)
    out = np.zeros_like(v)
    for i in range(16):
        out |= ((v >> np.uint64(i)) & np.uint64(1)) << np.uint64(3 * i)
    return out


def points_to_morton(p: np.ndarray) -> np.ndarray:
    """kal.ops.spc.points_to_morton (call site model/feature_octree.py:204): x->bit 3i+2, y->3i+1, z->3i."""
    p = np.asarray(p).astype(np.int64)
    m = (_part1by2(p[..., 0]) << np.uint64(2)) | (_part1by2(p[..., 1]) << np.uint64(1)) | _part1by2(p[..., 2])
    return m.astype(np.int64)


def morton_to_points(m: np.ndarray) -> np.ndarray:
    """kal.ops.spc.morton_to_points (call site model/feature_octree.py:97)."""
    m = np.asarray(m).astype(np.uint64)
    out = np.zeros(m.shape + (3,), dtype=np.int64)
    for axis, shift in ((0, 2), (1, 1), (2, 0)):
        v = m >> np.uint64(shift)
        acc = np.zeros_like(m)
        for i in range(16):
            acc |= ((v >> np.uint64(3 * i)) & np.uint64(1)) << np.uint64(i)
        out[..., axis] = acc.astype(np.int64)
    return out.astype(np.int16)


def points_to_corners(p: np.ndarray) -> np.ndarray:
    """kal.ops.spc.points_to_corners (call site model/feature_octree.py:131): corner i = p + ((i>>2)&1,
    (i>>1)&1, i&1).  The order is pinned by the weight order in model/feature_octree.py:186-195."""
    off = np.array([[(i >> 2) & 1, (i >> 1) & 1, i & 1] for i in range(8)], dtype=np.int16)
    return np.asarray(p, dtype=np.int16)[..., None, :] + off


def pointcloud_level_nodes(points: np.ndarray, max_level: int):
    """kal.ops.conversions.unbatched_pointcloud_to_spc as consumed at model/feature_octree.py:116-122:
    per level (root..leaf) the occupied nodes, int16 xyz in Morton order."""
    leaf = np.unique(points_to_morton(quantize_points(points, max_level)))
    return [morton_to_points(np.unique(leaf >> (3 * (max_level - l)))) for l in range(max_level + 1)]


# --------------------------------------------------------------------------------------------------
# FeatureOctree (model/feature_octree.py:29-298)
# --------------------------------------------------------------------------------------------------


class OracleOctree:
    """Restates FeatureOctree state + the methods on the hot path (model/feature_octree.py:31-74)."""

    def __init__(self, tree_level_world: int, tree_level_feat: int, feature_dim: int = 8,
                 feature_std: float = 0.05, poly_int_on: bool = True):
        if tree_level_feat < 1:  # model/feature_octree.py:58-59
            raise ValueError('No level with grid features!')
        self.max_level = tree_level_world
        self.featured_level_num = tree_level_feat
        self.free_level_num = self.max_level - self.featured_level_num + 1  # :39
        self.feature_dim = feature_dim
        self.feature_std = feature_std
        self.polynomial_interpolation = poly_int_on
        self.corners_lookup_tables = [dict() for _ in range(self.max_level + 1)]  # :46-52
        self.nodes_lookup_tables = [dict() for _ in range(self.max_level + 1)]
        self.hier_features: list[torch.Tensor] = []  # coarse -> fine, trailing trash row (:61-63)
        self.hierarchical_indices: list[torch.Tensor] = []  # bottom-up (:66-67)

    # model/feature_octree.py:114-166
    def update(self, surface_points) -> None:
        pts = np.asarray(torch.as_tensor(surface_points).detach().cpu().numpy(), dtype=np.float32)
        per_level = pointcloud_level_nodes(pts, self.max_level)
        for i in range(self.max_level + 1):
            if i < self.free_level_num:  # :119-120
                continue
            nodes = per_level[i]
            nodes_morton = points_to_morton(nodes).tolist()
            table = self.nodes_lookup_tables[i]
            new_idx = [k for k, m in enumerate(nodes_morton) if m not in table]  # :124-127
            if not new_idx:
                continue
            new_nodes = nodes[new_idx]
            corners = points_to_corners(new_nodes).reshape(-1, 3)
            corners_unique = np.unique(corners, axis=0)  # lexicographic x,y,z == torch.unique(dim=0) (:132)
            corners_morton = points_to_morton(corners_unique).tolist()
            ctab = self.corners_lookup_tables[i]
            if len(ctab) == 0:  # first frame (:135-142)
                ctab.update(zip(corners_morton, range(len(corners_morton))))
                fts = self.feature_std * torch.randn(len(ctab) + 1, self.feature_dim)
                fts[-1] = 0.0
                self.hier_features.append(fts.requires_grad_(True))
            else:  # later frames: append-only in that order (:146-156)
                pre = len(ctab)
                for m in corners_morton:
                    if m not in ctab:
                        ctab[m] = len(ctab)
                new_fts = self.feature_std * torch.randn(len(ctab) - pre + 1, self.feature_dim)
                new_fts[-1] = 0.0
                lvl = i - self.free_level_num
                self.hier_features[lvl] = torch.cat(
                    (self.hier_features[lvl].detach()[:-1], new_fts), 0).requires_grad_(True)
            corner_ids = np.array([ctab[m] for m in points_to_morton(corners).tolist()]).reshape(-1, 8)
            for k, m in enumerate(points_to_morton(new_nodes).tolist()):  # :162-166
                table[m] = corner_ids[k].tolist()

    # model/feature_octree.py:78-81
    def set_zero(self) -> None:
        with torch.no_grad():
            for f in self.hier_features:
                f[-1] = 0.0

    # model/feature_octree.py:172-196
    def interpolat(self, x: torch.Tensor, level: int, polynomial_on: bool = True) -> torch.Tensor:
        coords = (2 ** level) * (x * 0.5 + 0.5)
        d = torch.frac(coords)
        if polynomial_on:
            t = 3 * (d ** 2) - 2 * (d ** 3)
        else:
            t = d
        tx, ty, tz = t[:, 0], t[:, 1], t[:, 2]
        ux, uy, uz = 1 - tx, 1 - ty, 1 - tz
        p = torch.stack((ux * uy * uz, ux * uy * tz, ux * ty * uz, ux * ty * tz,
                         tx * uy * uz, tx * uy * tz, tx * ty * uz, tx * ty * tz), 0)
        return p.T.unsqueeze(2)  # [N, 8, 1]

    # model/feature_octree.py:199-218
    def get_indices(self, coord: torch.Tensor) -> list[torch.Tensor]:
        c = coord.detach().cpu().numpy()
        self.hierarchical_indices = []
        miss = [-1] * 8
        for i in range(self.featured_level_num):  # bottom-up
            level = self.max_level - i
            morton = points_to_morton(quantize_points(c, level)).tolist()
            table = self.nodes_lookup_tables[level]
            rows = [table.get(m, miss) for m in morton]  # the reference's "hash": Python dict (:209)
            self.hierarchical_indices.append(torch.tensor(rows, dtype=torch.int64).reshape(-1, 8))
        return self.hierarchical_indices

    # model/feature_octree.py:222-234
    def query_feature_with_indices(self, coord: torch.Tensor, hierarchical_indices) -> torch.Tensor:
        total = torch.zeros(coord.shape[0], self.feature_dim)
        for i in range(self.featured_level_num):
            level = self.max_level - i
            feat_level = self.featured_level_num - i - 1
            w = self.interpolat(coord, level, self.polynomial_interpolation)
            total = total + (self.hier_features[feat_level][hierarchical_indices[i]] * w).sum(1)
        return total

    # model/feature_octree.py:237-244
    def query_feature(self, coord: torch.Tensor) -> torch.Tensor:
        self.set_zero()
        return self.query_feature_with_indices(coord, self.get_indices(coord))


# --------------------------------------------------------------------------------------------------
# Decoder.sdf (model/decoder.py:29-36,49-63) and sdf_bce_loss (utils/loss.py:17-24)
# --------------------------------------------------------------------------------------------------


def make_decoder_params(feature_dim: int = 8, hidden: int = 32, mlp_level: int = 2, bias: bool = True):
    """Same layer shapes / torch default nn.Linear init as Decoder.__init__ (model/decoder.py:29-36):
    returns {'layers.k.weight','layers.k.bias','lout.weight','lout.bias'} leaf tensors."""
    params = {}
    for k in range(mlp_level):
        lin = torch.nn.Linear(feature_dim if k == 0 else hidden, hidden, bias)
        params[f"layers.{k}.weight"] = lin.weight.detach().clone().requires_grad_(True)
        if bias:
            params[f"layers.{k}.bias"] = lin.bias.detach().clone().requires_grad_(True)
    lout = torch.nn.Linear(hidden, 1, bias)
    params["lout.weight"] = lout.weight.detach().clone().requires_grad_(True)
    if bias:
        params["lout.bias"] = lout.bias.detach().clone().requires_grad_(True)
    return params


def decoder_sdf(feature: torch.Tensor, params: dict) -> torch.Tensor:
    """Decoder.sdf (model/decoder.py:49-63): (Linear+ReLU) x mlp_level, then lout -> [N] (negated-SDF sign)."""
    h = feature
    k = 0
    while f"layers.{k}.weight" in params:
        h = torch.relu(torch.nn.functional.linear(h, params[f"layers.{k}.weight"], params.get(f"layers.{k}.bias")))
        k += 1
    return torch.nn.functional.linear(h, params["lout.weight"], params.get("lout.bias")).squeeze(1)


def sdf_bce_loss(pred, label, sigma, weight, weighted=False, bce_reduction="mean"):
    """utils/loss.py:17-24: BCEWithLogits(pred, sigmoid(label / sigma)), optional per-sample weight."""
    target = torch.sigmoid(label / sigma)
    w = weight if weighted else None
    return torch.nn.functional.binary_cross_entropy_with_logits(pred, target, weight=w, reduction=bce_reduction)


def train_step(octree: OracleOctree, dec: dict, coord, label, weight, sigma: float,
               weighted: bool = False, reduction: str = "mean"):
    """The loop body shine_batch.py:123,128,172-174,208-209: query -> sdf -> |weight| -> bce -> backward.
    Returns dict(loss, pred, feature, table_grads (coarse->fine), dec_grads)."""
    for f in octree.hier_features:
        f.grad = None
    for p in dec.values():
        p.grad = None
    feature = octree.query_feature(coord)
    pred = decoder_sdf(feature, dec)
    w = torch.abs(weight) if weight is not None else None  # shine_batch.py:172
    loss = sdf_bce_loss(pred, label, sigma, w, weighted, reduction)
    loss.backward()
    return {
        "loss": loss.detach(), "pred": pred.detach(), "feature": feature.detach(),
        "table_grads": [f.grad if f.grad is not None else torch.zeros_like(f) for f in octree.hier_features],
        "dec_grads": {k: (p.grad if p.grad is not None else torch.zeros_like(p)) for k, p in dec.items()},
    }


# --------------------------------------------------------------------------------------------------
# continual-learning terms (BASELINE config 4): model/feature_octree.py:246-255, utils/incre_learning.py:8-40
# --------------------------------------------------------------------------------------------------


def cal_regularization(octree: OracleOctree, features_last_frame, importance_weight) -> torch.Tensor:
    """FeatureOctree.cal_regularization (model/feature_octree.py:246-255): over the UNIQUE rows touched by the last
    queried batch, sum Omega * (f - f_last)^2, per level."""
    reg = torch.zeros(())
    for i in range(octree.featured_level_num):
        k = octree.featured_level_num - i - 1
        u = octree.hierarchical_indices[i].flatten().unique()
        diff = octree.hier_features[k][u] - features_last_frame[k][u]
        reg = reg + (importance_weight[k][u] * diff ** 2).sum()
    return reg


def cal_feature_importance(octree: OracleOctree, dec: dict, coord_pool, label_pool, sigma, bs, down_rate=1,
                           reduction="sum"):
    """utils/incre_learning.py:8-40: sweep the pool in strides of bs*down_rate, accumulate |dL/dfeature| per row."""
    importance = [torch.zeros_like(f) for f in octree.hier_features]
    n = coord_pool.shape[0]
    interval = bs * down_rate
    for head in range(0, n, interval):
        c = coord_pool[head:min(head + interval, n):down_rate]
        l = label_pool[head:min(head + interval, n):down_rate]
        res = train_step(octree, dec, c, l, None, sigma, False, reduction)
        for k, g in enumerate(res["table_grads"]):
            importance[k] += g.abs()
            importance[k][-1] *= 0
    return importance


def train_step_eikonal(octree: OracleOctree, dec: dict, coord, label, weight, sigma: float, weight_e: float = 0.1,
                       weighted: bool = False, reduction: str = "mean", n_surface=None):
    """Loop body with ekional_loss_on (shine_batch.py:119-120,137-142,172-185,208-209): g = d pred / d coord (create_graph)
    * sigma_sigmoid; eikonal = mean over surface samples (weight > 0) of (1 - |g|)^2; loss = bce + weight_e * eikonal.
    BCE as shine_batch.py:172-174: |weight| applied only when `weighted`, with the given reduction.
    n_surface: denominator of the eikonal mean (default: this batch's surface count; pass the global count when the
    batch is one shard of a larger one).  Like the reference, a batch without a surface sample gives NaN (mean of empty).
    Besides the total's gradients, returns those of bce alone (`bce_*_grads`) and of the eikonal mean alone (`eik_*_grads`,
    i.e. at weight_e = 1)."""
    for f in octree.hier_features:
        f.grad = None
    for p in dec.values():
        p.grad = None
    coord = coord.clone().requires_grad_(True)
    feature = octree.query_feature(coord)
    pred = decoder_sdf(feature, dec)
    surface_mask = weight > 0
    g = torch.autograd.grad(pred, coord, torch.ones_like(pred), create_graph=True, retain_graph=True)[0] * sigma
    bce = sdf_bce_loss(pred, label, sigma, torch.abs(weight), weighted, reduction)
    sq = (1.0 - g[surface_mask].norm(2, dim=-1)) ** 2
    eik = sq.mean() if n_surface is None else sq.sum() / float(n_surface)
    loss = bce + weight_e * eik
    params = list(octree.hier_features) + list(dec.values())

    def grads(term):
        got = torch.autograd.grad(term, params, retain_graph=True, allow_unused=True)
        got = [torch.zeros_like(p) if d is None else d for p, d in zip(params, got)]
        L = len(octree.hier_features)
        return got[:L], dict(zip(dec.keys(), got[L:]))

    bce_t, bce_d = grads(bce)
    eik_t, eik_d = grads(eik) if bool(surface_mask.any()) else grads(0.0 * pred.sum())
    loss.backward()
    return {"loss": loss.detach(), "bce": bce.detach(), "eikonal": eik.detach(), "g": g.detach(), "pred": pred.detach(),
            "table_grads": [f.grad if f.grad is not None else torch.zeros_like(f) for f in octree.hier_features],
            "dec_grads": {k: (p.grad if p.grad is not None else torch.zeros_like(p)) for k, p in dec.items()},
            "bce_table_grads": bce_t, "bce_dec_grads": bce_d, "eik_table_grads": eik_t, "eik_dec_grads": eik_d}


# --------------------------------------------------------------------------------------------------
# the optimizer: utils/tools.py:57-83 (setup_optimizer) and torch.optim.Adam (shine_batch.py:210 `opt.step()`)
# --------------------------------------------------------------------------------------------------


def reference_param_groups(L: int, lr: float, weight_decay: float, lr_level_reduce_ratio: float):
    """setup_optimizer (utils/tools.py:57-83) without the semantic / ray-loss groups: the geometry decoder at `lr`
    with weight decay, then one group per table level, leaf first (hier_features[L - 1]), the lr multiplied by
    lr_level_reduce_ratio per level towards the coarse end, no decay.
    -> [{"params": "decoder" | table index into hier_features, "lr", "weight_decay"}, ...]"""
    groups = [{"params": "decoder", "lr": lr, "weight_decay": weight_decay}]
    lr_cur = lr
    for i in range(L):
        groups.append({"params": L - i - 1, "lr": lr_cur, "weight_decay": 0.0})
        lr_cur *= lr_level_reduce_ratio
    return groups


def adam_reference(params, grads, exp_avg, exp_avg_sq, step: int, lr: float, weight_decay: float,
                   betas=(0.9, 0.99), eps: float = 1e-15):
    """One step of torch.optim.Adam (amsgrad off, L2 weight decay added to the gradient) for the tensors of one
    parameter group, in float64.  `step` is the step number after this update (1 for the first).  Inputs are not
    modified.  -> (params, exp_avg, exp_avg_sq) after the step, float64 tensors (lists when lists were given)."""
    single = torch.is_tensor(params)
    if single:
        params, grads, exp_avg, exp_avg_sq = [params], [grads], [exp_avg], [exp_avg_sq]
    b1, b2 = float(betas[0]), float(betas[1])
    bc1 = 1.0 - b1 ** step
    bc2_sqrt = (1.0 - b2 ** step) ** 0.5
    out_p, out_m, out_v = [], [], []
    for p, g, m, v in zip(params, grads, exp_avg, exp_avg_sq):
        p, g, m, v = (t.detach().to(torch.float64) for t in (p, g, m, v))
        if weight_decay != 0.0:
            g = g + weight_decay * p
        m = b1 * m + (1.0 - b1) * g
        v = b2 * v + (1.0 - b2) * g * g
        p = p - (lr / bc1) * m / (v.sqrt() / bc2_sqrt + eps)
        out_p.append(p); out_m.append(m); out_v.append(v)
    if single:
        return out_p[0], out_m[0], out_v[0]
    return out_p, out_m, out_v
