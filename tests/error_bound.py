"""Shared pieces of the per-element error bounds of the GPU tests (the error model is stated in the module docstrings
of tests/test_gpu_replicas.py and tests/eikonal_bound.py): the unit roundoff, the 3xTF32 contraction error, the fp64
oracle of a case with its fp32 blend weights, the absolute-value decoder passes, the ReLU-kink filter and the row-sum
bound with its grading loop.  Test infrastructure, no GPU needed."""
from __future__ import annotations

import numpy as np
import torch

from tests.parity_utils import oracle_from_case

U = 2.0 ** -24
C_SLACK = 4
H = 32


def eps_mm(k, tf32x1=False):
    return (2.0 ** -9 if tf32x1 else 64 * U) + 8 * k * U


def subset(case, keep):
    out = dict(case)
    for k in ("coord", "label", "weight"):
        out[k] = np.ascontiguousarray(case[k][keep])
    return out


def oracle64(case):
    o, dec = oracle_from_case(case)
    o.hier_features = [t.detach().double().requires_grad_(True) for t in o.hier_features]
    return o, {k: v.detach().double().requires_grad_(True) for k, v in dec.items()}


def blend(o, coord):
    """Per level (bottom-up): the oracle's corner rows [N*8] and fp32 blend weights [N*8] as fp64."""
    idx = o.get_indices(coord)
    out = []
    for i in range(o.featured_level_num):
        w = o.interpolat(coord, o.max_level - i, o.polynomial_interpolation).reshape(-1).double()
        out.append((idx[i].reshape(-1), w))
    return out


def abs_feature(o, coord):
    """sum over levels and corners of |w| |row| (a coordinate outside [-1, 1] can have a negative blend weight)"""
    total = torch.zeros(coord.shape[0], o.feature_dim, dtype=torch.float64)
    for i, (ix, w) in enumerate(blend(o, coord)):
        t = o.hier_features[o.featured_level_num - 1 - i].detach().abs()
        total += (t[ix] * w.abs()[:, None]).reshape(coord.shape[0], 8, -1).sum(1)
    return total


def decoder_passes(feat, absfeat, dec, tf32x1, n_levels):
    """fp64 forward with the absolute-value passes of test_gpu_replicas' docstring -> dict of per-point quantities."""
    z = torch.zeros((), dtype=torch.float64)
    W1, W2, w3 = (dec[k].detach() for k in ("layers.0.weight", "layers.1.weight", "lout.weight"))
    b1, b2, b3 = (dec.get(k, z).detach() for k in ("layers.0.bias", "layers.1.bias", "lout.bias"))
    F = W1.shape[1]
    a1 = feat @ W1.T + b1
    m1 = (a1 > 0).double()
    a2 = (a1 * m1) @ W2.T + b2
    m2 = (a2 > 0).double()
    A1 = absfeat @ W1.abs().T + b1.abs()
    A2 = (A1 * m1) @ W2.abs().T + b2.abs()
    Ap = ((A2 * m2) @ w3.abs().T + b3.abs()).squeeze(1)
    e1 = (8 * n_levels + 2) * U + eps_mm(F, tf32x1) + U
    e2 = e1 + eps_mm(H, tf32x1) + U
    efwd = e2 + eps_mm(H, tf32x1) + U
    D = ((m2 * w3.abs()) @ W2.abs() * m1) @ W1.abs()
    # a unit whose absolute-value pass is 0 is an exact 0 in every precision (a point that misses every level, a decoder
    # without biases): its mask is exact, not a kink
    u1 = (a1.abs() <= 2 * e1 * A1) & (A1 > 0)
    m1_hi = ((m1 > 0) | u1).double()
    A2_hi = (A1 * m1_hi) @ W2.abs().T + b2.abs()
    u2 = (a2.abs() <= 2 * e2 * A2_hi) & (A2_hi > 0)
    kink = u1.any(1) | u2.any(1)
    # pred of a kink point, whichever branch the kernel takes: an uncertain unit is off by at most |a| + e A <= 3 e A of
    # its fp64 value (2 e A + e A), and the pass runs with the uncertain units live (A2_hi, m2_hi)
    Ap_hi = ((A2_hi * ((m2 > 0) | u2).double()) @ w3.abs().T + b3.abs()).squeeze(1)
    P = torch.where(kink, 3 * efwd * Ap_hi, efwd * Ap)
    return {"A0": absfeat, "P": P, "D": D, "kink": kink, "ebwd": 2 * eps_mm(H, tf32x1) + 2 * U,
            "A1": A1, "A2": A2, "A2_hi": A2_hi, "e1": e1, "e2": e2, "ef": (8 * n_levels + 2) * U * absfeat,
            "m1_hi": m1_hi, "m2_hi": ((m2 > 0) | u2).double()}


def drop_kinks(case, tf32x1=False):
    """The case without the points whose pre-activations lie within twice the forward error of a ReLU kink."""
    o, dec = oracle64(case)
    coord = torch.from_numpy(case["coord"])
    with torch.no_grad():
        feat = o.query_feature(coord)
        absfeat = abs_feature(o, coord)
        kink = decoder_passes(feat, absfeat, dec, tf32x1, o.featured_level_num)["kink"].numpy()
    return subset(case, ~kink), int(kink.sum())


class RowSums:
    """want, S, k and T of a scatter into the rows of each table: every term is a[m] * v[pts[m], f] added into row ix[m],
    with |a - a64| <= ea and |v - v64| <= ev.  The bound of test_gpu_replicas' docstring: (k_u + C) u S + T, with
    S = sum |a v| and T = sum (|a| ev + ea |v|) over the k_u terms of row u."""

    def __init__(self, rows, F, slack=C_SLACK):
        self.want = [np.zeros((r, F)) for r in rows]
        self.S = [np.zeros((r, F)) for r in rows]
        self.T = [np.zeros((r, F)) for r in rows]
        self.k = [np.zeros(r, dtype=np.int64) for r in rows]
        self.slack = slack

    def add(self, kk, ix, pts, a, v, ea=None, ev=None, count=True):
        """Terms of table kk; ix [M] rows (-1: a miss, skipped), pts [M] points, a / ea [M], v / ev [N, F] (fp64).
        count=False: the terms are parts of terms already added (one fp32 term per (point, corner)), k_u stays."""
        ix, pts, a = (np.asarray(x) for x in (ix, pts, a))
        hit = ix >= 0
        r, p, a = ix[hit], pts[hit], a[hit]
        v = np.asarray(v)
        np.add.at(self.want[kk], r, a[:, None] * v[p])
        np.add.at(self.S[kk], r, np.abs(a[:, None] * v[p]))
        t = np.zeros((r.shape[0], v.shape[1]))
        if ev is not None:
            t += np.abs(a)[:, None] * np.asarray(ev)[p]
        if ea is not None:
            t += np.asarray(ea)[hit][:, None] * np.abs(v[p])
        np.add.at(self.T[kk], r, t)
        if count:
            self.k[kk] += np.bincount(r, minlength=self.k[kk].shape[0])

    def bound(self, kk):
        return (self.k[kk][:, None] + self.slack) * U * self.S[kk] + self.T[kk]

    def grade(self, got_tables, what, tag="bounds"):
        return grade_tables(got_tables, self.want, [self.bound(kk) for kk in range(len(self.want))], self.k, self.S,
                            what, tag)


def grade_tables(got_tables, want, bounds, k, S, what, tag="bounds"):
    """Every element of every level (trash row excluded) against its bound -> worst error / bound."""
    worst = 0.0
    for kk, got in enumerate(got_tables):
        got = np.asarray(got, dtype=np.float64)[:-1]
        w, bound = want[kk][:-1], bounds[kk][:-1]
        err = np.abs(got - w)
        bad = np.argwhere(err > bound)
        if bad.size:
            r, f = bad[0]
            raise AssertionError(
                f"{what}: level {kk} has {len(bad)} elements outside the bound; first: row {r} channel {f} got "
                f"{got[r, f]:.9g} want {w[r, f]:.9g} bound {bound[r, f]:.3g} (k_u = {k[kk][r]}, S = {S[kk][r, f]:.3g})")
        if err.size:
            worst = max(worst, float((err / np.where(bound > 0, bound, 1.0)).max()))
    print(f"[{tag}] {what}: table grads worst {worst:.3f} of the bound")
    return worst


def grade_values(got, want, bound, what, name, tag="bounds"):
    """Per-element |got - want| <= bound of one array -> worst error / bound (printed)."""
    got, want, bound = (np.asarray(x, dtype=np.float64) for x in (got, want, bound))
    err = np.abs(got - want)
    bad = np.argwhere(err > bound)
    if bad.size:
        i = tuple(bad[0])
        raise AssertionError(f"{what}: {name} has {len(bad)} elements outside the bound; first {i}: got {got[i]:.9g} "
                             f"want {want[i]:.9g} bound {bound[i]:.3g}")
    worst = float((err / np.where(bound > 0, bound, 1.0)).max()) if err.size else 0.0
    print(f"[{tag}] {what}: {name} worst {worst:.3f} of the bound")
    return worst


def grouped_counts(ix, rows, max_runs=6, tile=16):
    """k_u of the voxel-grouped scatter (`grouped_scatter`): the fp32 adds that land on each row of one level.  ix [n, 8]
    corner rows of the level per point (-1: a miss).  Tiles are 16 consecutive points; a tile whose hitting points fall into
    at most `max_runs` (kMaxGroupedRuns) distinct nodes adds one term per (node, corner) row, its per-node sums formed by a
    tensor-core contraction; a scattered tile (more nodes) adds one term per (point, corner)."""
    ix = np.asarray(ix)
    n = ix.shape[0]
    pad = -n % tile
    node = np.concatenate((ix[:, 0], np.full(pad, -1, dtype=ix.dtype))).reshape(-1, tile)   # corner 0 names the node
    srt = np.sort(node, axis=1)
    nruns = ((srt >= 0) & np.concatenate((np.ones((srt.shape[0], 1), bool), srt[:, 1:] != srt[:, :-1]), 1)).sum(1)
    tile_of = np.arange(n) // tile
    hit = ix[:, 0] >= 0
    scattered = (nruns > max_runs)[tile_of] & hit
    k = np.bincount(ix[scattered].reshape(-1), minlength=rows)
    grouped = hit & ~scattered
    key = tile_of[grouped].astype(np.int64) * (int(node.max()) + 2) + ix[grouped, 0]
    _, first = np.unique(key, return_index=True)                       # one point per (tile, node)
    k += np.bincount(ix[grouped][first].reshape(-1), minlength=rows)
    return k
