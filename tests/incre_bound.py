"""fp64 reference of the continual-learning terms of incremental mapping with per-element error bounds: the three kernels of
csrc/shine_incre.cu (`shine_mark_touched`, `shine_regularization_apply`, `shine_importance_accumulate`) and the loop steps
built on them (`incre_loop.add_regularization`, `incre_loop.cal_feature_importance`).  Test infrastructure, no GPU needed.

The reference is an explicit restatement of FeatureOctree.cal_regularization (model/feature_octree.py:246-255) and
cal_feature_importance (utils/incre_learning.py:8-40) over the touched rows, not autograd; tests/test_incre_bound_host.py
checks it against the oracle's autograd versions.  Tables are coarse -> fine (index k), like hier_features.

Error model (u = 2^-24; extends the replica model of tests/test_gpu_replicas.py and tests/eikonal_bound.py):
  * touched set of level k: exact.  It is the unique non-negative rows of the oracle's get_indices on the batch; a miss
    (-1 on all 8 corners) marks nothing.  The reference's unique() also holds the -1 (trash) row, whose importance it keeps
    at 0, so that row adds nothing there either.
  * regulariser gradient: the kernel adds t = fl(fl(fl(2 lambda) Omega) fl(f - f_last)) to the gradient (nvcc may fuse the
    last product and the add into one FMA, which only drops a rounding).  The reference is t64 = 2 lambda Omega d with
    d = f - f_last in fp64 from the same fp32 values.  2 lambda rounded to fp32, the subtraction and the two products are
    four relative roundings: |t - t64| <= ((1 + u)^4 - 1) |t64| < 4.0001 u |t64|.  The add rounds once more, by at most
    u (|want64| + B + 4.0001 u |t64|), where B bounds the gradient the term lands on (the replica model's for the BCE step,
    EikRef's with the eikonal term, 0 when that gradient is an input).  So, with want64 = g64 + t64,
        |got - want64| <= (1 + u) B + 5 u |t64| + u |want64|.
  * regulariser value: the sum over touched rows and channels of q = Omega d^2.  Each q is off by 4 u |q| (the rounding of
    d counts twice, then two products).  The kernel sums them as (1) per item, the float4's four q in 3 adds, added into the
    thread's running sum, over the m grid-stride items the thread takes on its level; (2) a 5-step xor shuffle over the
    warp; (3) one atomicAdd per warp with a non-zero sum, over all levels, into *out_reg.  A warp whose threads own no item
    issues none, so there are at most N_a = sum over levels of min(blocks * 8, ceil(count F/4 / 32)) atomics.  Any q passes
    at most depth = 3 + m + 5 + N_a adds; the initial value of *out_reg is one more term and passes the N_a atomics, so
        |got - init - reg64| <= (depth + 4 + C) u (sum |q| + |init|),   C = C_SLACK,
    with blocks = min(ceil(max capacity * F/4 / 256), 8 * SM count) and m = ceil(count * F/4 / (blocks * 256)), the largest
    over the levels: both from the launch geometry (`launch_geometry`).
  * importance: every stride s adds |g_s| to Omega with one rounding; |g_s| is off by at most B_s (the replica bound of the
    unweighted step of that stride; 0 when the gradient is an input), so
        |Omega_got - Omega64| <= sum_s (B_s + u |Omega after stride s|).
  * ReLU kinks: the loop draws its own batches, so the points near a kink (error_bound.decoder_passes' criterion; EikRef's
    kink and ill-conditioned points with the eikonal term) cannot be left out of the batch.  The table rows such a point
    touches are left out of the per-element grade instead (`rows_of_points`); the tests count them and keep them under 5 %
    of the touched rows (0.3 % or more of the points are near a kink, and each takes its 8 L corner rows out).
"""
from __future__ import annotations

import numpy as np
import torch

from tests.error_bound import C_SLACK, U, oracle64


def touched_sets(o, coord):
    """Per table k (coarse -> fine): the sorted unique rows >= 0 of the oracle's get_indices on coord."""
    idx = o.get_indices(torch.as_tensor(np.asarray(coord, dtype=np.float32).reshape(-1, 3)))
    L = o.featured_level_num
    out = [None] * L
    for i in range(L):
        r = idx[i].reshape(-1).numpy()
        out[L - 1 - i] = np.unique(r[r >= 0])
    return out


def rows_of_points(o, coord, mask):
    """Per table k: boolean row mask of the rows that the points with mask set touch."""
    L = o.featured_level_num
    rows = [torch.zeros(t.shape[0], dtype=torch.bool).numpy() for t in o.hier_features]
    pts = np.asarray(coord, dtype=np.float32)[np.asarray(mask, dtype=bool)]
    if pts.shape[0]:
        for k, r in enumerate(touched_sets(o, pts)):
            rows[k][r] = True
    return rows


def launch_geometry(counts, capacities, F, sm_count):
    """The grid of the touched-row kernels (list_blocks) -> (blocks, m = most items per thread, N_a = most atomics)."""
    lp = F // 4
    blocks = max(1, min(-(-max(1, max(capacities)) * lp // 256), 8 * sm_count))
    threads = blocks * 256
    m = max([-(-c * lp // threads) for c in counts] + [0])
    n_atomics = sum(min(blocks * 8, -(-c * lp // 32)) for c in counts)
    return blocks, m, n_atomics


class RegRef:
    """The regulariser of one step in fp64: value and gradient term t = 2 lambda Omega (f - f_last) over the touched rows.
    tables / last / imp: fp32 arrays (coarse -> fine); rows: `touched_sets`; grads: the fp64 gradient the term lands on
    (None: zero) and B its bound (None: exact input)."""

    def __init__(self, tables, last, imp, rows, lam, grads=None, B=None):
        self.t, self.want, self.bound = [], [], []
        self.value, self.qabs, self.counts = 0.0, 0.0, [int(r.shape[0]) for r in rows]
        for kk, r in enumerate(rows):
            f, fl, w = (np.asarray(a[kk], dtype=np.float64) for a in (tables, last, imp))
            t = np.zeros_like(f)
            d = f[r] - fl[r]
            t[r] = 2.0 * lam * w[r] * d
            q = w[r] * d * d
            self.value += float(q.sum())
            self.qabs += float(np.abs(q).sum())
            g = np.zeros_like(f) if grads is None else np.asarray(grads[kk], dtype=np.float64)
            b = np.zeros_like(f) if B is None else np.asarray(B[kk], dtype=np.float64)
            want = g + t
            self.t.append(t)
            self.want.append(want)
            self.bound.append((1 + U) * b + 5 * U * np.abs(t) + U * np.abs(want))

    def value_bound(self, capacities, F, sm_count, init=0.0):
        _, m, n_atomics = launch_geometry(self.counts, capacities, F, sm_count)
        depth = 3 + m + 5 + n_atomics
        return (depth + 4 + C_SLACK) * U * (self.qabs + abs(init))


def importance_want(prior, strides, rows=None):
    """Omega after a sweep.  prior: fp32 Omega per table; strides: per stride (|g_s| fp64 per table, B_s per table or None);
    rows: per stride the touched sets (None: every row).  -> (want, bound) per table."""
    want = [np.asarray(p, dtype=np.float64).copy() for p in prior]
    bound = [np.zeros_like(w) for w in want]
    for s, (absg, B) in enumerate(strides):
        for kk in range(len(want)):
            add = np.asarray(absg[kk], dtype=np.float64)
            if rows is not None:
                r = rows[s][kk]
                want[kk][r] += add[r]
                if B is not None:
                    bound[kk][r] += np.asarray(B[kk], dtype=np.float64)[r]
                bound[kk][r] += U * np.abs(want[kk][r])
            else:
                want[kk] += add
                if B is not None:
                    bound[kk] += np.asarray(B[kk], dtype=np.float64)
                bound[kk] += U * np.abs(want[kk])
    return want, bound


def regularization64(o, last, imp, lam):
    """cal_regularization restated over touched_sets of the oracle's last get_indices: (value, gradient of lam * reg).
    o.hier_features, last and imp: tables coarse -> fine; the oracle's hierarchical_indices must be current."""
    L = o.featured_level_num
    value, grads = 0.0, []
    for kk in range(L):
        ix = o.hierarchical_indices[L - 1 - kk].reshape(-1).numpy()
        r = np.unique(ix[ix >= 0])
        f = o.hier_features[kk].detach().double().numpy()
        d = f[r] - np.asarray(last[kk], dtype=np.float64)[r]
        w = np.asarray(imp[kk], dtype=np.float64)[r]
        value += float((w * d * d).sum())
        g = np.zeros_like(f)
        g[r] = 2.0 * lam * w * d
        grads.append(g)
    return value, grads


def importance_sweep64(o, dec, coord, label, sigma, bs, down_rate=1):
    """cal_feature_importance restated with the touched sets: per stride of bs * down_rate samples (every down_rate-th),
    one unweighted BCE(sum) step in the oracle, then Omega[rows] += |g[rows]| on the rows the stride touched.
    -> (Omega per table, [(coord, label) of every stride])."""
    from oracle import shine_oracle as orc
    imp = [torch.zeros_like(f).double().numpy() for f in o.hier_features]
    n, interval = coord.shape[0], bs * down_rate
    strides = []
    for head in range(0, n, interval):
        c = coord[head:min(head + interval, n):down_rate]
        lab = label[head:min(head + interval, n):down_rate]
        res = orc.train_step(o, dec, c, lab, None, sigma, False, "sum")
        for kk, r in enumerate(touched_sets(o, c.numpy())):
            imp[kk][r] += res["table_grads"][kk].double().abs().numpy()[r]
        strides.append((c, lab))
    return imp, strides


# ---- the kernels' fp32 arithmetic, in their operation order (a yardstick for the bounds) -----------------------------------

def kernel_regularization32(tables, last, imp, grads, rows, lam, F, sm_count, capacities, init=0.0):
    """shine_regularization_apply in numpy fp32: rows per table in list order (a row listed twice is applied twice).
    -> (out_reg, gradient tables)."""
    f32 = np.float32
    L, lp = len(tables), F // 4
    blocks, _, _ = launch_geometry([len(r) for r in rows], capacities, F, sm_count)
    T = blocks * 256
    scale = f32(2.0 * lam)
    warp_sums, out = [], []
    for i in range(L):                                   # blockIdx.y: bottom-up
        kk = L - 1 - i
        r = np.asarray(rows[kk], dtype=np.int64)
        f = tables[kk][r].astype(f32).reshape(-1, 4)
        fl = last[kk][r].astype(f32).reshape(-1, 4)
        w = imp[kk][r].astype(f32).reshape(-1, 4)
        d = f - fl
        q = (w * d) * d
        term = ((q[:, 0] + q[:, 1]) + q[:, 2]) + q[:, 3]
        local = np.zeros(max(T, 32), dtype=f32)
        for p in range(0, term.shape[0], T):
            seg = term[p:p + T]
            local[:seg.shape[0]] = local[:seg.shape[0]] + seg
        lw = local.reshape(-1, 32)
        lane = np.arange(32)
        for o in (16, 8, 4, 2, 1):
            lw = lw + lw[:, lane ^ o]
        warp_sums.extend(float(s) for s in lw[:, 0] if s != 0)
        g = np.asarray(grads[kk], dtype=f32).copy()
        upd = ((scale * w) * d).reshape(-1, F)
        for j, u in enumerate(r):                        # plain RMW per list entry
            g[u] = g[u] + upd[j]
        out.append((kk, g))
    reg = f32(init)
    for s in warp_sums:
        reg = f32(reg + f32(s))
    gt = [None] * L
    for kk, g in out:
        gt[kk] = g
    return float(reg), gt


def kernel_importance32(imp, grads, rows, zero_grads=True, absolute=True):
    """shine_importance_accumulate in numpy fp32 -> (Omega, gradient tables)."""
    f32 = np.float32
    om, gs = [], []
    for kk, r in enumerate(rows):
        w = np.asarray(imp[kk], dtype=f32).copy()
        g = np.asarray(grads[kk], dtype=f32).copy()
        for u in np.asarray(r, dtype=np.int64):
            w[u] = w[u] + (np.abs(g[u]) if absolute else g[u])
            if zero_grads:
                g[u] = 0
        om.append(w)
        gs.append(g)
    return om, gs



def grade_rows(got_tables, want, bound, what, exclude=None, tag="incre bounds"):
    """Every element of every level (trash row excluded) against its bound; rows with exclude[k] set are left out."""
    from tests.error_bound import grade_tables
    if exclude is not None:
        bound = [np.where(np.asarray(x)[:, None], np.inf, b) for b, x in zip(bound, exclude)]
    zk = [np.zeros(w.shape[0], dtype=np.int64) for w in want]
    zs = [np.zeros_like(w) for w in want]
    return grade_tables(got_tables, want, bound, zk, zs, what, tag)


def decoder_kink_slack(case, kink):
    """Per decoder tensor: twice an upper bound of what the points with kink set add to the BCE gradients of the decoder.
    Either side of a kink gives a contribution within that bound (masks taken as all ones, |dL/dpred| <= the point's
    loss scale), so the kernel and the fp64 reference differ on such a point by at most twice it."""
    from tests.error_bound import abs_feature
    o, dec = oracle64(dict(case, coord=np.ascontiguousarray(case["coord"][kink])))
    c = case["cfg"]
    coord = torch.from_numpy(np.ascontiguousarray(case["coord"][kink]))
    n = case["coord"].shape[0]
    s = np.abs(case["weight"][kink]).astype(np.float64) if c["weighted"] else np.ones(coord.shape[0])
    s = torch.from_numpy(s / n if c["reduction"] == "mean" else s)
    z = torch.zeros((), dtype=torch.float64)
    W1, W2, w3 = (dec[k].detach().abs() for k in ("layers.0.weight", "layers.1.weight", "lout.weight"))
    b1, b2 = (dec.get(k, z).detach().abs() for k in ("layers.0.bias", "layers.1.bias"))
    with torch.no_grad():
        A0 = abs_feature(o, coord)
        A1 = A0 @ W1.T + b1
        A2 = A1 @ W2.T + b2
        c1 = w3 @ W2
        S = float(s.sum())
        out = {"lout.weight": (s[:, None] * A2).sum(0, keepdim=True), "lout.bias": torch.full((1,), S, dtype=torch.float64),
               "layers.1.weight": w3.T * (s[:, None] * A1).sum(0)[None, :], "layers.1.bias": w3[0] * S,
               "layers.0.weight": c1.T * (s[:, None] * A0).sum(0)[None, :], "layers.0.bias": c1[0] * S}
    return {k: 2 * v.numpy() for k, v in out.items() if k in dec}
