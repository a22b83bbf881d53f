"""fp64 reference of `sdf_grad_at` (csrc/shine_device.cuh) with per-point bounds, and of the registration normal
equations built on it (`shine_register_normal_eq`, csrc/shine_register.cu).  Test infrastructure, no GPU needed.

sdf_grad_at returns pred = Decoder.sdf(f(q)), g = dpred/dq (before sigma) and valid (q's voxel exists at lv[0]).  The
reference restates it in fp64 from the kernel's fp32 inputs, term by term in the kernel's order; u = 2^-24, first-order
propagation of absolute values, every bound an fp64 array beside the value it bounds.
  * Weights.  t, u = 1 - t and w = (X Y) Z are the fp32 values of `axis_td` / `BlendD` (eikonal_bound.level_geometry,
    bit-equal to the oracle's interpolat).  dt = t'(d) res / 2 from the fp32 fraction: poly (6d - 6d^2) s, which nvcc
    may contract, so 3 u (6|d| + 6 d^2) s absolute; linear dt = s exactly.  grad w_c = (dX Y) Z etc., two roundings:
    e_dw = |Y Z| (e_dt + 4 u |dt|).  All as EikRef (eikonal_bound.py docstring, "dt" and "grad w"); here the res of
    each bottom-up position is its own world level, so descriptors whose levels are not consecutive are covered.
  * Gather.  f and J = sum_c F_c (x) grad w_c are 8L-term FMA chains over the levels that hit (misses add nothing):
    (8L + 2) u A0 for f, sum |F| e_dw + (8L + 2) u sum |F| |dw| for J: eikonal_bound.gather, reused as is.
    A0 = sum |w| |F| is error_bound.abs_feature (|w|: a q outside the cube can have a negative weight).
  * Forward.  pre1 = b1 + W1 f as an 8-term FMA chain from b1, pre2 = b2 + W2 h1 a 32-term chain, pred = b3 + w3 . h2 a
    32-term chain: with A1 = |W1| A0 + |b1|, A2 = |W2| (m1 A1) + |b2|, Ap = |w3| (m2 A2) + |b3|,
        e1 = |W1| (8L + 2) u A0 + (F + 2) u A1,  e2 = |W2| (m1 e1) + (H + 2) u A2,  P = |w3| (m2 e2) + (H + 2) u Ap
    (EikRef's e1, e2, P; error_bound.decoder_passes has the same passes with tensor-core contraction constants, which
    this FMA-chain kernel does not need).
  * dq = W1^T D1 W2^T D2 w3.  Per live unit n, a_n is a 32-term chain over the masked w3 (exact inputs: (H + 2) u),
    folded into dq by 8 FMAs, one chain of up to H terms per component: e_dq = (2H + 4) u D, D = |W1|^T m1 |W2|^T m2
    |w3| (EikRef's e_q).
  * g = J^T dq in 8 FMAs per axis: e_g = sum_k (e_J |dq| + |J| e_dq + e_J e_dq) + (F + 2) u sum_k J_abs |dq|.
ReLU kinks are graded, not dropped.  A unit is uncertain where |pre| <= 2 e (and its absolute pass is non-zero: an exact
0 is no kink).  Elsewhere the kernel's mask is the fp64 one.  For a point with uncertain units, every assignment of
their masks is an alternative: layer 1 first, then the layer-2 units uncertain under that assignment.  An alternative's
fp64 values use h = m' pre (the linear continuation), so a kernel that took that branch is within the alternative's own
bounds, which are formed with its masks.  The kernel's (pred, g) must lie within the bounds of at least one alternative.
A point with more than MAX_UNCERTAIN uncertain units is left out and counted (`dropped`).

Registration (`RegBound`).  The kernel forms gv = fl(sigma g) and r = fl(sigma pred), then in fp64 Jr = [g, q x g]
(products of fp32 values are exact, each difference one rounding), w = (k^2 / (k^2 + r^2))^2 (three roundings) and the
point's share: H_ij = (w Jr_i) Jr_j, b_i = (w Jr_i) r, cost = (w r) r, count 1.  Per point:
  * e_r = sigma P + u (|r| + sigma P), e_g = sigma e_g + u (|sigma g| + sigma e_g); e_Jr = [e_g, |q| x e_g crosswise];
  * w is monotone in |r|: e_w = max(w(|r| - e_r) - w, w - w(|r| + e_r)), exact, so a tiny kappa does not blow it up;
  * a product X = a c: e_X = e_a |c| + |a| e_c + e_a e_c; a share w X: e_w (|X| + e_X) + w e_X + 8 2^-53 (|w X| + ...);
  * kink points: per element the interval [min, max] over the alternatives of (share -+ its bound).
The sums are fp64: each thread adds its points in order (m = ceil(n / (256 G)) terms, G = min(ceil(n / 256), 1024)
blocks), a 5-level shuffle tree, the 8 warps in order (the block partial, one scratch row), then the fold: lane l adds
blocks l, l + 32, .. (ceil(G / 32) terms) and a 5-level shuffle tree.  A term passes at most
    depth(n) = m + 5 + 8 + ceil(G / 32) + 5
roundings of 2^-53 (block partials m + 13), so |got - want| <= sum of the point bounds + (depth + 2) 2^-53 sum (|share| +
bound).  This replaces the flat 8 (n + 8) 2^-53 that test_gpu_odometry's RegRef used.  The count must be exact."""
from __future__ import annotations

import itertools

import numpy as np

from tests.eikonal_bound import _decoder, gather, level_geometry
from tests.error_bound import H, U, oracle64

E64 = 2.0 ** -53
MAX_UNCERTAIN = 4
REG_THREADS = 256
REG_MAX_BLOCKS = 1024
REG_OUT = 29


def reg_blocks(n):
    return max(1, min(-(-n // REG_THREADS), REG_MAX_BLOCKS))


def sum_depth(n):
    """fp64 roundings a term of the registration sums passes (module docstring)."""
    G = reg_blocks(n)
    m = -(-n // (G * REG_THREADS))
    return m + 5 + 8 + -(-G // 32) + 5


def block_depth(n):
    G = reg_blocks(n)
    return -(-n // (G * REG_THREADS)) + 5 + 8


class _Net:
    """The decoder as fp64 numpy with the passes of the module docstring, batched over rows (point, alternative)."""

    def __init__(self, dec, L, F):
        self.W1, self.b1, self.W2, self.b2, self.w3, self.b3 = _decoder(dec)
        self.aW1, self.aW2, self.aw3 = np.abs(self.W1), np.abs(self.W2), np.abs(self.w3)
        self.L, self.F = L, F

    def layer1(self, f, A0):
        pre1 = f @ self.W1.T + self.b1
        A1 = A0 @ self.aW1.T + np.abs(self.b1)
        e1 = ((8 * self.L + 2) * U * A0) @ self.aW1.T + (self.F + 2) * U * A1
        return pre1, A1, e1

    def layer2(self, pre1, A1, e1, m1):
        pre2 = (m1 * pre1) @ self.W2.T + self.b2
        A2 = (m1 * A1) @ self.aW2.T + np.abs(self.b2)
        e2 = (m1 * e1) @ self.aW2.T + (H + 2) * U * A2
        return pre2, A2, e2

    def out(self, pre2, A2, e2, m1, m2, J, Jabs, eJ):
        """-> pred, P, g, e_g of rows with masks m1, m2 (J, Jabs, eJ [M, F, 3] of each row's point)."""
        pred = (m2 * pre2) @ self.w3 + self.b3
        Ap = (m2 * A2) @ self.aw3 + abs(self.b3)
        P = (m2 * e2) @ self.aw3 + (H + 2) * U * Ap
        dq = (m1 * ((m2 * self.w3) @ self.W2)) @ self.W1
        edq = (2 * H + 4) * U * ((m1 * ((m2 * self.aw3) @ self.aW2)) @ self.aW1)
        g = np.einsum("nfa,nf->na", J, dq)
        eg = (np.einsum("nfa,nf->na", eJ, np.abs(dq)) + np.einsum("nfa,nf->na", np.abs(J) + eJ, edq) +
              (self.F + 2) * U * np.einsum("nfa,nf->na", Jabs, np.abs(dq)))
        return pred, P, g, eg


def uncertain(pre, A, e):
    return (np.abs(pre) <= 2 * e) & (A > 0)


class GradRef:
    """fp64 pred, g (before sigma), valid and their bounds at fp32 points `coord` (module docstring).

    Rows are (point, alternative): `pt` [M] the point of each row, `pred`, `P` [M], `g`, `eg` [M, 3].  A point without
    uncertain units has one row; `kink` [n] marks points with several, `dropped` [n] the points left out (no rows).
    `levels`: the world level of each bottom-up position (default: the oracle's `kept`, else max_level - i)."""

    def __init__(self, case, coord, levels=None, max_uncertain=MAX_UNCERTAIN):
        o, dec = oracle64(case)
        coord = np.ascontiguousarray(coord, dtype=np.float32)
        n = coord.shape[0]
        L, F = o.featured_level_num, o.feature_dim
        levels = levels if levels is not None else getattr(o, "kept", None)
        self.n, self.coord = n, coord
        geo = level_geometry(o, coord, levels=levels)
        self.valid = geo[0]["ix"][:, 0] >= 0
        self.hits = np.stack([g["ix"][:, 0] >= 0 for g in geo], 1)
        f, A0, J, Jabs, eJ = gather(o, geo)
        net = _Net(dec, L, F)
        pre1, A1, e1 = net.layer1(f, A0)
        m1 = (pre1 > 0).astype(np.float64)
        pre2, A2, e2 = net.layer2(pre1, A1, e1, m1)
        m2 = (pre2 > 0).astype(np.float64)
        u1, u2 = uncertain(pre1, A1, e1), uncertain(pre2, A2, e2)
        cand = np.flatnonzero(u1.any(1) | u2.any(1))
        plain = np.setdiff1d(np.arange(n), cand)
        # rows: every plain point once, then the alternatives of each candidate
        r_pt, r_m1, r_m2 = [plain], [m1[plain]], [m2[plain]]
        dropped = np.zeros(n, dtype=bool)
        kink = np.zeros(n, dtype=bool)
        for p in cand:
            rows1 = []
            idx1 = np.flatnonzero(u1[p])
            for bits in itertools.product((0.0, 1.0), repeat=idx1.size):
                mm = m1[p].copy()
                mm[idx1] = bits
                rows1.append(mm)
            M1 = np.stack(rows1)
            q2, a2, ee2 = net.layer2(pre1[p][None], A1[p][None], e1[p][None], M1)
            alts, too_many = [], False
            for k in range(M1.shape[0]):
                idx2 = np.flatnonzero(uncertain(q2[k], a2[k], ee2[k]))
                if idx1.size + idx2.size > max_uncertain:
                    too_many = True
                    break
                base2 = (q2[k] > 0).astype(np.float64)
                for bits in itertools.product((0.0, 1.0), repeat=idx2.size):
                    mm2 = base2.copy()
                    mm2[idx2] = bits
                    alts.append((M1[k], mm2))
            if too_many:
                dropped[p] = True
                continue
            kink[p] = len(alts) > 1
            r_pt.append(np.full(len(alts), p))
            r_m1.append(np.stack([a for a, _ in alts]))
            r_m2.append(np.stack([b for _, b in alts]))
        pt = np.concatenate(r_pt).astype(np.int64)
        M1, M2 = np.concatenate(r_m1), np.concatenate(r_m2)
        order = np.argsort(pt, kind="stable")
        pt, M1, M2 = pt[order], M1[order], M2[order]
        q2, a2, ee2 = net.layer2(pre1[pt], A1[pt], e1[pt], M1)
        self.pred, self.P, self.g, self.eg = net.out(q2, a2, ee2, M1, M2, J[pt], Jabs[pt], eJ[pt])
        self.pt, self.kink, self.dropped = pt, kink, dropped
        self.kinks, self.n_dropped = int(kink.sum()), int(dropped.sum())
        self.alternatives = int(pt.size)

    def row_ratio(self, got_g, got_pred=None):
        """per row: the largest |got - want| / bound over g (and pred) of the row's point"""
        gg = np.asarray(got_g, dtype=np.float64)[self.pt]
        err = np.abs(gg - self.g) / np.where(self.eg > 0, self.eg, 1e-300)
        r = err.max(1)
        if got_pred is not None:
            pp = np.asarray(got_pred, dtype=np.float64)[self.pt]
            r = np.maximum(r, np.abs(pp - self.pred) / np.where(self.P > 0, self.P, 1e-300))
        return r

    def grade(self, got_g, what, got_pred=None, points=None, tag="grad bounds"):
        """Every graded point's g (and pred) within the bounds of one of its alternatives -> worst ratio (printed)."""
        best = np.full(self.n, np.inf)
        np.minimum.at(best, self.pt, self.row_ratio(got_g, got_pred))
        sel = ~self.dropped if points is None else (np.asarray(points, bool) & ~self.dropped)
        bad = np.flatnonzero(sel & ~(best <= 1.0))
        if bad.size:
            i = bad[0]
            rows = np.flatnonzero(self.pt == i)
            raise AssertionError(
                f"{what}: g outside its bound at {bad.size} of {int(sel.sum())} points; first {i} (kink {self.kink[i]}, "
                f"{rows.size} alternatives): got {np.asarray(got_g)[i]} want {self.g[rows[0]]} bound {self.eg[rows[0]]}")
        worst = float(best[sel].max()) if sel.any() else 0.0
        print(f"[{tag}] {what}: worst {worst:.3f} of the bound, {int(sel.sum())} points graded "
              f"({int((self.kink & sel).sum())} kink, {self.n_dropped} left out with > {MAX_UNCERTAIN} uncertain units)")
        return worst


def gm_weight(r2, k2):
    wk = k2 / (k2 + r2)
    return wk * wk


def shares(g, r, q, kappa2):
    """The fp64 tail of the register kernel, op for op: [M, 28] (21 H, 6 b, cost) from gv = sigma g, r, q (fp64 arrays
    of fp32 values)."""
    g0, g1, g2 = g[:, 0], g[:, 1], g[:, 2]
    q0, q1, q2 = q[:, 0], q[:, 1], q[:, 2]
    Jr = [g0, g1, g2, q1 * g2 - q2 * g1, q2 * g0 - q0 * g2, q0 * g1 - q1 * g0]
    w = gm_weight(r * r, kappa2)
    out = []
    for i in range(6):
        wi = w * Jr[i]
        out += [wi * Jr[j] for j in range(i, 6)]
    out += [w * Jr[i] * r for i in range(6)]
    out.append(w * r * r)
    return np.stack(out, 1)


class RegBound:
    """Per point, the interval of its 28 fp64 shares (module docstring) from a GradRef at q = coord, the fp32 sigma the
    kernel gets and kappa (scaled units).  `expect(idx)` sums it over the launched points idx (indices into the ref's
    points, repeats allowed)."""

    def __init__(self, ref, sigma, kappa):
        self.ref = ref
        sigma = float(np.float32(sigma))
        k2 = float(kappa) * float(kappa)
        pt = ref.pt
        q = ref.coord.astype(np.float64)[pt]
        r = sigma * ref.pred
        er = sigma * ref.P + U * (np.abs(r) + sigma * ref.P)
        g = sigma * ref.g
        eg = sigma * ref.eg + U * (np.abs(g) + sigma * ref.eg)
        aq = np.abs(q)
        J = [g[:, 0], g[:, 1], g[:, 2], q[:, 1] * g[:, 2] - q[:, 2] * g[:, 1], q[:, 2] * g[:, 0] - q[:, 0] * g[:, 2],
             q[:, 0] * g[:, 1] - q[:, 1] * g[:, 0]]
        eJ = [eg[:, 0], eg[:, 1], eg[:, 2], aq[:, 1] * eg[:, 2] + aq[:, 2] * eg[:, 1],
              aq[:, 2] * eg[:, 0] + aq[:, 0] * eg[:, 2], aq[:, 0] * eg[:, 1] + aq[:, 1] * eg[:, 0]]
        eJ = [e + 2 * E64 * np.abs(j) for e, j in zip(eJ, J)]
        w = gm_weight(r * r, k2)
        ar = np.abs(r)
        ew = np.maximum(gm_weight(np.maximum(ar - er, 0.0) ** 2, k2) - w, w - gm_weight((ar + er) ** 2, k2)) + 4 * E64 * w

        def prod(a, ea, c, ec):
            X = np.abs(a * c)
            eX = ea * np.abs(c) + np.abs(a) * ec + ea * ec
            return ew * (X + eX) + w * eX + 8 * E64 * w * (X + eX)

        eb = []
        for i in range(6):
            eb += [prod(J[i], eJ[i], J[j], eJ[j]) for j in range(i, 6)]
        eb += [prod(J[i], eJ[i], r, er) for i in range(6)]
        eb.append(prod(r, er, r, er))
        val = shares(g, r, q, k2)
        e = np.stack(eb, 1)
        n = ref.n
        lo = np.full((n, 28), np.inf)
        hi = np.full((n, 28), -np.inf)
        np.minimum.at(lo, pt, val - e)
        np.maximum.at(hi, pt, val + e)
        use = ref.valid & ~ref.dropped
        lo[~use], hi[~use] = 0.0, 0.0
        self.mid, self.half = 0.5 * (lo + hi), 0.5 * (hi - lo)
        self.count = use.astype(np.float64)
        self.sigma, self.kappa = sigma, float(kappa)

    def sums(self, idx, weights=None):
        """(want [29], point-bound part [28], sum |share| + bound [28]) over the launched points idx"""
        c = np.bincount(np.asarray(idx, dtype=np.int64), minlength=self.ref.n).astype(np.float64)
        want = np.concatenate((c @ self.mid, [c @ self.count]))
        return want, c @ self.half, c @ (np.abs(self.mid) + self.half)

    def expect(self, idx, n_launched=None):
        """-> (want [29], bound [29]) of the kernel's out for launched points idx (count bound 0: exact)"""
        n = len(idx) if n_launched is None else n_launched
        want, half, mag = self.sums(idx)
        return want, np.concatenate((half + (sum_depth(n) + 2) * E64 * mag, [0.0]))

    def expect_blocks(self, idx):
        """-> (want [G, 29], bound [G, 29]) of the kernel's block partials (the scratch rows) for launched points idx"""
        idx = np.asarray(idx, dtype=np.int64)
        n = idx.size
        G = reg_blocks(n)
        blk = (np.arange(n) // REG_THREADS) % G
        want = np.zeros((G, 29))
        half = np.zeros((G, 28))
        mag = np.zeros((G, 28))
        for s in range(0, n, 1 << 17):
            b, p = blk[s:s + (1 << 17)], idx[s:s + (1 << 17)]
            np.add.at(want[:, :28], b, self.mid[p])
            np.add.at(want[:, 28], b, self.count[p])
            np.add.at(half, b, self.half[p])
            np.add.at(mag, b, np.abs(self.mid[p]) + self.half[p])
        bound = np.concatenate((half + (block_depth(n) + 2) * E64 * mag, np.zeros((G, 1))), 1)
        return want, bound


def grade_reg(got, want, bound, what, tag="register bounds"):
    """count exact, the 28 sums within their bounds -> worst ratio (printed)"""
    got, want, bound = (np.asarray(x, dtype=np.float64) for x in (got, want, bound))
    assert np.array_equal(got[..., 28], want[..., 28]), f"{what}: count {got[..., 28]} != {want[..., 28]}"
    err = np.abs(got[..., :28] - want[..., :28])
    bad = np.argwhere(~(err <= bound[..., :28]))
    names = [f"H{i}{j}" for i in range(6) for j in range(i, 6)] + [f"b{i}" for i in range(6)] + ["cost"]
    if bad.size:
        i = tuple(bad[0])
        raise AssertionError(f"{what}: {bad.shape[0]} sums outside the bound; first {names[i[-1]]} at {i}: got "
                             f"{got[..., :28][i]:.17g} want {want[..., :28][i]:.17g} bound {bound[..., :28][i]:.3g}")
    worst = float((err / np.where(bound[..., :28] > 0, bound[..., :28], 1.0)).max()) if err.size else 0.0
    print(f"[{tag}] {what}: worst {worst:.3f} of the bound, count {int(np.sum(want[..., 28]))}")
    return worst
