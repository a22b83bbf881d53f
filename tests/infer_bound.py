"""The fp64 reference and per-element bounds of the forward-only kernels (`shine_sdf_infer`, `shine_mesh_grid`,
`shine_sdf_fwd` / `shine_sdf_bce_fwd`).  Test infrastructure, no GPU needed.

Pred.  The fp64 oracle is error_bound.oracle64 (tables and decoder in fp64, the fp32 blend weights of the kernels) and the
bound P of error_bound.decoder_passes: the fp32 blend, three contractions (3xTF32 or, with tf32x1, plain TF32) and the
bias adds on the absolute-value passes.  A point within twice the forward error of a ReLU kink gets the kink bound (the
pass with the uncertain units live), so every point is graded.

Loss (`out_loss` of shine_sdf_fwd).  With s the loss scale (1 / n for a mean, 1 for a sum) and w_i the point's weight
(|weight| when weighted, else 1), the kernel adds fl(w_i l_i) over the lanes of a warp, sums each warp's lanes with
shuffles, multiplies by fl(s) and adds the warps' partials atomically.  Against the fp64 loss sum_i s w_i l_i(pred64_i):
  * the pred error: |l(p) - l(p64)| <= |dl/dp| P with |dl/dp| evaluated at p64 and widened by the curvature over P
    (BCE: |d2l/dp2| <= 1/4; sdf_l1: 1 / scale; sdf_l2: (2 |p64 - label| + P) / scale^2);
  * BCE's MUFU intrinsics, from the CUDA C Programming Guide's accuracy table (ulp(x) <= 2 u |x|):
      __fdividef  2 ulp;  __expf(x)  2 + floor(1.173 |x|) ulp;  __logf(x) for x in [0.5, 2]  2^-21.41 absolute.
    zt = 1 / (1 + __expf(-__fdividef(label, sigma))): the quotient's 2 ulp grow by |a| through exp (a = label / sigma),
    exp adds its own ulp, 1 + E one rounding, the reciprocal 2 ulp; dzt/dE = -zt (1 - zt) / E, so
        |zt - zt64| <= zt (1 - zt) ((2 + 1.173 |a|) 2u + 4u |a| + u) + 4u zt,
    and the term carries |p| times that.  e = __expf(-|p|) is off by (2 + 1.173 |p|) 2u e, log(1 + e) by 2^-21.41 + u
    (the add) + that e error (dlog/de <= 1);
  * the assembly max(p, 0) - p zt + log(1 + e): up to 3 roundings of its absolute parts; sdf_l1: the subtraction and the
    division, 2u |d|; sdf_l2: 5u d^2 (d = (p - label) / scale);
  * the summation: n fp32 adds in any order, the product by w_i and the product by fl(s) (fl(s) itself one rounding): at
    most (n + C) u sum_i |term_i|, C = C_SLACK, with |term_i| = s w_i |l_i| widened by its own bound.
All first order in u; C covers the rest."""
from __future__ import annotations

import numpy as np
import torch

from tests.error_bound import C_SLACK, U, abs_feature, decoder_passes, oracle64

LOG_ABS = 2.0 ** -21.41        # __logf on [0.5, 2], absolute
EXP_ULP0, EXP_ULP1 = 2.0, 1.173  # __expf(x): 2 + floor(1.173 |x|) ulp
DIV_ULP = 2.0                  # __fdividef


class PredRef:
    """pred64, P, kink and the oracle's corner rows (bottom-up [n, 8] per level) of a case's coordinates."""

    def __init__(self, case, coord=None, tf32x1=False):
        o, dec = oracle64(case)
        self.o, self.dec = o, {k: v.detach() for k, v in dec.items()}
        coord = torch.from_numpy(np.ascontiguousarray(case["coord"] if coord is None else coord, dtype=np.float32))
        with torch.no_grad():
            feat = o.query_feature(coord)
            self.indices = [t.numpy().copy() for t in o.hierarchical_indices]
            absfeat = abs_feature(o, coord)
            dp = decoder_passes(feat, absfeat, self.dec, tf32x1, o.featured_level_num)
            self.pred = self.sdf(feat)
        self.P, self.kink = dp["P"].numpy(), dp["kink"].numpy()
        self.n = coord.shape[0]

    def sdf(self, feat):
        from oracle.shine_oracle import decoder_sdf
        return decoder_sdf(feat, self.dec).numpy()

    def masks(self):
        """the validity mask at every mask level (index into the bottom-up levels): all 8 corner rows present"""
        return [(ix >= 0).all(1) for ix in self.indices]

    def grade(self, got, what, sign=1.0, tag="infer bounds"):
        """|got - sign pred64| <= P at every point -> worst ratio (printed with the number of graded points)."""
        got = np.asarray(got, dtype=np.float64)
        err = np.abs(got - sign * self.pred)
        bad = np.flatnonzero(~(err <= self.P))
        if bad.size:
            i = bad[0]
            raise AssertionError(f"{what}: pred outside its bound at {bad.size} of {self.n} points; first {i}: got "
                                 f"{got[i]:.9g} want {sign * self.pred[i]:.9g} bound {self.P[i]:.3g} (kink {self.kink[i]})")
        worst = float((err / np.where(self.P > 0, self.P, 1.0)).max()) if err.size else 0.0
        print(f"[{tag}] {what}: pred worst {worst:.3f} of the bound, {self.n} points graded ({int(self.kink.sum())} kink)")
        return worst

    def grade_masks(self, got_masks, what, levels=None, tag="infer bounds"):
        """got_masks[k] for mask level k (levels: which k were run): exactly the oracle's."""
        want = self.masks()
        levels = range(len(want)) if levels is None else levels
        for k, got in zip(levels, got_masks):
            got = np.asarray(got).astype(bool)
            bad = np.flatnonzero(got != want[k])
            assert bad.size == 0, f"{what}: mask level {k} differs at {bad.size} points; first {bad[0]}: got {got[bad[0]]}"
        print(f"[{tag}] {what}: masks exact at levels {list(levels)}, {self.n} points, "
              f"{[int(want[k].sum()) for k in levels]} present")


def loss_terms(pred64, P, label, weight, loss_type, sigma=1.0, scale=1.0, weighted=False, reduction="mean"):
    """-> (terms64 [n]: s w_i l_i(pred64_i), point bounds [n], s) of the module docstring.  sigma / scale as the kernel
    receives them (fp32)."""
    p = np.asarray(pred64, dtype=np.float64)
    P = np.asarray(P, dtype=np.float64)
    lb = np.asarray(label, dtype=np.float32).astype(np.float64)
    n = p.shape[0]
    if loss_type == "sdf_bce":
        w = np.abs(np.asarray(weight, dtype=np.float64)) if weighted else np.ones(n)
        s = 1.0 if reduction == "sum" else 1.0 / n
        sigma = float(np.float32(sigma))
        a = lb / sigma
        zt = 0.5 * (1.0 + np.tanh(0.5 * a))                                # sigmoid(a), no overflow
        ap = np.abs(p) + P
        e = np.exp(-np.abs(p))
        log1p_e = np.log1p(e)
        li = np.maximum(p, 0.0) - p * zt + log1p_e
        g = 0.5 * (1.0 + np.tanh(0.5 * p)) - zt                            # dl/dp = sigmoid(p) - zt
        e_zt = zt * (1 - zt) * ((EXP_ULP0 + EXP_ULP1 * np.abs(a)) * 2 * U + 2 * DIV_ULP * U * np.abs(a) + U) + \
            2 * DIV_ULP * U * zt
        e_e = (EXP_ULP0 + EXP_ULP1 * ap) * 2 * U * np.exp(-np.maximum(np.abs(p) - P, 0.0))
        e_log = LOG_ABS + U + e_e
        parts = np.maximum(p, 0.0) + ap * zt + log1p_e + P
        per = (np.abs(g) + P / 4) * P + ap * e_zt + e_log + 3 * U * parts
    elif loss_type in ("sdf_l1", "sdf_l2"):
        w = np.abs(np.asarray(weight, dtype=np.float64))
        s = 1.0 / n
        scale = float(np.float32(scale))
        d = np.abs(p - lb) / scale
        dP = P / scale
        if loss_type == "sdf_l1":
            li = d
            per = dP + 2 * U * (d + dP)
        else:
            li = d * d
            per = dP * (2 * d + dP) + 5 * U * (d + dP) ** 2
    else:
        raise ValueError(loss_type)
    return s * w * li, s * w * per, s


class LossRef:
    """The fp64 loss of a batch and its bound: sum of the point bounds + (n + C) u sum |term| (module docstring)."""

    def __init__(self, pred64, P, label, weight, loss_type, slack=C_SLACK, **kw):
        self.terms, self.per, self.s = loss_terms(pred64, P, label, weight, loss_type, **kw)
        self.n, self.loss_type = self.terms.shape[0], loss_type
        self.want = float(self.terms.sum())
        self.sum_abs = float((np.abs(self.terms) + self.per).sum())
        self.summation = (self.n + slack) * U * self.sum_abs
        self.bound = float(self.per.sum()) + self.summation

    def grade(self, got, what, tag="infer bounds"):
        err = abs(float(got) - self.want)
        assert err <= self.bound, (f"{what}: {self.loss_type} loss {float(got):.9g} vs fp64 {self.want:.9g}: error {err:.3g} "
                                   f"outside the bound {self.bound:.3g} (points {self.per.sum():.3g}, summation "
                                   f"{self.summation:.3g})")
        worst = err / self.bound
        print(f"[{tag}] {what}: {self.loss_type} loss worst {worst:.3f} of the bound, {self.n} points graded")
        return worst
