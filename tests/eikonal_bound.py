"""fp64 reference of the eikonal paths with per-element error bounds: the fused eikonal step (csrc/shine_eikonal.cu), the
class-surface recipe (`batch_loop.eikonal_iteration`) and the query kernels it is built from (query_fwd, query_coord_grad,
query_tangent_fwd, query_tangent_bwd).  Test infrastructure, no GPU needed.

The reference is an explicit restatement of the math in the header of shine_eikonal.cu, not autograd: the coordinates stay
fp32 for the lookup, and autograd would then differentiate the blend weights in fp32.  Per point j, level l, corner c:
  * lookup and weights: the oracle's corner rows and fp32 blend weights w (bit-equal to the kernels');
  * fraction d = c - trunc(c), c = fp32(res fp32(0.5 x + 0.5)) (exact, as axis_t), then t'(d) = 6d - 6d^2 (poly) or 1,
    dt = t'(d) res / 2 and grad w_c = (+-dt_x) Y Z, ... in fp64 with the fp32 blend factors Y, Z;
  * f, J = sum_c F_c (x) grad w_c, the decoder forward (masks m1, m2, pred), dp = dL/dpred, a2 = m2 w3, a1 = m1 W2^T a2,
    q = W1^T a1, g = sigma J^T q, |g|, gamma = 2 weight_e / N_surf (|g| - 1) g / |g|, and the scatter coefficient
    sc = dp w + sigma gamma . grad w: row u of a table gets sum_{(j,c) -> u} sc_{j,c} q_j.  Also the loss and eikonal
    scalars.
With `exact=True` the coordinates are fp64 too (t and w in fp64): that is the reference's autograd recipe in fp64.

Error model (extends the one in the docstring of tests/test_gpu_replicas.py; first-order propagation of absolute values,
u = 2^-24, every bound an fp64 array beside the value it bounds):
  * dt: fp32 (6d - 6d^2) s with s = res / 2 exact; nvcc may contract it into FMAs, so the bound is on absolute values,
    3 u (6|d| + 6 d^2) s, not relative to dt (near d -> 1 the subtraction cancels).  Linear: dt = s exactly.
    grad w = dX Y Z (two products; Y, Z within an ulp of the oracle's): e_dw = |Y Z| (e_dt + 4 u |dt|);
  * gather: f and J are 8L-term FMA chains: (8L + 2) u sum |w| |F| for f; J is off by sum |F| e_dw + (8L + 2) u sum |F| |dw|;
  * decoder: the fused eikonal step runs it as fp32 FMA chains (K-term chain: (K + 2) u of the sum of |terms|), the class
    surface as cuBLAS fp32 GEMMs with TF32 off, any-order K-term sums: the same (K + 2) u.  With A0 = sum w |F|,
    A1 = |W1| A0 + |b1|, A2 = |W2| (m1 A1) + |b2|, Ap = |w3| (m2 A2) + |b3|: e1 = |W1| e_f + (F + 2) u A1,
    e2 = |W2| (m1 e1) + (H + 2) u A2, P = |w3| (m2 e2) + (H + 2) u Ap bounds pred;
  * q: two 32-term chains on exact inputs: e_q = (2H + 4) u D, D = |W1|^T (m1 |W2|^T (m2 |w3|)) (as the replica model);
  * g = sigma J^T q: sigma (sum_k (e_J,k + (F + 8) u J_abs,k) |q_k| + |J_k| e_q,k) + 2 u |g| (the coordinate-gradient kernel
    sums the same terms in another order: per lane, then over the LP lanes of a point; sigma is rounded to fp32);
  * |g|: e_n = ||e_g|| + 3 u |g|.  gamma: coef = ce (|g| - 1) / |g|, ce = 2 weight_e / N_surf; where |g| > 2 e_n the
    division is off by at most 2 e_n / |g|^2 of ce, so e_coef = 2 |ce| e_n / |g|^2 + 6 u |coef|, and
    e_gamma = |coef| e_g + e_coef |g| + 4 u |gamma|;
  * dp: the rules of the replica model with P as above (BCE with the fast intrinsics, sdf_l2, sdf_l1 with the kernel's sign
    near the label);
  * sc: its two parts are bounded apart: e_sc1 = |w| e_dp + u |sc1| (sc1 = dp w) and e_sc2 = sigma sum_a (e_gamma,a |dw_a| +
    |gamma_a| e_dw,a) + 4 u sigma sum_a |gamma_a dw_a| + u |sc2|; the table rows then follow the k_u + C rule of the replica
    model with S = sum (|sc1| + |sc2|) |q| (a path may add the two parts apart) and T = sum (|sc1| + |sc2|) e_q + e_sc |q|.
    The class surface adds the parts apart (query_bwd of dp q, tangent_bwd of sigma gamma with q): both term sets count;
  * loss and eikonal scalars: sum |term errors| + (tiles + 8) u sum |terms| (a lane's running sum, five shuffles and the
    atomics of its warp; the class surface: (n + 8) u).  BCE terms use the fast intrinsics: per term
    |w| (P + 2^-21 + (12 + 2 |label / sigma|) u (1 + |pred|)).
Points left out, as the replica tests leave out ReLU kinks: points within twice the forward error of a ReLU kink, and
surface points with |g| <= 2 e_n (there g / |g| is ill-conditioned; the kernel's `nrm > 0 ? ... : 0` is the torch
subgradient).  `clean_case` drops them from the batch before the step runs.

The query kernels get the same treatment: query_fwd f = sum w F with (8L + 2) u A0; coord_grad G = sum grad w_c <F_c, d> with
sum (e_dw |F_c| |d| + (8L + F + 8) u |dw| |F_c| |d|); tangent_fwd sum (t . grad w_c) F_c with W_c = t . grad w_c off by
e_W = sum |t_a| e_dw,a + 3 u sum |t_a dw_a| and (8L + 2) u sum |t| |dw| |F| of rounding; tangent_bwd rows sum W_c d_j by
the k_u + C rule with T = sum e_W |d|.
"""
from __future__ import annotations

import numpy as np
import torch

from tests import sdf_diff_oracle as sdo
from tests.error_bound import C_SLACK, H, U, RowSums, grade_values, oracle64, subset


def _scale(case):
    """config.scale of a case (sdf_diff_loss): 1 / (leaf_vox_size 2^(tree_level_world - 1))."""
    c = case["cfg"]
    return 1.0 / (c["leaf_vox_size"] * 2 ** (c["tree_level_world"] - 1))


# ---- blend weights and their derivatives -----------------------------------------------------------------------------------

def level_geometry(o, coord, exact=False, levels=None):
    """Per level, bottom-up: dict(level, ix [N, 8] rows (-1: miss), w [N, 8], dw [N, 8, 3], edw [N, 8, 3]) as fp64 numpy.
    coord: fp32 array (exact=False: fp32 weights and factors, dt in fp64 from the fp32 fraction) or an fp64 array of
    fp32-representable points (exact=True: everything in fp64, edw = 0).  The rows come from the fp32 coordinates.
    levels: the world level of each bottom-up position when they are not max_level - i (an oracle of levels that are not
    consecutive, whose get_indices and interpolat already use them)."""
    c32 = torch.from_numpy(np.asarray(coord, dtype=np.float32))
    idx = o.get_indices(c32)
    poly = o.polynomial_interpolation
    out = []
    for i in range(o.featured_level_num):
        level = o.max_level - i
        res = 2.0 ** (level if levels is None else levels[i])
        if exact:
            x = np.asarray(coord, dtype=np.float64)
            cc = res * (x * 0.5 + 0.5)
            d = cc - np.trunc(cc)
            t = 3 * d ** 2 - 2 * d ** 3 if poly else d
            u = 1 - t
        else:
            cc = res * (c32 * 0.5 + 0.5)                    # the oracle's interpolat, op for op
            d32 = torch.frac(cc)
            t32 = 3 * (d32 ** 2) - 2 * (d32 ** 3) if poly else d32
            d, t, u = d32.double().numpy(), t32.double().numpy(), (1 - t32).double().numpy()
        s = res * 0.5
        if poly:
            dt = (6 * d - 6 * d * d) * s
            edt = 0.0 if exact else 3 * U * (6 * np.abs(d) + 6 * d * d) * s
        else:
            dt = np.full_like(d, s)
            edt = np.zeros_like(d)
        n = d.shape[0]
        w = np.empty((n, 8)); dw = np.empty((n, 8, 3)); edw = np.zeros((n, 8, 3))
        for c in range(8):
            bits = ((c >> 2) & 1, (c >> 1) & 1, c & 1)
            fac = [t[:, a] if bits[a] else u[:, a] for a in range(3)]
            sgn = [1.0 if bits[a] else -1.0 for a in range(3)]
            w[:, c] = fac[0] * fac[1] * fac[2]
            for a in range(3):
                other = fac[(a + 1) % 3] * fac[(a + 2) % 3]
                dw[:, c, a] = sgn[a] * dt[:, a] * other
                if not exact:
                    edw[:, c, a] = np.abs(other) * (edt[:, a] + 4 * U * np.abs(dt[:, a]))
        if not exact:     # the kernels' weights are the oracle's fp32 values
            w = o.interpolat(c32, level, poly).reshape(n, 8).double().numpy()
        ix = idx[i].numpy()
        miss = ix[:, 0] < 0
        w[miss], dw[miss], edw[miss] = 0.0, 0.0, 0.0
        out.append({"level": level, "ix": ix, "w": w, "dw": dw, "edw": edw})
    return out


def _rows(o, kk, ix):
    """Table kk's rows of the corner ids ix (fp64 numpy), zero for a miss."""
    t = o.hier_features[kk].detach().double().numpy()
    r = t[np.where(ix >= 0, ix, t.shape[0] - 1)]
    r[ix < 0] = 0.0
    return r


def gather(o, geo):
    """f, A0, J [N, F, 3], J_abs, e_J of the module docstring (fp64 numpy)."""
    L = o.featured_level_num
    F = o.feature_dim
    n = geo[0]["w"].shape[0]
    f = np.zeros((n, F)); A0 = np.zeros((n, F))
    J = np.zeros((n, F, 3)); Jabs = np.zeros((n, F, 3)); eJ = np.zeros((n, F, 3))
    for i, g in enumerate(geo):
        R = _rows(o, L - 1 - i, g["ix"])                          # [N, 8, F]
        f += np.einsum("nc,ncf->nf", g["w"], R)
        A0 += np.einsum("nc,ncf->nf", np.abs(g["w"]), np.abs(R))
        J += np.einsum("ncf,nca->nfa", R, g["dw"])
        Jabs += np.einsum("ncf,nca->nfa", np.abs(R), np.abs(g["dw"]))
        eJ += np.einsum("ncf,nca->nfa", np.abs(R), g["edw"])
    eJ += (8 * L + 2) * U * Jabs
    return f, A0, J, Jabs, eJ


# ---- the eikonal step ----------------------------------------------------------------------------------------------------------

def _decoder(dec):
    """W1, b1, W2, b2, w3, b3 as fp64 numpy (zero biases for a decoder without them)."""
    get = {k: v.detach().double().numpy() for k, v in dec.items()}
    W1, W2, w3 = get["layers.0.weight"], get["layers.1.weight"], get["lout.weight"].reshape(-1)
    b1 = get.get("layers.0.bias", np.zeros(W1.shape[0]))
    b2 = get.get("layers.1.bias", np.zeros(W2.shape[0]))
    b3 = float(get["lout.bias"].reshape(-1)[0]) if "lout.bias" in get else 0.0
    return W1, b1, W2, b2, w3, b3


class EikRef:
    """fp64 reference of one eikonal step of a case with the bounds of the module docstring.

    weight_e: the step's; loss_type: its first term; pred: the kernel's pred (sdf_l1: its sign near the label);
    n_surface: the eikonal mean's denominator (default: the batch's surface count); exact: fp64 coordinates;
    class_surface: bound the class-surface recipe (the two scatter parts added apart, torch sums of n terms)."""

    def __init__(self, case, weight_e=0.1, loss_type="sdf_bce", pred=None, n_surface=None, exact=False,
                 class_surface=False):
        c = case["cfg"]
        o, dec = oracle64(case)
        coord = np.asarray(case["coord"], dtype=np.float64 if exact else np.float32)
        label = np.asarray(case["label"], dtype=np.float64)
        weight = np.asarray(case["weight"], dtype=np.float64)
        n, L, F = coord.shape[0], c["tree_level_feat"], c["feature_dim"]
        sigma = float(c["sigma"])
        self.n, self.L, self.F, self.sigma, self.weight_e, self.loss_type = n, L, F, sigma, weight_e, loss_type
        self.geo = geo = level_geometry(o, coord, exact)
        f, A0, J, Jabs, eJ = gather(o, geo)
        W1, b1, W2, b2, w3, b3 = _decoder(dec)

        # ---- decoder forward and its absolute-value passes
        pre1 = f @ W1.T + b1
        m1 = (pre1 > 0).astype(np.float64)
        h1 = pre1 * m1
        pre2 = h1 @ W2.T + b2
        m2 = (pre2 > 0).astype(np.float64)
        pred64 = (pre2 * m2) @ w3 + b3
        A1 = A0 @ np.abs(W1).T + np.abs(b1)
        A2 = (m1 * A1) @ np.abs(W2).T + np.abs(b2)
        Ap = (m2 * A2) @ np.abs(w3) + abs(b3)
        e1 = ((8 * L + 2) * U * A0) @ np.abs(W1).T + (F + 2) * U * A1
        e2 = (m1 * e1) @ np.abs(W2).T + (H + 2) * U * A2
        P = (m2 * e2) @ np.abs(w3) + (H + 2) * U * Ap
        self.kink = (np.abs(pre1) <= 2 * e1).any(1) | (np.abs(pre2) <= 2 * e2).any(1)
        self.pred, self.P = pred64, P

        # ---- q = dpred / df, g = sigma J^T q
        a1 = m1 * ((m2 * w3) @ W2)
        q = a1 @ W1
        D = (m1 * ((m2 * np.abs(w3)) @ np.abs(W2))) @ np.abs(W1)
        eq = (2 * H + 4) * U * D
        g = sigma * np.einsum("nfa,nf->na", J, q)
        eg = sigma * (np.einsum("nfa,nf->na", eJ + (F + 8) * U * Jabs, np.abs(q)) +
                      np.einsum("nfa,nf->na", np.abs(J), eq)) + 2 * U * np.abs(g)
        self.q, self.eq, self.D, self.g, self.eg = q, eq, D, g, eg

        # ---- eikonal term and gamma
        surf = weight > 0
        nrm = np.linalg.norm(g, axis=1)
        en = np.linalg.norm(eg, axis=1) + 3 * U * nrm
        self.ill = surf & (nrm <= 2 * en)
        ns = int(surf.sum()) if n_surface is None else int(n_surface)
        ce = 2.0 * weight_e / ns if ns > 0 else 0.0
        safe = np.where(nrm > 0, nrm, 1.0)
        coef = np.where(surf & (nrm > 0), ce * (nrm - 1) / safe, 0.0)
        ecoef = np.where(surf & (nrm > 0), 2 * abs(ce) * en / safe ** 2 + 6 * U * np.abs(coef), 0.0)
        gam = coef[:, None] * g
        egam = np.abs(coef)[:, None] * eg + ecoef[:, None] * np.abs(g) + 4 * U * np.abs(gam)
        self.surf, self.nrm, self.gam, self.egam, self.n_surface = surf, nrm, gam, egam, ns
        E = np.where(surf, (1 - nrm) ** 2, 0.0)
        eE = np.where(surf, 2 * np.abs(1 - nrm) * en + 3 * U * (1 - nrm) ** 2, 0.0)
        depth = (n if class_surface else (n + 31) // 32) + 8
        self.eikonal = E.sum() / ns if ns > 0 else 0.0
        self.e_eikonal = ((eE.sum() + depth * U * E.sum()) / ns + 2 * U * self.eikonal) if ns > 0 else 0.0

        # ---- first term: dp and the loss value
        wabs = np.abs(weight)
        if loss_type == "sdf_bce":
            wgt = wabs if c["weighted"] else np.ones(n)
            ls = 1.0 / n if c["reduction"] == "mean" else 1.0
            zt = 1.0 / (1.0 + np.exp(-label / sigma))
            sp = 1.0 / (1.0 + np.exp(-pred64))
            dp = wgt * ls * (sp - zt)
            edp = wgt * ls * (P / 4 + 16 * U) + 4 * U * np.abs(dp)
            terms = wgt * (np.maximum(pred64, 0) - pred64 * zt + np.log1p(np.exp(-np.abs(pred64))))
            eterms = wgt * (P + 2.0 ** -21 + (12 + 2 * np.abs(label / sigma)) * U * (1 + np.abs(pred64)))
        else:
            scale = _scale(case)
            ls, wgt = 1.0 / n, wabs
            dm = (pred64 - label) / scale
            edm = (P + U * np.abs(pred64 - label)) / scale + U * np.abs(dm)
            if loss_type == "sdf_l2":
                dp = 2 * wgt * ls * dm / scale
                edp = 2 * wgt * ls * P / scale ** 2 + 8 * U * np.abs(dp)
                terms, eterms = wgt * dm ** 2, wgt * (2 * np.abs(dm) * edm + U * dm ** 2)
            else:
                if pred is not None:
                    sign = sdo.l1_sign(pred64, label, pred, P, 0.0)
                else:
                    sign = np.sign(dm)
                dp = wgt * ls * sign / scale
                edp = 6 * U * np.abs(dp)
                terms, eterms = wgt * np.abs(dm), wgt * edm
        self.dp, self.edp = dp, edp
        self.loss = ls * terms.sum()
        self.e_loss = ls * (eterms.sum() + depth * U * np.abs(terms).sum()) + U * abs(self.loss)

        # ---- the scatter: sc1 = dp w (first term), sc2 = sigma gamma . grad w (eikonal term)
        rows = [t.shape[0] for t in o.hier_features]
        self.rows = RowSums(rows, F, C_SLACK)
        self.eik_rows = RowSums(rows, F, C_SLACK)        # the eikonal term's own gradients (at weight_e = 1)
        pts = np.repeat(np.arange(n), 8)
        self.sc1, self.sc2 = [], []
        for i, gl in enumerate(geo):
            kk = L - 1 - i
            sc1 = dp[:, None] * gl["w"]
            sc2 = sigma * np.einsum("na,nca->nc", gam, gl["dw"])
            esc1 = np.abs(gl["w"]) * edp[:, None] + U * np.abs(sc1)
            esc2 = (sigma * (np.einsum("na,nca->nc", egam, np.abs(gl["dw"])) +
                             np.einsum("na,nca->nc", np.abs(gam), gl["edw"]) +
                             4 * U * np.einsum("na,nca->nc", np.abs(gam), np.abs(gl["dw"]))) + U * np.abs(sc2))
            ix = gl["ix"].reshape(-1)
            if class_surface:       # query_bwd of dfeat = dp q, tangent_bwd of sigma gamma with q
                dq = dp[:, None] * q
                edq = np.abs(dp)[:, None] * (eq + 2 * U * D) + edp[:, None] * np.abs(q)
                self.rows.add(kk, ix, pts, gl["w"].reshape(-1), dq, ev=edq)
            else:
                self.rows.add(kk, ix, pts, sc1.reshape(-1), q, esc1.reshape(-1), eq)
            self.rows.add(kk, ix, pts, sc2.reshape(-1), q, esc2.reshape(-1), eq, count=class_surface)
            if weight_e:
                self.eik_rows.add(kk, ix, pts, sc2.reshape(-1) / weight_e, q)
            self.sc1.append(sc1)
            self.sc2.append(sc2)

    @property
    def drop(self):
        """Points to leave out of the batch (module docstring): ReLU kinks and ill-conditioned surface gradients."""
        return self.kink | self.ill

    def grade(self, got, what, tag="eikonal bounds"):
        """got: dict with table_grads and any of pred, g, loss (the first term), eikonal -> worst error / bound per name."""
        worst = {"tables": self.rows.grade(got["table_grads"], what, tag)}
        if got.get("pred") is not None:
            worst["pred"] = grade_values(got["pred"], self.pred, self.P, what, "pred", tag)
        if got.get("g") is not None:
            worst["g"] = grade_values(got["g"], self.g, self.eg, what, "g", tag)
        if got.get("loss") is not None:
            worst["loss"] = grade_values(got["loss"], self.loss, self.e_loss, what, "loss", tag)
        if got.get("eikonal") is not None:
            worst["eikonal"] = grade_values(got["eikonal"], self.eikonal, self.e_eikonal, what, "eikonal", tag)
        return worst

    def eikonal_share(self):
        """min / max over touched rows of |eikonal part| / |total| of the table gradients (the weight_e of this ref)."""
        shares = []
        for kk in range(len(self.rows.want)):
            tot, eik = self.rows.want[kk][:-1], self.eik_rows.want[kk][:-1] * self.weight_e
            touched = np.abs(eik) > 0
            if touched.any():
                shares.append(np.abs(eik[touched]) / np.maximum(np.abs(tot[touched]), 1e-300))
        s = np.concatenate(shares) if shares else np.zeros(1)
        return float(np.median(s)), float(s.max())


def dominant_weight(case, loss_type="sdf_bce", factor=10.0):
    """A weight_e at which the eikonal term dominates the table rows the surface samples touch: `factor` x the largest
    ratio of first-term to eikonal maxima over the levels (at least 1)."""
    ref = EikRef(case, 1.0, loss_type)
    ratio = 1.0
    for tot, eik in zip(ref.rows.want, ref.eik_rows.want):
        if np.abs(eik[:-1]).max() > 0:
            ratio = max(ratio, float(np.abs(tot[:-1] - eik[:-1]).max() / np.abs(eik[:-1]).max()))
    return factor * ratio


def clean_case(case, loss_type="sdf_bce"):
    """The case without the points of EikRef.drop -> (case, number dropped)."""
    drop = EikRef(case, 0.1, loss_type).drop
    return subset(case, ~drop), int(drop.sum())


def autograd_decoder_grads(case, weight_e, loss_type="sdf_bce", l1_sign=None):
    """The oracle's double backward with fp64 tables and decoder (fp32 coordinates) -> decoder gradients (numpy)."""
    o, dec = oracle64(case)
    c = case["cfg"]
    coord, label, weight = (torch.from_numpy(case[k]) for k in ("coord", "label", "weight"))
    r = sdo.train_step_eikonal(o, dec, coord, label.double(), weight.double(), c["sigma"], weight_e, c["weighted"],
                               c["reduction"], loss_type=loss_type, scale=_scale(case), l1_sign=l1_sign)
    return {k: v.detach().numpy() for k, v in r["dec_grads"].items()}


# ---- the query kernels ---------------------------------------------------------------------------------------------------------

class QueryRef:
    """fp64 references of query_fwd, query_coord_grad (dfeat), query_tangent_fwd (tangent) and query_tangent_bwd (tangent,
    dfeat) with the bounds of the module docstring.  dfeat [N, F] and tangent [N, 3] are fp32 inputs (exact)."""

    def __init__(self, case, dfeat, tangent):
        c = case["cfg"]
        o, _ = oracle64(case)
        coord = np.asarray(case["coord"], dtype=np.float32)
        n, L, F = coord.shape[0], c["tree_level_feat"], c["feature_dim"]
        d = np.asarray(dfeat, dtype=np.float64)
        tg = np.asarray(tangent, dtype=np.float64)
        geo = level_geometry(o, coord)
        self.feat = np.zeros((n, F)); self.efeat = np.zeros((n, F))
        self.G = np.zeros((n, 3)); self.eG = np.zeros((n, 3))
        self.tfwd = np.zeros((n, F)); self.etfwd = np.zeros((n, F))
        self.rows = RowSums([t.shape[0] for t in o.hier_features], F, C_SLACK)
        pts = np.repeat(np.arange(n), 8)
        for i, g in enumerate(geo):
            kk = L - 1 - i
            R = _rows(o, kk, g["ix"])
            self.feat += np.einsum("nc,ncf->nf", g["w"], R)
            self.efeat += (8 * L + 2) * U * np.einsum("nc,ncf->nf", np.abs(g["w"]), np.abs(R))
            Rd = np.einsum("ncf,nf->nc", R, d)
            Rda = np.einsum("ncf,nf->nc", np.abs(R), np.abs(d))
            self.G += np.einsum("nca,nc->na", g["dw"], Rd)
            self.eG += np.einsum("nca,nc->na", g["edw"] + (8 * L + F + 8) * U * np.abs(g["dw"]), Rda)
            W = np.einsum("na,nca->nc", tg, g["dw"])
            Wabs = np.einsum("na,nca->nc", np.abs(tg), np.abs(g["dw"]))
            eW = np.einsum("na,nca->nc", np.abs(tg), g["edw"]) + 3 * U * Wabs
            self.tfwd += np.einsum("nc,ncf->nf", W, R)
            self.etfwd += np.einsum("nc,ncf->nf", eW + (8 * L + 2) * U * Wabs, np.abs(R))
            self.rows.add(kk, g["ix"].reshape(-1), pts, W.reshape(-1), d, ea=eW.reshape(-1))


def touched_ratio(bound, want):
    """median and worst bound / |want| over the elements a scatter touched with |want| > 0 (how tight a bound is)."""
    r = np.concatenate([b[:-1][w[:-1] != 0] / np.abs(w[:-1][w[:-1] != 0]) for b, w in zip(bound, want)])
    return float(np.median(r)), float(r.max())

