"""fp64 reference of the decoder gradients of the fused training step (csrc/shine_b200.cu, `sdf_fused_kernel`) with a
per-element error bound.  Test infrastructure, no GPU needed.

The reference is an explicit restatement of the backward, not autograd.  With the fp64 forward a1 = W1 f + b1,
m1 = [a1 > 0], h1 = m1 a1, a2 = W2 h1 + b2, m2 = [a2 > 0], h2 = m2 a2, and g_j = dL/dpred_j of point j:
    db3 = sum_j g_j                 dw3 = sum_j g_j h2_j
    dh2_j = g_j (w3 . m2_j)         db2 = sum_j dh2_j           dW2 = sum_j dh2_j h1_j^T
    dh1_j = m1_j . W2^T dh2_j       db1 = sum_j dh1_j           dW1 = sum_j dh1_j f_j^T
g is the loss's own (sdf_bce weighted or not, mean or sum; sdf_l1 with the sign rule of tests/test_gpu_replicas.py;
sdf_l2); a decoder without biases simply has no db entries.

Error model (extends the one in the docstring of tests/test_gpu_replicas.py; u = 2^-24).  Every element is a sum
e = sum_j a_j b_j over the batch, and
    |got - want64| <= (depth + C) u S + eps_mm S + T,   S = sum_j |a_j b_j|,   T = sum_j (|da_j| |b_j| + |a_j| |db_j|)
with the per-point, per-unit errors da, db of the operands (first-order propagation of absolute values, from the passes
of `error_bound.decoder_passes`: A0 = sum w |row|, A1, A2 and the relative forward errors e1, e2):
  * f: (8L + 2) u A0;  h1: e1 A1 on the live units;  h2: e2 A2 on the live units;  g: dg of the replica model;
  * dh2: m2 |w3| (dg + u |g|).  The per-point kernels round dp w3 once; the grouped kernel never forms dh2: it scales the
    A operand h1 by dp (one rounding, the same u |g| on the same terms) and applies w3 once per element in the epilogue,
    one rounding of the result that the depth counts;
  * dh1: both kernels form dp (M2 W2') with W2' = fp32(diag(w3) W2) (one rounding), M2 the exact 0/1 mask (a two-product
    3xTF32 contraction, EPS_MM2(32)) and the product by dp (one rounding): D1 (dg + (EPS_MM2(32) + 2 u) |g|) with
    D1 = m1 . |W2|^T (m2 . |w3|);
  * eps_mm: the weight contractions run over the 16 points of a tile on the tensor cores: dW1 and the per-point kernels'
    dW2 as three products, EPS_MM(16), the grouped kernel's dW2 = w3 . (dp h1)^T M2 with the exact mask as two, EPS_MM2(16)
    = (32 + 8 K) u (the one cut of lo, 2^-20 under truncation, rounded up, and the adds of two passes); plain TF32 cuts
    the other operand once: 2^-9 + 8 K u.  The bias and dw3 sums are plain fp32 adds, eps_mm = 0;
  * depth: the fp32 roundings a term passes after its product, from the launch geometry of `launch_fused_t`: grid
    B = min(SMs x per_sm, ceil(tiles / 8)), T = ceil(tiles / 8B) tiles per warp.  A warp's accumulators see at most 12
    roundings per tile (2 k-steps x 3 passes of mma.sync accumulation, 2 u each: the tensor cores truncate), the
    zero-tile sum of dL/dpred T lane adds, 5 shuffles and the 8 warps before it enters the virtual backward tile (1),
    then 5 lane shuffles, the sum of the 8 warp partials, the grouped epilogue's w3 product (1) and B global atomics per
    host chunk of `step_from_host`:
        depth = 12 T + (T + 13) + 1 + 5 + 8 + 1 + B chunks.
    The test does not see per_sm (the launcher picks 1..8 blocks/SM from the registers and shared memory of the
    instantiation), so `kernel_depth` takes the maximum over per_sm = 1..8;
  * C = 4 covers the second-order terms, as in the replica model.
The zero-tile shortcut needs no case of its own: a tile in which no point hits any level adds (sum_j g_j) q, q the
gradient of Decoder.sdf(0); each of its terms g_j q has the form a_j b_j above with f_j = 0 (exact), and the sum's extra
roundings are in the depth.  Elements whose S is 0 (dead units, w3 = 0) have a bound of 0: they must come back as exact
zeros.

ReLU kinks.  A point within twice the forward error of a kink (`error_bound.decoder_passes`) may take either branch in a
correct fp32 kernel.  The replica tests drop such points from their batches; the tests that lay batches out tile by tile
keep them, and there each kink point leaves the grade: its contribution to every element is bounded by an envelope
(masks 1 on the uncertain units, operands at their upper bounds, |dL/dpred| at its upper bound `gmax`), and kernel and
reference each stay within it, so the bound takes 2 x envelope for it instead of its terms.  Points that miss every level
have features of exactly 0 and exact masks: they are never kink points (`decoder_passes` flags a unit only where its
absolute-value pass is non-zero).
"""
from __future__ import annotations

import numpy as np
import torch

from tests.error_bound import C_SLACK, U, eps_mm

KEYS = ("layers.0.weight", "layers.0.bias", "layers.1.weight", "layers.1.bias", "lout.weight", "lout.bias")
W1, B1, W2, B2, W3, B3 = KEYS
MAX_PER_SM = 8
H100_SMS = 132
TILE = 16


def eps_mm2(k, tf32x1=False):
    """A k-term contraction on the tensor cores whose other operand is an exact 0/1 mask (two products in 3xTF32)."""
    return (2.0 ** -9 if tf32x1 else 32 * U) + 8 * k * U


def kernel_depth(n, chunks=1, sms=H100_SMS):
    """Roundings after a term's product (module docstring), maximised over the 1..8 blocks/SM the launcher may choose.
    n: the batch; chunks: the host chunks of `step_from_host` (each a launch over n / chunks points)."""
    tiles = max(1, -(-(-(-n // chunks)) // TILE))
    worst = 0
    for per_sm in range(1, MAX_PER_SM + 1):
        B = max(1, min(sms * per_sm, -(-tiles // 8)))
        T = -(-tiles // (8 * B))
        worst = max(worst, 12 * T + (T + 13) + 1 + 5 + 8 + 1 + B * chunks)
    return worst


def _np(x):
    return x.numpy() if torch.is_tensor(x) else np.asarray(x)


def restate(feat, dec, g):
    """The explicit fp64 backward of the module docstring -> (grads {key: array}, forward {m1, h1, m2, h2, dh2, dh1})."""
    z = torch.zeros((), dtype=torch.float64)
    W1_, W2_, w3 = (dec[k].detach().double() for k in (W1, W2, W3))
    b1, b2 = (dec[k].detach().double() if k in dec else z for k in (B1, B2))
    feat, g = feat.double(), g.double()
    a1 = feat @ W1_.T + b1
    m1 = (a1 > 0).double()
    h1 = a1 * m1
    a2 = h1 @ W2_.T + b2
    m2 = (a2 > 0).double()
    h2 = a2 * m2
    dh2 = g[:, None] * (w3 * m2)
    dh1 = m1 * (dh2 @ W2_)
    grads = {W1: dh1.T @ feat, B1: dh1.sum(0), W2: dh2.T @ h1, B2: dh2.sum(0), W3: (g @ h2)[None, :],
             B3: g.sum().reshape(1)}
    grads = {k: v.numpy() for k, v in grads.items() if k in dec}
    return grads, {"m1": m1, "h1": h1, "m2": m2, "h2": h2, "dh2": dh2, "dh1": dh1}


class DecoderRef:
    """want, S, T and the kink envelope of every decoder-gradient element of one step.
    feat [n, F] fp64 features, dp the dict of `error_bound.decoder_passes`, dec the fp64 decoder, g / dg / gmax [n] the
    fp64 dL/dpred, its error bound and (kink points) an upper bound of the kernel's |dL/dpred|."""

    def __init__(self, feat, dp, dec, g, dg, gmax=None, tf32x1=False, grouped=False):
        self.want, fw = restate(feat, dec, g)
        self.keys = list(self.want)
        self.tf32x1, self.grouped = tf32x1, grouped
        kink = dp["kink"].bool()
        keep = (~kink).double()[:, None]
        w3a, W2a = dec[W3].detach().double().abs(), dec[W2].detach().double().abs()
        g, dg = g.double(), dg.double()
        ga = g.abs()
        # operand magnitudes and errors of the graded (non-kink) points
        fa, ef = feat.abs() * keep, dp["ef"] * keep
        h1, eh1 = fw["h1"] * keep, dp["e1"] * dp["A1"] * fw["m1"] * keep
        h2, eh2 = fw["h2"] * keep, dp["e2"] * dp["A2"] * fw["m2"] * keep
        dh2, edh2 = fw["dh2"].abs() * keep, fw["m2"] * w3a * (dg + U * ga)[:, None] * keep
        D1 = fw["m1"] * ((fw["m2"] * w3a) @ W2a)
        dh1, edh1 = fw["dh1"].abs() * keep, D1 * (dg + (eps_mm2(32, tf32x1) + 2 * U) * ga)[:, None] * keep
        gk, egk = ga * keep[:, 0], dg * keep[:, 0]
        S = {W1: dh1.T @ fa, B1: dh1.sum(0), W2: dh2.T @ h1, B2: dh2.sum(0), W3: (gk @ h2)[None, :], B3: gk.sum().reshape(1)}
        T = {W1: edh1.T @ fa + dh1.T @ ef, B1: edh1.sum(0), W2: edh2.T @ h1 + dh2.T @ eh1, B2: edh2.sum(0),
             W3: (egk @ h2 + gk @ eh2)[None, :], B3: egk.sum().reshape(1)}
        # kink points: envelopes with the uncertain units live and every operand at its upper bound
        env = {k: torch.zeros_like(v) for k, v in S.items()}
        if bool(kink.any()):
            assert gmax is not None, "kink points need an upper bound of the kernel's |dL/dpred|"
            ix = torch.nonzero(kink).squeeze(1)
            mu1, mu2 = dp["m1_hi"][ix], dp["m2_hi"][ix]
            gA = gmax.double()[ix]
            fA = dp["A0"][ix] * (1 + 1e-5)
            h1A = mu1 * dp["A1"][ix] * (1 + 1e-5)
            h2A = mu2 * dp["A2_hi"][ix] * (1 + 1e-5)
            dh2A = gA[:, None] * mu2 * w3a * (1 + 1e-5)
            dh1A = mu1 * (dh2A @ W2a) * (1 + 1e-5)
            env = {W1: dh1A.T @ fA, B1: dh1A.sum(0), W2: dh2A.T @ h1A, B2: dh2A.sum(0), W3: (gA @ h2A)[None, :],
                   B3: gA.sum().reshape(1)}
        self.kinks = int(kink.sum())
        self.S = {k: (S[k] + env[k]).numpy() for k in self.keys}
        self.T = {k: (T[k] + 2 * env[k]).numpy() for k in self.keys}

    def eps(self, key):
        if key == W1:
            return eps_mm(TILE, self.tf32x1)
        if key == W2:
            return eps_mm2(TILE, self.tf32x1) if self.grouped else eps_mm(TILE, self.tf32x1)
        return 0.0

    def bound(self, key, depth):
        return (depth + C_SLACK) * U * self.S[key] + self.eps(key) * self.S[key] + self.T[key]

    def grade(self, got, depth, what, tag="decoder bounds"):
        """Every element of every decoder gradient against its bound -> {key: worst error / bound} (printed)."""
        worst = {}
        for k in self.keys:
            g = np.asarray(got[k], dtype=np.float64).reshape(self.want[k].shape)
            b = self.bound(k, depth)
            err = np.abs(g - self.want[k])
            bad = np.argwhere(err > b)
            if bad.size:
                i = tuple(bad[0])
                raise AssertionError(
                    f"{what}: decoder grad {k} has {len(bad)} elements outside the bound; first {i}: got {g[i]:.9g} "
                    f"want {self.want[k][i]:.9g} bound {b[i]:.3g} (S = {self.S[k][i]:.3g}, depth {depth})")
            worst[k] = float((err / np.where(b > 0, b, 1.0)).max())
        print(f"[{tag}] {what}: depth {depth}, kink points {self.kinks}, worst error / bound " +
              " ".join(f"{k}={v:.3f}" for k, v in worst.items()))
        return worst

    def median_ratio(self, depth):
        """Median bound / |want| per tensor over the elements with want != 0."""
        out = {}
        for k in self.keys:
            w = np.abs(self.want[k])
            nz = w > 0
            out[k] = float(np.median(self.bound(k, depth)[nz] / w[nz])) if nz.any() else float("nan")
        return out
