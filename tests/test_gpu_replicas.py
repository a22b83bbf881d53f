"""Gradient replicas against an fp64 oracle, element by element, at the replica counts that switch them on.

An unordered training batch spreads its table-gradient atomics over R replicas of every small, hot level
(`FeatureOctree._replicas_for`: R = pow2 <= min(8 n / (rows * _REPLICA_TARGET), _REPLICA_MAX)).  Warp w adds into replica
w & (R - 1) (the voxel-grouped kernel picks it by tile); replica 0 is the gradient table itself, replicas 1..R-1 live in the octree's scratch, and
`shine_reduce_grad_replicas` adds them back in the order 1..R-1 and re-zeroes them.  At the sizes of the parity cases R is 1
on every level, so the cases here lower `_REPLICA_TARGET` and raise `_REPLICA_MAX` (class attributes read at call time) on a
fresh octree, and every case asserts the R per level that its step's descriptor carried (a spy on `_reduce_replicas`): a
case that silently runs at R = 1 fails.  One case runs at a natural size without a patch.

Reference.  The oracle step (`oracle.shine_oracle.train_step`) runs in float64: tables, decoder and labels in float64, the
coordinates kept fp32, so the blend weights are the reference's fp32 values (the kernels compute the same expression in
the same fp32 operations) and everything after them is fp64.

Per-element bound, u = 2^-24.  Row u, channel f of a level's gradient is the sum over the k_u (point, corner) terms that land
on that row of w_{j,c} dfeat_{j,f}.  Every path forms a term as one fp32 product and adds terms with fp32 adds (atomics into
one of R partial sums, then the fold); an add into an exact zero is exact, so a term passes at most k_u - 1 roundings after
its product, whatever the order or the replica: the summation is off by at most k_u u S_{u,f}, S = sum_j w_{j,c} |dfeat_{j,f}|
(in fp64 from the oracle's indices and weights).  The slack C = 4 covers second-order terms.  The voxel-grouped kernel forms
the per-node sums of up to 16 points as a 3xTF32 contraction, so it adds EPS_MM(16) to C.
    |got - want64| <= (k_u + C) u S_{u,f} + T_{u,f}
For `query_bwd` dfeat is the input and T = 0.  The fused kernels compute dfeat themselves; T = sum_j w_{j,c} E_{j,f} carries
its error E_j:
  * decoder contractions are 3xTF32: x = hi + lo with hi cut to tf32 and lo = x - hi, x y ~ hi hi' + hi lo' + lo hi' with lo
    cut to tf32 too.  The dropped lo lo' and both cuts of lo stay below 2^-20 |x y| each (truncation, the worst case), so a
    K-term contraction is off by at most EPS_MM(K) = (64 + 8K) u of sum |x||y| (48 u for the products, up to 2 u per fp32 add in
    each of the three passes, rounded up).  Plain TF32 (tf32x1) cuts both operands once: 2^-9 + 8K u;
  * forward, on absolute values with the fp64 pass's ReLU masks (A0 = sum w |row|, A1 = |W1| A0 + |b1|, A2 = |W2| A1 + |b2|,
    Ap = |w3| A2 + |b3|): the blend is off by (8L + 2) u A0, layer k adds EPS_MM(K) and the bias add u, so
    |pred - pred64| <= P = EPS_FWD Ap (checked against the kernel's own pred);
  * dL/dpred = s (sigmoid(pred) - sigmoid(label / sigma)), s = loss scale x |weight|: off by dg = s (P / 4 + 16 u) + 4 u |g|;
  * sdf_l2 / sdf_l1 (`diff_point`): d = (pred - label) / scale, then dL/dpred = 2 d / scale or sign(d) / scale, times |w|,
    times the step's 1/n, every operation one fp32 rounding; scale and 1/n reach the kernel rounded to fp32.  s = |w| / n:
      L2: the subtraction, two divisions, the products by |w| and 1/n, 1/n itself and scale (twice) are 8 roundings, and
          pred is off by P: dg = 2 s P / scale^2 + 8 u |g|;
      L1: the sign is exact (pred - label rounds to 0 only when they are equal); one division, two products, 1/n and
          scale are 5 roundings: dg = 6 u |g|.  Where |pred64 - label| <= P the kernel's pred may lie on either side of the
          label, or on it (sign 0: dL/dpred exactly 0); there the reference takes sign(kernel pred - label), elsewhere
          sign(pred64 - label).  So the L1 reference is built after the step, from the pred it returned;
  * dfeat = W1^T (m1 . W2^T (m2 . w3 g)), two 32-term contractions: E = D ((2 EPS_MM(32) + 2 u) |g| + dg), D = |W1|^T (m1 .
    |W2|^T (m2 . |w3|)).
Points within twice the forward error of a ReLU kink are dropped from the fused cases: there a correct fp32 kernel may take
the other branch.  `compare_step` (2e-4 of the level maximum) runs as a second check, and each case prints its worst
error / bound.
The decoder gradients of every step are graded element by element too, by the model of tests/decoder_bound.py; the
grouped kernel's table rows count the adds that land on them (one per (tile, node) of a grouped tile, one per (point,
corner) of a scattered one: error_bound.grouped_counts) instead of the (point, corner) terms.
The eikonal paths extend this model (blend-weight derivatives, g, gamma and the eikonal scatter): tests/eikonal_bound.py.
The pieces both use (eps_mm, the fp32 blend, the decoder passes, the kink filter, the grading loop) live in
tests/error_bound.py.
"""
import copy
import ctypes as C

import numpy as np
import pytest
import torch

from oracle import shine_oracle as orc
from tests import sdf_diff_oracle as sdo
from tests.decoder_bound import DecoderRef, kernel_depth
from tests.error_bound import C_SLACK, U, drop_kinks, eps_mm, grade_tables, grouped_counts, subset
from tests.error_bound import abs_feature as _abs_feature
from tests.error_bound import blend as _blend
from tests.error_bound import decoder_passes as _decoder_passes
from tests.error_bound import oracle64 as _oracle64
from tests.parity_utils import (FROZEN_SENTINEL, build_cuda_models, compare_step, make_case, oracle_from_case,
                                sort_case_morton)
from tests.test_gpu_sdf_diff import _scale

DEV = "cuda:0"
INVALID = -1                            # SHINE_ERR_INVALID_ARG
gpu = pytest.mark.gpu
DIFF_LOSSES = ("sdf_l1", "sdf_l2")


# ---- forcing replicas and proving they were on ----------------------------------------------------------------------------

def expected_replicas(tables, n):
    """R per level, coarse -> fine, from the rule of the module docstring and the CURRENT class attributes."""
    from shine_mapping_b200 import FeatureOctree
    out = []
    for t in tables:
        want = (8 * n) // max(1, t.shape[0] * FeatureOctree._REPLICA_TARGET)
        r = 1
        while r * 2 <= min(want, FeatureOctree._REPLICA_MAX):
            r *= 2
        out.append(r)
    return out


@pytest.fixture
def force(monkeypatch):
    """force(target, rmax): switch replicas on at small batches for octrees that build their descriptors afterwards."""
    from shine_mapping_b200 import FeatureOctree

    def set_(target, rmax=64):
        monkeypatch.setattr(FeatureOctree, "_REPLICA_TARGET", target)
        monkeypatch.setattr(FeatureOctree, "_REPLICA_MAX", rmax)
    return set_


class FoldSpy:
    """Records the R per level (coarse -> fine) of every descriptor handed to the octree's fold."""

    def __init__(self, octree):
        self.calls = []
        fold = octree._reduce_replicas
        L = octree.featured_level_num

        def spy(desc, device):
            self.calls.append([max(1, desc.lv[L - 1 - k].num_replicas) for k in range(L)])   # 0 and 1: no replicas
            fold(desc, device)
        octree._reduce_replicas = spy

    def expect(self, want, what=""):
        assert self.calls, f"{what}: the step never called the replica fold"
        assert self.calls[-1] == want, f"{what}: the step ran with R = {self.calls[-1]} per level, expected {want}"
        assert max(want) > 1, f"{what}: the case does not switch replicas on"
        print(f"[replicas] {what}: R per level {want}")
        self.calls.clear()


def assert_scratch_zero(octree, what=""):
    torch.cuda.synchronize()
    assert octree._grad_scratch, f"{what}: no replica scratch was allocated"
    for k, buf in octree._grad_scratch.items():
        nz = int(torch.count_nonzero(buf))
        assert nz == 0, f"{what}: replica scratch of level {k} holds {nz} non-zero values after the step"


# ---- fp64 reference and the per-element bound -----------------------------------------------------------------------------

class Ref:
    """fp64 oracle step of a case (or the fp64 query backward of a given dfeat), with S, k and T per row.
    loss_type: the step's loss; sdf_l1 needs `pred`, the kernel's pred of the step being graded (module docstring)."""

    def __init__(self, case, dfeat=None, tf32x1=False, grouped=False, loss_type="sdf_bce", pred=None, replicas=None):
        c = case["cfg"]
        o, dec = _oracle64(case)
        coord = torch.from_numpy(case["coord"])
        n, L, F = coord.shape[0], c["tree_level_feat"], c["feature_dim"]
        self.n, self.tables, self.slack = n, case["tables"], C_SLACK + (eps_mm(16) / U if grouped else 0)
        self.dec = None
        env = torch.zeros(n, F, dtype=torch.float64)
        if dfeat is None:
            label = torch.from_numpy(case["label"]).double()
            weight = torch.from_numpy(case["weight"]).double()
            dd = {k: v.detach() for k, v in dec.items()}
            with torch.no_grad():
                feat = o.query_feature(coord)
                dp = _decoder_passes(feat, _abs_feature(o, coord), dd, tf32x1, L)
            scale, sign = _scale(case), None
            if loss_type == "sdf_l1":
                assert pred is not None, "the sdf_l1 reference needs the kernel's pred"
                sign = sdo.l1_sign(orc.decoder_sdf(feat, dd).numpy(), case["label"], pred, dp["P"].numpy(), 0.0)
            res = sdo.train_step(o, dec, coord, label, weight, c["sigma"], c["weighted"], c["reduction"], loss_type=loss_type,
                                 scale=scale, double=True, l1_sign=sign)
            self.want = [g.detach().numpy() for g in res["table_grads"]]
            self.pred = res["pred"].numpy()
            self.step = {"loss": float(res["loss"]), "dec_grads": {k: g.numpy() for k, g in res["dec_grads"].items()}}
            feat = res["feature"].clone().requires_grad_(True)
            pred64 = orc.decoder_sdf(feat, dd)
            if loss_type == "sdf_bce":
                loss = orc.sdf_bce_loss(pred64, label, c["sigma"], weight.abs(), c["weighted"], c["reduction"])
                dfeat64, g = torch.autograd.grad(loss, [feat, pred64])
            else:
                g = sdo.diff_dpred(pred64.detach(), label, weight.abs(), scale, loss_type == "sdf_l2", n,
                                   None if sign is None else torch.from_numpy(sign))
                dfeat64 = torch.autograd.grad(pred64, feat, g)[0]
            with torch.no_grad():
                if loss_type == "sdf_bce":
                    s = (weight.abs() if c["weighted"] else torch.ones(n, dtype=torch.float64))
                    s = s / n if c["reduction"] == "mean" else s
                    dg = s * (dp["P"] / 4 + 16 * U) + 4 * U * g.abs()
                elif loss_type == "sdf_l2":
                    dg = 2 * (weight.abs() / n) * dp["P"] / scale ** 2 + 8 * U * g.abs()
                else:
                    dg = 6 * U * g.abs()
                E = dp["D"] * (dp["ebwd"] * g.abs() + dg)[:, None]
                # kink points (kept only by the tile-layout tests): |dL/dpred| of the kernel at most gmax, dfeat within
                # the envelope with the uncertain units live, E = 2 x envelope (tests/decoder_bound.py)
                s_l = weight.abs() / n
                gmax = s_l / scale * (1 + 6 * U) if loss_type == "sdf_l1" else g.abs() + dg     # dg from the kink P
                kink = dp["kink"]
                if bool(kink.any()):
                    W1a, W2a, w3a = (dd[k].abs() for k in ("layers.0.weight", "layers.1.weight", "lout.weight"))
                    Dhi = (dp["m1_hi"] * ((dp["m2_hi"] * w3a) @ W2a)) @ W1a
                    env = torch.where(kink[:, None], Dhi * gmax[:, None] * (1 + 1e-5), env)
                    E = torch.where(kink[:, None], 2 * env, E)
                self.dec = DecoderRef(feat, dp, dd, g.detach(), dg, gmax, tf32x1, grouped)
                self.feat64, self.g64, self.dec64 = feat.detach(), g.detach(), dd     # for per-tile contributions
            self.P = dp["P"].numpy()
            self.kink = dp["kink"].numpy()
            self.kinks = int(dp["kink"].sum())
        else:
            dfeat64 = torch.from_numpy(dfeat).double()
            feat = o.query_feature(coord)
            feat.backward(dfeat64)
            self.want = [t.grad.numpy() for t in o.hier_features]
            E = torch.zeros(n, F, dtype=torch.float64)
            self.P, self.kink, self.kinks = None, np.zeros(n, dtype=bool), 0
        self.dfeat = dfeat64.detach().numpy()
        pts = torch.arange(n).repeat_interleave(8)
        self.S, self.k, self.T, self._ix = [None] * L, [None] * L, [None] * L, [None] * L
        for i, (ix, w) in enumerate(_blend(o, coord)):
            kk = L - 1 - i
            rows = self.want[kk].shape[0]
            hit = ix >= 0
            r, wj, pj = ix[hit], w[hit][:, None], pts[hit]
            mag = torch.maximum(dfeat64.detach().abs(), env)
            self.S[kk] = torch.zeros(rows, F, dtype=torch.float64).index_add_(0, r, wj * mag[pj]).numpy()
            self.T[kk] = torch.zeros(rows, F, dtype=torch.float64).index_add_(0, r, wj * E[pj]).numpy()
            self._ix[kk] = ix.numpy().reshape(n, 8)
            self.k[kk] = torch.bincount(r, minlength=rows).numpy()
        self._k_points = self.k
        if grouped:
            self.k = self._grouped_k(replicas)

    def _grouped_k(self, replicas):
        """k_u of the grouped kernel (error_bound.grouped_counts), plus the R - 1 adds of the replica fold."""
        out = []
        for kk, ix in enumerate(self._ix):
            kg = grouped_counts(ix, self.want[kk].shape[0])
            out.append(kg + np.where(kg > 0, (1 if replicas is None else replicas[kk]) - 1, 0))
        return out

    def for_kernel(self, grouped):
        """The same reference graded for the grouped kernel at R = 1 (its k_u, EPS_MM(16), two-product dW2) or for the
        per-point kernels."""
        out = copy.copy(self)
        out.slack = C_SLACK + (eps_mm(16) / U if grouped else 0)
        out.k = self._grouped_k(None) if grouped else self._k_points
        if self.dec is not None:
            out.dec = copy.copy(self.dec)
            out.dec.grouped = grouped
        return out

    def grade(self, got_tables, what, pred=None):
        """Every element of every level (trash row excluded) against its bound -> worst error / bound."""
        bounds = [(k[:, None] + self.slack) * U * S + T for S, k, T in zip(self.S, self.k, self.T)]
        worst = grade_tables(got_tables, self.want, bounds, self.k, self.S, what, "replica bounds")
        if pred is not None:      # every point, kink points with their wider P (error_bound.decoder_passes)
            e = np.abs(np.asarray(pred, dtype=np.float64) - self.pred)
            assert (e <= self.P).all(), f"{what}: pred outside its bound at {int((e > self.P).sum())} points"
            print(f"[replica bounds] {what}: pred worst {float((e / self.P).max()):.3f} of the bound")
        return worst

    def grade_decoder(self, dec_grads, what, chunks=1):
        """Every decoder-gradient element against the bound of tests/decoder_bound.py at the kernel's depth for this batch."""
        sms = torch.cuda.get_device_properties(0).multi_processor_count if torch.cuda.is_available() else None
        depth = kernel_depth(self.n, chunks, sms) if sms else kernel_depth(self.n, chunks)
        return self.dec.grade(dec_grads, depth, what)

    def compare(self, got_tables, pred, loss, dec_grads, tf32x1=False):
        """compare_step on the same step (fp32-graded quantities: loss, pred, decoder gradients)."""
        got = {"indices": [], "feature": np.zeros(0), "pred": pred, "loss": loss, "table_grads": got_tables,
               "dec_grads": dec_grads}
        want = {"indices": [], "feature": np.zeros(0), "pred": self.pred, "loss": self.step["loss"],
                "table_grads": self.want, "dec_grads": {k: self.step["dec_grads"][k] for k in dec_grads}}
        kw = dict(pred_atol=5e-3, pred_rtol=5e-3, grad_rel=3e-2) if tf32x1 else {}
        return compare_step(got, want, **kw)


def grade_run(case, got, what, loss_type="sdf_bce", morton_ordered=False, tf32x1=False, ref=None):
    """The per-element grade of one step's result (the dict of parity_utils.run_cuda_step / test_gpu_sdf_diff._cuda_step):
    pred, every table-gradient element (the grouped kernel's k_u where the Morton flag picks it: up to 4 levels, 3xTF32)
    and every decoder-gradient element unless the decoder was frozen.  ref: a Ref of the case to reuse (not for sdf_l1,
    whose reference follows the kernel's pred).  -> the Ref."""
    grouped = morton_ordered and case["cfg"]["tree_level_feat"] <= 4 and not tf32x1
    if ref is None:
        ref = Ref(case, tf32x1=tf32x1, loss_type=loss_type, pred=got["pred"])
    graded = ref.for_kernel(grouped)
    what = f"{what} {'grouped' if grouped else 'per-point'} {loss_type}"
    graded.grade(got["table_grads"], what, got["pred"])
    if got["dec_grads"]:
        graded.grade_decoder(got["dec_grads"], what)
    return ref


# ---- running the kernels -------------------------------------------------------------------------------------------------

def _dev(case):
    return tuple(torch.from_numpy(case[k]).to(DEV) for k in ("coord", "label", "weight"))


def trainer(case, freeze=False, main_loss_type="sdf_bce", **kw):
    from shine_mapping_b200 import SdfTrainer
    cfg, octree, dec = build_cuda_models(case, DEV, freeze_decoder=freeze)
    tr = SdfTrainer(cfg, octree, dec, main_loss_type=main_loss_type, **kw)
    tr.use_replicas = True
    return tr, FoldSpy(octree)


def train_step(tr, case, morton_ordered=None):
    """One step; a frozen decoder's gradient segment is filled with a sentinel first and must come back bit for bit."""
    coord, label, weight = _dev(case)
    tr.zero_grad()
    if not tr._dec_trainable:
        tr.dec_flat.fill_(FROZEN_SENTINEL)
        before = tr.dec_flat.clone()
    pred = torch.empty(coord.shape[0], device=DEV)
    loss = float(tr.forward_backward(coord, label, weight, pred_out=pred, morton_ordered=morton_ordered))
    torch.cuda.synchronize()
    if not tr._dec_trainable:
        assert torch.equal(tr.dec_flat.view(torch.int32), before.view(torch.int32)), \
            "a frozen decoder's gradient buffer was written"
    tables = [g.detach().cpu().numpy().copy() for g in tr.table_grads]
    return tables, pred.cpu().numpy(), loss, dec_grads(tr)


def dec_grads(tr):
    return {k: g.detach().cpu().numpy().copy() for k, g in zip(("layers.0.weight", "layers.0.bias", "layers.1.weight",
                                                                 "layers.1.bias", "lout.weight", "lout.bias"), tr.dec_grads)
            if g is not None and tr._dec_trainable}


def check_step(tr, spy, case, ref, what, tf32x1=False, morton_ordered=None, grouped=False, replicas=True):
    """One trainer step: R per level as expected, compare_step, every element within its bound (tables, pred and decoder
    gradients), scratch all zero.  ref None: the Ref of the trainer's loss, built after the step from the pred it
    returned.  replicas=False: a step that runs at R = 1 (no replica fold)."""
    tables, pred, loss, dec = train_step(tr, case, morton_ordered)
    if ref is None:
        ref = Ref(case, tf32x1=tf32x1, grouped=grouped, loss_type=tr.main_loss_type, pred=pred,
                  replicas=expected_replicas(case["tables"], case["coord"].shape[0]) if replicas else None)
    what = f"{what} {tr.main_loss_type}"
    if replicas:
        spy.expect(expected_replicas(case["tables"], ref.n), what)
    else:       # no fold with R > 1, and no replica scratch ever allocated
        assert all(max(r) == 1 for r in spy.calls), f"{what}: the step ran with replicas {spy.calls}"
        assert not tr.octree._grad_scratch, f"{what}: replica scratch was allocated"
        spy.calls.clear()
    print(what, ref.compare(tables, pred, loss, dec, tf32x1))
    worst = ref.grade(tables, what, pred)
    if tr._dec_trainable:
        ref.grade_decoder(dec, what)
    if replicas:
        assert_scratch_zero(tr.octree, what)
    return worst


def query_bwd(octree, case, dfeat):
    coord = torch.from_numpy(case["coord"]).to(DEV)
    feature = octree.query_feature(coord)
    grads = torch.autograd.grad(feature, list(octree.hier_features), torch.from_numpy(dfeat).to(DEV))
    torch.cuda.synchronize()
    return [g.cpu().numpy() for g in grads]


def random_dfeat(n, F, seed):
    g = np.random.default_rng(seed)
    return (g.standard_normal((n, F)) * 10.0 ** g.uniform(-2, 2, (n, F))).astype(np.float32)


def check_query_bwd(octree, spy, case, ref, dfeat, what):
    got = query_bwd(octree, case, dfeat)
    spy.expect(expected_replicas(case["tables"], ref.n), what)
    ref.grade(got, what)
    scale = [max(float(np.abs(w[:-1]).max()), 1e-30) for w in ref.want]
    for kk, (a, b) in enumerate(zip(got, ref.want)):
        assert float(np.abs(a[:-1] - b[:-1]).max()) <= 2e-4 * scale[kk], f"{what}: level {kk} beyond 2e-4 of its maximum"
    assert_scratch_zero(octree, what)


# ---- fused kernels at forced R ------------------------------------------------------------------------------------------

def with_weights(case, loss_type, seed):
    """sdf_l1 / sdf_l2 always weight by |w|: give the case weights other than +-1 (same points and labels)."""
    if loss_type == "sdf_bce":
        return case
    w = case["weight"] * np.random.default_rng(seed).uniform(0.5, 1.5, case["weight"].shape[0]).astype(np.float32)
    return dict(case, weight=w)


def with_own_pred_labels(tr, case, every=97):
    """sdf_l1: every `every`-th sample gets the kernel's own pred as label, an exact zero difference (dL/dpred = 0)."""
    if tr.main_loss_type != "sdf_l1":
        return case
    out = dict(case, label=case["label"].copy())
    out["label"][::every] = train_step(tr, case)[1][::every]
    return out


@gpu
@pytest.mark.parametrize("rmax,loss_type", [pytest.param(r, "sdf_bce", id=str(r)) for r in (2, 4, 8, 16, 32, 64)] +
                         [pytest.param(64, lt, id=f"64-{lt}") for lt in DIFF_LOSSES])
def test_general_kernel_at_every_replica_count(rmax, loss_type, force):
    """The LMAX = 8 general kernel (6 levels) with the coarsest level at R = rmax and the finer ones at smaller R: every tail
    split of the fold's 8-wide loop (nrep = 1, 3, 7, 15, 31, 63; R <= 64 takes them all at once)."""
    force(1, rmax)
    case, dropped = drop_kinks(with_weights(make_case(n_points=2500, n_batch=3000, feat_levels=6, seed=60 + rmax),
                                            loss_type, rmax))
    assert expected_replicas(case["tables"], case["coord"].shape[0])[0] == rmax
    tr, spy = trainer(case, main_loss_type=loss_type)
    case = with_own_pred_labels(tr, case)
    check_step(tr, spy, case, None, f"general L=6 R<={rmax} (kinks dropped: {dropped})")


VARIANTS = [("tf32x1", False, "mean"), ("frozen", True, "sum"), ("biasless", True, "mean"), ("plain", False, "sum")]


@gpu
@pytest.mark.parametrize("levels,variant,weighted,reduction,loss_type",
                         [pytest.param(lv, v, w, r, "sdf_bce", id=f"{v}-{w}-{r}-{lv}") for v, w, r in VARIANTS
                          for lv in (3, 8)] +
                         [pytest.param(lv, v, True, "mean", lt, id=f"{v}-{lv}-{lt}") for lt in DIFF_LOSSES
                          for lv, v in ((3, "tf32x1"), (8, "frozen"), (3, "biasless"), (8, "plain"))])
def test_general_kernel_variants(levels, variant, weighted, reduction, loss_type, force):
    """L <= 4 and L > 4 instantiations with plain TF32, a frozen decoder (no decoder gradients) and a bias-less decoder.
    Plain TF32 puts many points within its forward error of a ReLU kink, hence the larger batch.  sdf_l1 / sdf_l2 always
    weight by |w| with the mean: weighted / reduction do not apply to them."""
    force(1, 64)
    tf32x1 = variant == "tf32x1"
    case = make_case(n_points=2500, n_batch=12000 if tf32x1 else 3000, feat_levels=levels, seed=70 + levels,
                     weighted=weighted, reduction=reduction, bias=variant != "biasless", n_frames=2 if levels == 8 else 1)
    case, dropped = drop_kinks(case, tf32x1)
    tr, spy = trainer(case, freeze=variant == "frozen", tf32x1=tf32x1, main_loss_type=loss_type)
    check_step(tr, spy, case, None, f"general L={levels} {variant} (kinks dropped: {dropped})", tf32x1)


@gpu
@pytest.mark.parametrize("ordered,loss_type", [pytest.param(o, "sdf_bce", id=str(o)) for o in (True, False)] +
                         [pytest.param(o, lt, id=f"{o}-{lt}") for lt in DIFF_LOSSES for o in (True, False)])
def test_grouped_kernel_with_replicas(ordered, loss_type, force):
    """The voxel-grouped kernel with `grouped_replicas`: replica by tile, per-node 3xTF32 sums (Morton-ordered batch) and
    its per-point fall-back (batch in the order drawn)."""
    force(1, 64)
    case = with_weights(make_case(n_points=2500, n_batch=6000, feat_levels=4, seed=81), loss_type, 81)
    if ordered:
        case = sort_case_morton(case)
    case, dropped = drop_kinks(case)
    tr, spy = trainer(case, morton_ordered=True, main_loss_type=loss_type)
    tr.grouped_replicas = True
    check_step(tr, spy, case, None, f"grouped ordered={ordered} (kinks dropped: {dropped})", morton_ordered=True,
               grouped=True)


def _far_tiles(case, tiles, at, seed, weight=None):
    """The case with `tiles` tiles of points outside every node (zero tiles) inserted at tile `at`; weight: their weight
    (0: their dL/dpred is exactly 0), None: random weights in [0.5, 1.5)."""
    rng = np.random.default_rng(seed)
    m = 16 * tiles
    far = {"coord": rng.uniform(0.6, 0.9, size=(m, 3)).astype(np.float32),
           "label": rng.uniform(-0.2, 0.2, size=m).astype(np.float32),
           "weight": (rng.uniform(0.5, 1.5, size=m) if weight is None else np.full(m, weight)).astype(np.float32)}
    out = dict(case)
    for k in ("coord", "label", "weight"):
        out[k] = np.ascontiguousarray(np.concatenate((case[k][:16 * at], far[k], case[k][16 * at:])))
    return out


def _grouped_layout(layout, seed):
    """Morton-ordered batches for the grouped kernel at R = 1 (module docstring of the grouped cases below)."""
    from tests.test_gpu_rounds import _tiles_per_round
    per_round = _tiles_per_round()
    if layout == "zero-block":                  # one round: block 0 holds tiles 0-7, all zero tiles
        case = sort_case_morton(drop_kinks(make_case(n_points=2500, n_batch=(per_round // 2 - 16) * 16, feat_levels=4,
                                                     seed=seed, weighted=True))[0])
        return _far_tiles(case, 8, 0, seed)
    case = sort_case_morton(drop_kinks(make_case(n_points=2500, n_batch=2 * per_round * 16 + 40, feat_levels=4,
                                                 seed=seed, weighted=True))[0])
    if layout == "scattered":                   # 64 tiles in the order drawn: more than kMaxGroupedRuns nodes per tile
        rng = np.random.default_rng(seed)
        sl = np.arange(16 * per_round, 16 * (per_round + 64))
        perm = np.arange(case["coord"].shape[0])
        perm[sl] = rng.permutation(sl)
        case = subset(case, perm)
        return _far_tiles(case, 24, per_round // 2, seed)
    # zero-sum: block 0's tiles 0-7 are zero tiles of weight 0 (its dL/dpred sum is exactly 0), more zero tiles later
    return _far_tiles(_far_tiles(case, 40, per_round + 3, seed), 8, 0, seed + 1, weight=0.0)


@gpu
@pytest.mark.parametrize("layout,loss_type", [pytest.param(lo, "sdf_bce", id=lo) for lo in ("scattered", "zero-block",
                                                                                               "zero-sum")] +
                         [pytest.param("scattered", lt, id=f"scattered-{lt}") for lt in DIFF_LOSSES])
def test_grouped_kernel_at_one_replica(layout, loss_type):
    """The Morton-ordered kernel as the batch loop runs it, at R = 1: batches over more than two grid-stride rounds with
    a stretch of scattered tiles (more than kMaxGroupedRuns nodes on a level: per-point scatter inside the grouped kernel)
    and zero tiles in mid-batch; one round whose block 0 holds only zero tiles; and a block whose zero-tile dL/dpred sum is
    exactly 0 (weight 0), which skips its virtual backward tile."""
    from tests.error_bound import oracle64
    case = with_weights(_grouped_layout(layout, 500 + len(layout)), loss_type, 7)
    o, _ = oracle64(case)
    idx = o.get_indices(torch.from_numpy(case["coord"]))
    runs = [grouped_counts(ix.numpy().reshape(-1, 8), 1 + int(ix.max())).sum() for ix in idx]
    # the layout really is what it claims: zero tiles (every point misses every level) where they were put
    n = case["coord"].shape[0]
    miss = np.logical_and.reduce([(ix.numpy().reshape(n, -1) < 0).all(1) for ix in idx])
    zero = np.concatenate((miss, np.ones(-n % 16, bool))).reshape(-1, 16).all(1)
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    if layout == "zero-block":
        assert zero[:8].all() and not zero[8:].all(), "block 0 does not hold only zero tiles"
        assert zero.shape[0] <= 8 * sms, "more than one round: block 0 would get more tiles"
    elif layout == "zero-sum":
        assert zero[:8].all() and not case["weight"][:128].any(), "block 0's zero tiles do not sum to exactly 0"
        assert zero[8:].sum() >= 40 and np.abs(case["weight"][16 * 8:][np.repeat(zero[8:], 16)[:n - 128]]).min() > 0
    else:
        assert zero[1:-1].sum() >= 24, "no zero tiles in mid-batch"
    print(f"[grouped R=1] {layout}: {int(zero.sum())} zero tiles of {zero.shape[0]}")
    if layout == "scattered":
        leaf = idx[0].numpy().reshape(-1, 8)[:, 0]
        node = np.concatenate((leaf, np.full(-leaf.shape[0] % 16, -1))).reshape(-1, 16)
        nruns = [len(set(r[r >= 0].tolist())) for r in node]
        assert max(nruns) > 6, "no scattered tile"
        print(f"[grouped R=1] {layout}: {sum(x > 6 for x in nruns)} scattered tiles of {len(nruns)}; adds per level {runs}")
    tr, spy = trainer(case, morton_ordered=True, main_loss_type=loss_type)
    check_step(tr, spy, case, None, f"grouped R=1 {layout}", morton_ordered=True, grouped=True, replicas=False)


@gpu
@pytest.mark.parametrize("feature_dim", [4, 8, 16])
def test_query_bwd_with_replicas(feature_dim, force):
    """The class-surface backward (`shine_query_bwd`, LP = F / 4 lanes per point) with replicas."""
    force(1, 64)
    case = make_case(n_points=2000, n_batch=3000, feat_levels=4, seed=100 + feature_dim, feature_dim=feature_dim)
    cfg, octree, dec = build_cuda_models(case, DEV)
    spy = FoldSpy(octree)
    dfeat = random_dfeat(case["coord"].shape[0], feature_dim, feature_dim)
    check_query_bwd(octree, spy, case, Ref(case, dfeat=dfeat), dfeat, f"query_bwd F={feature_dim}")


# ---- natural size: no patch -----------------------------------------------------------------------------------------------

@pytest.fixture(scope="module")
def natural_case():
    return make_case(n_points=2500, n_batch=50000, feat_levels=8, seed=58, n_frames=2)


@gpu
def test_natural_size_general_kernel(natural_case):
    """50 000 points at L = 8 switch replicas on by themselves: R = 16 / 8 / 4 / 2 on the four coarsest levels; each loss
    on a trainer of its own."""
    case, dropped = drop_kinks(natural_case)
    assert expected_replicas(case["tables"], case["coord"].shape[0])[:4] == [16, 8, 4, 2]
    for loss_type in ("sdf_bce",) + DIFF_LOSSES:
        c = with_weights(case, loss_type, 58)
        tr, spy = trainer(c, main_loss_type=loss_type)
        check_step(tr, spy, c, None, f"natural L=8 general (kinks dropped: {dropped})")


@gpu
def test_natural_size_query_bwd(natural_case):
    case = natural_case
    assert expected_replicas(case["tables"], case["coord"].shape[0])[:4] == [16, 8, 4, 2]
    cfg, octree, dec = build_cuda_models(case, DEV)
    spy = FoldSpy(octree)
    dfeat = random_dfeat(case["coord"].shape[0], 8, 5)
    check_query_bwd(octree, spy, case, Ref(case, dfeat=dfeat), dfeat, "natural L=8 query_bwd")


# ---- scratch lifecycle ---------------------------------------------------------------------------------------------------

@gpu
def test_consecutive_steps(force):
    """Three steps in a row on the same trainer, the batch permuted in between (other warps, other replicas); a fold that
    leaves a replica dirty doubles that replica's share in the next step."""
    force(1, 64)
    case, _ = drop_kinks(make_case(n_points=2500, n_batch=3000, feat_levels=6, seed=111))
    tr, spy = trainer(case)
    rng = np.random.default_rng(0)
    for s in range(3):
        batch = case if s == 0 else subset(case, rng.permutation(case["coord"].shape[0]))
        check_step(tr, spy, batch, Ref(batch), f"consecutive step {s}")


@gpu
def test_batch_size_changes_replica_count(force):
    force(4, 64)
    case, _ = drop_kinks(make_case(n_points=2500, n_batch=6000, feat_levels=6, seed=112))
    small = subset(case, np.arange(0, case["coord"].shape[0], 5))
    assert expected_replicas(case["tables"], case["coord"].shape[0]) != expected_replicas(small["tables"],
                                                                                          small["coord"].shape[0])
    refs = {"full": Ref(case), "fifth": Ref(small)}
    tr, spy = trainer(case)
    for name in ("full", "fifth", "full", "fifth"):
        check_step(tr, spy, case if name == "full" else small, refs[name], f"batch {name}")


def _first_frame_case(case):
    """The case after its first frame only: the oracle's tables are append-only, so its rows are a prefix of the final ones."""
    c0 = dict(case)
    c0["frames"] = case["frames"][:1]
    o = orc.OracleOctree(case["cfg"]["tree_level_world"], case["cfg"]["tree_level_feat"], case["cfg"]["feature_dim"])
    o.update(torch.from_numpy(np.asarray(c0["frames"][0])))
    c0["tables"] = [np.concatenate((t[:f.shape[0] - 1], np.zeros_like(t[-1:]))) for t, f in zip(case["tables"], o.hier_features)]
    return c0


@gpu
def test_step_after_update_grows_the_tables(force):
    """update() grows every level: the replica stride (rows x F) changes, the scratch is either reused at the new stride
    (R lowered) or reallocated (R raised)."""
    force(1, 64)
    case, _ = drop_kinks(make_case(n_points=2500, n_batch=4000, feat_levels=4, seed=113, n_frames=2))
    c0 = _first_frame_case(case)
    assert all(a.shape[0] < b.shape[0] for a, b in zip(c0["tables"], case["tables"]))
    tr, spy = trainer(c0)
    octree = tr.octree
    check_step(tr, spy, c0, Ref(c0), "before update")
    before = {k: (b.data_ptr(), b.numel()) for k, b in octree._grad_scratch.items()}
    octree.update(torch.from_numpy(np.asarray(case["frames"][1])).to(DEV))
    with torch.no_grad():
        for p, t in zip(octree.hier_features, case["tables"]):
            p.copy_(torch.from_numpy(t))
    ref = Ref(case)
    force(1, 16)
    check_step(tr, spy, case, ref, "after update, R <= 16")
    reused = sum(before[k] == (b.data_ptr(), b.numel()) for k, b in octree._grad_scratch.items())
    force(1, 64)
    octree._desc_cache = {}
    check_step(tr, spy, case, ref, "after update, R <= 64")
    print("scratch buffers reused at the new stride:", reused, "of", len(before))


@gpu
def test_two_default_trainers_alternate_on_one_octree(force):
    """Two trainers on one octree share its replica scratch: each one's step still matches the oracle."""
    from shine_mapping_b200 import SdfTrainer
    force(1, 64)
    case, _ = drop_kinks(make_case(n_points=2500, n_batch=4000, feat_levels=4, seed=114))
    ref = Ref(case)
    tr1, spy = trainer(case)
    tr2 = SdfTrainer(tr1.config, tr1.octree, tr1.decoder)
    tr2.use_replicas = True
    for s, tr in enumerate((tr1, tr2, tr1, tr2)):
        check_step(tr, spy, case, ref, f"alternating step {s} (trainer {1 if tr is tr1 else 2})")


@gpu
def test_class_surface_backward_between_trainer_steps(force):
    force(1, 64)
    case, _ = drop_kinks(make_case(n_points=2500, n_batch=4000, feat_levels=5, seed=115))
    ref = Ref(case)
    dfeat = random_dfeat(case["coord"].shape[0], 8, 1)
    qref = Ref(case, dfeat=dfeat)
    tr, spy = trainer(case)
    check_step(tr, spy, case, ref, "trainer step before the class surface")
    check_query_bwd(tr.octree, spy, case, qref, dfeat, "class-surface backward")
    check_step(tr, spy, case, ref, "trainer step after the class surface")


@gpu
def test_step_from_host_chunks_with_different_replica_counts(force):
    """step_from_host(chunks=3) with n = 3m + 2: chunks of m, m + 1 and m + 1 points, and a target chosen so that the
    coarsest level flips from R = 32 to R = 64 between m and m + 1."""
    case, _ = drop_kinks(make_case(n_points=2500, n_batch=70000, feat_levels=4, seed=116, n_frames=2))
    rows0 = case["tables"][0].shape[0]
    target = max(1, round(8 * 22000 / (64 * rows0)))
    m = -(-64 * rows0 * target // 8) - 1                    # 8 m < 64 rows0 target <= 8 (m + 1)
    n = 3 * m + 2
    assert 65536 < n <= case["coord"].shape[0]
    case = subset(case, np.arange(n))
    force(target, 64)
    chunks = [(n * k // 3, n * (k + 1) // 3) for k in range(3)]
    want = [expected_replicas(case["tables"], e - b) for b, e in chunks]
    assert [r[0] for r in want] == [32, 64, 64], want
    for loss_type in ("sdf_bce",) + DIFF_LOSSES:
        # sdf_l1 / sdf_l2 read the weights: each chunk copies its own slice of them (weights other than +-1 show a wrong one)
        c = with_weights(case, loss_type, 116)
        tr, spy = trainer(c, main_loss_type=loss_type)
        what = f"step_from_host chunks=3 {loss_type}"
        pred = train_step(tr, c)[1] if loss_type == "sdf_l1" else None     # the kernel's pred for the L1 reference
        spy.calls.clear()
        coord_h, label_h, weight_h = (torch.from_numpy(c[k]).pin_memory() for k in ("coord", "label", "weight"))
        tr.step_from_host(coord_h, label_h, weight_h if loss_type != "sdf_bce" else None, chunks=3)
        torch.cuda.synchronize()
        assert spy.calls[:3] == want, f"{what}: chunks ran with R = {spy.calls[:3]}, expected {want}"
        print(f"[replicas] {what}: R per level of the chunks {want}")
        ref = Ref(c, loss_type=loss_type, pred=pred)
        ref.grade([g.detach().cpu().numpy() for g in tr.table_grads], what)
        ref.grade_decoder(dec_grads(tr), what, chunks=3)
        assert_scratch_zero(tr.octree, what)


@gpu
def test_capture_step_replays_on_changed_data(force):
    force(1, 64)
    case, _ = drop_kinks(make_case(n_points=2500, n_batch=6000, feat_levels=6, seed=117))
    n = case["coord"].shape[0] // 2
    for loss_type in ("sdf_bce",) + DIFF_LOSSES:
        c = with_weights(case, loss_type, 117)
        a, b = subset(c, np.arange(n)), subset(c, np.arange(n, 2 * n))
        tr, spy = trainer(a, main_loss_type=loss_type)
        # the kernel's pred of each half for the L1 reference (the replays write no pred)
        preds = {k: train_step(tr, v)[1] if loss_type == "sdf_l1" else None for k, v in (("A", a), ("B", b))}
        refs = {k: Ref(v, loss_type=loss_type, pred=preds[k]) for k, v in (("A", a), ("B", b))}
        coord, label, weight = _dev(a)
        graph = tr.capture_step(coord, label, weight, exchange=False)
        spy.expect(expected_replicas(a["tables"], n), f"capture {loss_type}")
        refs["A"].grade([g.detach().cpu().numpy() for g in tr.table_grads], f"capture warm-up on A {loss_type}")
        refs["A"].grade_decoder(dec_grads(tr), f"capture warm-up on A {loss_type}")
        for name in ("B", "A", "B"):
            src = _dev(b if name == "B" else a)
            for dst, s in zip((coord, label, weight), src):
                dst.copy_(s)
            graph.replay()
            torch.cuda.synchronize()
            refs[name].grade([g.detach().cpu().numpy() for g in tr.table_grads], f"replay on {name} {loss_type}")
            refs[name].grade_decoder(dec_grads(tr), f"replay on {name} {loss_type}")
            assert_scratch_zero(tr.octree, f"replay on {name} {loss_type}")


# ---- the fold kernel on its own, bit-exact ---------------------------------------------------------------------------------

F_FOLD = 8
BIG_ROWS = 150_000              # rows * F / 4 = 300 000 float4 > 132 SMs * 8 blocks * 256 threads: the grid-stride loop wraps


def fold_levels(rmax):
    """(rows, R, has_grads) of the hand-built descriptor: R = rmax, a second R, R = 1 (skipped), a level without
    gradients (skipped, its replicas untouched) and the big level."""
    return [(37, rmax, True), (1000, 1, True), (513, max(2, rmax // 4), True), (2000, rmax, False),
            (BIG_ROWS, rmax, True)]


def fold_data(rows, r, seed):
    """main [rows, F] and replicas [r - 1, rows, F], fp32 over twelve decades with both signs: sums depend on their order."""
    g = np.random.default_rng(seed)
    shape = (r, rows, F_FOLD)
    x = g.standard_normal(shape, dtype=np.float32)
    x *= np.power(np.float32(10), g.random(shape, dtype=np.float32) * np.float32(12) - np.float32(6))
    return x[0], x[1:]


def fold_model(main, reps):
    """The fold's fixed order in fp32: main, then replicas 0 .. nrep - 1."""
    acc = main.copy()
    for rep in reps:
        acc = acc + rep
    return acc


@pytest.mark.parametrize("r", [2, 4, 8, 16, 32, 64])
def test_fold_model_is_order_sensitive(r):
    """The numpy model of the fold, on the data the GPU test uses: within the fp64 bound of its nrep adds, and different
    (bit for bit) from a fold that skips a replica, adds them in another order, or sums the replicas before the main table,
    so that the bit-exact GPU comparison would see each of those."""
    main, reps = fold_data(513, r, r)
    got = fold_model(main, reps)
    exact = main.astype(np.float64) + reps.astype(np.float64).sum(0)
    mag = np.abs(main).astype(np.float64) + np.abs(reps).astype(np.float64).sum(0)
    assert (np.abs(got - exact) <= (r - 1) * U * mag * 1.0001).all()
    alternatives = {"skip last": fold_model(main, reps[:-1]), "reversed": fold_model(main, reps[::-1]),
                    "replicas first": fold_model(np.zeros_like(main), np.concatenate((reps, main[None]))),
                    "skip first": fold_model(main, reps[1:])}
    for name, alt in alternatives.items():
        if name in ("reversed", "replicas first") and r == 2:
            continue            # one replica: the order of two fp32 terms does not change their sum
        assert not np.array_equal(alt, got), f"R={r}: the data cannot tell the fold from '{name}'"


@gpu
@pytest.mark.parametrize("r", [2, 4, 8, 16, 32, 64])
def test_fold_kernel_is_bit_exact(r, built_lib):
    from shine_mapping_b200 import _abi
    levels = fold_levels(r)
    d = _abi.ShineOctree()
    d.num_levels, d.feature_dim = len(levels), F_FOLD
    keep, host = [], []
    hash_slots = torch.zeros(16 * _abi.HASH_SLOT_BYTES, dtype=torch.uint8, device=DEV)
    for i, (rows, rr, has_grads) in enumerate(levels):
        main, reps = fold_data(rows, rr, 1000 * r + i)
        feats = torch.zeros(rows, F_FOLD, device=DEV)
        g = torch.from_numpy(main).to(DEV) if has_grads else None
        rep = torch.from_numpy(np.ascontiguousarray(reps)).to(DEV) if rr > 1 else None
        lv = d.lv[i]
        lv.hash_slots, lv.features, lv.hash_capacity, lv.rows, lv.level = hash_slots.data_ptr(), feats.data_ptr(), 16, rows, 12 - i
        lv.feature_grads = g.data_ptr() if g is not None else None
        lv.num_replicas = rr
        lv.grad_replicas = rep.data_ptr() if rep is not None else None
        keep.append((feats, g, rep))
        host.append((main, reps))
    assert built_lib.shine_reduce_grad_replicas(C.byref(d), _abi.stream_ptr(DEV)) == 0
    torch.cuda.synchronize()
    for i, ((rows, rr, has_grads), (feats, g, rep), (main, reps)) in enumerate(zip(levels, keep, host)):
        if has_grads:
            want = fold_model(main, reps) if rr > 1 else main
            got = g.cpu().numpy()
            bad = np.argwhere(got.view(np.uint32) != want.view(np.uint32))
            assert bad.size == 0, f"level {i} (rows {rows}, R {rr}): {len(bad)} elements differ from the model, first {bad[0]}"
            if rep is not None:
                assert int(torch.count_nonzero(rep)) == 0, f"level {i}: replicas not re-zeroed"
        else:   # no gradient table: the level is skipped and its replicas stay as they were
            assert np.array_equal(rep.cpu().numpy(), reps), f"level {i} without gradients was touched"


# ---- ABI rejections (no GPU: the descriptor checks run before any device call) -------------------------------------------------

def _abi_call(lib, name, desc):
    """name: an entry, or "entry:main_loss_type" for the shine_sdf_* steps"""
    from shine_mapping_b200 import _abi
    from shine_mapping_b200.trainer import loss_flags
    dec = _abi.ShineDecoder()
    dec.w1 = dec.w2 = dec.w3 = 0x1000
    dec.in_dim, dec.hidden, dec.mlp_level = 8, 32, 2
    o = C.byref(desc)
    entry, _, loss = name.partition(":")
    if entry == "shine_query_bwd":
        return lib.shine_query_bwd(o, None, 0, None, None)
    if entry == "shine_reduce_grad_replicas":
        return lib.shine_reduce_grad_replicas(o, None)
    # sdf_l1 / sdf_l2 need their weights and a valid scale even for an empty batch
    weight, scale = (None, 1.0) if loss == "sdf_bce" else (0x3000, 0.01)
    if entry == "shine_sdf_step":
        return lib.shine_sdf_step(o, C.byref(dec), None, None, weight, 0, 1.0, scale, 1.0, None, None, None,
                                  loss_flags(loss), None)
    return lib.shine_sdf_eikonal_step(o, C.byref(dec), None, None, weight, 0, 1.0, scale, 1.0, 0.1, None, None, None, None,
                                      None, loss_flags(loss), None)

@pytest.mark.parametrize("name", ["shine_sdf_step:sdf_bce", "shine_query_bwd", "shine_reduce_grad_replicas",
                                  "shine_sdf_eikonal_step:sdf_bce", "shine_sdf_step:sdf_l1", "shine_sdf_step:sdf_l2",
                                  "shine_sdf_eikonal_step:sdf_l1", "shine_sdf_eikonal_step:sdf_l2"])
def test_abi_replica_checks(name, built_lib):
    """R must be a power of two up to 64 with a scratch pointer; R = 0 and 1 need no scratch.  Placeholder pointers and an
    empty batch: an accepted descriptor returns OK without touching the device."""
    from shine_mapping_b200 import _abi
    d = _abi.ShineOctree()
    d.num_levels, d.feature_dim = 2, 8
    for lv in d.lv[:2]:
        lv.hash_slots = lv.features = lv.feature_grads = 0x1000
        lv.hash_capacity, lv.rows, lv.level = 16, 10, 12
    for r in (0, 1):
        d.lv[1].num_replicas, d.lv[1].grad_replicas = r, None
        assert _abi_call(built_lib, name, d) == 0, f"R = {r} without scratch was refused"
    for r in (3, 65, 128):
        d.lv[1].num_replicas, d.lv[1].grad_replicas = r, 0x2000
        assert _abi_call(built_lib, name, d) == INVALID, f"R = {r} was accepted"
    d.lv[1].num_replicas, d.lv[1].grad_replicas = 2, None
    assert _abi_call(built_lib, name, d) == INVALID, "R = 2 without scratch was accepted"
    d.lv[1].grad_replicas = 0x2000
    d.lv[0].num_replicas, d.lv[0].grad_replicas = 64, None
    assert _abi_call(built_lib, name, d) == INVALID, "a bad first level was accepted"


# ---- the bound itself -------------------------------------------------------------------------------------------------------

def test_bound_passes_the_fp32_oracle_and_sees_one_lost_term():
    """For each loss, the fp32 oracle (a correct fp32 implementation in another summation order) is inside the bound; the
    same gradients with one (point, corner) term taken out of a row that several points touch, or added twice, are not.
    sdf_l1 takes the fp32 oracle's pred as the kernel's for its signs near the label."""
    for loss_type in ("sdf_bce",) + DIFF_LOSSES:
        case, _ = drop_kinks(with_weights(make_case(n_points=1500, n_batch=1500, feat_levels=3, seed=5), loss_type, 5))
        o, dec = oracle_from_case(case)
        res = sdo.train_step(o, dec, *(torch.from_numpy(case[k]) for k in ("coord", "label", "weight")),
                             case["cfg"]["sigma"], case["cfg"]["weighted"], case["cfg"]["reduction"], loss_type=loss_type,
                             scale=_scale(case))
        got, pred = [g.detach().numpy() for g in res["table_grads"]], res["pred"].numpy()
        ref = Ref(case, loss_type=loss_type, pred=pred)
        ref.grade(got, f"fp32 oracle {loss_type}", pred)
        o, dec = _oracle64(case)
        ix, w = _blend(o, torch.from_numpy(case["coord"]))[0]            # leaf level = table L - 1
        kk = len(got) - 1
        terms = w[:, None].numpy() * np.repeat(ref.dfeat, 8, 0)          # w_{j,c} dfeat_j of every (point, corner)
        rows = ix.numpy()
        # a median-sized term in a row that three or more terms touch
        cand = [j for j in range(len(rows)) if rows[j] >= 0 and ref.k[kk][rows[j]] >= 3 and np.abs(terms[j]).max() > 0]
        cand.sort(key=lambda j: np.abs(terms[j]).max())
        j = cand[len(cand) // 2]
        term = terms[j]
        for sign, name in ((-1.0, "lost"), (1.0, "duplicated")):
            bad = [t.copy() for t in got]
            bad[kk][rows[j]] += sign * term.astype(np.float32)
            with pytest.raises(AssertionError, match="outside the bound"):
                ref.grade(bad, f"one {name} term {loss_type}")
