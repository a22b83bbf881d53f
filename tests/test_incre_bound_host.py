"""The fp64 reference of the continual-learning terms and its per-element bounds (tests/incre_bound.py), checked without a GPU:
  * the explicit reference equals the oracle's autograd cal_regularization (value, and the gradient of lambda * reg) and
    its cal_feature_importance in fp64, at 1, 3 and 8 levels and F = 4 and 32;
  * an fp32 restatement of the kernels in their operation order lies inside every bound, over one grid pass and many;
  * seeded mistakes land outside the bound: the factor 2 missing from the gradient, a touched row dropped from the list, a
    row listed twice, importance adding g instead of |g|, Omega and f_last swapped.  The dropped row passes the normwise
    bar these terms had before (1e-5 of each level's maximum);
  * the bound is not vacuous: median and worst bound / |want| over the touched elements are printed."""
import numpy as np
import pytest
import torch

from oracle import shine_oracle as orc
from tests.eikonal_bound import touched_ratio
from tests.error_bound import oracle64
from tests.incre_bound import (RegRef, grade_rows, importance_sweep64, importance_want, kernel_importance32,
                               kernel_regularization32, regularization64, touched_sets)
from tests.parity_utils import make_case, oracle_from_case

LAM = 1e3
SHAPES = [(L, F) for L in (1, 3, 8) for F in (4, 32)]


def _case(L, F, seed=3):
    """A case with seeded f_last (f + 0.01 N), Omega of each row spread over six decades (trash row 0) and signed gradient tables."""
    case = make_case(n_points=1200, n_batch=1200, feat_levels=L, feature_dim=F, seed=seed, reduction="sum")
    g = np.random.default_rng(seed)
    tables = case["tables"]
    last = [(t + 0.01 * g.standard_normal(t.shape)).astype(np.float32) for t in tables]
    imp = [(10.0 ** g.uniform(-6, 0, (t.shape[0], 1)) * g.uniform(0.5, 1.0, t.shape)).astype(np.float32) for t in tables]
    for w in imp:
        w[-1] = 0.0
    grads = [(g.standard_normal(t.shape) * 10.0 ** g.uniform(-3, 1, t.shape)).astype(np.float32) for t in tables]
    return case, last, imp, grads


@pytest.mark.parametrize("L,F", SHAPES, ids=[f"L{L}-F{F}" for L, F in SHAPES])
def test_explicit_reference_equals_the_oracle(L, F):
    case, last, imp, _ = _case(L, F)
    o, dec = oracle64(case)
    coord, label = torch.from_numpy(case["coord"]), torch.from_numpy(case["label"])
    o.get_indices(coord)
    last64 = [torch.from_numpy(t).double() for t in last]
    imp64 = [torch.from_numpy(t).double() for t in imp]
    want = orc.cal_regularization(o, last64, imp64)
    (LAM * want).backward()
    value, grads = regularization64(o, last, imp, LAM)
    want = float(want.detach())
    assert abs(value - want) <= 1e-12 * abs(want)
    for kk, f in enumerate(o.hier_features):
        ref = f.grad.numpy()
        assert np.abs(grads[kk] - ref).max() <= 1e-12 * np.abs(ref).max(), kk
    rows = touched_sets(o, case["coord"])
    assert sum(r.shape[0] for r in rows) > 0
    for kk, r in enumerate(rows):
        assert r.max() < o.hier_features[kk].shape[0] - 1          # a miss marks nothing: the trash row is never touched
    imp_o = orc.cal_feature_importance(o, dec, coord, label.double(), case["cfg"]["sigma"], 256, 2, "sum")
    imp_x, strides = importance_sweep64(o, dec, coord, label.double(), case["cfg"]["sigma"], 256, 2)
    assert len(strides) == -(-coord.shape[0] // 512)
    for kk in range(L):
        ref = imp_o[kk].detach().numpy()
        assert np.abs(imp_x[kk] - ref).max() <= 1e-12 * np.abs(ref).max(), kk


@pytest.mark.parametrize("L,F", SHAPES, ids=[f"L{L}-F{F}" for L, F in SHAPES])
@pytest.mark.parametrize("sm_count", [1, 132])
def test_fp32_kernels_lie_inside_the_bounds(L, F, sm_count):
    """sm_count 1 puts up to 8 blocks on the grid: every thread takes several grid-stride items."""
    case, last, imp, grads = _case(L, F)
    o, _ = oracle_from_case(case)
    rows = touched_sets(o, case["coord"])
    caps = [t.shape[0] for t in case["tables"]]
    ref = RegRef(case["tables"], last, imp, rows, LAM, grads=grads)
    value, got = kernel_regularization32(case["tables"], last, imp, grads, rows, LAM, F, sm_count, caps, init=0.5)
    worst = grade_rows(got, ref.want, ref.bound, f"regularisation L={L} F={F} sm={sm_count}")
    vb = ref.value_bound(caps, F, sm_count, init=0.5)
    assert abs(value - 0.5 - ref.value) <= vb, (value, ref.value, vb)
    om, gz = kernel_importance32(imp, grads, rows)
    iw, ib = importance_want(imp, [([np.abs(g) for g in grads], None)], [rows])
    worst = max(worst, grade_rows(om, iw, ib, f"importance L={L} F={F}"))
    for kk, r in enumerate(rows):
        assert not gz[kk][r].any()
        keep = np.ones(gz[kk].shape[0], dtype=bool)
        keep[r] = False
        assert np.array_equal(gz[kk][keep], grads[kk][keep])
    med, hi = touched_ratio(ref.bound, ref.want)
    print(f"[incre bounds] L={L} F={F}: value error {abs(value - 0.5 - ref.value) / vb:.3f} of its bound; "
          f"gradient bound / |want| median {med:.2e} worst {hi:.2e}")
    assert worst <= 1.0


def _fails(fn):
    with pytest.raises(AssertionError):
        fn()


def test_seeded_mistakes_leave_the_bound():
    L, F = 3, 8
    case, last, imp, grads = _case(L, F, seed=11)
    o, _ = oracle_from_case(case)
    rows = touched_sets(o, case["coord"])
    caps = [t.shape[0] for t in case["tables"]]
    zero = [np.zeros_like(t) for t in case["tables"]]          # the regulariser alone, as the earlier normwise test ran it
    ref = RegRef(case["tables"], last, imp, rows, LAM)

    def reg(rows_=rows, lam=LAM, last_=last, imp_=imp):
        return kernel_regularization32(case["tables"], last_, imp_, zero, rows_, lam, F, 132, caps)

    value, got = reg()
    grade_rows(got, ref.want, ref.bound, "unmodified")
    vb = ref.value_bound(caps, F, 132)
    assert abs(value - ref.value) <= vb
    # the factor 2 missing from the gradient
    _fails(lambda: grade_rows(reg(lam=LAM / 2)[1], ref.want, ref.bound, "lambda instead of 2 lambda"))
    # Omega and f_last swapped
    v_sw, g_sw = reg(last_=imp, imp_=last)
    _fails(lambda: grade_rows(g_sw, ref.want, ref.bound, "Omega and f_last swapped"))
    assert abs(v_sw - ref.value) > vb
    # one row listed twice: the one with the largest term
    kk = L - 1
    r = rows[kk]
    twice = [x.copy() for x in rows]
    twice[kk] = np.concatenate([twice[kk], [r[np.argmax(np.abs(ref.t[kk][r]).max(1))]]])
    v_tw, g_tw = reg(rows_=twice)
    _fails(lambda: grade_rows(g_tw, ref.want, ref.bound, "row listed twice"))
    assert abs(v_tw - ref.value) > vb
    # one touched row dropped: the one with the smallest term, which the normwise bar cannot see
    drop = r[np.argmin(np.abs(ref.t[kk][r]).max(1))]
    dropped = [x.copy() for x in rows]
    dropped[kk] = dropped[kk][dropped[kk] != drop]
    _, g_dr = reg(rows_=dropped)
    _fails(lambda: grade_rows(g_dr, ref.want, ref.bound, "row dropped"))
    for a, b in zip(g_dr, ref.want):
        assert np.abs(a[:-1] - b[:-1]).max() <= 1e-5 * np.abs(b[:-1]).max() + 1e-12   # passes the old normwise bar
    # importance adding g instead of |g|
    iw, ib = importance_want(imp, [([np.abs(g) for g in grads], None)], [rows])
    grade_rows(kernel_importance32(imp, grads, rows)[0], iw, ib, "importance")
    _fails(lambda: grade_rows(kernel_importance32(imp, grads, rows, absolute=False)[0], iw, ib, "importance adds g"))
    med, hi = touched_ratio(ref.bound, ref.want)
    print(f"[incre bounds] gradient bound / |want|: median {med:.2e}, worst {hi:.2e}")
