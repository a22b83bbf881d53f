"""The fp64 reference of `sdf_grad_at` and of the registration sums (tests/grad_field_bound.py), checked without a GPU:
  * an fp32 numpy restatement of sdf_grad_at, op for op (FMAs as an fp64 multiply-add rounded to fp32), lies inside
    the bound on natural maps, poly and linear, fresh tables and x300, points outside the cube included, and at kink
    points placed on purpose (a bias set so that one point's pre-activation is 0 in fp64);
  * its registration sums in fp64 lie inside RegBound;
  * corrupted restatements land outside: one corner's dw sign flipped, one level left out, a non-kink unit's mask
    flipped, dt without its res / 2 factor, and one point's share counted twice in H."""
import numpy as np
import pytest
import torch

from tests.error_bound import oracle64
from tests.grad_field_bound import GradRef, RegBound, gm_weight, grade_reg, shares
from tests.parity_utils import make_case

F32 = np.float32


def fma(a, b, c):
    """fp32 fma(a, b, c): the product is exact in fp64, the sum rounds there, then to fp32 (a double rounding, within
    the bound's slack)"""
    return (np.asarray(a, np.float64) * np.asarray(b, np.float64) + np.asarray(c, np.float64)).astype(F32)


def sdf_grad_fp32(case, coord, flip_dw=None, drop_level=None, flip_mask=None, no_half_res=False):
    """sdf_grad_at in fp32 numpy, in the kernel's order -> (pred [n], g [n, 3], valid [n]).
    flip_dw=(level position, corner): that corner's dw with the wrong sign; drop_level: a level position skipped;
    flip_mask=n: layer-1 unit n's mask inverted in the dq loop; no_half_res: dt = t'(d) without res / 2."""
    o, dec = oracle64(case)
    x = np.ascontiguousarray(coord, dtype=F32)
    n, L = x.shape[0], o.featured_level_num
    levels = getattr(o, "kept", [o.max_level - i for i in range(L)])
    idx = o.get_indices(torch.from_numpy(x))
    tables = [t.detach().float().numpy() for t in o.hier_features]
    f = np.zeros((n, 8), F32)
    J = np.zeros((n, 8, 3), F32)
    valid = idx[0][:, 0].numpy() >= 0
    for i in range(L):
        if i == drop_level:
            continue
        ix = idx[i].numpy()
        hit = ix[:, 0] >= 0
        res = F32(2.0 ** levels[i])
        c = res * (x * F32(0.5) + F32(0.5))
        d = c - np.trunc(c)
        s = res * F32(0.5)
        if case["cfg"]["poly_int_on"]:
            d2 = d * d
            t = F32(3) * d2 - F32(2) * (d2 * d)
            dt = F32(6) * d - F32(6) * d2
            dt = dt if no_half_res else dt * s
        else:
            t = d
            dt = np.full_like(d, F32(1) if no_half_res else s)
        u = F32(1) - t
        rows = tables[L - 1 - i][np.where(hit[:, None], ix, 0)]
        for cc in range(8):
            bits = ((cc >> 2) & 1, (cc >> 1) & 1, cc & 1)
            fac = [t[:, a] if bits[a] else u[:, a] for a in range(3)]
            dfac = [dt[:, a] if bits[a] else -dt[:, a] for a in range(3)]
            if flip_dw == (i, cc):
                dfac = [-v for v in dfac]
            w = (fac[0] * fac[1]) * fac[2]
            dw = [(dfac[0] * fac[1]) * fac[2], (fac[0] * dfac[1]) * fac[2], (fac[0] * fac[1]) * dfac[2]]
            row = rows[:, cc]
            for k in range(8):
                f[:, k] = np.where(hit, fma(w, row[:, k], f[:, k]), f[:, k])
                for a in range(3):
                    J[:, k, a] = np.where(hit, fma(dw[a], row[:, k], J[:, k, a]), J[:, k, a])
    g = {k: v.detach().float().numpy() for k, v in dec.items()}
    W1, W2, w3 = g["layers.0.weight"], g["layers.1.weight"], g["lout.weight"].reshape(-1)
    b1 = g.get("layers.0.bias", np.zeros(32, F32))
    b2 = g.get("layers.1.bias", np.zeros(32, F32))
    b3 = g["lout.bias"].reshape(-1)[0] if "lout.bias" in g else F32(0)
    h1 = np.zeros((n, 32), F32)
    m1 = np.zeros((n, 32), bool)
    for u_ in range(32):
        a = np.full(n, b1[u_], F32)
        for k in range(8):
            a = fma(W1[u_, k], f[:, k], a)
        m1[:, u_] = a > 0
        h1[:, u_] = np.maximum(a, F32(0))
    pr = np.full(n, b3, F32)
    m2 = np.zeros((n, 32), bool)
    for j in range(32):
        a = np.full(n, b2[j], F32)
        for u_ in range(32):
            a = fma(W2[j, u_], h1[:, u_], a)
        m2[:, j] = a > 0
        pr = fma(np.maximum(a, F32(0)), w3[j], pr)
    if flip_mask is not None:
        m1[:, flip_mask] = ~m1[:, flip_mask]
    dq = np.zeros((n, 8), F32)
    for u_ in range(32):
        a = np.zeros(n, F32)
        for j in range(32):
            a = fma(W2[j, u_], np.where(m2[:, j], w3[j], F32(0)), a)
        for k in range(8):
            dq[:, k] = np.where(m1[:, u_], fma(a, W1[u_, k], dq[:, k]), dq[:, k])
    grad = np.zeros((n, 3), F32)
    for a in range(3):
        s = np.zeros(n, F32)
        for k in range(8):
            s = fma(J[:, k, a], dq[:, k], s)
        grad[:, a] = s
    return pr, grad, valid


def _case(levels, poly, scale, seed, bias=True, world=12):
    case = make_case(n_points=1500, n_batch=1200, feat_levels=levels, seed=seed, poly=poly, bias=bias, world_level=world)
    case["tables"] = [(t * F32(scale)).astype(F32) for t in case["tables"]]
    rng = np.random.default_rng(seed)
    surf = np.concatenate(case["frames"])
    near = surf[rng.integers(0, surf.shape[0], 600)] + rng.normal(0, 2.0 ** -world, (600, 3))
    out = np.array([[1.0, 0.1, 0.0], [-1.0, 0.0, 0.2], [1.25, -1.5, 0.3], [-1.3, 0.0, 0.0],
                    [np.nextafter(F32(1), F32(0)), 0.0, 0.0]])
    return case, np.concatenate((case["coord"], near, out)).astype(F32)


def _kinked(case, coord, units=(3, 11, 19, 27)):
    """The case with biases set so that, per listed unit, one point sits on a layer-1 (and then a layer-2) kink in fp64
    -> (case, the kink points)."""
    from tests.eikonal_bound import _decoder, gather, level_geometry
    o, dec = oracle64(case)
    geo = level_geometry(o, coord)
    f = gather(o, geo)[0]
    W1, b1, W2, b2, w3, b3 = _decoder(dec)
    hit = np.flatnonzero(geo[0]["ix"][:, 0] >= 0)
    pick = hit[:: max(1, hit.size // (2 * len(units)))][: 2 * len(units)]
    d = dict(case["dec"])
    nb1 = d["layers.0.bias"].astype(F32).copy()
    for u_, p in zip(units, pick[: len(units)]):
        nb1[u_] = F32(-(W1[u_] @ f[p]))
    d["layers.0.bias"] = nb1
    h1 = np.maximum(f @ W1.T + nb1.astype(np.float64), 0.0)
    nb2 = d["layers.1.bias"].astype(F32).copy()
    for j, p in zip(units, pick[len(units):]):
        nb2[j] = F32(-(W2[j] @ h1[p]))
    d["layers.1.bias"] = nb2
    return dict(case, dec=d), pick


CASES = [(3, True, 1.0, 3), (3, True, 300.0, 4), (2, False, 300.0, 5), (1, False, 1.0, 6), (4, True, 300.0, 7)]


@pytest.mark.parametrize("levels,poly,scale,seed", CASES)
def test_fp32_restatement_inside_the_bound(levels, poly, scale, seed):
    case, coord = _case(levels, poly, scale, seed)
    ref = GradRef(case, coord)
    pred, g, valid = sdf_grad_fp32(case, coord)
    assert np.array_equal(valid, ref.valid)
    assert ref.valid.sum() > 500 and (~ref.valid).sum() > 5
    ref.grade(g, f"L{levels} poly {poly} x{scale}", got_pred=pred)
    assert ref.n_dropped <= max(2, ref.n // 500)


@pytest.mark.parametrize("poly", [True, False])
def test_fp32_restatement_inside_the_bound_at_kinks(poly):
    case, coord = _case(3, poly, 300.0, 21)
    case, pick = _kinked(case, coord)
    ref = GradRef(case, coord)
    assert ref.kink[pick].sum() >= len(pick) - 1, "the placed kinks are uncertain units"
    pred, g, _ = sdf_grad_fp32(case, coord)
    ref.grade(g, f"kinks poly {poly}", got_pred=pred)
    assert ref.kinks >= 7


def _outside(ref, g, pred=None):
    """number of graded points outside every alternative's bound"""
    best = np.full(ref.n, np.inf)
    np.minimum.at(best, ref.pt, ref.row_ratio(g, pred))
    return int(((best > 1.0) & ~ref.dropped).sum())


@pytest.mark.parametrize("poly", [True, False])
def test_corruptions_land_outside(poly):
    case, coord = _case(3, poly, 300.0, 31)
    ref = GradRef(case, coord)
    pred, g, _ = sdf_grad_fp32(case, coord)
    assert _outside(ref, g, pred) == 0
    # a unit that is live and far from its kink at many points
    from tests.eikonal_bound import _decoder, gather, level_geometry
    o, dec = oracle64(case)
    f = gather(o, level_geometry(o, coord))[0]
    W1, b1 = _decoder(dec)[:2]
    pre = f @ W1.T + b1
    unit = int(np.argmax((np.abs(pre) > 1e-3 * np.abs(pre).max()).sum(0)))
    for name, kw in (("dw sign", dict(flip_dw=(1, 5))), ("level left out", dict(drop_level=2)),
                     ("mask flipped", dict(flip_mask=unit)), ("dt without res / 2", dict(no_half_res=True))):
        p2, g2, _ = sdf_grad_fp32(case, coord, **kw)
        bad = _outside(ref, g2, p2)
        print(f"poly {poly}: {name}: {bad} points outside")
        assert bad > 0, f"{name}: the corrupted restatement passes"


@pytest.mark.parametrize("poly,kappa", [(True, 0.05), (False, 0.5), (True, 1e15), (True, 1e-12)])
def test_registration_sums_inside_and_double_count_outside(poly, kappa):
    case, coord = _case(3, poly, 300.0 if poly else 1.0, 41)
    case, _ = _kinked(case, coord)
    ref = GradRef(case, coord)
    sigma = F32(case["cfg"]["sigma"])
    rb = RegBound(ref, sigma, kappa)
    pred, g, valid = sdf_grad_fp32(case, coord)
    use = valid & ~ref.dropped
    gv = (sigma * g).astype(F32).astype(np.float64)
    r = (sigma * pred).astype(F32).astype(np.float64)
    sh = shares(gv[use], r[use], coord[use].astype(np.float64), kappa * kappa)
    got = np.concatenate((sh.sum(0), [use.sum()]))
    idx = np.flatnonzero(~ref.dropped)
    want, bound = rb.expect(idx)
    grade_reg(got, want, bound, f"host sums poly {poly} kappa {kappa}")
    w = gm_weight(r[use] ** 2, kappa * kappa)
    if kappa > 1e10:
        assert np.all(w == 1.0)
        return
    if kappa < 1e-6:
        # most points have w < 2^-60; those within e_r of r = 0 keep w anywhere in [w(e_r), 1], and dominate the bound
        assert np.mean(w < 2.0 ** -60) > 0.5
        return
    # one point's share twice in H: the point with the largest H share
    k = int(np.argmax(np.abs(sh[:, :21]).max(1)))
    twice = got.copy()
    twice[:21] += sh[k, :21]
    with pytest.raises(AssertionError):
        grade_reg(twice, want, bound, "double count")
