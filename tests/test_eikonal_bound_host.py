"""The fp64 eikonal reference and its per-element bounds (tests/eikonal_bound.py), checked without a GPU:
  * the explicit reference equals the reference's own autograd recipe run entirely in fp64 (coordinates included);
  * an independent fp32 implementation, the fp32 oracle (autograd, exact expf, its own summation order), lies inside every
    bound;
  * seeded mistakes in one point's eikonal scatter land outside the bound while passing the normwise bar of the parity
    tests (1e-3 of each level's maximum);
  * the bound is not vacuous: median and worst bound / |want| over the touched elements are printed."""
import numpy as np
import pytest
import torch

from tests import sdf_diff_oracle as sdo
from tests.eikonal_bound import EikRef, QueryRef, _scale, clean_case, dominant_weight, touched_ratio
from tests.error_bound import grade_values, oracle64, subset
from tests.parity_utils import make_case, oracle_from_case

LOSSES = ("sdf_bce", "sdf_l1", "sdf_l2")


def _case(loss_type, levels=3, poly=True, scale=300.0, seed=5, weighted=False, reduction="mean", n_batch=1200):
    case = make_case(n_points=1500, n_batch=n_batch, feat_levels=levels, seed=seed, poly=poly,
                     weighted=weighted or loss_type != "sdf_bce", reduction=reduction)
    case["tables"] = [(t * np.float32(scale)).astype(np.float32) for t in case["tables"]]
    return case


def _same_cells(case):
    """Points whose fp32 and fp64 cell (integer part of res (0.5 x + 0.5)) agree on every level and axis."""
    c = case["cfg"]
    x32 = case["coord"].astype(np.float32)
    keep = np.ones(x32.shape[0], dtype=bool)
    for i in range(c["tree_level_feat"]):
        res = 2.0 ** (c["tree_level_world"] - i)
        c32 = np.float32(res) * (x32 * np.float32(0.5) + np.float32(0.5))
        c64 = res * (x32.astype(np.float64) * 0.5 + 0.5)
        keep &= (np.trunc(c32) == np.trunc(c64)).all(1)
    return keep


def _fp32_oracle(case, weight_e, loss_type):
    o, dec = oracle_from_case(case)
    c = case["cfg"]
    r = sdo.train_step_eikonal(o, dec, *(torch.from_numpy(case[k]) for k in ("coord", "label", "weight")), c["sigma"],
                               weight_e, c["weighted"], c["reduction"], loss_type=loss_type, scale=_scale(case))
    return {"table_grads": [t.detach().numpy() for t in r["table_grads"]], "pred": r["pred"].numpy(),
            "g": r["g"].numpy(), "loss": float(r["bce"]), "eikonal": float(r["eikonal"])}


@pytest.mark.parametrize("loss_type", LOSSES)
@pytest.mark.parametrize("poly", [True, False])
def test_explicit_reference_equals_fp64_autograd(loss_type, poly):
    case = _case(loss_type, levels=3, poly=poly, seed=11, weighted=True, reduction="sum" if poly else "mean")
    keep = _same_cells(case)
    case = subset(case, keep)
    ref = EikRef(case, 0.1, loss_type, exact=True)
    o, dec = oracle64(case)
    c = case["cfg"]
    coord = torch.from_numpy(case["coord"].astype(np.float64))
    label, weight = (torch.from_numpy(case[k]).double() for k in ("label", "weight"))
    r = sdo.train_step_eikonal(o, dec, coord, label, weight, c["sigma"], 0.1, c["weighted"], c["reduction"],
                               loss_type=loss_type, scale=_scale(case))
    pairs = [("pred", ref.pred, r["pred"]), ("g", ref.g, r["g"]), ("loss", ref.loss, r["bce"]),
             ("eikonal", ref.eikonal, r["eikonal"])]
    pairs += [(f"table {kk}", ref.rows.want[kk][:-1], t.detach().numpy()[:-1]) for kk, t in enumerate(r["table_grads"])]
    worst = 0.0
    for name, a, b in pairs:
        b = np.asarray(b.detach().numpy() if torch.is_tensor(b) else b, dtype=np.float64)
        rel = float(np.abs(np.asarray(a) - b).max() / max(np.abs(b).max(), 1e-300))
        assert rel <= 1e-10, f"{loss_type} poly={poly}: {name} differs from fp64 autograd by {rel:.2e} of its maximum"
        worst = max(worst, rel)
    print(f"{loss_type} poly={poly}: {int(keep.sum())} of {keep.shape[0]} points, worst {worst:.1e} relative")


@pytest.mark.parametrize("loss_type,levels,poly,scale,weighted,reduction", [
    ("sdf_bce", 3, True, 300.0, False, "mean"), ("sdf_bce", 4, False, 1.0, True, "sum"), ("sdf_bce", 1, True, 300.0, True, "mean"),
    ("sdf_l1", 3, True, 300.0, True, "mean"), ("sdf_l1", 2, False, 1.0, True, "mean"),
    ("sdf_l2", 3, False, 300.0, True, "mean"), ("sdf_l2", 4, True, 1.0, True, "mean"),
])
def test_fp32_oracle_is_inside_the_bound(loss_type, levels, poly, scale, weighted, reduction):
    """At weight_e = 0.1 and at 100: pred, g, loss, eikonal and every table-gradient element of the fp32 oracle."""
    case, dropped = clean_case(_case(loss_type, levels, poly, scale, 20 + levels, weighted, reduction), loss_type)
    for weight_e in (0.1, 100.0):
        got = _fp32_oracle(case, weight_e, loss_type)
        ref = EikRef(case, weight_e, loss_type, pred=got["pred"])
        what = f"fp32 oracle {loss_type} L={levels} poly={poly} x{scale:g} W={weight_e:g} (dropped {dropped})"
        ref.grade(got, what)
        med, worst = touched_ratio([ref.rows.bound(kk) for kk in range(levels)], ref.rows.want)
        print(f"{what}: bound / |want| over touched elements: median {med:.1e}, worst {worst:.1e}")
        assert med < 1e-2, f"{what}: the bound is loose (median {med:.1e} of |want|)"


def _normwise_passes(got, ref):
    """The normwise bar of the parity tests' eikonal checks on the table gradients: within 1e-3 of each level's maximum."""
    return all(np.abs(g[:-1] - w[:-1]).max() <= 1e-3 * np.abs(w[:-1]).max() + 1e-9 for g, w in zip(got, ref.rows.want))


def _mistakes(ref, j):
    """name -> [(table, rows, delta rows)] of seeded mistakes in point j's scatter (the last three on the coarsest level,
    where a row sums many points and one point's share stays below the normwise bar)."""
    q = ref.q[j]
    lv = [(ref.L - 1 - i, g["ix"][j], ref.sc1[i][j], ref.sc2[i][j], g["level"]) for i, g in enumerate(ref.geo)]
    out = {"eikonal term of one point dropped": [(kk, ix, -sc2[:, None] * q) for kk, ix, sc1, sc2, lev in lv]}
    kk, ix, sc1, sc2, lev = lv[-1]
    out["grad w without res/2 on one level"] = [(kk, ix, (2.0 ** (1 - lev) - 1) * sc2[:, None] * q)]
    sc = sc1 + sc2
    c = int(np.argsort(np.abs(sc))[4])                                  # a median-sized corner
    moved = np.zeros((8, q.shape[0]))
    moved[c], moved[c ^ 1] = -sc[c] * q, sc[c] * q
    out["sc scattered to the wrong corner"] = [(kk, ix, moved)]
    out["sigma missing from r"] = [(kk, ix, (1.0 / ref.sigma - 1) * sc2[:, None] * q)]
    return out


def _apply(got, mistake):
    bad = [t.astype(np.float64).copy() for t in got]
    for kk, ix, delta in mistake:
        np.add.at(bad[kk], ix, delta)
    return bad


@pytest.mark.parametrize("loss_type", LOSSES)
def test_seeded_mistakes_are_outside_the_bound(loss_type):
    """Each mistake, in one surface point's scatter of the fp32 oracle's result, changes too little for the normwise bar
    and leaves the per-element bound.  weight_e: the eikonal term at 1e-3 of the first term's maximum (0.005 for BCE on
    these x300 tables; sdf_l2's first term is 10^5 x larger).  The point: of the surface points whose mistake the normwise bar passes, the one of
    largest eikonal contribution (the largest such mistake the normwise bar cannot see); the share of all those points
    the bound catches is printed."""
    case, _ = clean_case(_case(loss_type, 3, True, 300.0, 31), loss_type)
    weight_e = dominant_weight(case, loss_type, 1e-3)
    got = _fp32_oracle(case, weight_e, loss_type)
    ref = EikRef(case, weight_e, loss_type, pred=got["pred"])
    ref.grade(got, f"fp32 oracle {loss_type}")
    hits = np.stack([g["ix"][:, 0] >= 0 for g in ref.geo], 1).all(1)
    cand = np.flatnonzero(ref.surf & hits & (np.abs(ref.gam).max(1) > 0))
    size = np.array([max(np.abs(s[j]).max() for s in ref.sc2) * np.abs(ref.q[j]).max() for j in cand])
    cand = cand[np.argsort(size)]
    names = list(_mistakes(ref, int(cand[0])))
    for name in names:
        passing = [j for j in cand if _normwise_passes(_apply(got["table_grads"], _mistakes(ref, int(j))[name]), ref)]
        assert passing, f"{loss_type}: every point's '{name}' fails the normwise bar already"
        j = int(passing[-1])
        bad = _apply(got["table_grads"], _mistakes(ref, j)[name])
        with pytest.raises(AssertionError, match="outside the bound"):
            ref.rows.grade(bad, f"{loss_type}: {name} (point {j})")
        caught = 0
        for jj in passing:
            try:
                ref.rows.grade(_apply(got["table_grads"], _mistakes(ref, int(jj))[name]), "", "quiet")
            except AssertionError:
                caught += 1
        print(f"{loss_type}: '{name}': normwise bar passes it at {len(passing)} of {len(cand)} surface points; "
              f"the bound catches {caught} of those")


def test_query_reference_matches_autograd_and_the_fp32_oracle():
    """The fp32 oracle's feature, coordinate gradient and both tangent products (autograd: its own order, exact fp32
    derivatives of the weights) inside QueryRef's bounds."""
    case = _case("sdf_bce", 3, True, 300.0, 41, n_batch=600)
    n = case["coord"].shape[0]
    rng = np.random.default_rng(0)
    dfeat = (rng.standard_normal((n, 8)) * 10.0 ** rng.uniform(-2, 2, (n, 8))).astype(np.float32)
    tangent = (rng.standard_normal((n, 3)) * 10.0 ** rng.uniform(-2, 2, (n, 3))).astype(np.float32)
    ref = QueryRef(case, dfeat, tangent)
    o, _ = oracle_from_case(case)
    coord = torch.from_numpy(case["coord"]).requires_grad_(True)
    d = torch.from_numpy(dfeat).requires_grad_(True)
    feat = o.query_feature(coord)
    G = torch.autograd.grad(feat, coord, d, create_graph=True)[0]
    tfwd, *rows = torch.autograd.grad(G, [d] + list(o.hier_features), torch.from_numpy(tangent))
    grade_values(feat.detach().numpy(), ref.feat, ref.efeat, "fp32 oracle", "query_fwd")
    grade_values(G.detach().numpy(), ref.G, ref.eG, "fp32 oracle", "coord_grad")
    grade_values(tfwd.numpy(), ref.tfwd, ref.etfwd, "fp32 oracle", "tangent_fwd")
    ref.rows.grade([r.numpy() for r in rows], "fp32 oracle tangent_bwd")
