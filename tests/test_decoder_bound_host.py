"""The fp64 decoder-gradient reference and its per-element bounds (tests/decoder_bound.py), checked without a GPU:
  * the explicit restatement equals the oracle's fp64 autograd decoder gradients, for every loss, weighted and not, mean
    and sum, and without biases;
  * an independent fp32 implementation, the fp32 oracle (autograd, BLAS summation in its own order), lies inside every
    bound at depth n - 1, the worst case of any summation order;
  * seeded mistakes of the kind a rewrite of the kernels' decoder-gradient scheme makes (a tile missing from dW1 / db1, a
    dW2 row scaled by another unit's w3, a zero-tile point missing from the zero-tile sum, a db2 entry without its w3
    factor) pass the normwise bar of the parity tests (2e-4 of each tensor's maximum) and land outside the bound at the
    kernel's depth;
  * the bound is not vacuous: the median bound / |want| per tensor is printed."""
import numpy as np
import pytest
import torch
from scipy.special import expit

from tests import sdf_diff_oracle as sdo
from tests.decoder_bound import B1, B2, KEYS, W1, W2, W3, kernel_depth
from tests.error_bound import drop_kinks
from tests.parity_utils import make_case, oracle_from_case
from tests.test_gpu_replicas import Ref, _far_tiles, with_weights
from tests.test_gpu_sdf_diff import _scale

LOSSES = ("sdf_bce", "sdf_l1", "sdf_l2")
CONFIGS = [pytest.param(lt, w, r, b, id=f"{lt}-{'w' if w else 'u'}-{r}-{'bias' if b else 'nobias'}")
           for lt, w, r, b in [("sdf_bce", False, "mean", True), ("sdf_bce", True, "sum", True),
                               ("sdf_bce", True, "mean", False), ("sdf_bce", False, "sum", False),
                               ("sdf_l1", True, "mean", True), ("sdf_l1", True, "mean", False),
                               ("sdf_l2", True, "mean", True), ("sdf_l2", True, "mean", False)]]


def _case(loss_type, weighted, reduction, bias, n_batch=1500, seed=9, far_tiles=3):
    case = make_case(n_points=1500, n_batch=n_batch, feat_levels=3, seed=seed, weighted=weighted, reduction=reduction,
                     bias=bias)
    case, _ = drop_kinks(with_weights(case, loss_type, seed))
    return _far_tiles(case, far_tiles, 5, seed)           # points that miss every level: exact zero features


def _fp32_oracle(case, loss_type):
    o, dec = oracle_from_case(case)
    c = case["cfg"]
    r = sdo.train_step(o, dec, *(torch.from_numpy(case[k]) for k in ("coord", "label", "weight")), c["sigma"],
                       c["weighted"], c["reduction"], loss_type=loss_type, scale=_scale(case))
    return r["pred"].numpy(), {k: v.detach().numpy() for k, v in r["dec_grads"].items()}


@pytest.mark.parametrize("loss_type,weighted,reduction,bias", CONFIGS)
def test_restatement_equals_fp64_autograd(loss_type, weighted, reduction, bias):
    case = _case(loss_type, weighted, reduction, bias)
    pred, _ = _fp32_oracle(case, loss_type)
    ref = Ref(case, loss_type=loss_type, pred=pred)
    assert sorted(ref.dec.keys) == sorted(k for k in KEYS if k in case["dec"])
    for k in ref.dec.keys:
        want = ref.step["dec_grads"][k]
        scale = max(float(np.abs(want).max()), 1e-300)
        err = float(np.abs(ref.dec.want[k] - want.reshape(ref.dec.want[k].shape)).max())
        assert err <= 1e-10 * scale, f"{k}: restatement off by {err:.3g} (max |want| {scale:.3g})"


@pytest.mark.parametrize("loss_type,weighted,reduction,bias", CONFIGS)
def test_fp32_oracle_is_inside_the_bound(loss_type, weighted, reduction, bias):
    case = _case(loss_type, weighted, reduction, bias)
    pred, got = _fp32_oracle(case, loss_type)
    ref = Ref(case, loss_type=loss_type, pred=pred)
    n = case["coord"].shape[0]
    ref.dec.grade(got, n - 1, f"fp32 oracle {loss_type}")
    print(f"[decoder bounds] median bound / |want| at depth {n - 1}:",
          {k: f"{v:.2e}" for k, v in ref.dec.median_ratio(n - 1).items()})


def _normwise_ok(got, want):
    """compare_step's bar on the decoder gradients: max |d| <= 2e-4 max |want| per tensor."""
    return all(float(np.abs(got[k] - want[k]).max()) <= 2e-4 * float(np.abs(want[k]).max()) for k in want)


def _outside(dref, got, depth):
    with pytest.raises(AssertionError, match="outside the bound"):
        dref.grade(got, depth, "seeded mistake")


@pytest.fixture(scope="module")
def big():
    """~50 k points, Morton-ordered, with zero tiles: the reference, its restated forward and the kernel's depth."""
    from tests.decoder_bound import restate
    from tests.error_bound import abs_feature, decoder_passes, oracle64
    from tests.parity_utils import sort_case_morton
    case = make_case(n_points=1500, n_batch=50000, feat_levels=3, seed=21, weighted=True)
    # layer-2 unit RARE fires on 0.05 % of the points (its bias at the 99.95th percentile of its input) with w3 = 0.95:
    # a small db2 entry and dW2 row next to the tensors' maxima, what a unit of a trained decoder often is
    o, dec = oracle64(case)
    with torch.no_grad():
        f = o.query_feature(torch.from_numpy(case["coord"]))
        _, fw = restate(f, {k: v.detach() for k, v in dec.items()}, torch.zeros(f.shape[0], dtype=torch.float64))
    case["dec"] = dict(case["dec"])
    b2 = np.array(case["dec"][B2], dtype=np.float32, copy=True)
    b2[RARE] = -np.quantile(fw["h1"].numpy() @ np.asarray(case["dec"][W2], dtype=np.float64)[RARE], 0.9995)
    case["dec"][B2] = b2
    w3 = np.array(case["dec"][W3], dtype=np.float32, copy=True)
    w3.reshape(-1)[RARE] = 0.95
    case["dec"][W3] = w3
    case = sort_case_morton(drop_kinks(case)[0])
    case = _far_tiles(case, 40, 1000, 21)
    ref = Ref(case, grouped=True)
    o, dec = oracle64(case)
    with torch.no_grad():
        feat = o.query_feature(torch.from_numpy(case["coord"]))
    g = torch.from_numpy(_g(ref, case))
    _, fw = restate(feat, {k: v.detach() for k, v in dec.items()}, g)
    n = case["coord"].shape[0]
    depth = kernel_depth(n)
    print(f"[decoder bounds] n = {n}, kernel depth {depth}; median bound / |want|:",
          {k: f"{v:.2e}" for k, v in ref.dec.median_ratio(depth).items()})
    return case, ref.dec, feat.numpy(), g.numpy(), fw, depth


RARE = 7


def _g(ref, case):
    """dL/dpred of the (weighted, mean) BCE case in fp64."""
    c = case["cfg"]
    n = case["coord"].shape[0]
    z = expit(case["label"].astype(np.float64) / c["sigma"])
    return np.abs(case["weight"].astype(np.float64)) / n * (expit(ref.pred) - z)


def _rounded(dref):
    return {k: v.astype(np.float32).astype(np.float64) for k, v in dref.want.items()}


def test_seeded_tile_missing_from_dW1_and_db1(big):
    case, dref, feat, g, fw, depth = big
    dh1 = fw["dh1"].numpy()
    n = feat.shape[0]
    tiles = n // 16
    c1 = np.einsum("tpk,tpc->tkc", dh1[:16 * tiles].reshape(tiles, 16, -1), feat[:16 * tiles].reshape(tiles, 16, -1))
    cb = dh1[:16 * tiles].reshape(tiles, 16, -1).sum(1)
    bw, bb = dref.bound(W1, depth), dref.bound(B1, depth)
    ok = ((np.abs(c1) <= 2e-4 * np.abs(dref.want[W1]).max()).all((1, 2)) &
          (np.abs(cb) <= 2e-4 * np.abs(dref.want[B1]).max()).all(1))
    score = np.maximum((np.abs(c1) / np.maximum(bw, 1e-300)).max((1, 2)), (np.abs(cb) / np.maximum(bb, 1e-300)).max(1))
    print(f"[seeded] one tile missing from dW1 / db1: seen by the bound in {int((score > 1).sum())} of {tiles} tiles, by the "
          f"normwise bar in {int((~ok).sum())}, by neither in {int(((score <= 1) & ok).sum())}")
    score[~ok] = 0
    t = int(np.argmax(score))
    assert score[t] > 1, "no tile both passes the normwise bar and leaves the bound"
    got = _rounded(dref)
    got[W1] = got[W1] - c1[t]
    got[B1] = got[B1] - cb[t]
    assert _normwise_ok(got, dref.want)
    _outside(dref, got, depth)
    print(f"[seeded] tile {t} missing from dW1 / db1: {score[t]:.1f} x the bound")


def test_seeded_dW2_row_scaled_by_another_units_w3(big):
    case, dref, feat, g, fw, depth = big
    w3 = np.asarray(case["dec"]["lout.weight"], dtype=np.float64).reshape(-1)
    want, b = dref.want[W2], dref.bound(W2, depth)
    top = np.abs(want).max()
    found = None
    for r in np.argsort(np.abs(want).max(1)):
        for r2 in range(w3.size):
            if r2 == r or w3[r] == 0:
                continue
            d = want[r] * (w3[r2] / w3[r] - 1.0)
            if np.abs(d).max() <= 2e-4 * top and (np.abs(d) > b[r]).any():
                found = (int(r), r2, d)
                break
        if found:
            break
    assert found, "no dW2 row whose wrong w3 passes the normwise bar"
    r, r2, d = found
    got = _rounded(dref)
    got[W2][r] += d
    assert _normwise_ok(got, dref.want)
    _outside(dref, got, depth)
    print(f"[seeded] dW2 row {r} scaled by w3[{r2}]: {float((np.abs(d) / np.maximum(b[r], 1e-300)).max()):.1f} x the bound")


def test_seeded_zero_tile_sum_missing_one_point(big):
    case, dref, feat, g, fw, depth = big
    miss = np.nonzero(np.abs(feat).sum(1) == 0)[0]
    assert miss.size >= 16 * 40
    j = int(miss[np.argmax(np.abs(g[miss]))])
    got = _rounded(dref)
    dh1, dh2, h1, h2 = (fw[k].numpy()[j] for k in ("dh1", "dh2", "h1", "h2"))
    terms = {W1: np.outer(dh1, feat[j]), B1: dh1, W2: np.outer(dh2, h1), B2: dh2, W3: (g[j] * h2)[None, :],
             "lout.bias": np.array([g[j]])}
    for k in got:
        got[k] = got[k] - terms[k].reshape(got[k].shape)
    assert _normwise_ok(got, dref.want)
    _outside(dref, got, depth)
    print(f"[seeded] zero-tile point {j} missing: worst "
          f"{max(float((np.abs(terms[k].reshape(got[k].shape)) / np.maximum(dref.bound(k, depth), 1e-300)).max()) for k in got):.1f}"
          " x the bound")


def test_seeded_db2_without_its_w3(big):
    case, dref, feat, g, fw, depth = big
    w3 = np.asarray(case["dec"]["lout.weight"], dtype=np.float64).reshape(-1)
    want, b = dref.want[B2], dref.bound(B2, depth)
    d = np.where(w3 != 0, want / np.where(w3 != 0, w3, 1.0) - want, 0.0)
    cand = np.nonzero((np.abs(d) <= 2e-4 * np.abs(want).max()) & (np.abs(d) > b))[0]
    assert cand.size, "no db2 entry whose missing w3 passes the normwise bar"
    u = int(cand[np.argmax(np.abs(d[cand]) / b[cand])])
    got = _rounded(dref)
    got[B2][u] += d[u]
    assert _normwise_ok(got, dref.want)
    _outside(dref, got, depth)
    print(f"[seeded] db2[{u}] without w3: {abs(d[u]) / b[u]:.1f} x the bound")


def test_kernel_depth_follows_the_launch_geometry():
    """depth = 13 T + 28 + B chunks, maximised over 1..8 blocks/SM (tests/decoder_bound.py)."""
    assert kernel_depth(16) == 13 + 28 + 1                       # one tile: one block, one tile per warp
    n = 132 * 8 * 8 * 16 * 3                                      # 25 344 tiles
    assert kernel_depth(n) == 13 * 3 + 28 + 1056                 # 8 blocks/SM: B = 1056, T = 3 (1 block/SM: T = 24, 13 T + 28 + 132 = 472)
    assert kernel_depth(n, chunks=3) == 13 * 1 + 28 + 3 * 1056   # 8 448 tiles per chunk: T = 1 at 8 blocks/SM
