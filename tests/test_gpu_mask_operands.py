"""The training kernels' layer-2 backward multiplies by the 0/1 ReLU mask M2 = [h2 > 0], which is exact in tf32: the dgrad
runs dh1 = dp * (M2 W2') with W2' = diag(w3) W2, and the Morton-ordered kernel forms dW2 = diag(w3) (dp h1)^T M2 and
db2 = diag(w3) M2^T dp.  These cases stress what that algebra rounds differently or relies on: zero and negative w3,
decoder weights far from 1, dead units of both hidden layers, batches of zero tiles only, a frozen decoder, and dL/dpred
spanning orders of magnitude.  Each is graded against the oracle for the per-point and the Morton-ordered kernels in
3xTF32, and for the 1xTF32 kernel at its own tolerance."""
import numpy as np
import pytest
import torch

from tests.parity_utils import (compare_step, drop_relu_kink_points, make_case, run_cuda_step, run_oracle_step,
                                sort_case_morton)
from tests.test_gpu_replicas import grade_run
from tests.test_gpu_rounds import TILE, _far, _tiles_per_round

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
W1, B1, W2, B2, W3, B3 = "layers.0.weight", "layers.0.bias", "layers.1.weight", "layers.1.bias", "lout.weight", "lout.bias"
# The plain-tf32 kernels on these 60-100 k-point batches: max-normalised table-gradient errors up to 0.17 (dead units) and
# 0.11 (frozen decoder, mixed-sign w3), the same with the three-product layer-2 backward.  The bound still catches a wrong
# index map or a missing scale, which are O(1).
TF32X1 = dict(pred_atol=5e-3, pred_rtol=5e-3, grad_rel=0.25)


@pytest.fixture(scope="module", autouse=True)
def _lib(built_lib):
    assert torch.cuda.is_available()
    return built_lib


def _case(seed, **kw):
    """Two rounds of the grid's warps (every warp folds more than one tile into its partial), Morton-ordered."""
    n = 2 * _tiles_per_round() * TILE + 7
    return sort_case_morton(make_case(n_points=2500, n_batch=n, feat_levels=3, seed=seed, **kw))


def _set_dec(case, **arrays):
    case = dict(case)
    case["dec"] = dict(case["dec"])
    for k, v in arrays.items():
        case["dec"][k] = np.ascontiguousarray(v, dtype=np.float32)
    return case


def _dec(case, key):
    return np.array(case["dec"][key], dtype=np.float32, copy=True)


def _grade(case, frozen=False, kink_eps=2e-6):
    """Every training flavour against the oracle, and element by element against the fp64 bounds
    (test_gpu_replicas.grade_run), on the points whose decoder pre-activations are farther than kink_eps
    from zero (tests/parity_utils.drop_relu_kink_points); returns the runs as {name: result}."""
    case, _ = drop_relu_kink_points(case, kink_eps)
    want = run_oracle_step(case)
    if frozen:
        want = dict(want); want["dec_grads"] = {}
    runs, ref = {}, None
    for name, kw in (("per-point", {}), ("grouped", {"morton_ordered": True})):
        runs[name] = run_cuda_step(case, DEV, freeze_decoder=frozen, **kw)
        print(name, compare_step(runs[name], want))
        ref = grade_run(case, runs[name], "mask operands", ref=ref, **kw)
    runs["tf32x1"] = run_cuda_step(case, DEV, freeze_decoder=frozen, tf32x1=True)
    print("tf32x1", compare_step(runs["tf32x1"], want, **TF32X1))
    grade_run(case, runs["tf32x1"], "mask operands", tf32x1=True)
    return runs


def _mixed_w3(case):
    """w3 with exact zeros on every fourth unit and alternating signs elsewhere."""
    w3 = _dec(case, W3)
    flat = w3.reshape(-1)
    flat[1::2] = -np.abs(flat[1::2]); flat[2::4] = np.abs(flat[2::4])
    zero = np.arange(0, flat.size, 4)
    flat[zero] = 0.0
    return _set_dec(case, **{W3: w3}), zero


def test_zero_and_mixed_sign_w3():
    """A unit with w3[n] = 0 has no gradient through layer 2: its dW2 row and db2 entry are exactly 0 in every flavour."""
    case, zero = _mixed_w3(_case(400, weighted=True))
    for name, got in _grade(case).items():
        g = got["dec_grads"]
        assert np.all(g[W2][zero] == 0.0), name
        assert np.all(g[B2][zero] == 0.0), name
        live = np.setdiff1d(np.arange(g[W2].shape[0]), zero)
        assert np.any(g[W2][live] != 0.0) and np.any(g[B2][live] != 0.0), name


@pytest.mark.parametrize("s", [1e3, 1e-3])
def test_scaled_decoder_weights(s):
    """W1, b1 and W2 times s, b2 times s^2, w3 over s^2: Decoder.sdf is unchanged (ReLU is positively homogeneous), while
    h1, w3 * W2 and dp * h1 move by orders of magnitude."""
    case = _case(401 + int(s > 1), weighted=True)
    w3 = _dec(case, W3) / np.float32(s * s)
    case = _set_dec(case, **{W1: _dec(case, W1) * np.float32(s), B1: _dec(case, B1) * np.float32(s),
                             W2: _dec(case, W2) * np.float32(s), B2: _dec(case, B2) * np.float32(s * s), W3: w3})
    _grade(case, kink_eps=2e-6 * max(s, s * s))   # pre-activations of layer 1 / 2 scale by s / s^2


def test_dead_units_of_both_layers():
    """Layer-1 unit a and layer-2 unit b never activate (zero weights, negative bias): dW1 row a, db1[a], dW2 column a,
    dW2 row b and db2[b] are exactly 0, and the other gradients still match."""
    a, b = 5, 22
    case = _case(403, weighted=True)
    w1, b1, w2, b2 = _dec(case, W1), _dec(case, B1), _dec(case, W2), _dec(case, B2)
    w1[a, :] = 0.0; b1[a] = -0.5
    w2[b, :] = 0.0; b2[b] = -0.5
    case = _set_dec(case, **{W1: w1, B1: b1, W2: w2, B2: b2})
    for name, got in _grade(case).items():
        g = got["dec_grads"]
        assert np.all(g[W1][a] == 0.0) and g[B1][a] == 0.0, name
        assert np.all(g[W2][:, a] == 0.0), name
        assert np.all(g[W2][b] == 0.0) and g[B2][b] == 0.0, name
        assert np.any(g[W2] != 0.0) and np.any(g[W1] != 0.0), name


@pytest.mark.parametrize("frozen", [False, True])
def test_zero_tiles_only(frozen):
    """Every point misses every level: the virtual backward tile carries the whole dL/dpred sum through the new dgrad
    and, with decoder gradients, through T = (dp h1)^T M2."""
    case, _ = _mixed_w3(make_case(n_points=2500, n_batch=64, feat_levels=3, seed=404, weighted=True, reduction="sum"))
    rng = np.random.default_rng(31)
    n = 3 * _tiles_per_round() * TILE + 3
    case["coord"] = _far(rng, n)
    case["label"] = rng.uniform(-0.2, 0.2, size=n).astype(np.float32)
    case["weight"] = rng.uniform(0.5, 1.5, size=n).astype(np.float32)
    _grade(case, frozen)


def test_frozen_decoder_table_grads():
    """Without decoder gradients the table gradients go only through the masked dgrad (mixed-sign w3 with zeros)."""
    case, _ = _mixed_w3(_case(405, weighted=True))
    _grade(case, frozen=True)


def test_sum_reduction_with_weights_over_six_decades():
    """loss_reduction 'sum' with sample weights 1e-4 .. 1e2: dL/dpred of the points of one tile spans six orders of
    magnitude, and so do the rows that dp scales after the masked products."""
    case = _case(406, weighted=True, reduction="sum")
    rng = np.random.default_rng(32)
    case["weight"] = (10.0 ** rng.uniform(-4.0, 2.0, size=case["weight"].shape[0])).astype(np.float32)
    _grade(case)
