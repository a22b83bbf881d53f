"""The oracle restatement (oracle/shine_oracle.py) must reproduce what the UNMODIFIED reference produced
(tests/golden/*.npz, minted by oracle/make_golden.py): this is what pins the oracle."""
import numpy as np
import pytest
import torch

from tests.parity_utils import (DEC_KEYS, GOLDEN_NAMES, compare_step, load_eikonal_golden, load_golden, oracle_from_case,
                                orc, run_oracle_step)


@pytest.mark.parametrize("name", GOLDEN_NAMES)
def test_oracle_matches_reference_golden(name):
    case, exp = load_golden(name)
    got = run_oracle_step(case)
    if case["cfg"]["decoder_frozen"]:
        got["dec_grads"] = {}
    # same CPU ops in the same order: essentially exact
    report = compare_step(got, exp, pred_atol=1e-6, pred_rtol=1e-6, grad_rel=1e-5, check_trash=True)
    print(name, report)


@pytest.mark.parametrize("name", GOLDEN_NAMES)
def test_oracle_update_reproduces_reference_row_numbering(name):
    """Replaying the frames must give the reference's table sizes, and every stored corner row must be in range."""
    case, exp = load_golden(name)
    o, _ = oracle_from_case(case)   # asserts row counts
    for lvl, table in enumerate(o.nodes_lookup_tables):
        if table:
            ids = np.array(list(table.values()))
            k = lvl - o.free_level_num
            assert ids.min() >= 0 and ids.max() < case["tables"][k].shape[0] - 1


def test_morton_known_answers():
    # SURVEY 8c KATs: Morton of (1,0,0)/(0,1,0)/(0,0,1) = 4/2/1; x is the most significant bit of each triplet
    p = np.array([[1, 0, 0], [0, 1, 0], [0, 0, 1], [1, 1, 1], [2, 0, 0], [4095, 4095, 4095], [0, 0, 4096]])
    m = orc.points_to_morton(p)
    assert m.tolist() == [4, 2, 1, 7, 32, (1 << 36) - 1, 1 << 36]
    assert np.array_equal(orc.morton_to_points(m), p.astype(np.int16))


def test_quantize_clamp_and_floor():
    x = np.array([[-1.0, 1.0, 0.0], [-3.0, 3.0, 0.999999], [2.0 ** -12, -(2.0 ** -12), 0.5]], dtype=np.float32)
    q = orc.quantize_points(x, 12)
    assert q.tolist() == [[0, 4095, 2048], [0, 4095, 4095], [2048, 2047, 3072]]
    assert q.dtype == np.int16


def test_corner_order_matches_weight_order():
    """Corner i of points_to_corners must be the corner weighted by p_i of interpolat (feature_octree.py:186-195)."""
    o = orc.OracleOctree(12, 1)
    x = torch.tensor([[0.3 * 2.0 ** -11 - 1 + 2.0 ** -11 * 7, 0.6 * 2.0 ** -11, 0.9 * 2.0 ** -11]])
    w = o.interpolat(x, 12, polynomial_on=False).reshape(8)
    coords = (2 ** 12) * (x * 0.5 + 0.5)
    d = (coords - torch.floor(coords)).reshape(3)
    for i, off in enumerate(orc.points_to_corners(np.zeros((1, 3), dtype=np.int16))[0]):
        expect = 1.0
        for a in range(3):
            expect *= float(d[a]) if off[a] else 1.0 - float(d[a])
        assert abs(float(w[i]) - expect) < 1e-6


def test_voxel_centre_has_equal_weights():
    o = orc.OracleOctree(12, 1)
    x = torch.tensor([[(100 + 0.5) * 2.0 ** -11 - 1, (7 + 0.5) * 2.0 ** -11 - 1, (4000 + 0.5) * 2.0 ** -11 - 1]])
    for poly in (True, False):
        assert torch.allclose(o.interpolat(x, 12, poly).reshape(8), torch.full((8,), 0.125))


def test_unseen_voxel_gives_zero_feature_and_mlp_of_zero():
    torch.manual_seed(0)
    o = orc.OracleOctree(12, 2)
    o.update(torch.rand(50, 3) * 0.01)
    dec = orc.make_decoder_params()
    far = torch.tensor([[-0.9, -0.9, -0.9], [0.95, 0.2, -0.4]])
    f = o.query_feature(far)
    assert torch.equal(f, torch.zeros(2, 8))
    assert all((i == -1).all() for i in o.hierarchical_indices)
    assert torch.allclose(orc.decoder_sdf(f, dec), orc.decoder_sdf(torch.zeros(2, 8), dec))


def test_raises_without_featured_level():
    with pytest.raises(ValueError):
        orc.OracleOctree(12, 0)


def test_oracle_eikonal_matches_reference_golden():
    """ekional_loss_on: d pred / d coord with create_graph=True on the reference's own classes (golden minted by
    oracle/make_golden.py::make_eikonal) vs the oracle's train_step_eikonal."""
    _check_oracle_against_eikonal_golden("ref_eikonal_l3")


def test_oracle_eikonal_matches_scaled_reference_golden():
    """The same on ref_eikonal_l3_sum_weighted: tables scaled x500 (median surface |g| ~1), weighted BCE with sum
    reduction, and the eikonal mean's own gradients (beside a summed BCE its share of the total is small)."""
    _check_oracle_against_eikonal_golden("ref_eikonal_l3_sum_weighted")


def _check_oracle_against_eikonal_golden(name):
    case, z = load_eikonal_golden(name)
    cfg = case["cfg"]
    o, dec = oracle_from_case(case)
    got = orc.train_step_eikonal(o, dec, torch.from_numpy(z["coord"]), torch.from_numpy(z["label"]),
                                 torch.from_numpy(z["weight"]), cfg["sigma"], cfg["weight_e"], cfg["weighted"],
                                 cfg["reduction"])
    assert np.abs(got["g"].numpy() - z["exp_g"]).max() <= 1e-5 * np.abs(z["exp_g"]).max()
    assert abs(float(got["eikonal"]) - float(z["exp_eikonal"])) <= 1e-5 * abs(float(z["exp_eikonal"]))
    assert abs(float(got["loss"]) - float(z["exp_loss"])) <= 1e-6 * abs(float(z["exp_loss"]))
    for k, g in enumerate(got["table_grads"]):
        want = z[f"exp_tgrad_{k}"]
        assert np.abs(g.numpy() - want).max() <= 1e-4 * np.abs(want).max() + 1e-12
    for k in DEC_KEYS:
        want = z["exp_dgrad_" + k]
        assert np.abs(got["dec_grads"][k].numpy() - want).max() <= 1e-4 * np.abs(want).max() + 1e-12
    if "exp_eik_tgrad_0" not in z.files:
        return
    for k, g in enumerate(got["eik_table_grads"]):
        want = z[f"exp_eik_tgrad_{k}"]
        assert np.abs(g.numpy() - want).max() <= 1e-4 * np.abs(want).max() + 1e-12, k
    for k in DEC_KEYS:
        want = z["exp_eik_dgrad_" + k]
        assert np.abs(got["eik_dec_grads"][k].numpy() - want).max() <= 1e-4 * np.abs(want).max() + 1e-12, k
