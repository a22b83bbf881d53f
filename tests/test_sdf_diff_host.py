"""CPU tests of training with the reference's sdf_l1 / sdf_l2 losses: the fp64 oracle against goldens minted from the
reference (oracle/make_sdf_diff_golden.py), the C-ABI argument checks of the shine_sdf_diff_* entries, and which loops
accept which main_loss_type."""
import ctypes as C
import os

import numpy as np
import pytest
import torch

from tests import sdf_diff_oracle as sdo
from tests.parity_utils import GOLDEN_DIR, make_config, oracle_from_case

DIFF_GOLDENS = ["ref_sdf_l1_l3_weighted", "ref_sdf_l2_l3"]
EIKONAL_GOLDENS = ["ref_sdf_l2_eikonal_l3", "ref_sdf_l1_eikonal_l3"]


def _rel(a, b):
    a, b = np.asarray(a, dtype=np.float64), np.asarray(b, dtype=np.float64)
    return float(np.abs(a - b).max() / max(np.abs(b).max(), 1e-30))


@pytest.mark.parametrize("name", DIFF_GOLDENS)
def test_oracle_matches_reference_golden(name):
    z = np.load(os.path.join(GOLDEN_DIR, name + ".npz"))
    case, cfg = sdo.golden_case(z)
    exp = sdo.expected(z, cfg["tree_level_feat"])
    o, dec = oracle_from_case(case)
    res = sdo.train_step(o, dec, torch.from_numpy(case["coord"]), torch.from_numpy(case["label"]),
                         torch.from_numpy(case["weight"]), cfg["sigma"], loss_type=cfg["loss_type"], scale=cfg["scale"],
                         double=True)
    got = sdo.as_numpy(res, o)
    for a, b in zip(got["indices"], exp["indices"]):
        assert np.array_equal(a, b)
    assert _rel(got["pred"], exp["pred"]) < 1e-5
    assert abs(got["loss"] - exp["loss"]) <= 1e-4 * abs(exp["loss"])
    for a, b in zip(got["table_grads"], exp["table_grads"]):
        assert _rel(a[:-1], b[:-1]) < 1e-4
    for k, b in exp["dec_grads"].items():
        assert _rel(got["dec_grads"][k], b) < 1e-4, k
    # the class-surface loss is the reference's function
    from shine_mapping_b200.loss import sdf_diff_loss
    p, lb, w = torch.from_numpy(exp["pred"]).double(), torch.from_numpy(case["label"]).double(), \
        torch.from_numpy(np.abs(case["weight"])).double()
    assert float(sdf_diff_loss(p, lb, w, cfg["scale"], cfg["loss_type"] == "sdf_l2")) == pytest.approx(exp["loss"], rel=1e-5)


@pytest.mark.parametrize("name", EIKONAL_GOLDENS)
def test_oracle_eikonal_matches_reference_golden(name):
    """Total and eikonal-only gradients.  The goldens are minted with labels and weight_e that give the eikonal term a
    real share of every gradient (0.03 to 0.93 of its max), so a step that dropped or mis-scaled it would fail."""
    z = np.load(os.path.join(GOLDEN_DIR, name + ".npz"))
    case, cfg = sdo.golden_case(z)
    o, dec = oracle_from_case(case)
    res = sdo.train_step_eikonal(o, dec, torch.from_numpy(case["coord"]), torch.from_numpy(case["label"]),
                                 torch.from_numpy(case["weight"]), cfg["sigma"], cfg["weight_e"],
                                 loss_type=cfg["loss_type"], scale=cfg["scale"])
    assert float(res["loss"]) == pytest.approx(float(z["exp_loss"]), rel=1e-5)
    assert float(res["eikonal"]) == pytest.approx(float(z["exp_eikonal"]), rel=1e-4)
    assert _rel(res["g"].numpy(), z["exp_g"]) < 1e-4
    for k, g in enumerate(res["table_grads"]):
        assert _rel(g.numpy()[:-1], z[f"exp_tgrad_{k}"][:-1]) < 1e-4
        assert _rel(res["eik_table_grads"][k].numpy()[:-1], z[f"exp_eik_tgrad_{k}"][:-1]) < 1e-4
        share = np.abs(cfg["weight_e"] * z[f"exp_eik_tgrad_{k}"]).max() / np.abs(z[f"exp_tgrad_{k}"]).max()
        assert share > 0.02, (k, share)      # the golden can see the eikonal term
    for k, g in res["dec_grads"].items():
        assert _rel(g.numpy(), z["exp_dgrad_" + k]) < 1e-4, k
        if np.abs(z["exp_eik_dgrad_" + k]).max() > 0:
            assert _rel(res["eik_dec_grads"][k].numpy(), z["exp_eik_dgrad_" + k]) < 1e-4, k


def test_l1_gradient_at_zero_difference_is_zero():
    pred = torch.tensor([0.5, 0.25, -1.0], dtype=torch.float64, requires_grad=True)
    label = torch.tensor([0.5, 0.0, 0.0], dtype=torch.float64)
    w = torch.tensor([2.0, 1.0, 3.0], dtype=torch.float64)
    sdo.sdf_diff_loss(pred, label, w, 0.01, l2_loss=False).backward()
    assert pred.grad[0] == 0.0                                              # torch: sign(0) = 0
    assert torch.allclose(pred.grad, sdo.diff_dpred(pred.detach(), label, w, 0.01, False, 3))
    pred.grad = None
    sdo.sdf_diff_loss(pred, label, w, 0.01, l2_loss=True).backward()
    assert torch.allclose(pred.grad, sdo.diff_dpred(pred.detach(), label, w, 0.01, True, 3))


def _fake_descriptors():
    """Octree / decoder descriptors that pass the argument checks (dummy host pointers): with n = 0 nothing is
    launched, so the checks before the launch can be exercised without a GPU."""
    from shine_mapping_b200 import _abi
    buf = (C.c_float * 64)()
    p = C.addressof(buf)
    o = _abi.ShineOctree()
    o.num_levels, o.feature_dim, o.poly_interp = 1, 8, 1
    lv = o.lv[0]
    lv.hash_slots, lv.features, lv.feature_grads, lv.hash_capacity, lv.rows, lv.level = p, p, p, 16, 2, 12
    d = _abi.ShineDecoder()
    d.w1 = d.w2 = d.w3 = p
    d.in_dim, d.hidden, d.mlp_level = 8, 32, 2
    return buf, o, d, p


def _calls(lib, o, d, p):
    """entry -> f(weight, scale, flags)"""
    oc, dc = C.byref(o), C.byref(d)
    cnt = C.c_int32(0)
    return {
        "shine_sdf_diff_fwd": lambda w, s, f: lib.shine_sdf_diff_fwd(oc, dc, None, None, w, 0, s, 1.0, None, None, f, None),
        "shine_sdf_diff_step": lambda w, s, f: lib.shine_sdf_diff_step(oc, dc, None, None, w, 0, s, 1.0, None, None, None,
                                                                       f, None),
        "shine_sdf_diff_eikonal_step": lambda w, s, f: lib.shine_sdf_diff_eikonal_step(
            oc, dc, None, None, w, 0, s, 0.01, 1.0, 0.1, C.addressof(cnt), None, None, None, None, f, None),
    }


def test_diff_entries_are_exported(built_lib):
    from shine_mapping_b200 import _abi
    for name in ("shine_sdf_diff_fwd", "shine_sdf_diff_step", "shine_sdf_diff_eikonal_step"):
        assert name in _abi.SYMBOLS and getattr(built_lib, name) is not None
    assert _abi.FLAG_LOSS_L2 == 32


def test_diff_entries_check_flags_weight_and_scale(built_lib):
    from shine_mapping_b200 import _abi
    buf, o, d, p = _fake_descriptors()
    accepted = {"shine_sdf_diff_fwd": _abi.FLAG_TF32X1 | _abi.FLAG_LOSS_L2,
                "shine_sdf_diff_step": _abi.FLAG_TF32X1 | _abi.FLAG_LOSS_L2 | _abi.FLAG_MORTON_ORDERED,
                "shine_sdf_diff_eikonal_step": _abi.FLAG_TF32X1 | _abi.FLAG_LOSS_L2}
    for name, call in _calls(built_lib, o, d, p).items():
        ok = accepted[name]
        for f in (0, _abi.FLAG_LOSS_L2, ok):
            assert call(p, 0.01, f) == 0, (name, f)                       # n = 0: valid arguments, nothing launched
        for bit in range(32):
            if not (1 << bit) & ok:   # REDUCTION_SUM, WEIGHTED, the retired bit 8, MORTON_ORDERED on the forward-only calls
                assert call(p, 0.01, 1 << bit) == -2, (name, bit)
        assert call(None, 0.01, 0) == -1, name                           # the weight is required
        for bad in (0.0, -0.01, float("inf"), float("nan")):
            assert call(p, bad, 0) == -1, (name, bad)
    # the BCE entries keep refusing the new bit
    oc, dc = C.byref(o), C.byref(d)
    assert built_lib.shine_sdf_bce_step(oc, dc, None, None, None, 0, 1.0, 1.0, None, None, None, _abi.FLAG_LOSS_L2, None) == -2


def test_sdf_diff_step_refuses_cpu_tensors(built_lib):
    from shine_mapping_b200 import Decoder, FeatureOctree, _abi
    from shine_mapping_b200.fused import sdf_diff_step
    cfg = make_config(2)
    octree, dec = FeatureOctree(cfg), Decoder(cfg)
    coord = torch.zeros(4, 3)
    with pytest.raises(_abi.ShineB200Error, match="no CPU fallback"):
        sdf_diff_step(octree, dec, coord, torch.zeros(4), torch.ones(4), cfg.scale)
    with pytest.raises(ValueError, match="weight"):
        sdf_diff_step(octree, dec, coord, torch.zeros(4), None, cfg.scale)


def test_batch_loop_accepts_the_point_losses_and_the_incremental_loop_does_not():
    from shine_mapping_b200.batch_loop import BATCH_LOSSES, check_supported
    from shine_mapping_b200.trainer import diff_loss_flags
    from shine_mapping_b200 import _abi
    cfg = make_config(2)
    for loss in ("sdf_bce", "sdf_l1", "sdf_l2"):
        cfg.main_loss_type = loss
        check_supported(cfg)
        if loss != "sdf_bce":
            with pytest.raises(NotImplementedError):
                check_supported(cfg, main_losses=("sdf_bce",))            # incre_loop's check
    assert [diff_loss_flags(t) for t in BATCH_LOSSES] == [None, 0, _abi.FLAG_LOSS_L2]
    with pytest.raises(NotImplementedError):
        diff_loss_flags("dr")
    for loss in ("dr", "dr_neus", "sdf_huber"):
        cfg.main_loss_type = loss
        with pytest.raises(NotImplementedError):
            check_supported(cfg)
        with pytest.raises(NotImplementedError):
            check_supported(cfg, main_losses=("sdf_bce",))
    cfg.main_loss_type = "sdf_l2"
    cfg.ray_loss = True
    with pytest.raises(NotImplementedError):
        check_supported(cfg)


def test_incre_loop_command_line_rejects_sdf_l2(tmp_path):
    from shine_mapping_b200 import incre_loop
    path = tmp_path / "incre.yaml"
    path.write_text("setting: {name: t, output_root: ./, pc_path: x, pose_path: x, calib_path: x}\n"
                    "loss: {main_loss_type: sdf_l2}\n")
    with pytest.raises(NotImplementedError, match="sdf_bce"):
        incre_loop.main([str(path)])
