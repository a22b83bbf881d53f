"""Parity of the sm_90a path (through the C ABI behind the package classes) against the CPU oracle and the
reference-minted golden vectors.  Tolerances are stated in tests/parity_utils.py."""
import ctypes as C

import numpy as np
import pytest
import torch

from tests.parity_utils import (DEC_KEYS, GOLDEN_NAMES, build_cuda_models, compare_step, load_eikonal_golden, load_golden,
                                make_case, run_cuda_step, run_oracle_step, sort_case_morton)
from tests.test_gpu_replicas import grade_run

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


@pytest.fixture(scope="module", autouse=True)
def _lib(built_lib):
    assert torch.cuda.is_available()
    return built_lib


# ---- against the reference's own outputs -----------------------------------------------------------------

@pytest.mark.parametrize("name", GOLDEN_NAMES)
def test_cuda_matches_reference_golden(name):
    case, exp = load_golden(name)
    got = run_cuda_step(case, DEV)
    if case["cfg"]["decoder_frozen"]:
        got["dec_grads"] = {}
    print(name, compare_step(got, exp))


# ---- against the oracle on seeded synthetic batches -----------------------------------------------------

@pytest.mark.parametrize("levels,poly,weighted,reduction,frames", [
    (1, True, False, "mean", 1), (2, True, False, "mean", 1), (3, False, True, "sum", 2),
    (4, True, False, "mean", 1), (4, True, True, "mean", 2), (4, False, False, "sum", 1),
    (6, True, False, "mean", 1), (8, True, True, "sum", 2),        # > 4 levels: the LMAX = 8 kernel instantiations
])
def test_fused_step_matches_oracle(levels, poly, weighted, reduction, frames):
    case = make_case(n_points=2500, n_batch=3000, feat_levels=levels, seed=10 + levels, n_frames=frames,
                     poly=poly, weighted=weighted, reduction=reduction)
    print(compare_step(run_cuda_step(case, DEV), run_oracle_step(case)))


@pytest.mark.parametrize("levels,poly,weighted,reduction,ordered", [
    (1, True, False, "mean", True), (2, False, True, "sum", True), (3, True, False, "mean", True),
    (4, True, True, "mean", True), (4, True, False, "mean", False), (3, False, False, "sum", False),
    (6, True, False, "mean", True),      # > 4 levels: the flag falls back to the general kernel
])
def test_grouped_scatter_matches_oracle(levels, poly, weighted, reduction, ordered):
    """SHINE_FLAG_MORTON_ORDERED: per-run tensor-core reduction of the table gradients.  Batches in Morton order (runs of
    equal node, several per tile) and in random order (the hint is wrong: every level of every tile takes the per-point
    path) must both match the oracle; a frozen decoder exercises the kernel flavour without the staging area."""
    case = make_case(n_points=2500, n_batch=6000, feat_levels=levels, seed=40 + levels, n_frames=1,
                     poly=poly, weighted=weighted, reduction=reduction)
    if ordered:
        case = sort_case_morton(case)
    want = run_oracle_step(case)
    got = run_cuda_step(case, DEV, morton_ordered=True)
    print(compare_step(got, want))
    ref = grade_run(case, got, f"grouped scatter L={levels} ordered={ordered}", morton_ordered=True)
    want_f = dict(want); want_f["dec_grads"] = {}
    got = run_cuda_step(case, DEV, morton_ordered=True, freeze_decoder=True)
    print(compare_step(got, want_f))
    grade_run(case, got, f"grouped scatter L={levels} ordered={ordered} frozen", morton_ordered=True, ref=ref)


@pytest.mark.parametrize("ordered,weighted,reduction,frozen", [(True, False, "mean", False), (False, True, "sum", False),
                                                              (True, True, "mean", True)])
def test_all_miss_tiles_match_oracle(ordered, weighted, reduction, frozen):
    """Whole 16-point tiles of free-space samples that miss every level (a third of the tiles of an ordered C2 batch): the
    kernel gives them Decoder.sdf(0) and folds their decoder gradients in by linearity.  Loss, predictions and every
    gradient must equal the oracle's, with the block of far points in the middle of a batch (order drawn) and spread by
    the Morton sort (ordered), general and grouped kernels, weighted / sum, and with a frozen decoder."""
    case = make_case(n_points=2500, n_batch=1500, feat_levels=3, seed=91, weighted=weighted, reduction=reduction)
    rng = np.random.default_rng(7)
    far = np.concatenate([rng.uniform(0.55, 0.95, size=(700, 3)), rng.uniform(-0.95, -0.6, size=(420, 3))]).astype(np.float32)
    k = 640                                     # a tile-aligned block of far points inside the batch
    case["coord"] = np.concatenate([case["coord"][:k], far, case["coord"][k:]]).astype(np.float32)
    case["label"] = np.concatenate([case["label"][:k], rng.uniform(-0.2, 0.2, size=far.shape[0]).astype(np.float32),
                                    case["label"][k:]])
    case["weight"] = np.concatenate([case["weight"][:k], rng.uniform(0.5, 1.5, size=far.shape[0]).astype(np.float32),
                                     case["weight"][k:]])
    if ordered:
        case = sort_case_morton(case)
    want = run_oracle_step(case)
    missed_everywhere = np.logical_and.reduce([(idx == -1).all(axis=1) for idx in want["indices"]])
    assert int(missed_everywhere.sum()) >= far.shape[0]                     # the far points really miss every level
    if not ordered:
        assert bool(missed_everywhere[k:k + far.shape[0]].all())
    if frozen:
        want = dict(want); want["dec_grads"] = {}
    ref = None
    for flag in (False, True):
        got = run_cuda_step(case, DEV, morton_ordered=flag, freeze_decoder=frozen)
        print(compare_step(got, want))
        ref = grade_run(case, got, f"all-miss tiles ordered={ordered}", morton_ordered=flag, ref=ref)


def test_all_miss_batch():
    """Every point misses every level: only virtual tiles reach the decoder."""
    case = make_case(n_points=2500, n_batch=64, feat_levels=2, seed=93)
    rng = np.random.default_rng(3)
    n = 1000
    case["coord"] = rng.uniform(0.6, 0.9, size=(n, 3)).astype(np.float32)
    case["label"] = rng.uniform(-0.1, 0.1, size=n).astype(np.float32)
    case["weight"] = np.ones(n, dtype=np.float32)
    print(compare_step(run_cuda_step(case, DEV), run_oracle_step(case)))


def test_grouped_scatter_dense_runs():
    """Many samples per voxel (16-point tiles inside ONE node at every level, runs crossing tile borders)."""
    case = make_case(n_points=2500, n_batch=64, feat_levels=3, seed=77)
    rng = np.random.default_rng(5)
    base = case["coord"][rng.integers(0, 64, size=24)]
    coord = (base[:, None, :] + rng.uniform(-2e-4, 2e-4, size=(24, 200, 3))).reshape(-1, 3).astype(np.float32)
    case["coord"] = coord
    case["label"] = rng.uniform(-0.05, 0.05, size=coord.shape[0]).astype(np.float32)
    case["weight"] = np.ones(coord.shape[0], dtype=np.float32)
    case = sort_case_morton(case)
    got = run_cuda_step(case, DEV, morton_ordered=True)
    print(compare_step(got, run_oracle_step(case)))
    grade_run(case, got, "dense runs", morton_ordered=True)


@pytest.mark.parametrize("n_batch", [0, 1, 15, 16, 17, 255])
def test_ragged_batch_sizes(n_batch):
    """Tile tails: 16 stragglers are always appended, so N = n_batch + 16 covers 16..271."""
    case = make_case(n_points=1500, n_batch=n_batch, feat_levels=2, seed=5)
    print(compare_step(run_cuda_step(case, DEV), run_oracle_step(case)))


def test_two_pass_mode_matches_oracle():
    case = make_case(n_points=2000, n_batch=2000, feat_levels=3, seed=21)
    print(compare_step(run_cuda_step(case, DEV, single_pass=False), run_oracle_step(case)))


def test_unfused_class_surface_matches_oracle():
    """query_feature kernel + torch MLP + torch loss (the reference call sequence verbatim)."""
    case = make_case(n_points=2000, n_batch=2000, feat_levels=4, seed=22)
    print(compare_step(run_cuda_step(case, DEV, unfused=True), run_oracle_step(case)))


@pytest.mark.parametrize("feature_dim", [4, 16])
def test_class_surface_other_feature_dims(feature_dim):
    """The generic query kernels take any feature_dim = 4*LP (here LP = 1 and 4); the fused decoder kernel is F=8 only
    and must say so."""
    from shine_mapping_b200 import _abi, sdf_bce_step
    case = make_case(n_points=2000, n_batch=2000, feat_levels=3, seed=25, feature_dim=feature_dim)
    print(compare_step(run_cuda_step(case, DEV, unfused=True), run_oracle_step(case)))
    cfg, octree, dec = build_cuda_models(case, DEV)
    with pytest.raises(_abi.ShineB200Error, match="feature_dim=8"):
        sdf_bce_step(octree, dec, torch.from_numpy(case["coord"]).to(DEV), torch.from_numpy(case["label"]).to(DEV), 0.01)


def test_plain_tf32_flag_is_close():
    case = make_case(n_points=2000, n_batch=2000, feat_levels=2, seed=23)
    got, want = run_cuda_step(case, DEV, tf32x1=True), run_oracle_step(case)
    print(compare_step(got, want, pred_atol=5e-3, pred_rtol=5e-3, grad_rel=3e-2))


def test_frozen_decoder_gives_only_table_grads():
    from shine_mapping_b200 import sdf_bce_step
    case = make_case(n_points=2000, n_batch=2000, feat_levels=4, seed=24)
    cfg, octree, dec = build_cuda_models(case, DEV, freeze_decoder=True)
    coord = torch.from_numpy(case["coord"]).to(DEV); label = torch.from_numpy(case["label"]).to(DEV)
    loss = sdf_bce_step(octree, dec, coord, label, case["cfg"]["sigma"])
    loss.backward()
    want = run_oracle_step(case)
    for p, w in zip(octree.hier_features, want["table_grads"]):
        g = p.grad.cpu().numpy()[:-1]
        assert np.abs(g - w[:-1]).max() <= 2e-4 * np.abs(w).max() + 1e-10
    assert all(p.grad is None for p in dec.parameters())


def test_empty_batch_is_ok():
    from shine_mapping_b200 import sdf_infer
    case = make_case(n_points=1500, n_batch=0, feat_levels=2, seed=5)
    cfg, octree, dec = build_cuda_models(case, DEV)
    empty = torch.empty(0, 3, device=DEV)
    assert octree.query_feature(empty).shape == (0, 8)
    assert [t.shape for t in octree.get_indices(empty)] == [(0, 8)] * 2
    assert sdf_infer(octree, dec, empty).shape == (0,)


def test_infer_and_mask_match_step_pred():
    from shine_mapping_b200 import sdf_infer
    case = make_case(n_points=2500, n_batch=3000, feat_levels=3, seed=31)
    cfg, octree, dec = build_cuda_models(case, DEV)
    coord = torch.from_numpy(case["coord"]).to(DEV)
    want = run_oracle_step(case)
    for lvl in range(3):
        pred, mask = sdf_infer(octree, dec, coord, mask_level=lvl)
        assert np.abs(pred.cpu().numpy() - want["pred"]).max() < 2e-5
        assert np.array_equal(mask.cpu().numpy(), (want["indices"][lvl] >= 0).all(1))
    case6 = make_case(n_points=2500, n_batch=3000, feat_levels=7, seed=37)       # LMAX = 8 instantiation
    cfg6, octree6, dec6 = build_cuda_models(case6, DEV)
    want6 = run_oracle_step(case6)
    pred6, mask6 = sdf_infer(octree6, dec6, torch.from_numpy(case6["coord"]).to(DEV), mask_level=5)
    assert np.abs(pred6.cpu().numpy() - want6["pred"]).max() < 2e-5
    assert np.array_equal(mask6.cpu().numpy(), (want6["indices"][5] >= 0).all(1))


# ---- ekional_loss_on: the fused double-backward kernel (csrc/shine_eikonal.cu) and the class surface ------------------
# Both are checked at the reference's weight_e = 0.1 (totals, the tolerances of the BCE tests) and, because the step is
# linear in weight_e, the eikonal term on its own: (gradients at weight_e = W - gradients at weight_e = 0) / W against the
# oracle's gradients of the eikonal mean alone, graded against that term's own maximum.  W (_eik_weight) is large enough
# that the fp32 reordering of the BCE part, which does not cancel in the difference, stays far below that bar even where
# the BCE part is a sum over the batch.  On freshly initialised tables
# |g| ~ 1e-3 and the eikonal term is ~1e-3 of the total, so the totals alone could not see it; scaling the tables
# (x300: median surface |g| ~0.6, a fifth of the samples above 1) puts |g| where a trained map has it.

def _eikonal_case(levels, poly, seed, weighted=False, reduction="mean", scale=1.0, n=None, ordered=False, bias=True,
                  n_batch=1500, feature_dim=8):
    """n: keep the last n points of the batch (the 10 surface points and 6 stragglers make_case appends come last)."""
    case = make_case(n_points=2000, n_batch=n_batch, feat_levels=levels, seed=seed, poly=poly, weighted=weighted,
                     reduction=reduction, bias=bias, feature_dim=feature_dim)
    if scale != 1.0:
        case["tables"] = [(t * np.float32(scale)).astype(np.float32) for t in case["tables"]]
    if n is not None:
        for k in ("coord", "label", "weight"):
            case[k] = np.ascontiguousarray(case[k][-n:])
    return sort_case_morton(case) if ordered else case


def _eik_weight(case, want=None):
    """sdf_bce: 100 (x N with the sum).  sdf_l1 / sdf_l2 (want: the oracle's outputs at weight_e = 0.1) put every sample's
    full-size dL/dpred into the first term, whose gradients reach 10^5 x the eikonal ones on x300 tables with L2: there
    W = 100 x the largest ratio of the two maxima (at least 100), so that the floor of the eikonal-only grading,
    1e-5 max|first| / W, stays at about 1e-4 of its 1e-3 bar."""
    if want is None:
        return 100.0 * (case["coord"].shape[0] if case["cfg"]["reduction"] == "sum" else 1)
    ratio = 1.0
    for tot, eik in _grad_pairs(want):
        if np.abs(eik).max() > 0:
            ratio = max(ratio, float(np.abs(tot - 0.1 * eik).max() / np.abs(eik).max()))
    return 100.0 * ratio


def _grad_pairs(want):
    """(total, eikonal-only) gradient pairs of an oracle result: table levels without the trash row, then the decoder."""
    pairs = [(t[:-1], e[:-1]) for t, e in zip(want["table_grads"], want["eik_table_grads"])]
    return pairs + [(want["dec_grads"][k], want["eik_dec_grads"][k]) for k in want["eik_dec_grads"]]


def _oracle_eikonal(case, weight_e=0.1, n_surface=None, loss_type="sdf_bce", l1_sign=None):
    """loss_type sdf_l1 / sdf_l2: the first term is sdf_diff_loss (tests/sdf_diff_oracle.py); l1_sign as there."""
    from tests import sdf_diff_oracle as sdo
    from tests.parity_utils import oracle_from_case
    from tests.test_gpu_sdf_diff import _scale
    o, odec = oracle_from_case(case)
    c = case["cfg"]
    r = sdo.train_step_eikonal(o, odec, torch.from_numpy(case["coord"]), torch.from_numpy(case["label"]),
                               torch.from_numpy(case["weight"]), c["sigma"], weight_e, c["weighted"], c["reduction"],
                               n_surface, loss_type=loss_type, scale=_scale(case), l1_sign=l1_sign)
    out = {k: float(r[k]) for k in ("loss", "bce", "eikonal")}
    out.update(g=r["g"].numpy(), pred=r["pred"].numpy(), table_grads=[t.numpy() for t in r["table_grads"]],
               eik_table_grads=[t.numpy() for t in r["eik_table_grads"]],
               dec_grads={k: v.numpy() for k, v in r["dec_grads"].items()},
               eik_dec_grads={k: v.numpy() for k, v in r["eik_dec_grads"].items()})
    return out


def _grads(tr, frozen):
    return ([t.cpu().numpy().copy() for t in tr.table_grads],
            {} if frozen else {k: g.cpu().numpy().copy() for k, g in zip(DEC_KEYS, tr.dec_grads) if g is not None})


def _fused_eikonal_runs(case, weights=None, frozen=False, outs=True, loss_type="sdf_bce"):
    """The fused step (SdfTrainer.forward_backward_eikonal, one launch) at each weight_e, on one trainer."""
    from shine_mapping_b200 import SdfTrainer
    cfg, octree, dec = build_cuda_models(case, DEV, freeze_decoder=frozen)
    coord = torch.from_numpy(case["coord"]).to(DEV); label = torch.from_numpy(case["label"]).to(DEV)
    weight = torch.from_numpy(case["weight"]).to(DEV)
    n = coord.shape[0]
    tr = SdfTrainer(cfg, octree, dec, main_loss_type=loss_type)
    runs = {}
    for w in weights or (0.1, 0.0, _eik_weight(case)):
        cfg.weight_e = w
        tr.zero_grad()
        g = torch.full((n, 3), float("nan"), device=DEV) if outs else None
        pred = torch.full((n,), float("nan"), device=DEV) if outs else None
        bce, eik = tr.forward_backward_eikonal(coord, label, weight, pred_out=pred, grad_out=g)
        torch.cuda.synchronize()
        tg, dg = _grads(tr, frozen)
        runs[w] = {"bce": float(bce), "eikonal": float(eik), "table_grads": tg, "dec_grads": dg,
                   "g": g.cpu().numpy() if outs else None, "pred": pred.cpu().numpy() if outs else None}
    if frozen:     # DEC_GRAD = false: the decoder segment of the flat buffer stays as zero_grad() left it
        assert all(float(g.abs().max()) == 0.0 for g in tr.dec_grads if g is not None)
        assert all(p.grad is None for p in dec.parameters())
    return runs


def _class_surface_eikonal_runs(case):
    """The reference's autograd recipe on the class surface (coordinate-gradient and tangent kernels + torch MLP)."""
    from shine_mapping_b200 import SdfTrainer
    from shine_mapping_b200.batch_loop import eikonal_iteration
    cfg, octree, dec = build_cuda_models(case, DEV)
    cfg.ekional_loss_on = True
    coord = torch.from_numpy(case["coord"]).to(DEV); label = torch.from_numpy(case["label"]).to(DEV)
    weight = torch.from_numpy(case["weight"]).to(DEV)
    tr = SdfTrainer(cfg, octree, dec)
    runs = {}
    for w in (0.1, 0.0, _eik_weight(case)):
        cfg.weight_e = w
        tr.zero_grad()
        total, eik, g = eikonal_iteration(cfg, octree, dec, tr, coord, label, weight)
        torch.cuda.synchronize()
        tg, dg = _grads(tr, False)
        runs[w] = {"bce": float(total) - w * float(eik), "eikonal": float(eik), "table_grads": tg, "dec_grads": dg,
                   "g": g.cpu().numpy(), "pred": None}
    return runs


def _check_eikonal(runs, want, weight_e=0.1, floor_share=None):
    """runs: {weight_e: outputs} at weight_e, 0 and W.  want: the oracle's (or a golden's) outputs at weight_e with the
    eikonal mean's own gradients.  Asserts parity; returns a line with the worst deviations, each relative to the
    maximum it is graded against (bars: 1e-4 for g / eikonal / loss, 1e-3 for the gradients).  floor_share: the largest
    share of its bar the floor of an eikonal-only gradient may take (a first term that swamps the eikonal one fails)."""
    big = max(runs)
    tot, r0, r1 = runs[weight_e], runs[0.0], runs[big]
    worst = {}

    def rel(name, got, exp, bound, floor=0.0):
        got, exp = np.asarray(got, dtype=np.float64), np.asarray(exp, dtype=np.float64)
        scale = float(np.abs(exp).max()) if exp.size else 0.0
        d = float(np.abs(got - exp).max()) if exp.size else 0.0
        assert d <= bound * scale + floor, f"{name}: max|d| {d:.3e} > {bound:g} x {scale:.3e} + {floor:.1e}"
        if scale > 0:        # lout.bias has no eikonal part: graded by the floor alone
            worst[name.split(" ")[0]] = max(worst.get(name.split(" ")[0], 0.0), d / scale)
            if floor_share is not None and name.startswith("eik_"):
                share = floor / (bound * scale)
                assert share <= floor_share, f"{name}: the floor is {share:.2e} of the bar (W = {big:g} is too small)"
                worst["floor/bar"] = max(worst.get("floor/bar", 0.0), share)

    if tot["g"] is not None:
        rel("g", tot["g"], want["g"], 1e-4, 1e-7)
    if tot["pred"] is not None:
        assert np.all(np.abs(tot["pred"] - want["pred"]) <= 2e-5 + 1e-5 * np.abs(want["pred"]))
    for r in (tot, r0, r1):
        rel("eikonal", r["eikonal"], want["eikonal"], 1e-4, 1e-7)
    rel("loss", tot["bce"] + weight_e * tot["eikonal"], want["loss"], 1e-4)
    for k, gt in enumerate(want["table_grads"]):
        rel(f"total_table level {k}", tot["table_grads"][k][:-1], gt[:-1], 1e-3, 1e-9)
    for name, gt in want["dec_grads"].items():
        if name in tot["dec_grads"]:
            rel(f"total_dec {name}", tot["dec_grads"][name], gt, 1e-3, 1e-9)
    # the eikonal term alone; what does not cancel between the two runs is fp32 reordering of the BCE part
    for k, gt in enumerate(want["eik_table_grads"]):
        base = r0["table_grads"][k][:-1]
        rel(f"eik_table level {k}", (r1["table_grads"][k][:-1] - base) / big, gt[:-1], 1e-3,
            1e-5 * float(np.abs(base).max()) / big + 1e-12)
    for name, gt in want["eik_dec_grads"].items():
        if name in r1["dec_grads"]:
            base = r0["dec_grads"][name]
            rel(f"eik_dec {name}", (r1["dec_grads"][name] - base) / big, gt, 1e-3,
                1e-5 * float(np.abs(base).max()) / big + 1e-12)
    return " ".join(f"{k}={v:.1e}" for k, v in worst.items())


@pytest.mark.parametrize("levels,poly,feature_dim,scale,bias,weighted,reduction", [
    pytest.param(2, True, 8, 1.0, True, False, "mean", id="2-True"),
    pytest.param(4, True, 8, 1.0, True, False, "mean", id="4-True"),
    pytest.param(3, False, 8, 1.0, True, False, "mean", id="3-False"),
    pytest.param(6, True, 8, 1.0, True, False, "mean", id="6-True"),
    pytest.param(3, True, 8, 300.0, True, True, "sum", id="3-True-weighted-sum-x300"),
    pytest.param(2, False, 8, 300.0, False, True, "mean", id="2-False-nobias-weighted-mean-x300"),
    # the coordinate-gradient and tangent kernels are generic in F
    pytest.param(3, True, 4, 300.0, True, False, "mean", id="3-True-F4-x300"),
    pytest.param(3, False, 16, 300.0, True, True, "sum", id="3-False-F16-weighted-sum-x300"),
])
def test_eikonal_through_class_surface_matches_oracle(levels, poly, feature_dim, scale, bias, weighted, reduction):
    """ekional_loss_on (reference shine_batch.py:141-142,183-185): d pred / d coord with create_graph=True through
    query_feature's coordinate-gradient kernels, and the second backward through the tangent kernels."""
    case = _eikonal_case(levels, poly, 100 + levels + (0 if scale == 1.0 else 20 + feature_dim), weighted, reduction, scale,
                         bias=bias, feature_dim=feature_dim)
    print(_check_eikonal(_class_surface_eikonal_runs(case), _oracle_eikonal(case)))


def test_eikonal_matches_reference_golden():
    """The CUDA eikonal path against the outputs of the reference's own classes (tests/golden/ref_eikonal_l3.npz)."""
    import json
    import os
    from shine_mapping_b200 import SdfTrainer
    from shine_mapping_b200.batch_loop import eikonal_iteration
    from tests.parity_utils import GOLDEN_DIR
    z = np.load(os.path.join(GOLDEN_DIR, "ref_eikonal_l3.npz"))
    cfg_j = json.loads(str(z["cfg_json"]))
    case = {"cfg": cfg_j, "frames": [z["frame_0"]], "tables": [z[f"table_{k}"] for k in range(cfg_j["tree_level_feat"])],
            "dec": {k: z["dec_" + k] for k in DEC_KEYS}, "coord": z["coord"], "label": z["label"], "weight": z["weight"]}
    cfg, octree, dec = build_cuda_models(case, DEV)
    cfg.ekional_loss_on, cfg.weight_e = True, cfg_j["weight_e"]
    tr = SdfTrainer(cfg, octree, dec)
    tr.zero_grad()
    total, eik, g = eikonal_iteration(cfg, octree, dec, tr, torch.from_numpy(z["coord"]).to(DEV),
                                      torch.from_numpy(z["label"]).to(DEV), torch.from_numpy(z["weight"]).to(DEV))
    assert np.abs(g.cpu().numpy() - z["exp_g"]).max() <= 1e-4 * np.abs(z["exp_g"]).max() + 1e-7
    assert abs(float(eik) - float(z["exp_eikonal"])) <= 1e-4 * abs(float(z["exp_eikonal"]))
    assert abs(float(total) - float(z["exp_loss"])) <= 1e-4 * abs(float(z["exp_loss"]))
    for k in range(cfg_j["tree_level_feat"]):
        want = z[f"exp_tgrad_{k}"]
        assert np.abs(tr.table_grads[k].cpu().numpy() - want)[:-1].max() <= 1e-3 * np.abs(want).max() + 1e-9
    for name, p in zip(DEC_KEYS, dec.fused_params()):
        want = z["exp_dgrad_" + name]
        assert np.abs(p.grad.cpu().numpy() - want).max() <= 1e-3 * np.abs(want).max() + 1e-9


def _fused_eikonal(case, weight_e):
    runs = _fused_eikonal_runs(case, (weight_e,))[weight_e]
    return runs, runs["bce"] + weight_e * runs["eikonal"], runs["eikonal"], runs["g"]


@pytest.mark.parametrize("levels,poly,weighted,reduction,scale,n,ordered,frozen,bias,outs,seed", [
    pytest.param(2, True, False, "mean", 1.0, None, False, False, True, True, 102, id="2-True"),
    pytest.param(3, False, False, "mean", 1.0, None, False, False, True, True, 103, id="3-False"),
    pytest.param(4, True, False, "mean", 1.0, None, False, False, True, True, 104, id="4-True"),
    pytest.param(1, True, False, "mean", 300.0, None, False, False, True, True, 111, id="L1-x300"),
    pytest.param(3, False, False, "mean", 300.0, None, False, False, True, True, 103, id="L3-linear-x300"),
    pytest.param(4, True, True, "mean", 300.0, None, False, False, True, False, 114, id="L4-weighted-mean-x300"),
    pytest.param(6, False, True, "sum", 300.0, None, False, False, True, True, 116, id="L6-linear-weighted-sum-x300"),
    pytest.param(8, True, True, "mean", 300.0, None, False, False, True, True, 118, id="L8-weighted-mean-x300"),
    pytest.param(2, True, True, "sum", 1.0, None, False, False, True, True, 112, id="L2-weighted-sum"),
    pytest.param(4, True, False, "mean", 300.0, None, False, True, True, True, 124, id="L4-frozen-x300"),
    pytest.param(2, False, False, "mean", 1.0, None, False, True, True, False, 122, id="L2-linear-frozen"),
    pytest.param(3, True, False, "mean", 300.0, None, False, False, False, True, 133, id="L3-nobias-x300"),
    pytest.param(2, False, True, "sum", 300.0, None, False, True, False, True, 132, id="L2-linear-nobias-frozen-x300"),
    pytest.param(4, True, False, "mean", 300.0, None, True, False, True, True, 144, id="L4-morton-x300"),
    pytest.param(3, False, True, "sum", 1.0, None, True, False, True, False, 143, id="L3-linear-morton-weighted-sum"),
    pytest.param(2, True, False, "mean", 300.0, 1, False, False, True, True, 152, id="n1"),
    pytest.param(3, False, False, "mean", 300.0, 31, False, False, True, True, 153, id="n31"),
    pytest.param(2, True, True, "sum", 300.0, 33, False, False, True, False, 152, id="n33"),
    pytest.param(4, True, False, "mean", 300.0, 129, False, False, True, True, 154, id="n129"),
    # > 2 blocks/SM x 4 warps x 32 points: warps loop over several tiles of the grid-stride loop
    pytest.param(4, True, True, "mean", 300.0, 60016, False, False, True, True, 164, id="n60016-x300"),
])
def test_fused_eikonal_step_matches_oracle(levels, poly, weighted, reduction, scale, n, ordered, frozen, bias, outs, seed):
    """ONE launch (shine_sdf_eikonal_step) against the oracle's autograd double backward, for every configuration
    the kernel takes: 1..8 levels, poly / linear interpolation, weighted BCE with mean / sum, the frozen-decoder
    instantiation (table gradients only), a decoder without biases, table scale 1 and x300, tile tails, the grid-stride
    loop, a Morton-ordered batch (lanes of a warp hit the same rows), pred_out / grad_out passed or not."""
    case = _eikonal_case(levels, poly, seed, weighted, reduction, scale, n=n, ordered=ordered, bias=bias,
                         n_batch=60000 if (n or 0) > 10000 else 1500)
    want = _oracle_eikonal(case)
    if frozen:
        want["dec_grads"], want["eik_dec_grads"] = {}, {}
    surf = case["weight"] > 0
    print(f"N={case['coord'].shape[0]} surface={int(surf.sum())} median|g|={np.median(np.linalg.norm(want['g'][surf], axis=1)):.3f}",
          _check_eikonal(_fused_eikonal_runs(case, frozen=frozen, outs=outs), want))


DIFF_LOSSES = ("sdf_l1", "sdf_l2")


def _diff_eikonal_runs(case, loss_type, frozen=False, outs=True):
    """The fused sdf_l1 / sdf_l2 + eikonal step (shine_sdf_eikonal_step) at weight_e = 0.1, 0 and W = _eik_weight(case,
    oracle), graded by _check_eikonal with the floor at most 0.1 of its bar.  The L1 oracle takes the kernel's sign near
    the label from a run with pred_out (the kernel's pred does not depend on the outputs asked for, so runs without
    them are graded against the same oracle).  -> (runs, oracle, report line with N, surface count and eikonal share)."""
    from tests import sdf_diff_oracle as sdo
    want = _oracle_eikonal(case, loss_type=loss_type)
    big = _eik_weight(case, want)
    runs = _fused_eikonal_runs(case, (0.1, 0.0, big), frozen, outs, loss_type)
    if loss_type == "sdf_l1":
        pred = runs[0.1]["pred"] if outs else _fused_eikonal_runs(case, (0.1,), frozen, True, loss_type)[0.1]["pred"]
        want = _oracle_eikonal(case, loss_type=loss_type, l1_sign=sdo.l1_sign(want["pred"], case["label"], pred, 2e-5, 1e-5))
    if frozen:
        want["dec_grads"], want["eik_dec_grads"] = {}, {}
    share = [0.1 * np.abs(e).max() / np.abs(t).max() for t, e in _grad_pairs(want) if np.abs(e).max() > 0] or [0.0]
    line = (f"{loss_type} N={case['coord'].shape[0]} surface={int((case['weight'] > 0).sum())} W={big:.3g} "
            f"eikonal share {min(share):.1e}..{max(share):.1e} " + _check_eikonal(runs, want, floor_share=0.1))
    return runs, want, line


DIFF_EIKONAL_CASES = [   # levels, poly, scale, n, ordered, frozen, bias, outs, seed
    pytest.param(1, True, 1.0, None, False, False, True, True, 201, id="L1"),
    pytest.param(2, True, 300.0, None, False, False, True, True, 202, id="L2-x300"),
    pytest.param(3, False, 1.0, None, False, False, True, True, 203, id="L3-linear"),
    pytest.param(4, True, 300.0, None, False, False, True, True, 204, id="L4-x300"),
    pytest.param(6, False, 300.0, None, False, False, True, True, 206, id="L6-linear-x300"),
    pytest.param(8, True, 300.0, None, False, False, True, True, 208, id="L8-x300"),
    pytest.param(4, True, 300.0, None, False, True, True, True, 214, id="L4-frozen-x300"),
    pytest.param(3, True, 300.0, None, False, False, False, True, 223, id="L3-nobias-x300"),
    pytest.param(4, True, 300.0, None, True, False, True, True, 234, id="L4-morton-x300"),
    pytest.param(2, False, 1.0, None, False, False, True, False, 242, id="L2-linear-no-outs"),
    pytest.param(2, True, 300.0, 1, False, False, True, True, 252, id="n1"),
    pytest.param(3, False, 300.0, 31, False, False, True, True, 253, id="n31"),
    pytest.param(2, True, 300.0, 33, False, False, True, False, 252, id="n33"),
    pytest.param(4, True, 300.0, 129, False, False, True, True, 254, id="n129"),
    pytest.param(4, True, 300.0, 60016, False, False, True, True, 264, id="n60016-x300"),
]


@pytest.mark.parametrize("loss_type", DIFF_LOSSES)
@pytest.mark.parametrize("levels,poly,scale,n,ordered,frozen,bias,outs,seed", DIFF_EIKONAL_CASES)
def test_fused_sdf_diff_eikonal_step_matches_oracle(loss_type, levels, poly, scale, n, ordered, frozen, bias, outs, seed):
    """ONE launch of shine_sdf_eikonal_step against the oracle's double backward, on the configurations of
    test_fused_eikonal_step_matches_oracle that apply to sdf_diff_loss (always |w|, always the mean): 1..8 levels, poly /
    linear interpolation, the frozen-decoder instantiation, a decoder without biases, a Morton-ordered batch, tables
    x1 and x300, tile tails, the grid-stride loop, pred_out / grad_out passed or not."""
    case = _eikonal_case(levels, poly, seed, True, "mean", scale, n=n, ordered=ordered, bias=bias,
                         n_batch=60000 if (n or 0) > 10000 else 1500)
    print(_diff_eikonal_runs(case, loss_type, frozen, outs)[2])


def test_fused_eikonal_step_without_surface_sample():
    """No sample with weight > 0: the eikonal value is exactly 0 (as include/shine_b200.h documents; the reference's
    torch mean over an empty selection would be NaN) and the gradients are those of the first term's step alone, for
    sdf_bce and sdf_l1 / sdf_l2."""
    from tests import test_gpu_sdf_diff as sdd
    case = _eikonal_case(3, True, 171, True, "mean", 300.0)
    case["weight"] = -np.abs(case["weight"])
    for loss_type in ("sdf_bce",) + DIFF_LOSSES:
        runs = _fused_eikonal_runs(case, loss_type=loss_type)
        want = run_oracle_step(case) if loss_type == "sdf_bce" else sdd._oracle(case, loss_type, runs[0.1]["pred"])
        for w, r in runs.items():
            assert r["eikonal"] == 0.0, (loss_type, w)
            assert abs(r["bce"] - want["loss"]) <= 1e-4 * abs(want["loss"]), (loss_type, w)
            assert np.all(np.abs(r["pred"] - want["pred"]) <= 2e-5 + 1e-5 * np.abs(want["pred"])), (loss_type, w)
            for k, gt in enumerate(want["table_grads"]):
                assert np.abs(r["table_grads"][k] - gt)[:-1].max() <= 2e-4 * np.abs(gt).max() + 1e-10, (loss_type, w, k)
            for k, gt in want["dec_grads"].items():
                assert np.abs(r["dec_grads"][k] - gt).max() <= 2e-4 * np.abs(gt).max() + 1e-10, (loss_type, w, k)
            for k in range(len(want["table_grads"])):   # weight_e does not enter: the same kernel arithmetic every time
                assert (np.abs(r["table_grads"][k] - runs[0.0]["table_grads"][k]).max() <=
                        1e-6 * np.abs(want["table_grads"][k]).max()), (loss_type, w, k)


def test_fused_eikonal_step_surface_samples_that_miss_every_level():
    """Surface samples outside the map: g = 0, so each adds (1 - 0)^2 = 1 to the mean and nothing to the gradients
    (torch's d|g|/dg is 0 at g = 0); with sdf_bce and with sdf_l1 / sdf_l2 as the first term."""
    case = _eikonal_case(3, False, 172, scale=300.0)
    rng = np.random.default_rng(11)
    far = rng.uniform(0.6, 0.9, size=(77, 3)).astype(np.float32)
    case["coord"] = np.concatenate([case["coord"], far])
    case["label"] = np.concatenate([case["label"], np.zeros(77, np.float32)])
    case["weight"] = np.concatenate([case["weight"], np.ones(77, np.float32)])
    n_surf = int((case["weight"] > 0).sum())
    for loss_type in ("sdf_bce",) + DIFF_LOSSES:
        if loss_type == "sdf_bce":
            want, runs = _oracle_eikonal(case), _fused_eikonal_runs(case)
            line = _check_eikonal(runs, want)
        else:
            runs, want, line = _diff_eikonal_runs(case, loss_type)
        assert np.all(want["g"][-77:] == 0.0) and np.all(runs[0.1]["g"][-77:] == 0.0), loss_type
        assert want["eikonal"] >= 77.0 / n_surf, loss_type
        print(loss_type, line)


def test_fused_eikonal_shards_add_up_to_the_global_batch():
    """A batch in two uneven parts accumulated into one trainer, with n_norm and n_surface of the whole batch, gives the
    full batch's gradients, and the two eikonal values add up to its mean: what a rank of a data-parallel run computes."""
    from shine_mapping_b200 import SdfTrainer
    case = _eikonal_case(3, True, 181, scale=300.0, n_batch=3000)
    want = _oracle_eikonal(case, weight_e=1.0)
    cfg, octree, dec = build_cuda_models(case, DEV)
    cfg.weight_e = 1.0
    coord = torch.from_numpy(case["coord"]).to(DEV); label = torch.from_numpy(case["label"]).to(DEV)
    weight = torch.from_numpy(case["weight"]).to(DEV)
    n, n_surf = coord.shape[0], int((case["weight"] > 0).sum())
    tr = SdfTrainer(cfg, octree, dec)
    tr.zero_grad()
    bce = eik = 0.0
    for sl in (slice(0, 2 * n // 5), slice(2 * n // 5, n)):
        b, e = tr.forward_backward_eikonal(coord[sl], label[sl], weight[sl], n_norm=n, n_surface=n_surf)
        bce, eik = bce + float(b), eik + float(e)
    torch.cuda.synchronize()
    parts = _grads(tr, False)
    tr.zero_grad()
    b, e = tr.forward_backward_eikonal(coord, label, weight)
    torch.cuda.synchronize()
    full = _grads(tr, False)
    assert abs(eik - float(e)) <= 1e-5 * abs(float(e)) and abs(bce - float(b)) <= 1e-5 * abs(float(b))
    assert abs(eik - want["eikonal"]) <= 1e-4 * want["eikonal"]
    assert abs(bce + eik - want["loss"]) <= 1e-4 * want["loss"]
    for got, ful, gt in zip(parts[0], full[0], want["table_grads"]):
        assert np.abs(got - ful)[:-1].max() <= 1e-5 * np.abs(ful).max()
        assert np.abs(got - gt)[:-1].max() <= 1e-3 * np.abs(gt).max()
    for k, gt in want["dec_grads"].items():
        assert np.abs(parts[1][k] - full[1][k]).max() <= 1e-5 * np.abs(full[1][k]).max(), k
        assert np.abs(parts[1][k] - gt).max() <= 1e-3 * np.abs(gt).max(), k


def test_fused_eikonal_step_matches_scaled_reference_golden():
    """The fused entry against the reference's own classes on tables scaled x500 (median surface |g| ~1), weighted BCE
    with sum reduction (tests/golden/ref_eikonal_l3_sum_weighted.npz, which also holds the eikonal mean's own gradients)."""
    case, z = load_eikonal_golden("ref_eikonal_l3_sum_weighted")
    w = case["cfg"]["weight_e"]
    L = case["cfg"]["tree_level_feat"]
    want = {"g": z["exp_g"], "pred": z["exp_pred"], "eikonal": float(z["exp_eikonal"]), "loss": float(z["exp_loss"]),
            "table_grads": [z[f"exp_tgrad_{k}"] for k in range(L)], "eik_table_grads": [z[f"exp_eik_tgrad_{k}"] for k in range(L)],
            "dec_grads": {k: z["exp_dgrad_" + k] for k in DEC_KEYS}, "eik_dec_grads": {k: z["exp_eik_dgrad_" + k] for k in DEC_KEYS}}
    print(_check_eikonal(_fused_eikonal_runs(case, (w, 0.0, _eik_weight(case))), want, w))


def test_fused_eikonal_step_matches_reference_golden_and_beats_class_surface():
    """The fused entry against the outputs of the reference's own classes (tests/golden/ref_eikonal_l3.npz), and its
    time against the class-surface composition (query kernels + cuBLAS + autograd double backward)."""
    import json
    import os
    from shine_mapping_b200 import SdfTrainer
    from shine_mapping_b200.batch_loop import eikonal_iteration
    from tests.parity_utils import GOLDEN_DIR
    z = np.load(os.path.join(GOLDEN_DIR, "ref_eikonal_l3.npz"))
    cfg_j = json.loads(str(z["cfg_json"]))
    case = {"cfg": cfg_j, "frames": [z["frame_0"]], "tables": [z[f"table_{k}"] for k in range(cfg_j["tree_level_feat"])],
            "dec": {k: z["dec_" + k] for k in DEC_KEYS}, "coord": z["coord"], "label": z["label"], "weight": z["weight"]}
    run, total, eik, g = _fused_eikonal(case, cfg_j["weight_e"])
    assert np.abs(g - z["exp_g"]).max() <= 1e-4 * np.abs(z["exp_g"]).max() + 1e-7
    assert abs(eik - float(z["exp_eikonal"])) <= 1e-4 * abs(float(z["exp_eikonal"]))
    assert abs(total - float(z["exp_loss"])) <= 1e-4 * abs(float(z["exp_loss"]))
    for k in range(cfg_j["tree_level_feat"]):
        want = z[f"exp_tgrad_{k}"]
        assert np.abs(run["table_grads"][k] - want)[:-1].max() <= 1e-3 * np.abs(want).max() + 1e-9
    for name, gd in run["dec_grads"].items():
        want = z["exp_dgrad_" + name]
        assert np.abs(gd - want).max() <= 1e-3 * np.abs(want).max() + 1e-9
    # timing at the KITTI batch size (config/kitti/kitti_batch.yaml: batch_size 16384)
    big = make_case(n_points=3000, n_batch=16384, feat_levels=4, seed=7)
    cfg, octree, dec2 = build_cuda_models(big, DEV)
    cfg.ekional_loss_on, cfg.weight_e = True, 0.1
    coord = torch.from_numpy(big["coord"]).to(DEV); label = torch.from_numpy(big["label"]).to(DEV)
    weight = torch.from_numpy(big["weight"]).to(DEV)
    tr2 = SdfTrainer(cfg, octree, dec2)

    def timed(fn, reps=10):
        for _ in range(3):
            tr2.zero_grad(); fn()
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(reps):
            tr2.zero_grad(); fn()
        e1.record(); torch.cuda.synchronize()
        return e0.elapsed_time(e1) / reps
    t_fused = timed(lambda: tr2.forward_backward_eikonal(coord, label, weight))
    t_class = timed(lambda: eikonal_iteration(cfg, octree, dec2, tr2, coord, label, weight))
    print(f"eikonal step, {coord.shape[0]} points: fused {t_fused:.3f} ms, class surface {t_class:.3f} ms, x{t_class / t_fused:.1f}")
    assert t_class > 2.0 * t_fused


def test_points_to_morton_bit_exact():
    from shine_mapping_b200 import _abi
    from oracle import shine_oracle as orc
    g = torch.Generator().manual_seed(3)
    x = (torch.rand(200000, 3, generator=g) * 2.4 - 1.2)
    x[:8] = torch.tensor([[-1, -1, -1], [1, 1, 1], [0, 0, 0], [1 - 2 ** -12, 2 ** -12, -2 ** -12], [0.5, -0.5, 0.25],
                          [-1.0000001, 0.99999994, 0.9999999], [3, -3, 0], [2 ** -11, 2 ** -10, 2 ** -9]])
    xd = x.to(DEV).contiguous()
    for level in (1, 5, 9, 12, 15):
        out = torch.empty(x.shape[0], dtype=torch.int64, device=DEV)
        _abi.check(_abi.lib().shine_points_to_morton(_abi.ptr(xd), x.shape[0], level, _abi.ptr(out),
                                                     _abi.stream_ptr()), "morton")
        want = orc.points_to_morton(orc.quantize_points(x.numpy(), level))
        assert np.array_equal(out.cpu().numpy(), want), level


# ---- size-independent properties at BASELINE scale ------------------------------------------------------

def test_large_batch_properties():
    """1M points, L=4: (a) interpolation weights sum to 1 => per level, the column sums of the table gradient
    equal the column sums of dL/dfeature over the points that hit that level; (b) two runs give identical
    indices and (up to atomic ordering) identical gradients; (c) pred of the step == pred of the inference
    kernel bit-for-bit."""
    from shine_mapping_b200 import SdfTrainer, sdf_infer, synth
    from tests.parity_utils import make_config
    from shine_mapping_b200 import Decoder, FeatureOctree
    torch.manual_seed(1)
    cfg = make_config(4, device=DEV, pc_radius=50.0)
    octree, dec = FeatureOctree(cfg), Decoder(cfg)
    pool = synth.build_scene_map(cfg, octree, n_azimuth=512, n_frames=2, seed=1, device=DEV)
    n = 1 << 20
    coord, label, weight = pool.get_batch(n)
    tr = SdfTrainer(cfg, octree, dec)
    pred = torch.empty(n, device=DEV)
    tr.zero_grad(); tr.forward_backward(coord, label, weight, pred_out=pred)
    g1 = tr.flat_grad.clone()
    tr.zero_grad(); tr.forward_backward(coord, label, weight)
    g2 = tr.flat_grad.clone()
    assert (g1 - g2).abs().max() <= 1e-4 * g1.abs().max()
    assert torch.equal(pred, sdf_infer(octree, dec, coord))
    # (a) with the unfused autograd path giving dL/dfeature
    feat = octree.query_feature(coord).detach().requires_grad_(True)
    loss = torch.nn.functional.binary_cross_entropy_with_logits(
        dec.sdf(feat), torch.sigmoid(label / cfg.sigma_sigmoid))
    loss.backward()
    idx = octree.get_indices(coord)
    for i in range(4):
        hit = (idx[i] >= 0).all(1)
        want = feat.grad[hit].double().sum(0)
        got = tr.table_grads[4 - i - 1].double().sum(0)
        assert torch.allclose(got, want, rtol=2e-3, atol=1e-7), (i, got, want)
    # loss value agrees with the torch composition
    assert abs(float(tr.loss) - float(loss)) <= 2e-5 * abs(float(loss))


# ---- optimizer + trainer ---------------------------------------------------------------------------------

def test_adam_kernel_matches_torch_adam():
    from shine_mapping_b200 import SdfTrainer
    case = make_case(n_points=2000, n_batch=4096, feat_levels=3, seed=41)
    cfg, octree, dec = build_cuda_models(case, DEV)
    cfg.lr, cfg.weight_decay, cfg.lr_level_reduce_ratio = 0.01, 1e-7, 0.7
    cfg2, octree2, dec2 = build_cuda_models(case, DEV)
    coord = torch.from_numpy(case["coord"]).to(DEV); label = torch.from_numpy(case["label"]).to(DEV)
    tr = SdfTrainer(cfg, octree, dec)
    # torch reference optimiser with the reference grouping (utils/tools.py:57-83)
    groups = [{"params": list(dec2.fused_params()), "lr": cfg.lr, "weight_decay": cfg.weight_decay}]
    lr = cfg.lr
    feats = list(octree2.parameters())
    for i in range(3):
        groups.append({"params": feats[3 - i - 1], "lr": lr}); lr *= cfg.lr_level_reduce_ratio
    opt = torch.optim.Adam(groups, betas=(0.9, 0.99), eps=cfg.adam_eps)
    from shine_mapping_b200 import sdf_bce_step
    for it in range(5):
        tr.zero_grad() if it == 0 else None
        tr.train_step(coord, label)
        opt.zero_grad(set_to_none=True)
        sdf_bce_step(octree2, dec2, coord, label, cfg.sigma_sigmoid).backward()
        opt.step()
    for a, b in zip(octree.hier_features, octree2.hier_features):
        assert torch.allclose(a[:-1], b[:-1], rtol=2e-3, atol=2e-5), (a[:-1] - b[:-1]).abs().max()
    for a, b in zip(dec.fused_params(), dec2.fused_params()):
        assert torch.allclose(a, b, rtol=2e-3, atol=2e-5)


def test_training_reduces_loss():
    from shine_mapping_b200 import SdfTrainer
    case = make_case(n_points=3000, n_batch=8192, feat_levels=4, seed=42)
    cfg, octree, dec = build_cuda_models(case, DEV)
    cfg.lr = 0.01
    coord = torch.from_numpy(case["coord"]).to(DEV); label = torch.from_numpy(case["label"]).to(DEV)
    tr = SdfTrainer(cfg, octree, dec)
    tr.zero_grad()
    first = float(tr.train_step(coord, label))
    for _ in range(60):
        last = float(tr.train_step(coord, label))
    assert last < 0.9 * first, (first, last)


def test_cpu_tensor_is_rejected_loudly():
    from shine_mapping_b200 import _abi
    case = make_case(n_points=1500, n_batch=10, feat_levels=2, seed=5)
    cfg, octree, dec = build_cuda_models(case, DEV)
    with pytest.raises(_abi.ShineB200Error):
        octree.query_feature(torch.zeros(4, 3))


def test_abi_rejects_bad_arguments():
    from shine_mapping_b200 import _abi
    lib = _abi.lib()
    d = _abi.ShineOctree()
    d.num_levels = 0
    assert lib.shine_query_fwd(C.byref(d), None, 4, None, None) == -1
    assert b"invalid" in lib.shine_error_string(-1)


def test_biasless_decoder_matches_oracle_in_every_default_kernel():
    """geo_mlp_bias_on: False — every fused kernel reads the biases through null-pointer branches: the general and the
    grouped (Morton-ordered) kernels of sdf_bce_step, its two-pass mode, and the inference kernel."""
    from shine_mapping_b200 import sdf_infer
    from tests.parity_utils import drop_relu_kink_points
    case = make_case(n_points=2500, n_batch=3000, feat_levels=3, seed=57, weighted=True, reduction="sum", bias=False)
    case, dropped = drop_relu_kink_points(case)
    want = run_oracle_step(case)
    assert sorted(want["dec_grads"]) == ["layers.0.weight", "layers.1.weight", "lout.weight"]
    print("general", compare_step(run_cuda_step(case, DEV), want))
    print("two-pass", compare_step(run_cuda_step(case, DEV, single_pass=False), want))
    want_f = dict(want); want_f["dec_grads"] = {}
    print("frozen", compare_step(run_cuda_step(case, DEV, freeze_decoder=True), want_f))
    ordered = sort_case_morton(case)
    print("grouped", compare_step(run_cuda_step(ordered, DEV, morton_ordered=True), run_oracle_step(ordered)))
    cfg, octree, dec = build_cuda_models(case, DEV)
    assert all(p is None for p in dec.fused_params()[1::2])
    pred = sdf_infer(octree, dec, torch.from_numpy(case["coord"]).to(DEV))
    torch.cuda.synchronize()
    assert np.abs(pred.cpu().numpy() - want["pred"]).max() < 2e-5


def test_two_queries_before_one_backward():
    """ADVICE r01: the reference queries `coord_near` while the first query's graph is still alive (shine_batch.py:155-160);
    re-zeroing the trash row inside query_feature must not invalidate the tensors autograd saved for the first query."""
    case = make_case(n_points=1500, n_batch=600, feat_levels=3, seed=12)
    cfg, octree, dec = build_cuda_models(case, DEV)
    c = torch.from_numpy(case["coord"]).to(DEV)
    f1 = octree.query_feature(c[:300])
    f2 = octree.query_feature(c[300:600] + 1e-4)
    (f1.sum() + 2.0 * f2.sum()).backward()
    g = [p.grad.clone() for p in octree.hier_features]
    for p in octree.hier_features:
        p.grad = None
    octree.query_feature(c[:300]).sum().backward()
    ga = [p.grad.clone() for p in octree.hier_features]
    for p in octree.hier_features:
        p.grad = None
    (2.0 * octree.query_feature(c[300:600] + 1e-4).sum()).backward()
    for a, b, p in zip(g, ga, octree.hier_features):
        assert torch.allclose(a, b + p.grad, rtol=1e-5, atol=1e-7)
