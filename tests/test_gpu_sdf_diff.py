"""Training with the reference's sdf_l1 / sdf_l2 losses on the GPU: the fused kernels against the fp64 oracle
(tests/sdf_diff_oracle.py) and against goldens minted from the reference, shards, and both mapping loops."""
import os

import numpy as np
import pytest
import torch

from tests import sdf_diff_oracle as sdo
from tests.parity_utils import (GOLDEN_DIR, build_cuda_models, check_frozen_grads, compare_step, drop_relu_kink_points,
                                fill_frozen_grads, make_case, make_config, oracle_from_case, sort_case_morton)

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
PRED_ATOL, PRED_RTOL = 2e-5, 1e-5          # compare_step's pred tolerance


def _with_far_points(case, k=80, seed=0):
    """k more samples far from the map (a miss on every level): whole zero tiles once the batch is in Morton order."""
    rng = np.random.default_rng(seed)
    out = dict(case)
    far = rng.uniform(0.80, 0.95, size=(k, 3)).astype(np.float32)
    out["coord"] = np.concatenate([case["coord"], far])
    out["label"] = np.concatenate([case["label"], rng.uniform(-1e-3, 1e-3, k).astype(np.float32)])
    out["weight"] = np.concatenate([case["weight"], rng.uniform(-1.5, -0.5, k).astype(np.float32)])
    return out


def _scale(case):
    c = case["cfg"]
    return 1.0 / (c["leaf_vox_size"] * 2 ** (c["tree_level_world"] - 1))


def _cuda_step(case, loss_type, **kw):
    from shine_mapping_b200.fused import sdf_diff_step
    freeze = kw.pop("freeze_decoder", False)
    cfg, octree, dec = build_cuda_models(case, DEV, freeze_decoder=freeze)
    frozen = fill_frozen_grads(dec) if freeze else None
    coord, label, weight = (torch.from_numpy(np.ascontiguousarray(case[k])).to(DEV) for k in ("coord", "label", "weight"))
    indices = [t.cpu().numpy() for t in octree.get_indices(coord)]
    feature = octree.query_feature(coord)
    loss, pred = sdf_diff_step(octree, dec, coord, label, weight, cfg.scale, l2_loss=loss_type == "sdf_l2",
                               return_pred=True, **kw)
    loss.backward()
    torch.cuda.synchronize()
    if frozen is not None:
        check_frozen_grads(dec, frozen)
    named = dict(dec.named_parameters())
    return {"indices": indices, "feature": feature.detach().cpu().numpy(), "pred": pred.cpu().numpy(),
            "loss": float(loss.detach()), "table_grads": [p.grad.cpu().numpy() for p in octree.hier_features],
            "dec_grads": {} if freeze else {k: named[k].grad.cpu().numpy() for k in case["dec"]}}


def _oracle(case, loss_type, got_pred=None, atol=PRED_ATOL, rtol=PRED_RTOL):
    """fp64 oracle; for L1, samples whose |pred - label| lies inside the pred tolerance (atol, rtol) take the sign of
    the CUDA pred's fp32 difference (either side is right there), exact zeros included."""
    o, dec = oracle_from_case(case)
    label = case["label"]
    sign = None
    if loss_type == "sdf_l1" and got_pred is not None:
        o2, dec2 = oracle_from_case(case)
        ref = sdo.train_step(o2, dec2, torch.from_numpy(case["coord"]), torch.from_numpy(label),
                             torch.from_numpy(case["weight"]), 1.0, loss_type=loss_type, scale=_scale(case), double=True)
        sign = sdo.l1_sign(ref["pred"].numpy(), label, got_pred, atol, rtol)
    res = sdo.train_step(o, dec, torch.from_numpy(case["coord"]), torch.from_numpy(label), torch.from_numpy(case["weight"]),
                         1.0, loss_type=loss_type, scale=_scale(case), double=True, l1_sign=sign)
    return sdo.as_numpy(res, o)


def _drop_frozen(want, freeze):
    return dict(want, dec_grads={}) if freeze else want


# (levels, batch, morton order, single_pass, tf32x1, frozen decoder, biases)
CONFIGS = [
    (2, 2037, False, True, False, False, True),      # order drawn, tile tail
    (3, 2037, True, True, False, False, True),       # Morton order: grouped kernel, zero tiles
    (4, 1500, True, True, False, True, True),        # grouped kernel, frozen decoder
    (3, 1500, True, True, False, False, False),      # grouped kernel, bias-less decoder
    (1, 1200, False, True, False, False, True),
    (5, 1500, True, True, False, False, True),       # L > 4: the general kernel takes Morton-ordered batches
    (8, 1200, True, True, False, False, True),
    (6, 1200, False, False, False, False, True),     # forward kernel + recomputing backward
    (3, 1500, True, False, False, True, True),
    (4, 1500, False, True, True, False, True),       # TF32X1
    (7, 1200, False, True, True, False, False),
]


@pytest.mark.parametrize("loss_type", ["sdf_l1", "sdf_l2"])
@pytest.mark.parametrize("levels,n_batch,morton,single_pass,tf32x1,frozen,bias", CONFIGS)
def test_fused_step_matches_oracle(loss_type, levels, n_batch, morton, single_pass, tf32x1, frozen, bias, built_lib):
    case = make_case(n_points=3000, n_batch=n_batch, feat_levels=levels, seed=100 + levels, weighted=True, bias=bias)
    case, _ = drop_relu_kink_points(_with_far_points(case, seed=levels))
    if morton:
        case = sort_case_morton(case)
    kw = dict(morton_ordered=morton, single_pass=single_pass, tf32x1=tf32x1, freeze_decoder=frozen)
    got = _cuda_step(case, loss_type, **kw)
    if loss_type == "sdf_l1":
        # exact-zero differences: give some samples their own CUDA prediction as label (dL/dpred = 0 there)
        case = dict(case, label=case["label"].copy())
        case["label"][::97] = got["pred"][::97]
        got = _cuda_step(case, loss_type, **kw)
        assert np.array_equal(got["pred"][::97], case["label"][::97])
    # TF32X1: plain TF32 products (10-bit mantissa); the bar of test_gpu_mask_operands.py's TF32X1 grading.  Every L1
    # sample carries a full-size dL/dpred, so cancellation in the table sums shows more than with BCE (L=7: 7.5e-2)
    tol = dict(pred_atol=5e-3, pred_rtol=5e-3, grad_rel=0.25) if tf32x1 else {}
    want = _drop_frozen(_oracle(case, loss_type, got["pred"], tol.get("pred_atol", PRED_ATOL),
                                tol.get("pred_rtol", PRED_RTOL)), frozen)
    print(loss_type, levels, compare_step(got, want, **tol))


def test_l1_zero_difference_gives_zero_gradient(built_lib):
    """One sample, its label its own prediction: the step leaves every gradient at 0 (torch's sign(0) = 0)."""
    case = make_case(n_points=1500, n_batch=1, feat_levels=2, seed=5)
    case = dict(case, coord=case["coord"][:1], label=case["label"][:1].copy(), weight=np.ones(1, np.float32))
    pred = _cuda_step(case, "sdf_l1")["pred"]
    case["label"][:] = pred
    got = _cuda_step(case, "sdf_l1")
    assert got["loss"] == 0.0
    assert all(not g.any() for g in got["table_grads"]) and all(not g.any() for g in got["dec_grads"].values())


@pytest.mark.parametrize("name", ["ref_sdf_l1_l3_weighted", "ref_sdf_l2_l3"])
@pytest.mark.parametrize("morton", [False, True])
def test_fused_step_matches_reference_golden(name, morton, built_lib):
    z = np.load(os.path.join(GOLDEN_DIR, name + ".npz"))
    case, cfg = sdo.golden_case(z)
    want = sdo.expected(z, cfg["tree_level_feat"])
    if morton:
        sorted_case = sort_case_morton(case)
        from shine_mapping_b200.feature_octree import points_to_morton, quantize_points
        order = torch.argsort(points_to_morton(quantize_points(torch.from_numpy(case["coord"]), 12)), stable=True).numpy()
        case = sorted_case
        want = dict(want, indices=[i[order] for i in want["indices"]], feature=want["feature"][order],
                    pred=want["pred"][order])
    got = _cuda_step(case, cfg["loss_type"], morton_ordered=morton)
    print(name, compare_step(got, want))


def _trainer(case, loss_type, eikonal=False, weight_e=0.1):
    from shine_mapping_b200 import SdfTrainer
    cfg, octree, dec = build_cuda_models(case, DEV)
    cfg.main_loss_type, cfg.ekional_loss_on, cfg.weight_e = loss_type, eikonal, weight_e
    return cfg, octree, dec, SdfTrainer(cfg, octree, dec)


def _tensors(case):
    return [torch.from_numpy(np.ascontiguousarray(case[k])).to(DEV) for k in ("coord", "label", "weight")]


def _eik_step(tr, coord, label, weight, weight_e):
    """One fused eikonal step at weight_e -> (total loss, eikonal mean, pred, table grads, decoder grads) on the host."""
    tr.config.weight_e = weight_e
    tr.zero_grad()
    pred = torch.empty(coord.shape[0], device=DEV)
    first, eik = tr.forward_backward_eikonal(coord, label, weight, pred_out=pred)
    torch.cuda.synchronize()
    return (float(first) + weight_e * float(eik), float(eik), pred.cpu().numpy(),
            [g.cpu().numpy()[:-1] for g in tr.table_grads],
            [g.cpu().numpy() for g in tr.dec_grads] if tr._dec_trainable else [])


def _close_rel(got, want, tol, what):
    scale = max(float(np.abs(want).max()), 1e-30)
    err = float(np.abs(np.asarray(got, np.float64) - want).max()) / scale
    assert err <= tol, f"{what}: rel err {err:.3e}"
    return err


@pytest.mark.parametrize("name", ["ref_sdf_l1_eikonal_l3", "ref_sdf_l2_eikonal_l3"])
@pytest.mark.parametrize("frozen", [False, True])
def test_eikonal_step_matches_oracle_golden_and_class_surface(name, frozen, built_lib):
    """The fused sdf_diff_loss + eikonal step (trainable and frozen decoder) against the reference's golden, the fp32
    oracle and the class-surface route (query_feature -> decoder.sdf -> sdf_diff_loss, double backward).  The eikonal
    part is graded on its own too: the step at weight_e minus the step at weight_e = 0 against weight_e times the
    eikonal mean's gradients.  The goldens give the eikonal term 0.03 to 0.93 of every gradient's max."""
    from shine_mapping_b200 import SdfTrainer
    from shine_mapping_b200.batch_loop import eikonal_iteration
    z = np.load(os.path.join(GOLDEN_DIR, name + ".npz"))
    case, cfg = sdo.golden_case(z)
    c, octree, dec = build_cuda_models(case, DEV, freeze_decoder=frozen)
    c.main_loss_type, c.ekional_loss_on = cfg["loss_type"], True
    tr = SdfTrainer(c, octree, dec)
    coord, label, weight = _tensors(case)
    we = cfg["weight_e"]
    total, eik, pred, tg, dg = _eik_step(tr, coord, label, weight, we)
    _, _, _, tg0, dg0 = _eik_step(tr, coord, label, weight, 0.0)
    keys = [k for k in case["dec"]]
    # the reference's golden
    assert total == pytest.approx(float(z["exp_loss"]), rel=1e-4)
    assert eik == pytest.approx(float(z["exp_eikonal"]), rel=1e-3)
    for k in range(len(tg)):
        _close_rel(tg[k], z[f"exp_tgrad_{k}"][:-1], 2e-4, f"golden table grad {k}")
        _close_rel(tg[k] - tg0[k], we * z[f"exp_eik_tgrad_{k}"][:-1], 2e-3, f"golden eikonal table grad {k}")
    for j, k in enumerate(keys if dg else []):
        _close_rel(dg[j], z["exp_dgrad_" + k], 2e-4, f"golden decoder grad {k}")
        if np.abs(z["exp_eik_dgrad_" + k]).max() > 0:
            _close_rel(dg[j] - dg0[j], we * z["exp_eik_dgrad_" + k], 2e-3, f"golden eikonal decoder grad {k}")
    # the oracle, with the L1 sign of the CUDA pred where |pred - label| is inside the pred tolerance
    o, odec = oracle_from_case(case)
    sign = None
    if cfg["loss_type"] == "sdf_l1":
        near = np.abs(z["exp_pred"] - case["label"]) <= PRED_ATOL + PRED_RTOL * np.abs(z["exp_pred"])
        sign = np.sign(z["exp_pred"] - case["label"])
        sign[near] = np.sign(pred[near] - case["label"][near])
    ref = sdo.train_step_eikonal(o, odec, torch.from_numpy(case["coord"]), torch.from_numpy(case["label"]),
                                 torch.from_numpy(case["weight"]), cfg["sigma"], we, loss_type=cfg["loss_type"],
                                 scale=cfg["scale"], l1_sign=sign)
    assert total == pytest.approx(float(ref["loss"]), rel=1e-4)
    for k in range(len(tg)):
        _close_rel(tg[k], ref["table_grads"][k].numpy()[:-1], 2e-4, f"oracle table grad {k}")
        _close_rel(tg[k] - tg0[k], we * ref["eik_table_grads"][k].numpy()[:-1], 2e-3, f"oracle eikonal table grad {k}")
    for j, k in enumerate(keys if dg else []):
        _close_rel(dg[j], ref["dec_grads"][k].numpy(), 2e-4, f"oracle decoder grad {k}")
    # the class-surface route
    tr.config.weight_e = we
    tr.zero_grad()
    total2, eik2, _ = eikonal_iteration(c, octree, dec, tr, coord, label, weight)
    assert float(total2) == pytest.approx(total, rel=1e-4)
    assert float(eik2) == pytest.approx(eik, rel=1e-3)
    for k, g in enumerate(tr.table_grads):
        _close_rel(g.cpu().numpy()[:-1], tg[k], 2e-4, f"class surface table grad {k}")
    for j, g in enumerate(tr.dec_grads if dg else []):
        _close_rel(g.cpu().numpy(), dg[j], 2e-4, f"class surface decoder grad {keys[j]}")


@pytest.mark.parametrize("loss_type", ["sdf_l1", "sdf_l2"])
@pytest.mark.parametrize("eikonal", [False, True])
def test_shards_add_up(loss_type, eikonal, built_lib):
    """Two half batches with n_norm = N (and, eikonal, the whole batch's surface count) sum to the whole batch."""
    case = make_case(n_points=2500, n_batch=4000, feat_levels=3, seed=9, weighted=True)
    n = case["coord"].shape[0]
    coord, label, weight = _tensors(case)
    _, _, _, tr = _trainer(case, loss_type, eikonal, 1.0)

    def step(sl, n_surface=None):
        if eikonal:
            a, b = tr.forward_backward_eikonal(coord[sl], label[sl], weight[sl], n_norm=n, n_surface=n_surface)
            return float(a) + float(b)
        return float(tr.forward_backward(coord[sl], label[sl], weight[sl], n_norm=n))

    tr.zero_grad()
    whole = step(slice(0, n))
    g_whole = tr.flat_grad.clone()
    tr.zero_grad()
    ns = int((weight > 0).sum())
    parts = step(slice(0, n // 2), ns) + step(slice(n // 2, n), ns)
    assert parts == pytest.approx(whole, rel=2e-5)
    assert float((tr.flat_grad - g_whole).abs().max()) <= 2e-5 * float(g_whole.abs().max())


# MaiCity's thresholds (eval/evaluator.py), with 10^6 instead of 10^7 mesh samples
STREET_EVAL = dict(down_sample_res=0.02, threshold=0.1, truncation_acc=0.2, truncation_com=2.0, gt_bbx_mask_on=True,
                   mesh_sample_point=1_000_000, seed=11)


@pytest.mark.parametrize("loss_type", ["sdf_l1", "sdf_l2"])
def test_batch_loop_trains_meshes_and_evaluates(loss_type, built_lib):
    from shine_mapping_b200 import Decoder, FeatureOctree, Mesher, synth
    from shine_mapping_b200.batch_loop import run_shine_mapping_batch
    from shine_mapping_b200.evaluate import eval_mesh
    # the street of test_gpu_eval.py (default lr 1e-3: at 1e-2 the L1 map of 300 iterations has no surface yet)
    base = dict(tree_level_world=12, tree_level_feat=3, leaf_vox_size=0.3, device=DEV, bs=8192, iters=300,
                mc_res_m=0.15, surface_sample_range_m=0.3, free_sample_end_dist_m=1.0, min_range=2.0, pc_radius=25.0,
                main_loss_type=loss_type, continual_learning_reg=False, window_replay_on=False)
    for graphed, host in ((True, False), (False, False), (True, True), (False, True)):
        cfg = make_config(**dict(base, pc_count_gpu_limit=2 if host else 100))
        torch.manual_seed(0)
        octree, dec = FeatureOctree(cfg), Decoder(cfg)
        pool = synth.build_scene_map(cfg, octree, 512, 10 if not host else 4, frame_step_m=1.0, seed=3, pool="auto")
        assert isinstance(pool, synth.HostSamplePool) == host
        out = run_shine_mapping_batch(cfg, octree, dec, pool, iters=300 if not host else 100, use_cuda_graph=graphed)
        assert np.isfinite(out["loss_last"]) and out["loss_last"] < 0.8 * out["loss_first"], (graphed, host, out)
        if graphed and not host:
            verts, faces, _ = Mesher(cfg, octree, dec).recon_bbx_mesh(pool.map_bbx[0], pool.map_bbx[1], cfg.mc_res_m)
            gt = synth.scene_surface_points(-10.0, 20.0, 0.1).to(DEV)
            m = eval_mesh((verts, faces), gt, device=DEV, **STREET_EVAL)
            print(loss_type, {k: round(float(v), 4) for k, v in m.items()})
            assert m["F-score (%)"] > 0, m
    # the eikonal variant of the loop
    cfg = make_config(**dict(base, ekional_loss_on=True, weight_e=0.1, bs=2048))
    torch.manual_seed(0)
    octree, dec = FeatureOctree(cfg), Decoder(cfg)
    pool = synth.build_scene_map(cfg, octree, 256, 2, seed=3)
    out = run_shine_mapping_batch(cfg, octree, dec, pool, iters=100)
    assert np.isfinite(out["loss_last"]) and out["loss_last"] < out["loss_first"], out


def test_scans_command_line_writes_checkpoint_and_mesh(tmp_path, capsys, built_lib):
    from shine_mapping_b200 import batch_loop
    from tests.test_gpu_scans import _yaml, write_sequence
    paths = write_sequence(str(tmp_path), "bin", n_frames=4)
    run = tmp_path / "run"
    over = {"loss__main_loss_type": "sdf_l2", "eval__save_freq_iters": 100, "eval__vis_freq_iters": 100,
            "eval__mc_res_m": 0.2}
    batch_loop.main([_yaml(tmp_path, paths, **over), "--scans", "--iters", "100", "--run-path", str(run)])
    out = capsys.readouterr().out
    assert "loss_first" in out
    assert (run / "model" / "model_iter_100.pth").exists()
    meshes = list((run / "mesh").glob("mesh_iter_100.ply"))
    assert meshes and meshes[0].stat().st_size > 1000


def test_incremental_loop_trains_bce_whatever_main_loss_type_says(built_lib):
    """run_shine_mapping_incremental trains sdf_bce as the reference's shine_incre.py:150 does, also when the config says
    sdf_l1 / sdf_l2, with the regularisation mode's feature importance (an unweighted BCE sweep) included."""
    from shine_mapping_b200 import Decoder, FeatureOctree, synth
    from shine_mapping_b200.incre_loop import run_shine_mapping_incremental
    hists = {}
    for loss in ("sdf_bce", "sdf_l2", "sdf_l1"):
        cfg = make_config(3, device=DEV, bs=2048, lr=0.01, iters=20, continual_learning_reg=True, lambda_forget=1e3,
                          main_loss_type=loss)
        torch.manual_seed(1)
        octree, decoder = FeatureOctree(cfg), Decoder(cfg)
        dirs, boxes = synth.lidar_directions(128, device=DEV), synth.default_boxes(DEV)
        gen = torch.Generator(device=DEV).manual_seed(3)
        frames = []
        for f in range(2):
            origin = torch.tensor([2.0 * f, 0.0, 0.0], device=DEV)
            hits = synth.raycast_scene(origin, dirs, boxes, cfg.min_range, cfg.pc_radius)
            frames.append(synth.sample_rays(hits * cfg.scale, origin * cfg.scale, cfg, gen))
        hists[loss] = run_shine_mapping_incremental(cfg, octree, decoder, frames)
    for loss in ("sdf_l2", "sdf_l1"):
        assert len(hists[loss]) == 2
        # the first batch's loss before any step: BCE (about 0.69), not the L1 / L2 value of the same batch
        assert hists[loss][0]["bce_first"] == pytest.approx(hists["sdf_bce"][0]["bce_first"], rel=1e-5), hists[loss]
        assert all(h["bce_last"] < h["bce_first"] for h in hists[loss]), hists[loss]


@pytest.mark.parametrize("loss_type", ["sdf_l1", "sdf_l2"])
def test_host_memory_entries_take_the_weights(loss_type, built_lib):
    """step_from_host / submit_host_step copy the weights for sdf_l1 / sdf_l2 whatever loss_weight_on says, and give
    the loss and gradients of the device-tensor step."""
    case = make_case(n_points=2500, n_batch=3000, feat_levels=3, seed=21, weighted=True)
    _, _, _, tr = _trainer(case, loss_type)
    tr.config.loss_weight_on = False                 # weighted=True above only makes the weights non-trivial
    coord, label, weight = _tensors(case)
    tr.zero_grad()
    want = float(tr.forward_backward(coord, label, weight))
    g_want = tr.flat_grad.clone()
    ch, lh, wh = (t.cpu().pin_memory() for t in (coord, label, weight))
    for use_graph in (False, True):
        got = tr.step_from_host(ch, lh, wh, chunks=1, use_graph=use_graph)
        assert got == pytest.approx(want, rel=1e-5)
        assert float((tr.flat_grad - g_want).abs().max()) <= 2e-5 * float(g_want.abs().max())
    got = tr.submit_host_step(ch, lh, wh).result()
    assert got == pytest.approx(want, rel=1e-5)
