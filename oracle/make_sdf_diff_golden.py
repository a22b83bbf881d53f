"""Mint tests/golden/ref_sdf_l1_l3_weighted.npz, ref_sdf_l2_l3.npz, ref_sdf_l2_eikonal_l3.npz and ref_sdf_l1_eikonal_l3.npz
from the UNMODIFIED reference.  *** TEST INFRASTRUCTURE ***

Same conventions as oracle/make_golden.py (whose `import_reference`, `reference_config` and `DEC_KEYS` this uses, and
whose goldens it leaves alone): runs only where the reference checkout is available, on the CPU, with oracle/kaolin_shim
in place of kaolin.  The reference's own `FeatureOctree`, `Decoder` and `utils/loss.py::sdf_diff_loss` are driven like
the loop body of shine_batch.py:123,128,171-179,183-185,208-209 with main_loss_type sdf_l1 / sdf_l2; the npz keys are
those of make_golden.make (plain step) and make_golden.make_eikonal (eikonal step), plus `scale` and `loss_type` in
cfg_json.

    python oracle/make_sdf_diff_golden.py            # mints all four
    python oracle/make_sdf_diff_golden.py NAME ...   # only the named ones
"""
from __future__ import annotations

import json
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from make_golden import DEC_KEYS, REF, ROOT, import_reference, reference_config  # noqa: E402


def make(name, loss_type, feat_levels, n_azimuth, n_batch, seed, weighted=False, eikonal=False, weight_e=0.1,
         table_scale=1.0, label_noise=None):
    """label_noise: labels = the reference's own prediction + label_noise * N(0, 1) instead of the sampler's labels.  With
    small differences the sdf term's gradients shrink (L2) or keep a fixed size (L1), so that the eikonal term's share
    of the gradient is large enough for a test to see it (printed when minted)."""
    SHINEConfig, FeatureOctree, Decoder, dataSampler, _ = import_reference()
    from utils.loss import sdf_diff_loss
    sys.path.insert(0, ROOT)
    from shine_mapping_b200 import synth   # scene ray-caster only (inputs); everything after is the reference

    torch.manual_seed(seed)
    cfg = reference_config(SHINEConfig, feat_levels, 0.2, True, weighted, "mean")
    octree, decoder, sampler = FeatureOctree(cfg), Decoder(cfg), dataSampler(cfg)
    dirs, boxes = synth.lidar_directions(n_azimuth), synth.default_boxes()
    origin = torch.zeros(3)
    hits = synth.raycast_scene(origin, dirs, boxes, 3.0, 30.0)
    coord, label, _, _, weight, _, _ = sampler.sample(hits * cfg.scale, origin * cfg.scale, None, None)
    surface = coord[weight > 0, :]
    octree.update(surface, False)                                          # dataset/lidar_dataset.py:212-218
    index = torch.randint(0, coord.shape[0], (n_batch,))                   # dataset/lidar_dataset.py:431-448
    coord, label, weight = coord[index].clone(), label[index], weight[index]
    extra = torch.tensor([[0.9, 0.9, 0.9], [-1.0, -1.0, -1.0], [0.0, 0.0, 0.0]])   # misses: pred = Decoder.sdf(0)
    coord = torch.cat((coord, extra))
    label = torch.cat((label, torch.zeros(3)))
    weight = torch.cat((weight, -torch.ones(3)))
    if weighted:
        weight = weight * (0.5 + torch.rand(weight.shape[0]))
    with torch.no_grad():
        for p in octree.hier_features:
            p.mul_(table_scale)
    sigma = cfg.logistic_gaussian_ratio * cfg.sigma_sigmoid_m * cfg.scale   # shine_batch.py:87
    if label_noise is not None:
        with torch.no_grad():
            label = (decoder.sdf(octree.query_feature(coord.detach())) + label_noise * torch.randn(coord.shape[0])).detach()
    tables_before = [p.detach().numpy().copy() for p in octree.hier_features]
    # ---- the loop body, shine_batch.py:119-120,123,128,137-142,171-185,208-209 ----
    if eikonal:
        coord.requires_grad_(True)
    feature = octree.query_feature(coord)
    pred = decoder.sdf(feature)
    surface_mask = weight > 0
    loss = sdf_diff_loss(pred, label, torch.abs(weight), cfg.scale, l2_loss=loss_type == "sdf_l2")
    total = loss
    out = {}
    params = list(octree.hier_features) + [dict(decoder.named_parameters())[k] for k in DEC_KEYS]
    if eikonal:
        g = torch.autograd.grad(outputs=pred, inputs=coord, grad_outputs=torch.ones_like(pred), create_graph=True,
                                retain_graph=True, only_inputs=True)[0] * sigma   # get_gradient(coord, pred) * sigma_sigmoid
        eikonal_loss = ((1.0 - g[surface_mask].norm(2, dim=-1)) ** 2).mean()
        total = loss + weight_e * eikonal_loss
        eik_grads = torch.autograd.grad(eikonal_loss, params, retain_graph=True, allow_unused=True)
        eik_grads = [torch.zeros_like(p) if d is None else d for p, d in zip(params, eik_grads)]
        out.update({"exp_g": g.detach().numpy(), "exp_eikonal": np.array(float(eikonal_loss.detach()))})
    total.backward()
    out.update({
        "cfg_json": np.array(json.dumps(dict(
            tree_level_world=12, tree_level_feat=feat_levels, feature_dim=cfg.feature_dim, poly_int_on=True,
            leaf_vox_size=0.2, sigma=float(sigma), scale=float(cfg.scale), loss_type=loss_type, weighted=weighted,
            reduction="mean", decoder_frozen=False, n_frames=1, eikonal=eikonal, weight_e=weight_e,
            table_scale=table_scale))),
        "frame_0": surface.numpy().copy(), "coord": coord.detach().numpy(), "label": label.numpy(),
        "weight": weight.numpy(), "exp_feature": feature.detach().numpy(), "exp_pred": pred.detach().numpy(),
        "exp_loss": np.array(float(total.detach())), "exp_sdf_loss": np.array(float(loss.detach())),
    })
    for i, idx in enumerate(octree.hierarchical_indices):
        out[f"exp_indices_{i}"] = idx.numpy().astype(np.int32)
    for k, t in enumerate(tables_before):
        out[f"table_{k}"] = t
        out[f"exp_tgrad_{k}"] = octree.hier_features[k].grad.numpy()
        if eikonal:
            out[f"exp_eik_tgrad_{k}"] = eik_grads[k].numpy()
    sd, named = decoder.state_dict(), dict(decoder.named_parameters())
    for j, k in enumerate(DEC_KEYS):
        out["dec_" + k] = sd[k].numpy()
        out["exp_dgrad_" + k] = named[k].grad.numpy()
        if eikonal:
            out["exp_eik_dgrad_" + k] = eik_grads[len(tables_before) + j].numpy()
    path = os.path.join(ROOT, "tests", "golden", name + ".npz")
    np.savez_compressed(path, **out)
    share = ""
    if eikonal:   # the eikonal term's share of every gradient tensor: max |weight_e * d eik| / max |d total|
        tot = [p.grad for p in params]
        share = " eikonal share " + " ".join(f"{float((weight_e * e).abs().max() / t.abs().max()):.2g}"
                                              for e, t in zip(eik_grads, tot) if float(t.abs().max()) > 0)
    print(f"{name}: N={coord.shape[0]} rows={[t.shape[0] for t in tables_before]} scale={cfg.scale:.3e} "
          f"loss={float(total):.6f}{share} -> {path} ({os.path.getsize(path) / 1e6:.2f} MB)")


WE_L2, NOISE_L2, WE_L1 = 3000.0, 1e-2, 3000.0

GOLDENS = {
    "ref_sdf_l1_l3_weighted": lambda n: make(n, "sdf_l1", 3, n_azimuth=10, n_batch=1000, seed=61, weighted=True),
    "ref_sdf_l2_l3": lambda n: make(n, "sdf_l2", 3, n_azimuth=10, n_batch=1000, seed=62),
    # tables x500 as ref_eikonal_l3_sum_weighted: surface |g| near 1.  The sdf term's gradient carries 1 / scale (L1) or
    # diff / scale^2 (L2): a weight_e that gives the eikonal term a share of every gradient a test can see and, for L2,
    # labels at 1e-2 from the prediction: small enough for that weight_e, large against the fp32 rounding of |pred| <= 8
    "ref_sdf_l2_eikonal_l3": lambda n: make(n, "sdf_l2", 3, n_azimuth=10, n_batch=1000, seed=63, eikonal=True,
                                            table_scale=500.0, weight_e=WE_L2, label_noise=NOISE_L2),
    "ref_sdf_l1_eikonal_l3": lambda n: make(n, "sdf_l1", 3, n_azimuth=10, n_batch=1000, seed=64, eikonal=True,
                                            table_scale=500.0, weight_e=WE_L1, weighted=True),
}


if __name__ == "__main__":
    if not os.path.isdir(REF):
        sys.exit(f"{REF} not found: goldens can only be minted where the reference is mounted")
    for golden in sys.argv[1:] or list(GOLDENS):
        GOLDENS[golden](golden)
