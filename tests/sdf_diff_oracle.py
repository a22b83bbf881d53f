"""fp64 oracle of the training step with the reference's sdf_diff_loss (utils/loss.py:6-14; main_loss_type sdf_l1 /
sdf_l2, shine_batch.py:171-185), on the restated octree and decoder of oracle/shine_oracle.py.  Test infrastructure.

`train_step` / `train_step_eikonal` take the same arguments as shine_oracle's and a `loss_type`: "sdf_bce" calls
shine_oracle's own step unchanged, "sdf_l1" / "sdf_l2" replace the BCE term by sdf_diff_loss.  With `double=True` the
tables, decoder, labels and weights are promoted to fp64 first; the coordinates, and so the octree lookup and the fp32
interpolation weights of the reference, stay as they are.
"""
from __future__ import annotations

import numpy as np
import torch

from oracle import shine_oracle as orc

LOSS_TYPES = ("sdf_bce", "sdf_l1", "sdf_l2")


def sdf_diff_loss(pred, label, weight, scale, l2_loss=True):
    """utils/loss.py:6-14: sum(weight * |diff_m|) or sum(weight * diff_m^2) over count = len(pred), diff_m in metres."""
    count = pred.shape[0]
    diff_m = (pred - label) / scale
    return (weight * (diff_m ** 2 if l2_loss else diff_m.abs())).sum() / count


def diff_dpred(pred, label, weight, scale, l2_loss, count, sign=None):
    """dL/dpred of sdf_diff_loss per sample: 2 w diff_m / scale / count (L2) or w sign(diff_m) / scale / count (L1).
    sign: the L1 sign to use instead of sign(diff_m) (grading an fp32 kernel whose pred lands on the other side of the
    label)."""
    diff_m = (pred - label) / scale
    if l2_loss:
        return 2.0 * weight * diff_m / scale / count
    s = torch.sign(diff_m) if sign is None else sign
    return weight * s / scale / count


def l1_sign(pred, label, got_pred, atol, rtol):
    """The L1 sign per sample for grading an fp32 kernel: sign(pred - label) of the oracle's pred, and the sign of the
    kernel's own difference (0 where its pred equals the label) where |pred - label| <= atol + rtol |pred|: there either
    side of the label is right."""
    pred, label = np.asarray(pred, np.float64), np.asarray(label)
    near = np.abs(pred - label) <= atol + rtol * np.abs(pred)
    sign = np.sign(pred - label)
    sign[near] = np.sign(np.asarray(got_pred, np.float32)[near] - label[near])
    return sign


def _promote(octree, dec, coord, label, weight):
    octree.hier_features = [f.detach().double().requires_grad_(True) for f in octree.hier_features]
    dec = {k: v.detach().double().requires_grad_(True) for k, v in dec.items()}
    return octree, dec, coord, label.double(), weight.double()


def train_step(octree, dec, coord, label, weight, sigma, weighted=False, reduction="mean", loss_type="sdf_bce",
               scale=None, n_norm=None, double=False, l1_sign=None):
    """shine_batch.py:123,128,171-179,208-209 -> dict(loss, pred, feature, table_grads, dec_grads) like
    shine_oracle.train_step.  scale: config.scale (sdf_l1 / sdf_l2).  n_norm: the loss's count (default len(coord)).
    l1_sign: per-sample sign replacing sign(diff_m) in the L1 backward (the loss value keeps |diff_m|)."""
    if loss_type not in LOSS_TYPES:
        raise ValueError(loss_type)
    if loss_type == "sdf_bce":
        return orc.train_step(octree, dec, coord, label, weight, sigma, weighted, reduction)
    if double:
        octree, dec, coord, label, weight = _promote(octree, dec, coord, label, weight)
    for f in octree.hier_features:
        f.grad = None
    for p in dec.values():
        p.grad = None
    # the interpolation weights stay fp32, as the reference computes them from fp32 coordinates
    feature = octree.query_feature_with_indices(coord, octree.get_indices(coord))
    pred = orc.decoder_sdf(feature, dec)
    w = torch.abs(weight).to(pred.dtype)                                  # shine_batch.py:172
    l2 = loss_type == "sdf_l2"
    count = float(n_norm if n_norm else pred.shape[0])
    loss = sdf_diff_loss(pred, label, w, scale, l2) * (pred.shape[0] / count)
    dp = diff_dpred(pred.detach(), label, w, scale, l2, count,
                    None if l1_sign is None else torch.as_tensor(l1_sign, dtype=pred.dtype))
    pred.backward(dp)
    return {
        "loss": loss.detach(), "pred": pred.detach(), "feature": feature.detach(),
        "table_grads": [f.grad if f.grad is not None else torch.zeros_like(f) for f in octree.hier_features],
        "dec_grads": {k: (p.grad if p.grad is not None else torch.zeros_like(p)) for k, p in dec.items()},
    }


def train_step_eikonal(octree, dec, coord, label, weight, sigma, weight_e=0.1, weighted=False, reduction="mean",
                       n_surface=None, loss_type="sdf_bce", scale=None, n_norm=None, l1_sign=None):
    """shine_oracle.train_step_eikonal with the first term chosen by loss_type (sdf_diff_loss with |weight|, count =
    n_norm or len(coord)); g = sigma * d pred / d coord whatever the loss (shine_batch.py:141-142).  The returned `bce`
    entry holds that first term; `eik_table_grads` / `eik_dec_grads` are the gradients of the eikonal mean alone (at
    weight_e = 1).  l1_sign: as in train_step, the sign of the L1 term's backward per sample."""
    if loss_type == "sdf_bce":
        return orc.train_step_eikonal(octree, dec, coord, label, weight, sigma, weight_e, weighted, reduction, n_surface)
    for f in octree.hier_features:
        f.grad = None
    for p in dec.values():
        p.grad = None
    coord = coord.clone().requires_grad_(True)
    feature = octree.query_feature(coord)
    pred = orc.decoder_sdf(feature, dec)
    surface_mask = weight > 0
    g = torch.autograd.grad(pred, coord, torch.ones_like(pred), create_graph=True, retain_graph=True)[0] * sigma
    count = float(n_norm if n_norm else pred.shape[0])
    first = sdf_diff_loss(pred, label, torch.abs(weight), scale, loss_type == "sdf_l2") * (pred.shape[0] / count)
    if loss_type == "sdf_l1" and l1_sign is not None:   # the same value where the signs agree, the given sign's gradient
        s = torch.as_tensor(l1_sign, dtype=pred.dtype)
        first = (torch.abs(weight) * s * (pred - label) / scale).sum() / count
    sq = (1.0 - g[surface_mask].norm(2, dim=-1)) ** 2
    eik = sq.mean() if n_surface is None else sq.sum() / float(n_surface)
    loss = first + weight_e * eik
    params = list(octree.hier_features) + list(dec.values())
    eg = torch.autograd.grad(eik, params, retain_graph=True, allow_unused=True)
    eg = [torch.zeros_like(p) if d is None else d for p, d in zip(params, eg)]
    L = len(octree.hier_features)
    loss.backward()
    return {"loss": loss.detach(), "bce": first.detach(), "eikonal": eik.detach(), "g": g.detach(), "pred": pred.detach(),
            "table_grads": [f.grad if f.grad is not None else torch.zeros_like(f) for f in octree.hier_features],
            "dec_grads": {k: (p.grad if p.grad is not None else torch.zeros_like(p)) for k, p in dec.items()},
            "eik_table_grads": eg[:L], "eik_dec_grads": dict(zip(dec.keys(), eg[L:]))}


def as_numpy(res, octree):
    """The dict of train_step -> the layout of tests.parity_utils.run_oracle_step (numpy, indices included)."""
    return {"indices": [t.numpy() for t in octree.hierarchical_indices], "feature": res["feature"].numpy(),
            "pred": res["pred"].numpy(), "loss": float(res["loss"]),
            "table_grads": [g.detach().numpy() for g in res["table_grads"]],
            "dec_grads": {k: g.detach().numpy() for k, g in res["dec_grads"].items()}}


def golden_case(z):
    """-> (case, cfg) of a golden minted by oracle/make_sdf_diff_golden.py, in the layout of parity_utils.make_case."""
    import json
    cfg = json.loads(str(z["cfg_json"]))
    keys = [k[4:] for k in z.files if k.startswith("dec_")]
    case = {"cfg": cfg, "frames": [z["frame_0"]], "tables": [z[f"table_{k}"] for k in range(cfg["tree_level_feat"])],
            "dec": {k: z["dec_" + k] for k in keys}, "coord": z["coord"], "label": z["label"], "weight": z["weight"]}
    return case, cfg


def expected(z, L):
    """The reference's outputs frozen in a golden of oracle/make_sdf_diff_golden.py (numpy)."""
    return {"indices": [z[f"exp_indices_{i}"].astype(np.int64) for i in range(L)], "feature": z["exp_feature"],
            "pred": z["exp_pred"], "loss": float(z["exp_loss"]),
            "table_grads": [z[f"exp_tgrad_{k}"] for k in range(L)],
            "dec_grads": {k[10:]: z[k] for k in z.files if k.startswith("exp_dgrad_")}}
