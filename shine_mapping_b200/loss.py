"""Losses of the hot path — reference utils/loss.py:17-24 (`sdf_bce_loss`) and :6-14 (`sdf_diff_loss`).

Class-surface versions (they take a `pred` tensor); the fused kernels compute the same expressions per point in
registers (`csrc/shine_b200.cu`, the `loss_point` lambda; `csrc/shine_device.cuh`, `diff_point`)."""
import torch
import torch.nn.functional as F


def sdf_bce_loss(pred, label, sigma, weight, weighted=False, bce_reduction="mean"):
    """BCE-with-logits between the predicted logits and the occupancy target sigmoid(label / sigma)."""
    target = torch.sigmoid(label / sigma)
    return F.binary_cross_entropy_with_logits(pred, target, weight=weight if weighted else None,
                                              reduction=bce_reduction)


def sdf_diff_loss(pred, label, weight, scale, l2_loss=True):
    """main_loss_type sdf_l1 / sdf_l2: the weighted L1 or L2 distance in metres, diff_m = (pred - label) / scale, summed and
    divided by the batch size.  The weight is always applied (the caller passes |weight|, shine_batch.py:172)."""
    count = pred.shape[0]
    diff_m = (pred - label) / scale
    return (weight * (diff_m ** 2 if l2_loss else diff_m.abs())).sum() / count
