"""The loss bound of the forward-only kernels (tests/infer_bound.py), checked without a GPU:
  * an independent fp32 implementation, the fp32 oracle (torch's fused BCE-with-logits, or sdf_diff_loss, reduced in
    torch's own order), lies inside the pred bound P at every point and inside the loss bound, for BCE mean / sum /
    weighted, sdf_l1 and sdf_l2, on fresh tables and on tables x300;
  * one point's term changed by twice the bound, or one point left out of the sum, lands outside it;
  * the bound is not vacuous: its size relative to the loss is printed."""
import numpy as np
import pytest
import torch

from oracle import shine_oracle as orc
from tests import sdf_diff_oracle as sdo
from tests.infer_bound import LossRef, PredRef
from tests.parity_utils import make_case, oracle_from_case
from tests.test_gpu_replicas import with_weights
from tests.test_gpu_sdf_diff import _scale

CONFIGS = [pytest.param(lt, w, r, id=f"{lt}-{'w' if w else 'u'}-{r}")
           for lt, w, r in [("sdf_bce", False, "mean"), ("sdf_bce", True, "sum"), ("sdf_bce", True, "mean"),
                            ("sdf_l1", True, "mean"), ("sdf_l2", True, "mean")]]


def loss_case(loss_type, weighted, reduction, table_scale, seed=3, n_batch=1500, feat_levels=3):
    case = make_case(n_points=1500, n_batch=n_batch, feat_levels=feat_levels, seed=seed, weighted=weighted,
                     reduction=reduction)
    if table_scale != 1:
        case["tables"] = [(t * np.float32(table_scale)).astype(np.float32) for t in case["tables"]]
    return with_weights(case, loss_type, seed)


def loss_ref(case, loss_type, pred, tf32x1=False):
    """(PredRef, LossRef) of a case for the loss the kernel computes with the case's config"""
    c = case["cfg"]
    pr = PredRef(case, tf32x1=tf32x1)
    lr = LossRef(pr.pred, pr.P, case["label"], case["weight"], loss_type, sigma=c["sigma"], scale=_scale(case),
                 weighted=c["weighted"], reduction=c["reduction"])
    return pr, lr


def _fp32_terms(case, loss_type):
    """the fp32 oracle: pred and the per-point loss terms (loss scale included) and the loss as torch reduces it"""
    c = case["cfg"]
    o, dec = oracle_from_case(case)
    coord, label, weight = (torch.from_numpy(case[k]) for k in ("coord", "label", "weight"))
    with torch.no_grad():
        pred = orc.decoder_sdf(o.query_feature(coord), dec)
        n = pred.shape[0]
        if loss_type == "sdf_bce":
            w = weight.abs() if c["weighted"] else None
            tgt = torch.sigmoid(label / np.float32(c["sigma"]))
            loss = orc.sdf_bce_loss(pred, label, np.float32(c["sigma"]), weight.abs(), c["weighted"], c["reduction"])
            terms = torch.nn.functional.binary_cross_entropy_with_logits(pred, tgt, weight=w, reduction="none")
            terms = terms / n if c["reduction"] == "mean" else terms
        else:
            scale = np.float32(_scale(case))
            loss = sdo.sdf_diff_loss(pred, label, weight.abs(), scale, loss_type == "sdf_l2")
            d = (pred - label) / scale
            terms = weight.abs() * (d * d if loss_type == "sdf_l2" else d.abs()) / n
    return pred.numpy(), float(loss), terms.double().numpy()


@pytest.mark.parametrize("table_scale", [1, 300])
@pytest.mark.parametrize("loss_type,weighted,reduction", CONFIGS)
def test_fp32_oracle_is_inside_the_loss_bound(loss_type, weighted, reduction, table_scale):
    case = loss_case(loss_type, weighted, reduction, table_scale)
    pred32, loss32, terms32 = _fp32_terms(case, loss_type)
    pr, lr = loss_ref(case, loss_type, pred32)
    pr.grade(pred32, f"fp32 oracle x{table_scale}")
    lr.grade(loss32, f"fp32 oracle x{table_scale}")
    print(f"[infer bounds] {loss_type}: bound / |loss| = {lr.bound / abs(lr.want):.2e} (points {lr.per.sum():.2e}, "
          f"summation {lr.summation:.2e})")
    # one point's term off by twice the bound
    with pytest.raises(AssertionError, match="outside the bound"):
        lr.grade(loss32 + 2 * lr.bound, "one term changed by 2 x bound")
    with pytest.raises(AssertionError, match="outside the bound"):
        lr.grade(loss32 - 2 * lr.bound, "one term changed by -2 x bound")
    # one point missing from the sum (the largest term: a dropped tile loses at least one like it)
    j = int(np.argmax(np.abs(terms32)))
    assert abs(terms32[j]) > 2 * lr.bound, (terms32[j], lr.bound)
    with pytest.raises(AssertionError, match="outside the bound"):
        lr.grade(loss32 - terms32[j], "one point missing")


def test_kernel_error_model_terms_are_each_needed():
    """Each part of the BCE point bound is positive where its source is: the MUFU log error on every point, the zt error
    where labels are far from 0, the pred part where P is."""
    from tests.infer_bound import loss_terms
    p = np.array([0.0, 3.0, -40.0, 1e-3])
    lb = np.array([0.0, 50.0, -50.0, 1.0], dtype=np.float32)
    t, per, s = loss_terms(p, np.zeros(4), lb, np.ones(4), "sdf_bce", sigma=1.0, reduction="sum")
    assert s == 1.0 and np.all(per > 0) and np.all(t >= 0)
    t2, per2, _ = loss_terms(p, np.full(4, 1e-6), lb, np.ones(4), "sdf_bce", sigma=1.0, reduction="sum")
    assert np.all(per2 > per)
    assert np.allclose(t, t2)
