"""The fused hot path: reference shine_batch.py:123 (`query_feature`) + :128 (`Decoder.sdf`) + :174
(`sdf_bce_loss`) + :209 (`backward`) as ONE sm_90a kernel launch (`shine_sdf_bce_step`); `sdf_diff_step` is the same
with the reference's other point-wise losses (:176-179, `sdf_diff_loss`, main_loss_type sdf_l1 / sdf_l2).

`sdf_bce_step(...)` returns the loss with autograd attached.  Because the loss gradient of a sample depends only
on that sample, the kernel computes forward, loss AND the full backward (table scatter-add + decoder grads) in one
pass while the gathered rows, interpolation weights and activations are still in registers; `loss.backward()`
then only scales the stashed gradients by the upstream scalar.  `single_pass=False` gives the classical two
launches (forward kernel; backward kernel that recomputes) for callers that want it.
"""
from __future__ import annotations

import ctypes as C

import torch

from . import _abi
from .decoder import Decoder
from .feature_octree import FeatureOctree


def _flags(weighted: bool, reduction: str, extra) -> int:
    """extra: True / False (plain-TF32 decoder) or an int of further SHINE_FLAG_* bits (TF32X1, MORTON_ORDERED)."""
    if reduction not in ("mean", "sum"):
        raise ValueError(f"loss_reduction must be 'mean' or 'sum', got {reduction!r}")
    f = 0
    if reduction == "sum":
        f |= _abi.FLAG_REDUCTION_SUM
    if weighted:
        f |= _abi.FLAG_WEIGHTED
    if extra is True:
        f |= _abi.FLAG_TF32X1
    elif extra:
        f |= int(extra)
    return f


def _prep(t, name):
    if t is None:
        return None
    _abi.require_cuda(t, name)
    t = t.detach()
    if t.dtype != torch.float32 or not t.is_contiguous():
        t = t.float().contiguous()
    return t


class _SdfBce(torch.autograd.Function):
    @staticmethod
    def forward(ctx, octree, decoder, coord, label, weight, sigma, weighted, reduction, n_norm, single_pass,
                tf32x1, *params):
        L = octree.featured_level_num
        tables, dparams = params[:L], params[L:]
        n = coord.shape[0]
        dev = coord.device
        lib = _abi.lib()
        stream = _abi.stream_ptr(dev)
        flags = _flags(weighted, reduction, tf32x1)
        scale = 1.0 if reduction == "sum" else 1.0 / float(n_norm if n_norm else n)
        pred = torch.empty(n, dtype=torch.float32, device=dev)
        loss = torch.zeros((), dtype=torch.float32, device=dev)
        need_t = [p.requires_grad for p in tables]
        need_d = [p is not None and p.requires_grad for p in dparams]
        # forward() runs under no_grad; needs_input_grad already folds in the caller's grad mode
        need_t = [bool(x) for x in ctx.needs_input_grad[11:11 + L]]
        need_d = [bool(x) for x in ctx.needs_input_grad[11 + L:]]
        want_grad = any(need_t) or any(need_d)
        ctx.octree, ctx.decoder = octree, decoder
        ctx.cfg = (sigma, scale, flags, n, need_t, need_d)
        if want_grad and single_pass:
            tgrads = [torch.zeros_like(p) for p in tables]
            dgrads = [torch.zeros_like(p) if (p is not None and any(need_d)) else None for p in dparams]
            od = octree._descriptor(tables, tgrads)
            dd = decoder.c_descriptor(dgrads if any(need_d) else None)
            _abi.check(lib.shine_sdf_bce_step(C.byref(od), C.byref(dd), _abi.ptr(coord), _abi.ptr(label),
                                              _abi.ptr(weight), n, sigma, scale, None, _abi.ptr(pred),
                                              _abi.ptr(loss), flags, stream), "shine_sdf_bce_step")
            ctx.stash = (tgrads, dgrads)
        else:
            od = octree._descriptor(tables, None)
            dd = decoder.c_descriptor(None)
            _abi.check(lib.shine_sdf_bce_fwd(C.byref(od), C.byref(dd), _abi.ptr(coord), _abi.ptr(label),
                                             _abi.ptr(weight), n, sigma, scale, _abi.ptr(pred), _abi.ptr(loss),
                                             flags, stream), "shine_sdf_bce_fwd")
            ctx.stash = None
            if want_grad:
                ctx.save_for_backward(coord, label, weight if weight is not None else coord.new_empty(0), *params)
        ctx.mark_non_differentiable(pred)
        return loss, pred

    @staticmethod
    def backward(ctx, dloss, _dpred):
        sigma, scale, flags, n, need_t, need_d = ctx.cfg
        octree, decoder = ctx.octree, ctx.decoder
        L = octree.featured_level_num
        if ctx.stash is not None:
            tgrads, dgrads = ctx.stash
            ctx.stash = None
            for g in list(tgrads) + [g for g in dgrads if g is not None]:
                g.mul_(dloss)
        else:
            coord, label, weight, *params = ctx.saved_tensors
            weight = weight if weight.numel() else None
            tables, dparams = params[:L], params[L:]
            tgrads = [torch.zeros_like(p) for p in tables]
            dgrads = [torch.zeros_like(p) if (p is not None and any(need_d)) else None for p in dparams]
            od = octree._descriptor(tables, tgrads)
            dd = decoder.c_descriptor(dgrads if any(need_d) else None)
            dl = dloss.detach().float().contiguous()
            _abi.check(_abi.lib().shine_sdf_bce_step(
                C.byref(od), C.byref(dd), _abi.ptr(coord), _abi.ptr(label), _abi.ptr(weight), n, sigma, scale,
                _abi.ptr(dl), None, None, flags, _abi.stream_ptr(coord.device)), "shine_sdf_bce_step")
        out_t = [g if need else None for g, need in zip(tgrads, need_t)]
        out_d = [g if need else None for g, need in zip(dgrads, need_d)]
        return (None,) * 11 + tuple(out_t) + tuple(out_d)


def sdf_bce_step(octree: FeatureOctree, decoder: Decoder, coord, sdf_label, sigma, weight=None, weighted=False,
                 bce_reduction="mean", n_norm=None, single_pass=True, tf32x1=False, return_pred=False,
                 morton_ordered=False):
    """loss (= sdf_bce_loss(decoder.sdf(octree.query_feature(coord)), sdf_label, sigma, |weight|, weighted,
    reduction)) with autograd to `octree.hier_features` and the decoder parameters.

    n_norm: denominator of the "mean" (defaults to len(coord); pass the GLOBAL batch when sharding points).
    morton_ordered: the batch is in Morton order (see SdfTrainer.forward_backward); a performance hint."""
    if coord.requires_grad:
        raise NotImplementedError("gradients w.r.t. coordinates are not part of the fused sm_90a path")
    coord, sdf_label = _prep(coord, "coord"), _prep(sdf_label, "sdf_label")
    weight = _prep(weight, "weight") if weighted else None
    if weighted and weight is None:
        raise ValueError("weighted=True needs a weight tensor")
    params = list(octree.hier_features) + list(decoder.fused_params())
    octree._last_coord, octree._hier_idx = coord, []
    # autograd.Function cannot take None among *tensor* args transparently for needs_input_grad bookkeeping,
    # so bias-less decoders pass None placeholders which are skipped in backward.
    loss, pred = _SdfBce.apply(octree, decoder, coord, sdf_label, weight, float(sigma), bool(weighted),
                               bce_reduction, n_norm, single_pass,
                               (_abi.FLAG_TF32X1 if tf32x1 else 0) | (_abi.FLAG_MORTON_ORDERED if morton_ordered else 0), *params)
    return (loss, pred) if return_pred else loss


class _SdfDiff(torch.autograd.Function):
    """`_SdfBce` with sdf_diff_loss (`shine_sdf_diff_fwd` / `shine_sdf_diff_step`)."""

    @staticmethod
    def forward(ctx, octree, decoder, coord, label, weight, scale, flags, n_norm, single_pass, *params):
        L = octree.featured_level_num
        tables, dparams = params[:L], params[L:]
        n = coord.shape[0]
        dev = coord.device
        lib = _abi.lib()
        stream = _abi.stream_ptr(dev)
        loss_scale = 1.0 / float(n_norm if n_norm else n)         # utils/loss.py:7,12-14: sum / count
        pred = torch.empty(n, dtype=torch.float32, device=dev)
        loss = torch.zeros((), dtype=torch.float32, device=dev)
        need_t = [bool(x) for x in ctx.needs_input_grad[9:9 + L]]
        need_d = [bool(x) for x in ctx.needs_input_grad[9 + L:]]
        want_grad = any(need_t) or any(need_d)
        ctx.octree, ctx.decoder = octree, decoder
        ctx.cfg = (scale, loss_scale, flags, n, need_t, need_d)
        if want_grad and single_pass:
            tgrads = [torch.zeros_like(p) for p in tables]
            dgrads = [torch.zeros_like(p) if (p is not None and any(need_d)) else None for p in dparams]
            od = octree._descriptor(tables, tgrads)
            dd = decoder.c_descriptor(dgrads if any(need_d) else None)
            _abi.check(lib.shine_sdf_diff_step(C.byref(od), C.byref(dd), _abi.ptr(coord), _abi.ptr(label), _abi.ptr(weight),
                                               n, scale, loss_scale, None, _abi.ptr(pred), _abi.ptr(loss), flags, stream),
                       "shine_sdf_diff_step")
            ctx.stash = (tgrads, dgrads)
        else:
            od = octree._descriptor(tables, None)
            dd = decoder.c_descriptor(None)
            _abi.check(lib.shine_sdf_diff_fwd(C.byref(od), C.byref(dd), _abi.ptr(coord), _abi.ptr(label), _abi.ptr(weight),
                                              n, scale, loss_scale, _abi.ptr(pred), _abi.ptr(loss),
                                              flags & ~_abi.FLAG_MORTON_ORDERED, stream), "shine_sdf_diff_fwd")
            ctx.stash = None
            if want_grad:
                ctx.save_for_backward(coord, label, weight, *params)
        ctx.mark_non_differentiable(pred)
        return loss, pred

    @staticmethod
    def backward(ctx, dloss, _dpred):
        scale, loss_scale, flags, n, need_t, need_d = ctx.cfg
        octree, decoder = ctx.octree, ctx.decoder
        L = octree.featured_level_num
        if ctx.stash is not None:
            tgrads, dgrads = ctx.stash
            ctx.stash = None
            for g in list(tgrads) + [g for g in dgrads if g is not None]:
                g.mul_(dloss)
        else:
            coord, label, weight, *params = ctx.saved_tensors
            tables, dparams = params[:L], params[L:]
            tgrads = [torch.zeros_like(p) for p in tables]
            dgrads = [torch.zeros_like(p) if (p is not None and any(need_d)) else None for p in dparams]
            od = octree._descriptor(tables, tgrads)
            dd = decoder.c_descriptor(dgrads if any(need_d) else None)
            dl = dloss.detach().float().contiguous()
            _abi.check(_abi.lib().shine_sdf_diff_step(
                C.byref(od), C.byref(dd), _abi.ptr(coord), _abi.ptr(label), _abi.ptr(weight), n, scale, loss_scale,
                _abi.ptr(dl), None, None, flags, _abi.stream_ptr(coord.device)), "shine_sdf_diff_step")
        out_t = [g if need else None for g, need in zip(tgrads, need_t)]
        out_d = [g if need else None for g, need in zip(dgrads, need_d)]
        return (None,) * 9 + tuple(out_t) + tuple(out_d)


def sdf_diff_step(octree: FeatureOctree, decoder: Decoder, coord, sdf_label, weight, scale, l2_loss=True, n_norm=None,
                  single_pass=True, tf32x1=False, return_pred=False, morton_ordered=False):
    """loss (= sdf_diff_loss(decoder.sdf(octree.query_feature(coord)), sdf_label, |weight|, scale, l2_loss), the
    reference's main_loss_type sdf_l2 / sdf_l1) with autograd to `octree.hier_features` and the decoder parameters.

    weight: the per-sample weights (required; their magnitude always multiplies the loss).  scale: config.scale.
    n_norm: the loss's count (defaults to len(coord); pass the GLOBAL batch when sharding points).  The other arguments
    as in `sdf_bce_step`."""
    if coord.requires_grad:
        raise NotImplementedError("gradients w.r.t. coordinates are not part of the fused sm_90a path")
    if weight is None:
        raise ValueError("sdf_diff_step needs the per-sample weight tensor")
    coord, sdf_label, weight = _prep(coord, "coord"), _prep(sdf_label, "sdf_label"), _prep(weight, "weight")
    flags = (_abi.FLAG_LOSS_L2 if l2_loss else 0) | (_abi.FLAG_TF32X1 if tf32x1 else 0) | \
            (_abi.FLAG_MORTON_ORDERED if morton_ordered else 0)
    params = list(octree.hier_features) + list(decoder.fused_params())
    octree._last_coord, octree._hier_idx = coord, []
    loss, pred = _SdfDiff.apply(octree, decoder, coord, sdf_label, weight, float(scale), flags, n_norm, single_pass,
                                *params)
    return (loss, pred) if return_pred else loss


@torch.no_grad()
def sdf_infer(octree: FeatureOctree, decoder: Decoder, coord, mask_level=None, tf32x1=False):
    """decoder.sdf(octree.query_feature(coord)) in one kernel, forward only (the mesher's query, reference
    utils/mesher.py:60-72).  With mask_level (index into hierarchical_indices, 0 = leaf) also returns the
    validity mask the mesher derives from hierarchical_indices[level] >= 0 (utils/mesher.py:82-89)."""
    coord = _prep(coord, "coord")
    n = coord.shape[0]
    pred = torch.empty(n, dtype=torch.float32, device=coord.device)
    mask = torch.empty(n, dtype=torch.uint8, device=coord.device) if mask_level is not None else None
    od = octree._descriptor(None, None)
    dd = decoder.c_descriptor(None)
    _abi.check(_abi.lib().shine_sdf_infer(C.byref(od), C.byref(dd), _abi.ptr(coord), n, _abi.ptr(pred),
                                          _abi.ptr(mask), int(mask_level or 0),
                                          _abi.FLAG_TF32X1 if tf32x1 else 0,
                                          _abi.stream_ptr(coord.device)),
               "shine_sdf_infer")
    return (pred, mask.bool()) if mask is not None else pred
