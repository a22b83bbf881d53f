"""`SdfTrainer` — the training-step engine behind the `shine_batch.py`-equivalent loop (reference
shine_batch.py:105-210) without autograd in the way.

One flat fp32 gradient buffer holds every table level and the decoder (each segment 16-byte aligned), so that
  * zeroing the gradients is ONE memset (or free: fused into the Adam kernel),
  * the data-parallel exchange is ONE NCCL all-reduce over NVLink (decoder 1 377 floats + table rows),
  * `param.grad` of every parameter is a view into it, so stock torch optimizers still work.
`forward_backward()` = one `shine_sdf_bce_step` launch (`shine_sdf_diff_step` with main_loss_type sdf_l1 / sdf_l2);
`optimizer_step()` = one `shine_adam_step` launch with the
reference's grouping (utils/tools.py:57-83: Adam betas (0.9, 0.99), eps 1e-15, weight decay on the decoder only,
per-level lr scaled leaf -> coarse by lr_level_reduce_ratio).
"""
from __future__ import annotations

import ctypes as C
import os

import torch

from . import _abi
from .config import SHINEConfig
from .decoder import Decoder
from .feature_octree import FeatureOctree


def _align4(n: int) -> int:
    return (n + 3) & ~3


def diff_loss_flags(main_loss_type: str):
    """main_loss_type -> None for sdf_bce, else the loss bit of the shine_sdf_diff_* calls (sdf_l1: 0, sdf_l2:
    FLAG_LOSS_L2; shine_batch.py:176-179)."""
    kinds = {"sdf_bce": None, "sdf_l1": 0, "sdf_l2": _abi.FLAG_LOSS_L2}
    if main_loss_type not in kinds:
        raise NotImplementedError(f"main_loss_type {main_loss_type!r}: the trainer has {sorted(kinds)}")
    return kinds[main_loss_type]


class SdfTrainer:
    def __init__(self, config: SHINEConfig, octree: FeatureOctree, decoder: Decoder, process_group=None,
                 tf32x1: bool = False, shard_mode: str = "replicated", boundary=None, comm=None, p2p=None,
                 morton_ordered: bool = False, main_loss_type: str | None = None):
        """main_loss_type: the loss every step trains, None = config.main_loss_type (the incremental loop passes
        "sdf_bce": the reference's shine_incre.py:150 trains it whatever the config says).
        shard_mode (multi-GPU, see dist.py / partition.py): "replicated" = every rank holds the whole table and a
        slice of the point batch -> all-reduce the whole flat gradient; "spatial" = every rank owns a Morton-prefix
        range of ONE map and the samples inside it (BASELINE config 5) -> ONE all-reduce over
        [decoder gradients | gradients of the corner rows shared with other ranks] (`boundary`: partition.BoundaryPlan).
        comm: dist.NcclComm (the C-ABI collective); None = torch.distributed (gloo in the CPU tests)."""
        if shard_mode not in ("replicated", "spatial"):
            raise ValueError(shard_mode)
        self.config, self.octree, self.decoder = config, octree, decoder
        self.shard_mode = shard_mode
        self.boundary, self.comm = boundary, comm
        self.p2p = p2p              # dist.P2PExchange: the spatial exchange as one NVLink peer-memory kernel
        # gradient replicas for small hot levels (see FeatureOctree._replicas_for); on by default for big batches
        self.use_replicas = os.environ.get("SHINE_FUSED_REPLICAS", "1") != "0"
        self.grouped_replicas = os.environ.get("SHINE_GROUPED_REPLICAS", "0") != "0"   # replicas for ordered batches too (A/B)
        self.group = process_group
        self.morton_ordered = bool(morton_ordered)   # default for every step: batches come from a Morton-sorted SamplePool
        self.tf32x1 = tf32x1
        self.lr = config.lr
        self.step_count = 0
        self._sig = None
        self.sigma = config.sigma_sigmoid
        self.main_loss_type = config.main_loss_type if main_loss_type is None else main_loss_type
        self._diff = diff_loss_flags(self.main_loss_type)   # None: sdf_bce
        self._sync()

    # ---- flat buffers --------------------------------------------------------------------------------------

    def _params(self):
        tables = list(self.octree.hier_features)
        dec = [p for p in self.decoder.fused_params()]
        return tables, dec

    def _sync(self):
        """(Re)bind the flat grad / Adam-state buffers after `octree.update()` replaced the Parameters
        (reference model/feature_octree.py:156; the reference rebuilds its optimizer too, shine_incre.py:108-109)."""
        tables, dec = self._params()
        sig = tuple((p.data_ptr(), tuple(p.shape)) for p in tables + [p for p in dec if p is not None])
        if sig == self._sig:
            return
        dev = tables[0].device
        _abi.require_cuda(tables[0], "SdfTrainer")
        sizes = [p.numel() for p in tables] + [p.numel() if p is not None else 0 for p in dec]
        offs, total = [], 0
        for s in sizes:
            offs.append(total)
            total += _align4(s)
        # after the decoder segment: the boundary-row exchange slots of a spatial partition (so that ONE in-place
        # all-reduce covers [decoder | boundary]), then 4 floats for the loss accumulator: zero_grad() clears all of it
        nb = 0
        if self.boundary is not None:
            dec_seg = total - offs[len(tables)]
            if self.boundary.dec_floats != dec_seg:
                raise ValueError(f"BoundaryPlan was built for a {self.boundary.dec_floats}-float decoder segment, "
                                 f"this trainer's is {dec_seg}")
            nb = self.boundary.total_floats - self.boundary.dec_floats
        self._flat_all = torch.zeros(total + nb + 4, dtype=torch.float32, device=dev)
        self.flat_grad = self._flat_all[:total]
        self.exchange = self._flat_all[offs[len(tables)]:total + nb]     # [decoder | boundary rows]
        self.exp_avg = torch.zeros(total, dtype=torch.float32, device=dev)
        self.exp_avg_sq = torch.zeros(total, dtype=torch.float32, device=dev)
        self.step_count = 0   # fresh Adam state, like a rebuilt torch optimizer
        self.adam_state = torch.zeros(3, dtype=torch.int32, device=dev)   # {step, bc1, bc2_sqrt} for graph replay
        self._device_steps = 0   # what adam_state[0] holds (host-step Adam advances step_count alone)
        views = []
        for p, o, s in zip(tables + dec, offs, sizes):
            views.append(self.flat_grad[o:o + s].view(p.shape) if p is not None else None)
        L = len(tables)
        self.table_grads, self.dec_grads = views[:L], views[L:]
        self.dec_flat = self.flat_grad[offs[L]:]          # contiguous decoder segment (1 377 floats + padding)
        self._offs, self._sizes = offs, sizes
        self._dec_trainable = any(p is not None and p.requires_grad for p in dec)
        for p, g in zip(tables + dec, views):
            if p is not None and p.requires_grad:
                p.grad = g
        self._sig = sig
        self.loss = self._flat_all[total + nb:total + nb + 1].view(())
        self._loss_clean = True

    def zero_grad(self):
        self._flat_all.zero_()       # gradients AND the loss accumulator: one memset
        self._loss_clean = True

    # ---- the hot path --------------------------------------------------------------------------------------

    def forward_backward(self, coord, sdf_label, weight=None, n_norm=None, pred_out=None, accumulate_loss=False,
                         weighted=None, mid_event=None, morton_ordered=None):
        """One fused launch: loss value (device scalar, accumulated into self.loss which is zeroed here) and
        gradients accumulated into the flat buffer.  Caller zeroes grads (zero_grad / fused in optimizer_step).
        weighted: None = config.loss_weight_on (the loop, shine_batch.py:174); False = unweighted BCE whatever the
        config says (what cal_feature_importance uses, utils/incre_learning.py:33).
        morton_ordered: the batch comes in Morton order of its coordinates (`DataPool.get_batch(..., ordered=True)`):
        the kernel then sums the table gradients per run of equal node before the atomics (same result up to fp32
        summation order; a hint only, any batch is handled correctly).  None = the trainer's `morton_ordered` default."""
        self._sync()
        cfg = self.config
        n = coord.shape[0]
        diff = self._diff
        if diff is not None and weight is None:
            raise ValueError(f"main_loss_type {self.main_loss_type} needs the per-sample weight tensor")
        weighted = bool(cfg.loss_weight_on) if weighted is None else bool(weighted)
        if weighted and weight is None:
            raise ValueError("loss_weight_on needs the per-sample weight tensor")
        flags = (_abi.FLAG_REDUCTION_SUM if cfg.loss_reduction == "sum" else 0) | \
                (_abi.FLAG_WEIGHTED if weighted else 0) | (_abi.FLAG_TF32X1 if self.tf32x1 else 0) | \
                (_abi.FLAG_MORTON_ORDERED if (self.morton_ordered if morton_ordered is None else morton_ordered) else 0)
        scale = 1.0 if cfg.loss_reduction == "sum" else 1.0 / float(n_norm if n_norm else n)
        # gradient replicas spread same-row atomics of unordered batches; the grouped scatter of ordered batches issues one
        # red per run and row, so it goes straight to the gradient table (and there is no fold kernel)
        replicas = self.use_replicas and (self.grouped_replicas or not (flags & _abi.FLAG_MORTON_ORDERED))
        od = self.octree._descriptor(None, self.table_grads, n_points=n if replicas else 0)
        dd = self.decoder.c_descriptor(self.dec_grads if self._dec_trainable else None)
        if not accumulate_loss and not self._loss_clean:
            self.loss.zero_()
        self._loss_clean = False
        if diff is None:
            _abi.check(_abi.lib().shine_sdf_bce_step(
                C.byref(od), C.byref(dd), _abi.ptr(coord), _abi.ptr(sdf_label),
                _abi.ptr(weight) if weighted else None, n, float(self.sigma), scale, None,
                _abi.ptr(pred_out), _abi.ptr(self.loss), flags, _abi.stream_ptr(coord.device)), "shine_sdf_bce_step")
        else:   # sdf_diff_loss: always weighted, divided by the batch size whatever loss_reduction says
            flags = diff | (flags & (_abi.FLAG_TF32X1 | _abi.FLAG_MORTON_ORDERED))
            _abi.check(_abi.lib().shine_sdf_diff_step(
                C.byref(od), C.byref(dd), _abi.ptr(coord), _abi.ptr(sdf_label), _abi.ptr(weight), n, float(cfg.scale),
                1.0 / float(n_norm if n_norm else n), None, _abi.ptr(pred_out), _abi.ptr(self.loss), flags,
                _abi.stream_ptr(coord.device)), "shine_sdf_diff_step")
        if mid_event is not None:          # lets a profiler time the fused kernel and the replica fold separately
            mid_event.record()
        if replicas:
            self.octree._reduce_replicas(od, coord.device)
        return self.loss

    def forward_backward_eikonal(self, coord, sdf_label, weight, n_norm=None, pred_out=None, grad_out=None,
                                 n_surface=None):
        """The step with `ekional_loss_on` (reference shine_batch.py:119-142,172-185,208-209) as ONE launch
        (`shine_sdf_bce_eikonal_step`): BCE + weight_e * mean over surface samples of (1 - |sigma d pred/d coord|)^2,
        gradients of both terms accumulated into the flat buffer.  -> (bce loss, eikonal mean) device scalars;
        the loop's total loss is bce + config.weight_e * eikonal.  With main_loss_type sdf_l1 / sdf_l2 the first term is
        sdf_diff_loss (`shine_sdf_diff_eikonal_step`) and the first scalar its value.
        n_surface: denominator of the eikonal mean, the analogue of n_norm: the number of surface samples (weight > 0) in
        the GLOBAL batch when this call sees one part of it.  None = counted on the device from this batch and, when the
        trainer runs on several ranks, summed over them, so that the per-rank eikonal values and gradients add up to those
        of the global batch.  A batch without surface sample contributes 0 (not the NaN of torch's mean of nothing)."""
        self._sync()
        cfg = self.config
        n = coord.shape[0]
        dev = coord.device
        weighted = bool(cfg.loss_weight_on)
        flags = (_abi.FLAG_REDUCTION_SUM if cfg.loss_reduction == "sum" else 0) | (_abi.FLAG_WEIGHTED if weighted else 0)
        scale = 1.0 if cfg.loss_reduction == "sum" else 1.0 / float(n_norm if n_norm else n)
        aux = getattr(self, "_eik_aux", None)
        if aux is None or aux[0].device != dev:
            aux = (torch.zeros(1, dtype=torch.int32, device=dev), torch.zeros(1, dtype=torch.float32, device=dev))
            self._eik_aux = aux
        count, eik = aux
        eik.zero_()
        if not self._loss_clean:
            self.loss.zero_()
        self._loss_clean = False
        od = self.octree._descriptor(None, self.table_grads)
        dd = self.decoder.c_descriptor(self.dec_grads if self._dec_trainable else None)
        lib, st = _abi.lib(), _abi.stream_ptr(dev)
        if n_surface is not None:
            count.fill_(int(n_surface))
        else:
            count.zero_()
            _abi.check(lib.shine_count_positive(_abi.ptr(weight), n, _abi.ptr(count), st), "shine_count_positive")
            if self._world() > 1:
                total = count.float()                 # exact below 2^24 samples; the collectives here sum fp32
                self._all_reduce(total)
                count.copy_(total.round())
        diff = self._diff
        if diff is None:
            _abi.check(lib.shine_sdf_bce_eikonal_step(
                C.byref(od), C.byref(dd), _abi.ptr(coord), _abi.ptr(sdf_label), _abi.ptr(weight), n, float(self.sigma), scale,
                float(cfg.weight_e), _abi.ptr(count), _abi.ptr(pred_out), _abi.ptr(grad_out), _abi.ptr(self.loss),
                _abi.ptr(eik), flags, st), "shine_sdf_bce_eikonal_step")
        else:
            _abi.check(lib.shine_sdf_diff_eikonal_step(
                C.byref(od), C.byref(dd), _abi.ptr(coord), _abi.ptr(sdf_label), _abi.ptr(weight), n, float(cfg.scale),
                float(self.sigma), 1.0 / float(n_norm if n_norm else n), float(cfg.weight_e), _abi.ptr(count),
                _abi.ptr(pred_out), _abi.ptr(grad_out), _abi.ptr(self.loss), _abi.ptr(eik), diff, st),
                "shine_sdf_diff_eikonal_step")
        return self.loss, eik.view(())

    def _all_reduce(self, buf):
        if self.comm is not None:
            self.comm.all_reduce(buf)
        elif torch.distributed.is_available() and torch.distributed.is_initialized():
            torch.distributed.all_reduce(buf, group=self.group)

    def _world(self) -> int:
        if self.comm is not None:
            return self.comm.world
        if torch.distributed.is_available() and torch.distributed.is_initialized():
            return torch.distributed.get_world_size(self.group)
        return 1

    def all_reduce_grads(self):
        """The step's exchange, ONE sum collective (the 1/N_global is already in the per-point gradient scale):
        replicated -> the whole flat gradient; spatial -> [decoder | rows shared with other ranks]."""
        if self.p2p is not None and self.shard_mode == "spatial":
            if self.p2p.world > 1:
                self.p2p.exchange(self.dec_flat, self.boundary, self.table_grads)
            return
        if self._world() <= 1:
            return
        if self.shard_mode == "replicated":
            self._all_reduce(self.flat_grad)
            return
        if self.boundary is not None and self.boundary.total_floats > self.boundary.dec_floats:
            self.boundary.pack(self.table_grads, self.exchange)
            self._all_reduce(self.exchange)
            self.boundary.unpack(self.table_grads, self.exchange)
        elif self._dec_trainable:
            self._all_reduce(self.dec_flat)

    def optimizer_step(self, zero_grad: bool = True, device_step: bool = False):
        """Dense Adam with the reference's groups (utils/tools.py:57-83) as one multi-tensor launch.  With
        device_step the step number / bias corrections live on the device (CUDA-graph replayable)."""
        cfg = self.config
        tables, dec = self._params()
        capturing = torch.cuda.is_current_stream_capturing()
        if not capturing:             # a captured call executes nothing: whoever replays the graph counts its step
            if device_step:
                self._align_device_step()
                self._device_steps += 1
            self.step_count += 1
        entries = []
        L = len(tables)

        def add(p, idx, lr, wd):
            o, s = self._offs[idx], self._sizes[idx]
            t = _abi.ShineAdamTensor()
            t.param, t.grad = p.data_ptr(), self.flat_grad.data_ptr() + 4 * o
            t.exp_avg, t.exp_avg_sq = self.exp_avg.data_ptr() + 4 * o, self.exp_avg_sq.data_ptr() + 4 * o
            t.numel, t.lr, t.weight_decay = s, lr, wd
            entries.append(t)

        for j, p in enumerate(dec):
            if p is not None and p.requires_grad:
                add(p, L + j, self.lr, cfg.weight_decay)
        lr_cur = self.lr
        for i in range(L):   # leaf first, lr shrinking towards coarse levels (utils/tools.py:68-72)
            k = L - i - 1
            if tables[k].requires_grad:
                add(tables[k], k, lr_cur, 0.0)
            lr_cur *= cfg.lr_level_reduce_ratio
        arr = (_abi.ShineAdamTensor * len(entries))(*entries)
        if device_step:
            _abi.check(_abi.lib().shine_adam_step_dev(arr, len(entries), 0.9, 0.99, float(cfg.adam_eps),
                                                      _abi.ptr(self.adam_state), 1 if zero_grad else 0,
                                                      _abi.stream_ptr(tables[0].device)), "shine_adam_step_dev")
            return
        _abi.check(_abi.lib().shine_adam_step(arr, len(entries), 0.9, 0.99, float(cfg.adam_eps), self.step_count,
                                              1 if zero_grad else 0, _abi.stream_ptr(tables[0].device)),
                   "shine_adam_step")

    def _align_device_step(self):
        """The host step_count is the single source of truth.  Host-step Adam advances it alone, so before a device-step
        Adam runs (eagerly or in a replayed graph) the device counter is set to it (the bump kernel recomputes the bias
        corrections from the step number on every call).  While only device-step Adam runs, as in the graphed loop,
        the two agree and this launches nothing."""
        if self._device_steps != self.step_count:
            self.adam_state[0] = self.step_count
            self._device_steps = self.step_count

    def _replay_with_adam(self, graph):
        """Replay a CUDA graph that holds one device-step Adam, counted like an eager call."""
        self._align_device_step()
        graph.replay()
        self._device_steps += 1
        self.step_count += 1

    def train_step(self, coord, sdf_label, weight=None, n_norm=None):
        """shine_batch.py:123-210: fwd + loss + bwd (+ all-reduce when data parallel) + Adam."""
        loss = self.forward_backward(coord, sdf_label, weight, n_norm)
        self.all_reduce_grads()
        self.optimizer_step(zero_grad=True)
        return loss

    # ---- host-buffer entry (the reference-facing call with HOST memory) -----------------------------------------

    def _host_step_body(self, coord_h, label_h, weight_h, n, chunks, weighted, optimizer):
        dev = self.flat_grad.device
        coord_d, label_d, weight_d = (t[:n] for t in self._h2d)
        main = torch.cuda.current_stream(dev)
        bounds = [(n * k // chunks, n * (k + 1) // chunks) for k in range(chunks)]
        self._copy_stream.wait_stream(main)          # previous consumers of the staging buffers are done
        events = []
        with torch.cuda.stream(self._copy_stream):
            for b, e in bounds:
                coord_d[b:e].copy_(coord_h[b:e], non_blocking=True)
                label_d[b:e].copy_(label_h[b:e], non_blocking=True)
                if weighted:
                    weight_d[b:e].copy_(weight_h[b:e], non_blocking=True)
                ev = torch.cuda.Event()
                ev.record(self._copy_stream)
                events.append(ev)
        self.zero_grad()
        for (b, e), ev in zip(bounds, events):
            main.wait_event(ev)
            if e > b:
                self.forward_backward(coord_d[b:e], label_d[b:e], weight_d[b:e] if weighted else None, n_norm=n,
                                      accumulate_loss=True)
        if optimizer:
            self.all_reduce_grads()
            self.optimizer_step(zero_grad=False, device_step=True)

    def _uses_weight(self) -> bool:
        """Whether the steps read the per-sample weights: sdf_bce with loss_weight_on, sdf_l1 / sdf_l2 always."""
        return bool(self.config.loss_weight_on) or self._diff is not None

    # ---- pipelined host-buffer entry ------------------------------------------------------------------------

    class StepGraph:
        """One whole step on device tensors as a CUDA graph (see `capture_step`)."""

        def __init__(self, trainer, graph, launches, optimizer):
            self.trainer, self.graph, self.launches, self.optimizer = trainer, graph, launches, optimizer

        def replay(self):
            if self.optimizer:
                self.trainer._replay_with_adam(self.graph)
            else:
                self.graph.replay()
            self.trainer._loss_clean = False
            _abi.LAUNCHES["count"] += self.launches       # the replayed kernels are this library's launches too
            return self.trainer.loss

    def capture_step(self, coord, sdf_label, weight=None, n_norm=None, exchange: bool = True, optimizer: bool = False):
        """{zero gradients -> fused fwd + loss + bwd -> the multi-GPU exchange (-> Adam)} on DEVICE tensors, captured once
        as a CUDA graph: `replay()` re-runs it on whatever the tensors hold then, without the host in the loop (the
        peer-memory exchange keeps its step number on the device for this).  One real step runs as warm-up before the
        capture: with several ranks every rank has to call this the same number of times."""
        self._sync()
        dev = coord.device

        def body():
            self.zero_grad()
            self.forward_backward(coord, sdf_label, weight, n_norm=n_norm)
            if exchange:
                self.all_reduce_grads()
            if optimizer:
                self.optimizer_step(zero_grad=False, device_step=True)

        side = torch.cuda.Stream(device=dev)
        side.wait_stream(torch.cuda.current_stream(dev))
        with torch.cuda.stream(side):
            body()
        torch.cuda.current_stream(dev).wait_stream(side)
        torch.cuda.synchronize(dev)
        graph = torch.cuda.CUDAGraph()
        before = _abi.LAUNCHES["count"]
        with torch.cuda.graph(graph):
            body()
        launches = _abi.LAUNCHES["count"] - before
        _abi.LAUNCHES["count"] = before                  # capturing launched nothing
        return SdfTrainer.StepGraph(self, graph, launches, optimizer)

    class HostStepHandle:
        """Result of `submit_host_step`: `.result()` blocks until that step's loss is on the host."""

        def __init__(self, event, loss_host):
            self._event, self._loss_host = event, loss_host

        def result(self) -> float:
            self._event.synchronize()
            return float(self._loss_host.item())

    def submit_host_step(self, coord_h, label_h, weight_h=None, n_norm=None, optimizer: bool = False,
                         exchange: bool = False):
        """Asynchronous variant of `step_from_host` for loops that do not need step k's loss before building step k+1
        (the reference loop reads the loss only for logging, shine_batch.py:215-226).  Two device staging slots: the
        host->device copy of this batch runs on a copy stream while the previous step's kernels run on the main stream;
        the loss is copied to a pinned host scalar and an event tells when it is there.  Every step still copies its
        own inputs and reads its own result; only the waiting is overlapped."""
        dev = self.flat_grad.device
        n = coord_h.shape[0]
        weighted = self._uses_weight() and weight_h is not None
        self._sync()
        pl = getattr(self, "_pipe", None)
        if pl is None or pl["cap"] < n or pl["sig"] != self._sig:
            pl = {"cap": n, "sig": self._sig, "k": 0, "copy": torch.cuda.Stream(device=dev),
                  "copy2": torch.cuda.Stream(device=dev),
                  "slots": [{"coord": torch.empty(n, 3, device=dev), "label": torch.empty(n, device=dev),
                             "weight": torch.empty(n, device=dev), "free": None,
                             "loss_h": torch.zeros(1).pin_memory()} for _ in range(2)]}
            self._pipe = pl
        slot = pl["slots"][pl["k"] & 1]
        pl["k"] += 1
        main, copy, copy2 = torch.cuda.current_stream(dev), pl["copy"], pl["copy2"]
        if slot["free"] is not None:
            copy.wait_event(slot["free"])            # the kernels that read this slot two steps ago are done
            copy2.wait_event(slot["free"])
        # two copy streams: the coordinates (3/4 of the bytes) are split in halves that travel concurrently
        half = (n // 2) & ~63
        with torch.cuda.stream(copy):
            slot["coord"][:half].copy_(coord_h[:half], non_blocking=True)
            slot["label"][:n].copy_(label_h, non_blocking=True)
            copied = torch.cuda.Event()
            copied.record(copy)
        with torch.cuda.stream(copy2):
            slot["coord"][half:n].copy_(coord_h[half:], non_blocking=True)
            if weighted:
                slot["weight"][:n].copy_(weight_h, non_blocking=True)
            copied2 = torch.cuda.Event()
            copied2.record(copy2)
        main.wait_event(copied2)
        main.wait_event(copied)
        self.zero_grad()
        self.forward_backward(slot["coord"][:n], slot["label"][:n], slot["weight"][:n] if weighted else None,
                              n_norm=n_norm or n)
        if exchange or optimizer:
            self.all_reduce_grads()
        slot["loss_h"].copy_(self.loss.view(1), non_blocking=True)
        done = torch.cuda.Event()
        done.record(main)
        slot["free"] = done
        if optimizer:
            self.optimizer_step(zero_grad=False)
        return SdfTrainer.HostStepHandle(done, slot["loss_h"])

    def step_from_host(self, coord_h, label_h, weight_h=None, optimizer: bool = False, chunks: int = 0,
                       use_graph: bool = True) -> float:
        """coord/label(/weight) are PINNED host tensors.  The batch is cut into `chunks` slices: slice k+1 is copied
        host->device on a copy stream while the fused kernel runs on slice k (gradients and the loss accumulate across
        slices; the per-point scale uses the whole batch), then the loss is read back.  With use_graph the whole
        sequence (copies, memset, kernels) is captured once per (host buffers, size) as a CUDA graph and replayed, which
        removes the host launch overhead (measured: 0.65 -> 0.48 ms for 776 k points; 2 chunks is the optimum, finer chunking
        pays a fixed ~20 us of kernel prologue/epilogue per slice)."""
        dev = self.flat_grad.device
        n = coord_h.shape[0]
        weighted = self._uses_weight() and weight_h is not None
        self._sync()
        if getattr(self, "_h2d", None) is None or self._h2d[0].shape[0] < n:
            self._h2d = (torch.empty(n, 3, device=dev), torch.empty(n, device=dev), torch.empty(n, device=dev))
            self._copy_stream = torch.cuda.Stream(device=dev)
            self._host_graphs = {}
        graphable = use_graph and coord_h.is_pinned() and label_h.is_pinned() and not (
            optimizer and torch.distributed.is_initialized() and torch.distributed.get_world_size() > 1)
        if chunks <= 0:
            chunks = 2
        chunks = max(1, min(chunks, (n + 32767) // 32768))
        if not graphable:
            self._host_step_body(coord_h, label_h, weight_h, n, chunks, weighted, optimizer)
            return float(self.loss.item())
        key = (coord_h.data_ptr(), label_h.data_ptr(), weight_h.data_ptr() if weighted else 0, n, chunks, optimizer,
               self._sig, self.lr)
        graph = self._host_graphs.get(key)
        if graph is None:
            if len(self._host_graphs) >= 16:
                self._host_graphs.clear()
            self._host_step_body(coord_h, label_h, weight_h, n, chunks, weighted, False)   # warm-up outside capture
            torch.cuda.synchronize(dev)
            graph = torch.cuda.CUDAGraph()
            with torch.cuda.graph(graph):
                self._host_step_body(coord_h, label_h, weight_h, n, chunks, weighted, optimizer)
            self._host_graphs[key] = graph
        if optimizer:
            self._replay_with_adam(graph)
        else:
            graph.replay()
        return float(self.loss.item())
