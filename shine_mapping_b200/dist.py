"""Multi-GPU plumbing: one process per GPU, `torch.distributed` (NCCL over NVLink 5 / NVSwitch; gloo in the CPU
tests).  The reference has no multi-GPU code (SURVEY.md §2.2) — this is new design, two modes:

* "replicated": tables replicated, the POINT BATCH is sharded (`shard_range`); every per-point gradient already
  carries 1/N_global, so one sum all-reduce of the flat gradient buffer (tables + 1 377 decoder floats) yields
  exactly the single-GPU gradient of the global batch.
* "spatial" (BASELINE config 5): every rank owns a Morton-prefix range of ONE map and the samples that fall inside it.
  Corner rows on the faces between ranges exist on every rank that holds a node touching them (`partition.BoundaryPlan`);
  every step their gradients travel with the decoder gradients in ONE exchange ([decoder | boundary rows]: pack ->
  all-reduce -> unpack through `NcclComm`, or the one-kernel peer-memory `P2PExchange`), which sums them in a fixed rank
  order so that the duplicates stay bit-identical.  The other rows are private to their rank (DESIGN.md §6).
"""
from __future__ import annotations

import os

import torch
import torch.distributed as dist


def init_from_env(backend: str | None = None):
    """Initialise from torchrun's env (RANK / WORLD_SIZE / LOCAL_RANK / MASTER_*).  -> (rank, world, local_rank)."""
    world = int(os.environ.get("WORLD_SIZE", "1"))
    rank = int(os.environ.get("RANK", "0"))
    local = int(os.environ.get("LOCAL_RANK", "0"))
    if world > 1 and not dist.is_initialized():
        os.environ.setdefault("MASTER_ADDR", "127.0.0.1")
        if backend is None:
            backend = "nccl" if torch.cuda.is_available() else "gloo"
        if backend == "nccl":
            torch.cuda.set_device(local)
        dist.init_process_group(backend=backend, rank=rank, world_size=world)
    return rank, world, local


class NcclComm:
    """NCCL communicator created and driven through the C ABI (`shine_nccl_comm_create`,
    `shine_allreduce_decoder_grads`): the step's collective does not go through torch.distributed.  The 128-byte unique
    id travels over whatever process group is already up (set-up only)."""

    def __init__(self, rank: int, world: int, device: torch.device, group=None):
        import ctypes as C
        from . import _abi
        self.rank, self.world, self.device = rank, world, torch.device(device)
        lib = _abi.lib()
        uid = (C.c_ubyte * 128)()
        if rank == 0:
            _abi.check(lib.shine_nccl_unique_id(uid), "shine_nccl_unique_id")
        box = [bytes(uid)]
        if world > 1:
            dist.broadcast_object_list(box, src=0, group=group)
        uid = (C.c_ubyte * 128).from_buffer_copy(box[0])
        comm = C.c_void_p()
        _abi.check(lib.shine_nccl_comm_create(uid, world, rank, self.device.index or 0, C.byref(comm)),
                   "shine_nccl_comm_create")
        self._comm, self._lib, self._abi = comm, lib, _abi

    def all_reduce(self, t: torch.Tensor) -> torch.Tensor:
        """In-place sum over all ranks, asynchronous on the current stream."""
        if t.dtype != torch.float32 or not t.is_contiguous() or not t.is_cuda:
            raise ValueError("NcclComm.all_reduce: contiguous fp32 CUDA tensor expected")
        self._abi.check(self._lib.shine_allreduce_decoder_grads(self._comm, self._abi.ptr(t), t.numel(),
                                                                self._abi.stream_ptr(t.device)),
                        "shine_allreduce_decoder_grads")
        return t

    def close(self):
        if self._comm:
            self._lib.shine_nccl_comm_destroy(self._comm)
            self._comm = None


class P2PExchange:
    """The step's exchange as one kernel over NVLink peer memory (`csrc/shine_p2p.cu`): IPC-shared buffers, flags instead of
    a collective library.  `SdfTrainer(p2p=...)` uses it for [decoder | boundary rows] in place of pack -> NCCL -> unpack."""

    def __init__(self, rank: int, world: int, device: torch.device, max_floats: int, group=None):
        import ctypes as C
        from . import _abi
        self.rank, self.world, self.device = rank, world, torch.device(device)
        lib = _abi.lib()
        handle = (C.c_ubyte * 64)()
        ctx = C.c_void_p()
        # every rank walks through the same collectives whatever happens locally, then all agree on the outcome
        rc = lib.shine_p2p_create(world, rank, self.device.index or 0, int(max_floats), handle, C.byref(ctx))
        mine = (rc, bytes(handle))
        everyone = [None] * world
        if world > 1:
            dist.all_gather_object(everyone, mine, group=group)
        else:
            everyone = [mine]
        if rc == 0 and all(r == 0 for r, _ in everyone):
            blob = (C.c_ubyte * (64 * world)).from_buffer_copy(b"".join(h for _, h in everyone))
            rc = lib.shine_p2p_connect(ctx, blob)
        elif rc == 0:
            rc = -1
        ok = torch.tensor([1 if rc == 0 else 0], dtype=torch.int32, device=self.device if dist.is_initialized() and
                          dist.get_backend(group) == "nccl" else "cpu")
        if world > 1:
            dist.all_reduce(ok, op=dist.ReduceOp.MIN, group=group)      # also: every rank has mapped every buffer
        self._ctx, self._lib, self._abi, self._C = ctx, lib, _abi, C
        if int(ok.item()) == 0:
            self.close()
            raise _abi.ShineB200Error(f"peer-memory exchange could not be set up (local code {rc}: "
                                      f"{lib.shine_error_string(rc).decode() if rc > -1000 else rc})")

    def exchange(self, dec_flat: torch.Tensor, plan, table_grads):
        """In place: dec_flat and the plan's rows of table_grads become the sums over all ranks."""
        C = self._C
        if plan is not None and plan.total_floats > plan.dec_floats:
            # the descriptors point at the plan's index tensors and at the tables: rebuilt when either changes (another
            # plan, a plan moved by .to(), tables re-allocated by octree.update)
            key = (tuple(t.data_ptr() for t in table_grads),
                   tuple(t.data_ptr() for ts in (plan.rows, plan.slots, plan.inverse, plan.holders) for t in ts))
            cached = getattr(self, "_desc", None)
            if cached is None or cached[0] != key or cached[-1] is not plan:   # building the ctypes structs costs tens of us
                cached = (key, plan.descriptor(table_grads), plan.inverse_descriptor(), len(table_grads), plan.feature_dim,
                          plan)
                self._desc = cached
            _, desc, inv, levels, fdim, _ = cached
            arg, iarg = C.byref(desc), C.byref(inv)
        else:
            arg, iarg, levels, fdim = None, None, 0, 8
        dec_n = plan.dec_floats if plan is not None else dec_flat.numel()
        self._abi.check(self._lib.shine_p2p_exchange(self._ctx, self._abi.ptr(dec_flat), dec_n, arg, iarg, levels, fdim,
                                                     self._abi.stream_ptr(dec_flat.device)), "shine_p2p_exchange")

    def timeouts(self) -> int:
        n = self._C.c_int32(0)
        self._abi.check(self._lib.shine_p2p_timeouts(self._ctx, self._C.byref(n)), "shine_p2p_timeouts")
        return int(n.value)

    def close(self):
        if getattr(self, "_ctx", None):
            self._lib.shine_p2p_destroy(self._ctx)
            self._ctx = None


def shard_range(n: int, rank: int, world: int) -> tuple[int, int]:
    """Contiguous, balanced slice [begin, end) of an n-point batch for `rank` (sizes differ by at most 1)."""
    base, rem = divmod(n, world)
    begin = rank * base + min(rank, rem)
    return begin, begin + base + (1 if rank < rem else 0)


def all_reduce_sum(t: torch.Tensor, group=None) -> torch.Tensor:
    if dist.is_initialized() and dist.get_world_size(group) > 1:
        dist.all_reduce(t, group=group)
    return t


def max_over_ranks(value: float, device) -> float:
    if dist.is_initialized() and dist.get_world_size() > 1:
        t = torch.tensor([value], dtype=torch.float64, device=device)
        dist.all_reduce(t, op=dist.ReduceOp.MAX)
        return float(t.item())
    return value


def barrier(device=None):
    if dist.is_initialized() and dist.get_world_size() > 1:
        if device is not None and torch.device(device).type == "cuda":
            dist.barrier(device_ids=[torch.device(device).index or 0])
        else:
            dist.barrier()


def gpu_numa_node(local_rank: int) -> int | None:
    """NUMA node of GPU `local_rank` (sysfs numa_node of its PCI device, via NVML's bus id); None when unknown."""
    try:
        import pynvml
        pynvml.nvmlInit()
        vis = os.environ.get("CUDA_VISIBLE_DEVICES")
        index = local_rank
        if vis:
            ids = [v.strip() for v in vis.split(",") if v.strip()]
            if local_rank < len(ids) and ids[local_rank].isdigit():
                index = int(ids[local_rank])
        handle = pynvml.nvmlDeviceGetHandleByIndex(index)
        bus = pynvml.nvmlDeviceGetPciInfo(handle).busId
        bus = bus.decode() if isinstance(bus, bytes) else bus
        bus = bus.lower()
        if len(bus.split(":")[0]) == 8:            # NVML prints an 8-digit PCI domain, sysfs uses 4
            bus = bus[4:]
        with open(f"/sys/bus/pci/devices/{bus}/numa_node") as f:
            node = int(f.read().strip())
        return node if node >= 0 else None
    except Exception:
        return None


def _parse_cpulist(text: str) -> set[int]:
    cpus: set[int] = set()
    for part in text.strip().split(","):
        if not part:
            continue
        lo, _, hi = part.partition("-")
        cpus.update(range(int(lo), int(hi or lo) + 1))
    return cpus


def pin_to_gpu_numa_node(local_rank: int) -> dict:
    """Bind this process (and what it allocates afterwards: pinned staging buffers are first-touched locally) to the
    CPUs of the NUMA node its GPU hangs off.  Eight ranks feeding eight GPUs from one socket halve the host->device
    rate of the far GPUs (r01: e2e efficiency 0.61 at N=8).  No-op when the topology cannot be read."""
    node = gpu_numa_node(local_rank)
    info = {"numa_node": node, "cpus": None}
    if node is None or not hasattr(os, "sched_setaffinity"):
        return info
    try:
        with open(f"/sys/devices/system/node/node{node}/cpulist") as f:
            cpus = _parse_cpulist(f.read())
        allowed = os.sched_getaffinity(0)
        cpus = cpus & allowed
        if len(cpus) >= 4:                      # never squeeze a rank onto a sliver of a cgroup-restricted node
            os.sched_setaffinity(0, cpus)
            info["cpus"] = len(cpus)
    except Exception:
        pass
    return info
