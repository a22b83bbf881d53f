#!/usr/bin/env python
"""Experiment: the fused step reading its batch straight from PINNED HOST memory (unified addressing: the kernel's
cp.async input prefetch pulls coord/label over PCIe while it computes) against staged copies.  Prints ms per step."""
import ctypes as C, os, statistics, sys, time
import torch
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import bench
from shine_mapping_b200 import SdfTrainer, _abi

dev = torch.device("cuda", 0)
cfg, octree, decoder, pool = bench.build_workload(str(dev), 0, 1, 2048)
n = len(pool)
tr = SdfTrainer(cfg, octree, decoder)
gen = torch.Generator(device=dev).manual_seed(1)
host = [tuple(t.cpu().pin_memory() for t in pool.get_batch(n, gen)[:2]) for _ in range(12)]
lib, st = _abi.lib(), _abi.stream_ptr(dev)

def zero_copy_step(c_h, l_h):
    tr.zero_grad()
    od = tr.octree._descriptor(None, tr.table_grads, n_points=n)
    dd = tr.decoder.c_descriptor(tr.dec_grads)
    _abi.check(lib.shine_sdf_step(C.byref(od), C.byref(dd), C.c_void_p(c_h.data_ptr()), C.c_void_p(l_h.data_ptr()), None, n,
                                  float(tr.sigma), 1.0, 1.0 / n, None, None, _abi.ptr(tr.loss), 0, st), "step")
    tr.octree._reduce_replicas(od, dev)
    return float(tr.loss.item())

def timeit(fn, name, reps=20):
    for i in range(4): fn(i)
    torch.cuda.synchronize(); t0 = time.perf_counter()
    for i in range(reps): fn(i)
    torch.cuda.synchronize(); ms = (time.perf_counter() - t0) / reps * 1e3
    print(f"{name:44s} {ms:8.4f} ms/step  {n / ms / 1e6:8.1f} Mpts/s", flush=True)

timeit(lambda i: zero_copy_step(*host[i % 12]), "zero-copy (kernel reads pinned host)")
timeit(lambda i: tr.step_from_host(*host[i % 4]), "step_from_host (graph, 2 chunks)")
def pipe(reps):
    pend = None
    for i in range(reps):
        h = tr.submit_host_step(*host[i % 12])
        if pend is not None: pend.result()
        pend = h
    pend.result()
pipe(4); torch.cuda.synchronize(); t0 = time.perf_counter(); pipe(40); torch.cuda.synchronize()
ms = (time.perf_counter() - t0) / 40 * 1e3
print(f"{'submit_host_step pipelined depth 2':44s} {ms:8.4f} ms/step  {n / ms / 1e6:8.1f} Mpts/s")
# raw pinned H2D rate for reference
buf = torch.empty(n, 3, device=dev)
torch.cuda.synchronize(); t0 = time.perf_counter()
for i in range(20): buf.copy_(host[i % 12][0], non_blocking=True)
torch.cuda.synchronize(); dt = (time.perf_counter() - t0) / 20
print(f"raw H2D coord copy: {n * 12 / dt / 1e9:.1f} GB/s")
