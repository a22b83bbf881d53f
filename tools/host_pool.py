#!/usr/bin/env python
"""Measure the batch-mode sample pool in pinned host memory (synth.HostSamplePool) against the device pool and the
reference's CPU path, on a pool of >= 10^8 samples (the C2 scan's samples, repeated).

    python tools/host_pool.py [--samples 100000000] [--out DIR]

get_batch at bs 4 096 / 65 536 / 1 048 576 for
  host    HostSamplePool: torch.randint on the GPU + one gather launch reading 32-byte records over PCIe
  device  SamplePool: torch.randint + three index kernels on device memory
  ref     the reference's CPU pools (dataset/lidar_dataset.py:431-448): CPU randint, CPU indexing, .to(cuda)
and one graphed batch_loop iteration (get_batch -> fused step -> Adam) at bs 4 096 on the host and the device pool.
Times are host clocks around work that ends in a device synchronise, median of 3 rounds that alternate the cases.  The
gather rate counts useful bytes (coord, label, weight: 20 B per sample) over the whole get_batch time.
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import subprocess
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.dont_write_bytecode = True

USEFUL_BYTES = 20
BATCH_SIZES = (4096, 65536, 1048576)


def gpu_info():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
    except (OSError, subprocess.SubprocessError, IndexError):
        q = torch.cuda.get_device_name(0) + ", power limit unknown"
    return q


def timed(fn, reps, dev):
    torch.cuda.synchronize(dev)
    t0 = time.perf_counter()
    for _ in range(reps):
        fn()
    torch.cuda.synchronize(dev)
    return (time.perf_counter() - t0) / reps


def main(argv=None):
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--samples", type=int, default=100_000_000)
    ap.add_argument("--out", default=None, help="directory for host_pool.json")
    args = ap.parse_args(argv)
    import bench
    from shine_mapping_b200 import SdfTrainer, synth
    from shine_mapping_b200.batch_loop import _GraphedIteration
    assert torch.cuda.is_available(), "tools/host_pool.py measures on the GPU"
    dev = torch.device("cuda", 0)
    info = gpu_info()
    print("GPU:", info, flush=True)

    cfg, octree, decoder, scan = bench.build_workload(str(dev), 0, 1, 2048)
    c, l, w = scan.coord_pool, scan.sdf_label_pool, scan.weight_pool
    reps = -(-args.samples // len(scan))
    n = reps * len(scan)
    host = synth.HostSamplePool(dev)
    t0 = time.perf_counter()
    for _ in range(reps):
        host.append(c, l, w)                       # one launch per frame
    torch.cuda.synchronize(dev)
    fill_s = time.perf_counter() - t0
    device_pool = synth.SamplePool(dev)
    device_pool.coord_pool, device_pool.sdf_label_pool, device_pool.weight_pool = c.repeat(reps, 1), l.repeat(reps), w.repeat(reps)
    cpu_c, cpu_l, cpu_w = device_pool.coord_pool.cpu(), device_pool.sdf_label_pool.cpu(), device_pool.weight_pool.cpu()
    print(f"pool: {n} samples ({reps} x {len(scan)}); host pool {len(host._chunks)} chunks of {host.chunk_records} records "
          f"= {len(host._chunks) * host.chunk_records * 32 / 2**30:.2f} GiB pinned, filled in {fill_s:.2f} s "
          f"({n * USEFUL_BYTES / fill_s / 1e9:.2f} GB/s of samples)", flush=True)

    def ref_batch(bs):
        index = torch.randint(0, n, (bs,))        # lidar_dataset.py:433-441 with pool_device = "cpu"
        return cpu_c[index, :].to(dev), cpu_l[index].to(dev), cpu_w[index].to(dev)

    cases = {"host": lambda bs: host.get_batch(bs), "device": lambda bs: device_pool.get_batch(bs), "ref": ref_batch}
    results = {"gpu": info, "samples": n, "get_batch": {}, "graphed_iteration": {}}
    for bs in BATCH_SIZES:
        count = max(5, min(400, (1 << 24) // bs * 4))
        for fn in cases.values():
            for _ in range(3):
                fn(bs)
        rounds = {k: [] for k in cases}
        for _ in range(3):
            for k, fn in cases.items():
                r = count if k != "ref" else max(3, count // 8)
                rounds[k].append(timed(lambda: fn(bs), r, dev))
        row = {}
        for k, ts in rounds.items():
            s = statistics.median(ts)
            row[k] = {"ms": s * 1e3, "spread_ms": (max(ts) - min(ts)) * 1e3, "GB_per_s_useful": bs * USEFUL_BYTES / s / 1e9,
                      "Msamples_per_s": bs / s / 1e6}
            print(f"get_batch bs {bs:8d} {k:6s} {s * 1e3:9.4f} ms (spread {row[k]['spread_ms']:.4f})  "
                  f"{row[k]['Msamples_per_s']:9.1f} Msamples/s  {row[k]['GB_per_s_useful']:7.2f} GB/s useful", flush=True)
        results["get_batch"][bs] = row

    # gather kernel alone (indices drawn beforehand): the PCIe read rate of random 32-byte records
    for bs in BATCH_SIZES:
        idx = torch.randint(0, n, (bs,), device=dev)
        for _ in range(3):
            host.gather(idx)
        count = max(5, min(400, (1 << 24) // bs * 4))
        s = statistics.median(timed(lambda: host.gather(idx), count, dev) for _ in range(3))
        results["get_batch"][bs]["host_gather_only"] = {"ms": s * 1e3, "GB_per_s_useful": bs * USEFUL_BYTES / s / 1e9,
                                                        "GB_per_s_records": bs * 32 / s / 1e9}
        print(f"gather only bs {bs:8d}        {s * 1e3:9.4f} ms  {bs * USEFUL_BYTES / s / 1e9:7.2f} GB/s useful, "
              f"{bs * 32 / s / 1e9:7.2f} GB/s of records", flush=True)

    # one graphed batch_loop iteration at bs 4096, BCE and eikonal
    for eik in (False, True):
        cfg.ekional_loss_on, cfg.weight_e = eik, 0.1
        trainer = SdfTrainer(cfg, octree, decoder)
        trainer.zero_grad()
        its = {k: _GraphedIteration(trainer, p, 4096) for k, p in (("host", host), ("device", device_pool))}
        for it in its.values():
            for _ in range(5):
                it.run()
        rounds = {k: [] for k in its}
        for _ in range(3):
            for k, it in its.items():
                rounds[k].append(timed(it.run, 300, dev))
        name = "eikonal" if eik else "bce"
        results["graphed_iteration"][name] = {}
        for k, ts in rounds.items():
            s = statistics.median(ts)
            results["graphed_iteration"][name][k] = {"ms": s * 1e3, "spread_ms": (max(ts) - min(ts)) * 1e3}
            print(f"graphed iteration bs 4096 {name:7s} {k:6s} {s * 1e3:8.4f} ms (spread {(max(ts) - min(ts)) * 1e3:.4f})",
                  flush=True)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "host_pool.json"), "w") as fh:
            json.dump(results, fh, indent=1)
    print(json.dumps(results))
    del host
    torch._C._host_emptyCache()


if __name__ == "__main__":
    sys.exit(main())
