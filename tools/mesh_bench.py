"""Time the mesher on the GPU: grid query, marching cubes, and normals + cluster filter + compaction, separately.

    python tools/mesh_bench.py [--iters 300] [--reps 3]

Two maps: the C2 map of bench.py (one synthetic scan, L=4) and a 20-frame synthetic street (frames 2 m apart).  Each
is trained briefly (the timings do not depend on how well, only on the mesh's size), meshed once as warm-up, then
`--reps` times in each mode (octree, bbx) with CUDA events around each phase of every chunk; the median is reported.
One JSON line per map and mode, with the card's name and power limit read in the same run.  Writes nothing.
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def street_workload(device):
    from bench import workload_config
    from shine_mapping_b200 import Decoder, FeatureOctree, synth
    cfg = workload_config(device)
    cfg.name = "street_20_frames"
    torch.manual_seed(42)
    octree, decoder = FeatureOctree(cfg), Decoder(cfg)
    pool = synth.build_scene_map(cfg, octree, n_azimuth=1024, n_frames=20, frame_step_m=2.0, seed=42, device=device)
    return cfg, octree, decoder, pool


def time_mesh(mesher, grid, min_tris):
    """-> dict of GPU milliseconds per phase and mesh sizes, one reconstruction (events around every phase)."""
    from shine_mapping_b200 import _abi
    from shine_mapping_b200.mesher import compact, normals_and_clusters
    import ctypes as C
    dev = grid["bricks"].device
    lib, st = _abi.lib(), _abi.stream_ptr(dev)
    ev = lambda: torch.cuda.Event(enable_timing=True)
    grid_ms = mc_ms = 0.0
    cap = mesher.edge_capacity(grid)
    slots = torch.full((cap * 16,), 0xFF, dtype=torch.uint8, device=dev)
    counters = torch.zeros(4, dtype=torch.int32, device=dev)
    verts = torch.empty(0, 3, dtype=torch.float32, device=dev)
    faces = []
    it = iter(mesher.chunks(grid))
    while True:
        e0, e1, e2 = ev(), ev(), ev()
        e0.record()
        try:
            _, _, _, g = next(it)
        except StopIteration:
            break
        e1.record()
        counters[1:3].zero_()
        _abi.check(lib.shine_marching_cubes(C.byref(g), _abi.ptr(slots), cap, _abi.ptr(counters), None, 0, None, 0, st), "count")
        nv, nt, _, lost = counters.tolist()
        if lost or 2 * nv > cap:
            raise RuntimeError("edge table too small for the bench's map; raise Mesher.edge_capacity")
        if nv > verts.shape[0]:
            grown = torch.empty(max(nv, 2 * verts.shape[0]), 3, dtype=torch.float32, device=dev)
            grown[:verts.shape[0]] = verts
            verts = grown
        f = torch.empty(nt, 3, dtype=torch.int32, device=dev)
        _abi.check(lib.shine_marching_cubes(C.byref(g), _abi.ptr(slots), cap, _abi.ptr(counters), _abi.ptr(verts),
                                            verts.shape[0], _abi.ptr(f), nt, st), "emit")
        faces.append(f)
        e2.record()
        torch.cuda.synchronize(dev)
        grid_ms += e0.elapsed_time(e1)
        mc_ms += e1.elapsed_time(e2)
    nv = int(counters[0])
    verts = verts[:nv]
    faces = torch.cat(faces) if faces else torch.zeros(0, 3, dtype=torch.int32, device=dev)
    e0, e1 = ev(), ev()
    e0.record()
    normals, keep = normals_and_clusters(verts, faces, min_tris)
    v, f, _ = compact(verts, faces, normals, keep)
    e1.record()
    torch.cuda.synchronize(dev)
    return {"grid_ms": grid_ms, "mc_ms": mc_ms, "filter_ms": e0.elapsed_time(e1), "verts_raw": nv,
            "tris_raw": int(faces.shape[0]), "verts": int(v.shape[0]), "tris": int(f.shape[0])}


def main():
    from bench import build_workload, device_info
    from shine_mapping_b200 import Mesher
    from shine_mapping_b200.batch_loop import run_shine_mapping_batch
    from shine_mapping_b200.mesher import OCTREE_MIN_CLUSTER
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--iters", type=int, default=300)
    ap.add_argument("--reps", type=int, default=3)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("mesh_bench.py times the sm_90a kernels: it needs a GPU")
    dev = "cuda:0"
    card = device_info(0)
    for name, build in (("c2_maicity_like_single_scan", lambda: build_workload(dev, 0, 1, 2048)),
                        ("street_20_frames", lambda: street_workload(dev))):
        cfg, octree, decoder, pool = build()
        run_shine_mapping_batch(cfg, octree, decoder, pool, iters=args.iters)
        mesher = Mesher(cfg, octree, decoder)
        bbx = getattr(pool, "map_bbx", None)
        for mode in ("octree", "bbx"):
            if mode == "octree":
                grid, min_tris = mesher.octree_grid(octree.free_level_num, cfg.mc_res_m), OCTREE_MIN_CLUSTER
            else:
                grid, min_tris = mesher.bbx_grid(bbx[0], bbx[1], cfg.mc_res_m), cfg.min_cluster_vertices
            time_mesh(mesher, grid, min_tris)                                       # warm-up
            runs = [time_mesh(mesher, grid, min_tris) for _ in range(args.reps)]
            med = {k: statistics.median(r[k] for r in runs) for k in ("grid_ms", "mc_ms", "filter_ms")}
            n1 = grid["n"] + 1
            points = int(grid["bricks"].shape[0]) * n1 ** 3
            print(json.dumps({
                "workload": name, "mode": mode, "mc_res_m": cfg.mc_res_m, "train_iters": args.iters,
                "bricks": int(grid["bricks"].shape[0]), "cubes_per_brick_side": grid["n"], "grid_points": points,
                "grid_points_per_s": points / (med["grid_ms"] * 1e-3) if med["grid_ms"] > 0 else None,
                **med, "total_ms": sum(med.values()),
                **{k: runs[-1][k] for k in ("verts_raw", "tris_raw", "verts", "tris")},
                "reps": args.reps, "stat": "median of GPU event times", "device": card}))


if __name__ == "__main__":
    main()
