#!/usr/bin/env python
"""Kernel-variant timings on the bench workload (development aid; prints one line per variant)."""
import argparse, ctypes as C, os, statistics, sys
import torch
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import bench
from shine_mapping_b200 import SdfTrainer, _abi, sdf_infer

ap = argparse.ArgumentParser()
ap.add_argument("--n-azimuth", type=int, default=2048)
ap.add_argument("--frames", type=int, default=1)
ap.add_argument("--points", type=int, default=0)
ap.add_argument("--reps", type=int, default=10)
ap.add_argument("--leaf-vox", type=float, default=0.2)
ap.add_argument("--step-m", type=float, default=2.0)
ap.add_argument("--sorted", action="store_true", help="Morton-sort the batch (locality experiment)")
ap.add_argument("--quick", action="store_true", help="only the step / frozen / infer lines")
ap.add_argument("--free-last", action="store_true", help="with --sorted: samples that see no node go behind all others")
args = ap.parse_args()
dev = torch.device("cuda", 0)
from shine_mapping_b200 import Decoder, FeatureOctree, synth
cfg = bench.workload_config(str(dev))
cfg.leaf_vox_size = args.leaf_vox; cfg.calculate_world_scale()
torch.manual_seed(42)
octree, decoder = FeatureOctree(cfg), Decoder(cfg)
pool = synth.build_scene_map(cfg, octree, n_azimuth=args.n_azimuth, n_frames=args.frames, frame_step_m=args.step_m, seed=42, device=str(dev))
n = args.points or len(pool)
gen = torch.Generator(device=dev).manual_seed(1)
coord, label, weight = pool.get_batch(n, gen)
if args.sorted:
    from shine_mapping_b200.feature_octree import points_to_morton, quantize_points
    key = points_to_morton(quantize_points(coord, 12))
    if args.free_last:
        key = key | ((~octree.sees_a_node(coord)).long() << 62)
    order = torch.argsort(key)
    coord, label, weight = coord[order].contiguous(), label[order].contiguous(), weight[order].contiguous()
print(f"table MB={sum(p.numel() for p in octree.hier_features)*4/1e6:.1f}", end=" "); print(f"N={n} rows={[int(p.shape[0]) for p in octree.hier_features]} pool={len(pool)}")
flush = torch.empty(256 << 20, dtype=torch.uint8, device=dev)

def timeit(fn, name, bytes_per_pt=None):
    for _ in range(3): fn()
    ts = []
    for k in range(args.reps):
        flush.fill_(k); e0 = torch.cuda.Event(enable_timing=True); e1 = torch.cuda.Event(enable_timing=True)
        e0.record(); fn(); e1.record(); torch.cuda.synchronize(); ts.append(e0.elapsed_time(e1))
    ms = statistics.median(ts)
    print(f"{name:34s} {ms:8.4f} ms  {n / ms / 1e6:9.1f} Mpts/s")

tr3 = SdfTrainer(cfg, octree, decoder)
tr1 = SdfTrainer(cfg, octree, decoder, tf32x1=True)
timeit(lambda: tr3.forward_backward(coord, label), "step 3xTF32 dec_grad")
timeit(lambda: tr3.forward_backward(coord, label, morton_ordered=True), "step 3xTF32 dec_grad grouped")
if not args.quick: timeit(lambda: tr1.forward_backward(coord, label), "step 1xTF32 dec_grad")
for p in decoder.parameters(): p.requires_grad = False
trf3 = SdfTrainer(cfg, octree, decoder); trf1 = SdfTrainer(cfg, octree, decoder, tf32x1=True)
timeit(lambda: trf3.forward_backward(coord, label), "step 3xTF32 frozen decoder")
timeit(lambda: trf3.forward_backward(coord, label, morton_ordered=True), "step 3xTF32 frozen grouped")
timeit(lambda: sdf_infer(octree, decoder, coord), "infer 3xTF32")
if args.quick: sys.exit(0)
timeit(lambda: trf1.forward_backward(coord, label), "step 1xTF32 frozen decoder")
timeit(lambda: sdf_infer(octree, decoder, coord, tf32x1=True), "infer 1xTF32")
feat = torch.empty(n, 8, device=dev); od = octree._descriptor(None, tr3.table_grads, n_points=n)
lib = _abi.lib(); st = _abi.stream_ptr(dev)
timeit(lambda: lib.shine_query_fwd(C.byref(od), _abi.ptr(coord), n, _abi.ptr(feat), st), "query_fwd (gather only)")
timeit(lambda: lib.shine_query_bwd(C.byref(od), _abi.ptr(coord), n, _abi.ptr(feat), st), "query_bwd (scatter only)")
idx = torch.empty(4, n, 8, dtype=torch.int64, device=dev)
timeit(lambda: lib.shine_get_indices(C.byref(od), _abi.ptr(coord), n, _abi.ptr(idx), st), "get_indices")
timeit(lambda: tr3.flat_grad.zero_(), "zero grads")
for p in decoder.parameters(): p.requires_grad = True
tr = SdfTrainer(cfg, octree, decoder)
tr.forward_backward(coord, label)
timeit(lambda: tr.optimizer_step(zero_grad=True), "adam (all tables + decoder)")
