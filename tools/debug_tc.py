import os, sys, ctypes as C
import numpy as np, torch
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__))); sys.path.insert(0, ROOT)
import __graft_entry__ as ge; ge.build()
from tests.parity_utils import make_case, build_cuda_models
from shine_mapping_b200 import SdfTrainer, _abi, sdf_bce_loss
DEV = "cuda:0"
case = make_case(n_points=2500, n_batch=60000, feat_levels=4, seed=44, n_frames=2)
cfg, octree, dec = build_cuda_models(case, DEV)
coord = torch.from_numpy(case["coord"]).to(DEV)[:37888].contiguous(); label = torch.from_numpy(case["label"]).to(DEV)[:37888].contiguous()
n = coord.shape[0]
# reference dL/dfeature through the class surface (query kernel + torch MLP/loss autograd)
feat = octree.query_feature(coord).detach().requires_grad_(True)
loss = sdf_bce_loss(dec.sdf(feat), label, cfg.sigma_sigmoid, None, False, "mean"); loss.backward()
ref = feat.grad.cpu().numpy()
dbg = torch.zeros(n, 8, device=DEV)
lib = _abi.lib(); lib.shine_debug_set_dx.argtypes = [C.c_void_p]; lib.shine_debug_set_dx(C.c_void_p(dbg.data_ptr()))
tr = SdfTrainer(cfg, octree, dec, tcgen05=True); tr.use_replicas = False; tr.zero_grad()
tr.forward_backward(coord, label, None); torch.cuda.synchronize()
lib.shine_debug_set_dx(None)
got = dbg.cpu().numpy()
err = np.abs(got - ref).max(1) / np.abs(ref).max()
bad = np.nonzero(err > 1e-4)[0]
n_sm = torch.cuda.get_device_properties(0).multi_processor_count   # one CTA per SM: tile -> CTA, round
print("dX: max rel err", err.max(), "points off:", bad.size)
for i in bad[:40]:
    tile = i // 128; row = i % 128
    print(f"  point {i}: tile {tile} (cta {tile % n_sm}, round {tile // n_sm}) row {row} (gs warp {row // 16}, ep warp {row // 32}) err {err[i]:.3e} got {got[i][:3]} ref {ref[i][:3]}")
if bad.size:
    t = bad // 128
    print("tiles affected:", np.unique(t).size, "rounds:", np.unique(t // n_sm, return_counts=True), "rows hist (by 16):", np.bincount((bad % 128) // 16, minlength=8))
