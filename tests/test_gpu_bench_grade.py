"""The step `bench.py` times, graded element by element at full size: the C2 workload (`bench.build_workload`, one
64 x 2048 scan, 776 616 pool samples) with batches of the whole pool's size.

  (a) the batch the benchmark times: drawn from the Morton-sorted pool (`pool.sort_morton(octree=...)`, free-space samples
      last), `SdfTrainer(..., morton_ordered=True)`: the grouped kernel at R = 1;
  (b) a batch in the order drawn: the per-point kernel, with gradient replicas switching on by themselves;
  (c) batch (a) with sentinel tiles: a few whole tiles weigh 2^12 and every other point 1 (both exact), at the first tile,
      the last (partial) tile, the first and the last zero tile of the free-space run, a scattered tile (more than
      kMaxGroupedRuns nodes on a level) and a tile next to the end, in the grid's last round.  Dropping or doubling one
      sentinel tile's decoder gradients lands outside the bound, by orders of magnitude (checked on the host).
For each batch every pred (bound P), every table-gradient element (the grouped kernel's k_u for (a) and (c)) and every
decoder-gradient element (tests/decoder_bound.py at the kernel's depth for the batch) is graded against the fp64 oracle,
whose lookup tables are the octree's own dict views (test_gpu_scale checks the oracle's own update loops against them).
Points near a ReLU kink stay in the batch and are bounded by their envelope.  Each case prints its worst error / bound
and the process's peak host memory."""
import resource

import numpy as np
import pytest
import torch

import bench
from tests.decoder_bound import restate
from tests.error_bound import grouped_counts
from tests.test_gpu_replicas import FoldSpy, Ref, dec_grads, expected_replicas
from tests.test_gpu_scale import _oracle_with_tables

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(900)]
DEV = "cuda:0"
SENTINEL = 2.0 ** 12


@pytest.fixture(scope="module", autouse=True)
def _lib(built_lib):
    assert torch.cuda.is_available()
    return built_lib


@pytest.fixture(scope="module")
def workload():
    cfg, octree, decoder, pool = bench.build_workload(DEV, 0, 1, 2048)
    pool.sort_morton(octree=octree)
    o, dec = _oracle_with_tables(octree, decoder)
    return cfg, octree, decoder, pool, o, dec


def _case(cfg, o, dec, coord, label, weight, weighted):
    keys = ("layers.0.weight", "layers.0.bias", "layers.1.weight", "layers.1.bias", "lout.weight", "lout.bias")
    return {"cfg": dict(tree_level_world=cfg.tree_level_world, tree_level_feat=cfg.tree_level_feat,
                        feature_dim=cfg.feature_dim, poly_int_on=cfg.poly_int_on, leaf_vox_size=cfg.leaf_vox_size,
                        sigma=float(cfg.sigma_sigmoid), weighted=weighted, reduction=cfg.loss_reduction,
                        bias=cfg.geo_mlp_bias_on),
            "oracle": o, "frames": [], "tables": [t.detach().numpy() for t in o.hier_features],
            "dec": {k: dec[k].detach().numpy() for k in keys if k in dec},
            "coord": coord.cpu().numpy(), "label": label.cpu().numpy(), "weight": weight.cpu().numpy()}


def _step(tr, coord, label, weight, weighted):
    tr.zero_grad()
    pred = torch.empty(coord.shape[0], device=DEV)
    tr.forward_backward(coord, label, weight, pred_out=pred, weighted=weighted)
    torch.cuda.synchronize()
    return [g.detach().cpu().numpy() for g in tr.table_grads], pred.cpu().numpy(), dec_grads(tr)


def _peak_gb():
    return resource.getrusage(resource.RUSAGE_SELF).ru_maxrss / 2 ** 20


def _grade(case, got, what, grouped, replicas=None):
    tables, pred, dec = got
    ref = Ref(case, grouped=grouped, pred=pred, replicas=replicas)
    ref.grade(tables, what, pred)
    ref.grade_decoder(dec, what)
    print(f"[bench grade] {what}: N = {ref.n}, kink points {ref.kinks}, peak host memory {_peak_gb():.2f} GB")
    return ref


def _layout(o, coord):
    """Per tile: zero tile (every point misses every level) and scattered (more than 6 nodes on some level)."""
    idx = o.get_indices(torch.from_numpy(coord))
    n = coord.shape[0]
    pad = -n % 16
    miss = np.logical_and.reduce([(ix.numpy().reshape(n, -1) < 0).all(1) for ix in idx])
    zero = np.concatenate((miss, np.ones(pad, bool))).reshape(-1, 16).all(1)
    scattered = np.zeros(zero.shape[0], bool)
    for ix in idx:
        node = np.concatenate((ix.numpy().reshape(n, -1)[:, 0], np.full(pad, -1))).reshape(-1, 16)
        srt = np.sort(node, 1)
        runs = ((srt >= 0) & np.concatenate((np.ones((srt.shape[0], 1), bool), srt[:, 1:] != srt[:, :-1]), 1)).sum(1)
        scattered |= runs > 6
    return zero, scattered


def test_bench_ordered_batch(workload):
    """(a): the timed step, grouped kernel at R = 1, and its R = 1 really asserted."""
    from shine_mapping_b200 import SdfTrainer
    cfg, octree, decoder, pool, o, dec = workload
    n = len(pool)
    coord, label, weight = pool.get_batch(n, torch.Generator(device=DEV).manual_seed(1000))
    tr = SdfTrainer(cfg, octree, decoder, shard_mode="spatial", morton_ordered=True)
    spy = FoldSpy(octree)
    got = _step(tr, coord, label, weight, None)
    assert all(max(r) == 1 for r in spy.calls), f"the ordered step ran with replicas {spy.calls}"
    _grade(_case(cfg, o, dec, coord, label, weight, cfg.loss_weight_on), got, "bench (a) Morton-ordered", True)


def test_bench_drawn_order_batch(workload):
    """(b): the per-point kernel with the replicas the batch size switches on."""
    from shine_mapping_b200 import SdfTrainer
    cfg, octree, decoder, pool, o, dec = workload
    n = len(pool)
    coord, label, weight = pool.get_batch(n, torch.Generator(device=DEV).manual_seed(1001), ordered=False)
    tr = SdfTrainer(cfg, octree, decoder, shard_mode="spatial", morton_ordered=False)
    spy = FoldSpy(octree)
    got = _step(tr, coord, label, weight, None)
    case = _case(cfg, o, dec, coord, label, weight, cfg.loss_weight_on)
    assert spy.calls and max(spy.calls[-1]) > 1, f"the drawn-order step ran without replicas: {spy.calls}"
    print(f"[bench grade] (b) R per level {spy.calls[-1]}")
    _grade(case, got, "bench (b) order drawn", False)


def test_bench_sentinel_tiles(workload):
    """(c): sentinel tiles of weight 2^12 in batch (a); a dropped or doubled sentinel tile leaves the bound."""
    from shine_mapping_b200 import SdfTrainer
    cfg, octree, decoder, pool, o, dec = workload
    n = len(pool)
    coord, label, _ = pool.get_batch(n, torch.Generator(device=DEV).manual_seed(1000))
    zero, scattered = _layout(o, coord.cpu().numpy())
    tiles = zero.shape[0]
    assert n % 16 != 0, "the last tile is not partial"
    zt = np.nonzero(zero[:-1])[0]
    st = np.nonzero(scattered & ~zero)[0]
    assert zt.size > 2 and st.size, f"zero tiles {zt.size}, scattered tiles {st.size}"
    sentinels = sorted({0, tiles - 1, int(zt[0]), int(zt[-1]), int(st[st.size // 2]), tiles - 3})
    print(f"[bench grade] (c) {tiles} tiles, {int(zero.sum())} zero, {int(scattered.sum())} scattered; sentinels {sentinels}")
    w = np.ones(n, dtype=np.float32)
    for t in sentinels:
        w[16 * t:16 * (t + 1)] = SENTINEL
    weight = torch.from_numpy(w).to(DEV)
    tr = SdfTrainer(cfg, octree, decoder, shard_mode="spatial", morton_ordered=True)
    got = _step(tr, coord, label, weight, True)
    ref = _grade(_case(cfg, o, dec, coord, label, weight, True), got, "bench (c) sentinel tiles", True)
    graded = ref.for_kernel(True)
    depth_ref = graded.dec
    from tests.decoder_bound import kernel_depth
    depth = kernel_depth(n, 1, torch.cuda.get_device_properties(0).multi_processor_count)
    for t in sentinels:
        sl = slice(16 * t, min(n, 16 * (t + 1)))
        part = restate(ref.feat64[sl], ref.dec64, ref.g64[sl])[0]
        worst = max(float((np.abs(part[k]) / np.maximum(depth_ref.bound(k, depth), 1e-300)).max()) for k in part)
        for sign in (-1.0, 1.0):
            bad = {k: v + sign * part[k].reshape(v.shape) for k, v in got[2].items()}
            with pytest.raises(AssertionError, match="outside the bound"):
                depth_ref.grade(bad, depth, f"sentinel tile {t} {'dropped' if sign < 0 else 'doubled'}")
        print(f"[bench grade] sentinel tile {t}: {worst:.3g} x the bound when dropped or doubled")
