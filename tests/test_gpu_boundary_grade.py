"""The spatially partitioned training step and its exchange kernels, graded on one GPU (tests/boundary_oracle.py).

A. `shine_boundary_pack` / `shine_boundary_unpack` bit for bit against numpy indexing, at F = 4 .. 32, 1 / 3 / 8 levels,
   empty levels first, in the middle and last, one row, and a level past 4 x SMs x 256 quads (a second grid-stride
   pass); every float outside the plan's slots and rows keeps its sentinel bits.  Refused descriptors write nothing.
B. Every rank of a 2, 3 and 5-way partition of one global batch, run in turn, the collective replaced by the exchange's
   rank-order fp32 sum: pred equal to inference on the single-GPU map bit for bit, every table element within the bound
   of a partitioned step, decoder gradients and loss within theirs, shared rows bitwise equal on every rank.  For the
   per-point kernel, the Morton-ordered grouped kernel and the per-point kernel with forced gradient replicas.
C. `BoundaryPlan.unify_values` through the CUDA pack / unpack: duplicates that start out different end up with their
   lowest holder's bits.
D. `shine_p2p_exchange` with 2 and 3 ranks, one process each, all on this GPU (gloo for set-up, CUDA IPC for the
   buffers): plans sized for the single-block branch, the arrive-counter hand-shake and the 128-block cap with its tail
   loop; five eager exchanges (both buffer parities twice) and replays of a captured one, every output bit for bit
   against the model, every other float untouched, no timeout.
E. The step `bench.py --gpus N` times, 2 and 3 rank processes on this GPU set up as `build_partitioned_workload` does
   (gloo in place of NCCL): the Morton-ordered grouped kernel and the peer-memory exchange in one captured graph.  Four
   replays, each graded against the fp64 step of the global batch and bitwise equal across ranks on every shared corner;
   then three eager steps with Adam, after which the duplicates' features, moments and gradients are still bit-identical.
   Replays are not bitwise equal to each other: the grouped scatter's fp32 atomics land in any order, so every replay is
   graded on its own.
D and E skip, and say why, when CUDA IPC cannot map the peers' buffers."""
import copy
import ctypes as C
import os
import socket

import numpy as np
import pytest
import torch

from oracle import shine_oracle as orc
from tests.boundary_oracle import PartitionBound, check_plans, exchange_model, global_rows, pack_host
from tests.error_bound import drop_kinks
from tests.parity_utils import DEC_KEYS
from tests.partition_utils import check_rank_against_global, global_case, global_scene

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
INVALID = -1                                     # SHINE_ERR_INVALID_ARG
SENTINEL = np.uint32(0x7FA5A5A5)                 # a NaN payload: any float written over it shows


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _bits(t):
    return np.asarray(t.cpu().numpy() if torch.is_tensor(t) else t, dtype=np.float32).view(np.uint32)


# ---- A. pack / unpack --------------------------------------------------------------------------------------------------

def _pack_levels(n_levels, F):
    """(count, table rows, slots) per level: empty levels first / mid / last, one row, and one big level."""
    big = -(-4 * _sms() * 256 * 4 // F) + 1000          # rows: more than 4 x SMs x 256 quads
    pattern = {1: [big], 3: [0, 1, big], 8: [37, 0, 1, big, 5, 0, 200, 0]}[n_levels]
    return [(c, c + 7 + c // 3, 2 * c + 3) for c in pattern]


def _pack_case(n_levels, F, seed):
    from shine_mapping_b200 import _abi
    rng = np.random.default_rng(seed)
    base = 1384
    levels = _pack_levels(n_levels, F)
    d = _abi.ShineBoundary()
    keep, host, off = [], [], base
    for i, (count, rows, slots) in enumerate(levels):
        table = rng.standard_normal((rows + 1, F)).astype(np.float32)     # last row: the trash row
        r = rng.permutation(rows)[:count].astype(np.int32)                 # random order, never the trash row
        s = rng.permutation(slots)[:count].astype(np.int32)                # sparse slots
        t_dev, r_dev, s_dev = (torch.from_numpy(x).to(DEV) for x in (table, r, s))
        lv = d.lv[i]
        lv.table, lv.rows, lv.slots = t_dev.data_ptr(), r_dev.data_ptr(), s_dev.data_ptr()
        lv.offset, lv.count = off, count
        keep.append((t_dev, r_dev, s_dev))
        host.append((table, r, s, off))
        off += slots * F
    return d, keep, host, off + 64


def _call(name, d, n_levels, F, buf):
    from shine_mapping_b200 import _abi
    return getattr(_abi.lib(), name)(C.byref(d), n_levels, F, _abi.ptr(buf), _abi.stream_ptr(DEV))


@pytest.mark.parametrize("F", [4, 8, 16, 32])
@pytest.mark.parametrize("n_levels", [1, 3, 8])
def test_pack_unpack_bit_for_bit(n_levels, F, built_lib):
    d, keep, host, total = _pack_case(n_levels, F, 10 * F + n_levels)
    quads = max(c * F // 4 for c, _, _ in _pack_levels(n_levels, F))
    assert quads > 4 * _sms() * 256, "no level takes a second grid-stride pass"
    # pack: sentinel buffer, every slot of the plan gets its row, everything else keeps its bits
    buf = torch.from_numpy(np.full(total, SENTINEL, dtype=np.uint32).view(np.float32)).to(DEV)
    assert _call("shine_boundary_pack", d, n_levels, F, buf) == 0
    torch.cuda.synchronize()
    want = np.full(total, SENTINEL, dtype=np.uint32)
    for table, r, s, off in host:
        want[off:off + (s.max(initial=-1) + 1) * F].reshape(-1, F)[s] = table[r].view(np.uint32) if r.size else 0
    got = _bits(buf)
    bad = np.flatnonzero(got != want)
    assert bad.size == 0, f"pack: {bad.size} floats differ, first at {bad[0]}"
    for (t_dev, _, _), (table, _, _, _) in zip(keep, host):
        assert np.array_equal(_bits(t_dev), table.view(np.uint32)), "pack wrote a table"
    # unpack: random buffer, sentinel tables; the plan's rows get their slots, the trash row and other rows keep their bits
    data = np.random.default_rng(F).standard_normal(total).astype(np.float32)
    buf = torch.from_numpy(data).to(DEV)
    for t_dev, _, _ in keep:
        t_dev.view(torch.int32).fill_(int(SENTINEL))
    assert _call("shine_boundary_unpack", d, n_levels, F, buf) == 0
    torch.cuda.synchronize()
    for i, ((t_dev, _, _), (table, r, s, off)) in enumerate(zip(keep, host)):
        want_t = np.full(table.shape, SENTINEL, dtype=np.uint32)
        if r.size:
            want_t[r] = data[off:off + (s.max() + 1) * F].reshape(-1, F)[s].view(np.uint32)
        bad = np.argwhere(_bits(t_dev) != want_t)
        assert bad.size == 0, f"unpack level {i}: {len(bad)} floats differ, first at {bad[0]}"
    assert np.array_equal(_bits(buf), data.view(np.uint32)), "unpack wrote the buffer"
    print(f"[pack] F={F} levels={n_levels}: counts {[c for c, _, _ in _pack_levels(n_levels, F)]}, "
          f"largest level {quads} quads ({-(-quads // (4 * _sms() * 256))} grid-stride passes): bit for bit")


@pytest.mark.parametrize("name", ["shine_boundary_pack", "shine_boundary_unpack"])
def test_pack_unpack_refusals_write_nothing(name, built_lib):
    from shine_mapping_b200 import _abi
    d, keep, host, total = _pack_case(3, 8, 3)
    buf = torch.from_numpy(np.full(total, SENTINEL, dtype=np.uint32).view(np.float32)).to(DEV)
    before = [_bits(t) for t, _, _ in keep]
    refusals = {"0 levels": (d, 0, 8), "9 levels": (d, 9, 8), "F = 6": (d, 3, 6)}
    odd = _abi.ShineBoundary.from_buffer_copy(d)
    odd.lv[2].offset += 2
    null_rows = _abi.ShineBoundary.from_buffer_copy(d)
    null_rows.lv[1].rows = None
    refusals.update({"offset not a multiple of 4": (odd, 3, 8), "count > 0 with null rows": (null_rows, 3, 8)})
    for what, (desc, nl, F) in refusals.items():
        assert _call(name, desc, nl, F, buf) == INVALID, f"{name}: {what} was accepted"
    torch.cuda.synchronize()
    assert np.all(_bits(buf) == SENTINEL), f"{name}: a refused call wrote the buffer"
    for t, b in zip(keep, before):
        assert np.array_equal(_bits(t[0]), b), f"{name}: a refused call wrote a table"


# ---- B. the partitioned step -------------------------------------------------------------------------------------------

@pytest.fixture(scope="module")
def scene():
    """The global scene of the 3-range test, its oracle octree, the global batch without ReLU-kink points as a case, its
    fp64 Ref, the fp32 oracle step (the second check) and the single-GPU map for inference."""
    from tests.test_gpu_partition import _build_rank
    from tests.test_gpu_replicas import Ref
    cfg0, pool, batch, dec = global_scene(levels=4, n_azimuth=128, n_frames=3, n_batch=20000)
    assert not cfg0.loss_weight_on and cfg0.loss_reduction == "mean"
    o = orc.OracleOctree(cfg0.tree_level_world, cfg0.tree_level_feat, cfg0.feature_dim, cfg0.feature_std, cfg0.poly_int_on)
    torch.manual_seed(11)
    o.update(pool[0][pool[2] > 0])
    key_to_row = [o.corners_lookup_tables[o.free_level_num + k] for k in range(o.featured_level_num)]
    case, kinks = drop_kinks(global_case(cfg0, o, batch, dec))
    ref = Ref(case)
    d = {k: v.detach().clone().requires_grad_(True) for k, v in dec.items()}
    og = copy.copy(o)
    og.hier_features = [t.detach().clone().requires_grad_(True) for t in o.hier_features]
    res32 = orc.train_step(og, d, torch.from_numpy(case["coord"]), torch.from_numpy(case["label"]), None,
                           float(cfg0.sigma_sigmoid), False, "mean")
    _, g_oct, g_dec, _ = _build_rank(cfg0, pool, dec, key_to_row, o, DEV, 0)
    from shine_mapping_b200.fused import sdf_infer
    pred_infer = sdf_infer(g_oct, g_dec, torch.from_numpy(case["coord"]).to(DEV)).cpu().numpy()
    print(f"[partition] global batch {case['coord'].shape[0]} points ({kinks} kink points dropped)")
    return {"cfg0": cfg0, "pool": pool, "dec": dec, "o": o, "key_to_row": key_to_row, "case": case, "ref": ref,
            "res32": res32, "pred_infer": pred_infer}


def _ranks(scene, world):
    """Per rank: (cfg, octree, decoder, corner keys), the plans, and the global batch indices of each rank."""
    from shine_mapping_b200.partition import BoundaryPlan, coarse_keys, owner_of, partition_pool
    from tests.test_gpu_partition import _build_rank
    cfg0, case = scene["cfg0"], scene["case"]
    bounds, parts = partition_pool(*scene["pool"], cfg0, world)
    built = [_build_rank(cfg0, parts[r], scene["dec"], scene["key_to_row"], scene["o"], DEV, r) for r in range(world)]
    keys = [b[3] for b in built]
    plans = [BoundaryPlan(r, keys, cfg0.feature_dim, 1380) for r in range(world)]
    check_plans(plans, keys, cfg0.feature_dim, 1380)
    plans = [p.to(DEV) for p in plans]
    coord = torch.from_numpy(case["coord"])
    owner = owner_of(coarse_keys(coord, cfg0.tree_level_world - cfg0.tree_level_feat + 1), bounds).numpy()
    points = [np.flatnonzero(owner == r) for r in range(world)]
    return built, plans, points


def _morton_order(coord, idx):
    from shine_mapping_b200.feature_octree import points_to_morton, quantize_points
    key = points_to_morton(quantize_points(torch.from_numpy(coord[idx]), 12))
    return idx[torch.argsort(key, stable=True).numpy()]


def _check_shared_rows(plans, tables_by_rank, total, what):
    """Every holder of every shared corner carries the exchange's value bit for bit (so all holders agree)."""
    for r, (p, tables) in enumerate(zip(plans, tables_by_rank)):
        mine = pack_host(p, tables)
        for lvl, n in enumerate(p.counts):
            s = p.slots[lvl].cpu().numpy()
            seg = slice(p.offsets[lvl], p.offsets[lvl] + n * p.feature_dim)
            a = mine[seg].reshape(-1, p.feature_dim)[s].view(np.uint32)
            b = total[seg].reshape(-1, p.feature_dim)[s].view(np.uint32)
            bad = np.argwhere(a != b)
            assert bad.size == 0, f"{what}: rank {r} level {lvl}: {len(bad)} shared floats differ from the other ranks'"


MODES = ("per-point", "grouped", "replicas")


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("world", [2, 3, 5])
def test_partitioned_step_against_fp64(world, mode, scene, monkeypatch, built_lib):
    from shine_mapping_b200 import FeatureOctree, SdfTrainer
    from tests.test_gpu_replicas import FoldSpy, dec_grads
    if mode == "replicas":
        monkeypatch.setattr(FeatureOctree, "_REPLICA_TARGET", 1)
        monkeypatch.setattr(FeatureOctree, "_REPLICA_MAX", 64)
    grouped = mode == "grouped"
    case, ref = scene["case"], scene["ref"].for_kernel(grouped)
    built, plans, points = _ranks(scene, world)
    if grouped:
        points = [_morton_order(case["coord"], idx) for idx in points]
    n_global = case["coord"].shape[0]
    trainers, preds, spies, Rs = [], [], [], []
    for r, (cfg, octree, decoder, keys) in enumerate(built):
        tr = SdfTrainer(cfg, octree, decoder, shard_mode="spatial", boundary=plans[r], morton_ordered=grouped)
        spy = FoldSpy(octree)
        idx = points[r]
        coord, label = (torch.from_numpy(case[k][idx]).to(DEV) for k in ("coord", "label"))
        pred = torch.empty(idx.size, device=DEV)
        tr.zero_grad()
        tr.forward_backward(coord, label, None, n_norm=n_global, pred_out=pred)
        plans[r].pack(tr.table_grads, tr.exchange)
        torch.cuda.synchronize()
        if mode == "replicas":
            assert spy.calls and max(spy.calls[-1]) > 1, f"rank {r}: the step ran without replicas ({spy.calls})"
            Rs.append(spy.calls[-1])
        else:       # the bound below is the one of R = 1: no fold with R > 1 ran
            assert all(max(c) == 1 for c in spy.calls), f"rank {r}: the {mode} step ran with replicas {spy.calls}"
        trainers.append(tr); preds.append(pred.cpu().numpy())
    what = f"{world} ranges {mode}"
    if Rs:
        print(f"[replicas] {what}: R per level (coarse -> fine) and rank {Rs}")
    # the collective: the rank-order fp32 sum of every rank's packed buffer
    total = exchange_model([t.exchange.cpu().numpy() for t in trainers], plans[0])
    loss = np.float32(0)
    for tr in trainers:
        loss = loss + np.float32(float(tr.loss))
    rank_rows = [[global_rows(k, scene["key_to_row"][kk]) for kk, k in enumerate(b[3])] for b in built]
    pb = PartitionBound(ref, points, rank_rows, grouped)
    sms = _sms()
    tables_by_rank = []
    for r, tr in enumerate(trainers):
        tr.exchange.copy_(torch.from_numpy(total))
        plans[r].unpack(tr.table_grads, tr.exchange)
        torch.cuda.synchronize()
        got_pred = preds[r]
        want_pred = scene["pred_infer"][points[r]]
        bad = np.flatnonzero(got_pred.view(np.uint32) != want_pred.view(np.uint32))
        assert bad.size == 0, f"{what} rank {r}: pred differs from inference on the single-GPU map at {bad.size} points"
        tables = [g.detach().cpu().numpy().copy() for g in tr.table_grads]
        tables_by_rank.append(tables)
        pb.grade_rank(r, tables, f"{what} rank {r}")
        dg = dec_grads(tr)
        ref.dec.grade(dg, pb.decoder_depth([p.size for p in points], sms), f"{what} rank {r}")
        check_rank_against_global(tables, built[r][3], scene["key_to_row"], scene["res32"])
        assert np.array_equal(_bits(tr.exchange[:1380]), total[:1380].view(np.uint32))
    pb.loss_ref(case).grade(loss, what)
    _check_shared_rows(plans, tables_by_rank, total, what)
    print(f"[partition] {what}: shared corners per level {plans[0].counts}, rows bitwise equal on every holder")


# ---- C. unify_values ----------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("world", [2, 3])
def test_unify_values_copies_the_lowest_holder(world, scene, built_lib):
    import threading
    from shine_mapping_b200 import FeatureOctree
    from shine_mapping_b200.partition import BoundaryPlan, corner_keys_of, partition_pool
    from tests.parity_utils import make_config
    cfg0 = scene["cfg0"]
    _, parts = partition_pool(*scene["pool"], cfg0, world)
    octrees, keys = [], []
    for r in range(world):
        torch.manual_seed(100 + r)              # every rank draws its own initial features: duplicates differ
        oc = FeatureOctree(make_config(cfg0.tree_level_feat, device=DEV, pc_radius=30.0))
        c, _, w = parts[r]
        oc.update(c[w > 0].to(DEV))
        octrees.append(oc)
        keys.append([k.cpu() for k in corner_keys_of(oc)])
    plans = [BoundaryPlan(r, keys, cfg0.feature_dim, 1380).to(DEV) for r in range(world)]
    before = [[p.detach().cpu().numpy().copy() for p in oc.hier_features] for oc in octrees]
    key_rows = [[{int(k): i for i, k in enumerate(ks.tolist())} for ks in kr] for kr in keys]
    barrier, bufs, errors = threading.Barrier(world), [None] * world, []

    def all_reduce(r):
        def reduce(buf):
            bufs[r] = buf
            barrier.wait()
            if r == 0:
                acc = torch.zeros_like(buf)
                for b in bufs:
                    acc += b
                for b in bufs:
                    b.copy_(acc)
                torch.cuda.synchronize()
            barrier.wait()
        return reduce

    def run(r):
        try:
            plans[r].unify_values(list(octrees[r].hier_features), all_reduce(r))
            torch.cuda.synchronize()
        except Exception as exc:       # noqa: BLE001 — reported below
            errors.append(exc)
            barrier.abort()
    threads = [threading.Thread(target=run, args=(r,)) for r in range(world)]
    for t in threads:
        t.start()
    for t in threads:
        t.join()
    assert not errors, errors
    after = [[p.detach().cpu().numpy() for p in oc.hier_features] for oc in octrees]
    differed = 0
    for lvl in range(len(keys[0])):
        for r in range(world):
            got, old = after[r][lvl].view(np.uint32), before[r][lvl].view(np.uint32)
            shared = np.zeros(got.shape[0], dtype=bool)
            for j, k in enumerate(keys[r][lvl].tolist()):
                holders = [q for q in range(world) if k in key_rows[q][lvl]]
                if len(holders) < 2:
                    continue
                shared[j] = True
                low = holders[0]
                want = before[low][lvl][key_rows[low][lvl][k]].view(np.uint32)
                assert np.array_equal(got[j], want), f"rank {r} level {lvl} key {k}: not the lowest holder's ({low}) bits"
                differed += int(r != low and not np.array_equal(old[j], want))
            assert np.array_equal(got[~shared], old[~shared]), f"rank {r} level {lvl}: a row that is not shared changed"
    assert differed > 0, "no duplicate started out different"
    print(f"[unify] {world} ranks: shared per level {plans[0].counts}, {differed} duplicate rows took their owner's bits")


# ---- D. the peer-memory exchange, every rank a process on this GPU ---------------------------------------------------------

def _p2p_launch_constants():
    """(threads per block, quads per thread before the tail loop, block cap) of `shine_p2p_exchange`'s launch, read from
    csrc/shine_p2p.cu so that the branch each plan is sized for follows the launcher if its sizing changes."""
    import re
    src = open(os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "shine_mapping_b200", "csrc",
                            "shine_p2p.cu")).read()
    threads = int(re.search(r"constexpr int kP2PThreads = (\d+);", src).group(1))
    items = int(re.search(r"constexpr int kItems = (\d+);", src).group(1))
    cap = re.search(r"if \(blocks > (\d+)\) blocks = (\d+);", src)
    assert cap and cap.group(1) == cap.group(2), "the launcher's block cap is no longer where this test reads it"
    per_block = re.search(r"int64_t blocks = \(most \+ (\d+) \* kP2PThreads - 1\) / \((\d+) \* kP2PThreads\);", src)
    assert per_block and int(per_block.group(1)) == int(per_block.group(2)) == items, \
        "the launcher no longer sizes the grid for kItems quads per thread"
    return threads, items, int(cap.group(1))


# (name, F, decoder floats, per level (shared corners, private corners per rank)); the shared corners of the level marked
# "no-last" are never held by the last rank
P2P_CASES = [
    ("single-block", 4, 64, [(0, 20), (300, 50), (200, 10)]),
    ("arrive-counter", 8, 1380, [(7000, 500), (0, 300), (12800, 1000)]),
    ("block-cap-tail", 16, 1380, [(15000, 100), (25000, 100), (0, 100)]),
]


def p2p_branch(total_floats):
    """The grid `shine_p2p_exchange` launches for a buffer of total_floats (blocks = ceil(quads / (kItems x threads)),
    capped) and the branch of `p2p_exchange_kernel` it takes: one block skips the arrive counter, more blocks hand over
    through it, and past the cap the quads beyond kItems per thread go through the tail loop."""
    threads, items, cap = _p2p_launch_constants()
    quads = total_floats // 4
    blocks = min(max(-(-quads // (items * threads)), 1), cap)
    if blocks == 1:
        return blocks, "single block"
    return blocks, "arrive counter" + (" + 128-block cap, tail loop" if quads > items * threads * blocks else "")


def p2p_keys(case_i, world):
    """Per rank, per level shuffled int64 corner keys of P2P_CASES[case_i]: shared corners held by 2 or more ranks (with 3
    ranks: some by two, some by all three; on level 1 of the single-block case never by the last rank), private ones by
    one rank."""
    _, F, dec, levels = P2P_CASES[case_i]
    rng = np.random.default_rng(1000 + 10 * case_i + world)
    out = [[] for _ in range(world)]
    for lvl, (n_shared, n_private) in enumerate(levels):
        keys = rng.choice(1 << 40, size=n_shared + world * n_private, replace=False)
        allowed = world - 1 if (case_i == 0 and lvl == 1 and world == 3) else world
        held = [[] for _ in range(world)]
        for j, k in enumerate(keys[:n_shared].tolist()):
            size = 2 if allowed == 2 else int(rng.integers(2, allowed + 1))
            for r in rng.choice(allowed, size=size, replace=False).tolist():
                held[r].append(k)
        for r in range(world):
            held[r].extend(keys[n_shared + r * n_private:n_shared + (r + 1) * n_private].tolist())
            out[r].append(torch.from_numpy(rng.permutation(np.array(held[r], dtype=np.int64))))
    return out


def p2p_data(case_i, world, rank, step, rows_per_level, F, dec):
    """Decoder segment and tables (with trash row) of one exchange: magnitudes over eleven decades, both signs, so that
    another add order changes the bits."""
    rng = np.random.default_rng([case_i, world, rank, step])

    def draw(shape):
        x = rng.standard_normal(shape).astype(np.float32)
        return x * np.power(np.float32(10), rng.uniform(-3, 8, shape).astype(np.float32))
    return draw(dec), [draw((n + 1, F)) for n in rows_per_level]


def _free_port():
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        return s.getsockname()[1]


def _p2p_worker(rank, world, port, out_dir):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    import torch.distributed as dist
    from shine_mapping_b200 import _abi, dist as sdist
    from shine_mapping_b200.partition import BoundaryPlan
    dist.init_process_group("gloo", rank=rank, world_size=world)
    torch.cuda.set_device(0)
    dev = torch.device(DEV)
    plans = [BoundaryPlan(rank, p2p_keys(i, world), c[1], c[2]) for i, c in enumerate(P2P_CASES)]
    try:
        p2p = sdist.P2PExchange(rank, world, dev, max(p.total_floats for p in plans))
    except _abi.ShineB200Error as exc:            # every rank agrees before raising
        if rank == 0:
            open(os.path.join(out_dir, "skip"), "w").write(str(exc))
        dist.barrier()
        dist.destroy_process_group()
        return

    def go(fn):
        dist.barrier()
        torch.cuda.synchronize()
        fn()
        torch.cuda.synchronize()

    for i, ((name, F, dec_n, levels), plan) in enumerate(zip(P2P_CASES, plans)):
        plan.to(dev)
        rows = [k.numel() for k in p2p_keys(i, world)[rank]]
        dec = torch.zeros(dec_n, device=dev)
        tables = [torch.zeros(n + 1, F, device=dev) for n in rows]

        def load(step):
            d, ts = p2p_data(i, world, rank, step, rows, F, dec_n)
            dec.copy_(torch.from_numpy(d))
            for t, x in zip(tables, ts):
                t.copy_(torch.from_numpy(x))

        def save(step):
            np.savez(os.path.join(out_dir, f"c{i}_s{step}_r{rank}.npz"), dec=dec.cpu().numpy(),
                     **{f"t{lvl}": t.cpu().numpy() for lvl, t in enumerate(tables)})

        for step in range(5):
            load(step)
            go(lambda: p2p.exchange(dec, plan, tables))
            save(step)
        load(5)
        torch.cuda.synchronize()
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph):
            p2p.exchange(dec, plan, tables)
        for step in (5, 6):
            load(step)
            go(graph.replay)
            save(step)
        del graph
    open(os.path.join(out_dir, f"timeouts_r{rank}"), "w").write(str(p2p.timeouts()))
    dist.barrier()
    p2p.close()
    dist.destroy_process_group()


def _spawn(fn, world, *args):
    """One daemon process per rank; joined in a finally, and any still alive then is terminated."""
    import torch.multiprocessing as mp
    ctx = mp.get_context("spawn")
    port = _free_port()
    procs = [ctx.Process(target=fn, args=(r, world, port, *args), daemon=True) for r in range(world)]
    try:
        for p in procs:
            p.start()
        for p in procs:
            p.join(timeout=240)
    finally:
        for p in procs:
            if p.is_alive():
                p.terminate()
                p.join()
    codes = [p.exitcode for p in procs]
    assert codes == [0] * world, f"rank processes exited with {codes}"


@pytest.mark.timeout(600)
@pytest.mark.parametrize("world", [2, 3])
def test_p2p_exchange_bit_for_bit_on_one_gpu(world, tmp_path, built_lib):
    from shine_mapping_b200.partition import BoundaryPlan
    _spawn(_p2p_worker, world, str(tmp_path))
    if (tmp_path / "skip").exists():
        reason = (tmp_path / "skip").read_text()
        print(f"[p2p] {world} ranks: skipped, peer-memory exchange unavailable: {reason}")
        pytest.skip(f"peer-memory exchange could not be set up: {reason}")
    timeouts = [int((tmp_path / f"timeouts_r{r}").read_text()) for r in range(world)]
    for i, (name, F, dec_n, levels) in enumerate(P2P_CASES):
        keys = p2p_keys(i, world)
        plans = [BoundaryPlan(r, keys, F, dec_n) for r in range(world)]
        check_plans(plans, keys, F, dec_n)
        blocks, branch = p2p_branch(plans[0].total_floats)
        want_branch = {"single-block": "single block", "arrive-counter": "arrive counter",
                       "block-cap-tail": "arrive counter + 128-block cap, tail loop"}[name]
        assert branch == want_branch, f"{name}: the plan takes '{branch}'"
        rows = [[k.numel() for k in keys[r]] for r in range(world)]
        for step in range(7):
            ins = [p2p_data(i, world, r, step, rows[r], F, dec_n) for r in range(world)]
            bufs = []
            for r in range(world):
                b = pack_host(plans[r], ins[r][1])
                b[:dec_n] = ins[r][0]
                bufs.append(b)
            total = exchange_model(bufs, plans[0])
            for r in range(world):
                z = np.load(tmp_path / f"c{i}_s{step}_r{r}.npz")
                what = f"{world} ranks {name} step {step}{' (graph replay)' if step >= 5 else ''} rank {r}"
                assert np.array_equal(z["dec"].view(np.uint32), total[:dec_n].view(np.uint32)), f"{what}: decoder segment"
                for lvl, t_in in enumerate(ins[r][1]):
                    want = t_in.copy()
                    p = plans[r]
                    seg = total[p.offsets[lvl]:p.offsets[lvl] + p.counts[lvl] * F].reshape(-1, F)
                    want[p.rows[lvl].numpy()] = seg[p.slots[lvl].numpy()]
                    bad = np.argwhere(z[f"t{lvl}"].view(np.uint32) != want.view(np.uint32))
                    assert bad.size == 0, (f"{what} level {lvl}: {len(bad)} floats differ, first at row {bad[0][0]} "
                                           f"({'shared' if bad[0][0] in set(p.rows[lvl].tolist()) else 'not shared'})")
        print(f"[p2p] {world} ranks {name}: F={F}, slots per level {plans[0].counts}, {plans[0].total_floats // 4} quads, "
              f"{blocks} blocks ({branch}): 5 exchanges + 2 graph replays bit for bit")
    assert timeouts == [0] * world, f"timeouts {timeouts}"
    print(f"[p2p] {world} ranks: timeouts = {sum(timeouts)}")


# ---- E. the bench's N > 1 step, every rank a process on this GPU --------------------------------------------------------

BENCH_AZIMUTH = 256         # the bench's scans at a quarter of their azimuth steps: the fp64 oracle of the batch stays small
BENCH_BS = 6144             # points per rank and step


def _shared_agree(plans, arrays_by_rank, what):
    """For every pair of ranks, the rows of every corner both hold are bitwise equal (arrays: per rank, per level [rows + 1,
    F] in the rank's row order)."""
    packed, held = [], []
    for p, arrays in zip(plans, arrays_by_rank):
        packed.append(pack_host(p, arrays).view(np.uint32))
        h = np.zeros(p.total_floats, dtype=bool)
        for lvl, n in enumerate(p.counts):
            h[p.offsets[lvl]:p.offsets[lvl] + n * p.feature_dim].reshape(-1, p.feature_dim)[p.slots[lvl].numpy()] = True
        held.append(h)
    pairs = 0
    for r in range(len(plans)):
        for q in range(r + 1, len(plans)):
            both = held[r] & held[q]
            bad = np.flatnonzero(packed[r][both] != packed[q][both])
            assert bad.size == 0, f"{what}: ranks {r} and {q} differ in {bad.size} floats of the corners they share"
            pairs += int(both.sum())
    assert pairs > 0, f"{what}: no corner is shared"
    return pairs


def _bench_worker(rank, world, port, out_dir):
    """build_partitioned_workload with gloo in place of NcclComm, then the bench's step: captured with the peer-memory
    exchange and replayed, then eager steps with Adam."""
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    import torch.distributed as dist
    import bench
    from shine_mapping_b200 import Decoder, FeatureOctree, SdfTrainer, _abi, dist as sdist, partition, synth
    from tests.test_gpu_replicas import FoldSpy, dec_grads
    dist.init_process_group("gloo", rank=rank, world_size=world)
    torch.cuda.set_device(0)
    dev = torch.device(DEV)
    cfg = bench.workload_config(DEV)
    torch.manual_seed(42)                       # the decoder is replicated: the same initial weights on every rank
    octree, decoder = FeatureOctree(cfg), Decoder(cfg)
    frames = synth.generate_scans(cfg, BENCH_AZIMUTH, world, bench.SCAN_SPACING_M, 42, DEV,
                                  origin_x0=-(world - 1) * bench.SCAN_SPACING_M / 2)
    coord = torch.cat([f[0] for f in frames]); label = torch.cat([f[1] for f in frames])
    weight = torch.cat([f[2] for f in frames])
    level = cfg.tree_level_world - cfg.tree_level_feat + 1
    box = [partition.balanced_key_bounds(partition.coarse_keys(coord, level).cpu(), world)]
    dist.broadcast_object_list(box, src=0)
    _, parts = partition.partition_pool(coord, label, weight, cfg, world, bounds=box[0])
    if rank == 0:
        np.save(os.path.join(out_dir, "surface.npy"), coord[weight > 0].cpu().numpy())
    pool = partition.build_rank_map(cfg, octree, parts[rank], dev)
    plan = partition.BoundaryPlan(rank, partition.gather_corner_keys(octree), cfg.feature_dim,
                                  partition.decoder_segment_floats(decoder)).to(dev)

    def gloo_sum(buf):
        host = buf.cpu()
        dist.all_reduce(host)
        buf.copy_(host)
    plan.unify_values(list(octree.hier_features), gloo_sum)
    try:
        p2p = sdist.P2PExchange(rank, world, dev, plan.total_floats)
    except _abi.ShineB200Error as exc:            # every rank agrees before raising
        if rank == 0:
            open(os.path.join(out_dir, "skip"), "w").write(str(exc))
        dist.barrier()
        dist.destroy_process_group()
        return
    tr = SdfTrainer(cfg, octree, decoder, shard_mode="spatial", boundary=plan, p2p=p2p, morton_ordered=True)
    spy = FoldSpy(octree)
    pool.sort_morton(octree=octree)
    gen = torch.Generator(device=dev).manual_seed(7 + rank)
    coord_b, label_b, _ = pool.get_batch(BENCH_BS, generator=gen)
    n_global = BENCH_BS * world
    keys = [k.cpu().numpy() for k in partition.corner_keys_of(octree)]
    save = {f"k{l}": k for l, k in enumerate(keys)}
    save.update({f"f{l}": p.detach().cpu().numpy() for l, p in enumerate(octree.hier_features)})
    save.update({"coord": coord_b.cpu().numpy(), "label": label_b.cpu().numpy()})
    save.update({"dec_" + k: v.detach().cpu().numpy() for k, v in decoder.state_dict().items()})

    def go(fn):
        dist.barrier()
        torch.cuda.synchronize()
        out = fn()
        torch.cuda.synchronize()
        return out

    graph = go(lambda: tr.capture_step(coord_b, label_b, None, n_norm=n_global, exchange=True))
    for k in range(4):
        go(graph.replay)
        save.update({f"r{k}_g{l}": g.detach().cpu().numpy() for l, g in enumerate(tr.table_grads)})
        save.update({f"r{k}_dec_" + name: g for name, g in dec_grads(tr).items()})
        save[f"r{k}_loss"] = np.float32(float(tr.loss))
    del graph
    for s in range(3):                          # eager steps on fresh batches, Adam after each exchange
        cb, lb, _ = pool.get_batch(BENCH_BS, generator=gen)

        def step():
            tr.zero_grad()
            tr.forward_backward(cb, lb, None, n_norm=n_global)
            tr.all_reduce_grads()
        go(step)
        tr.optimizer_step(zero_grad=False)
    torch.cuda.synchronize()
    L = len(tr.table_grads)
    save.update({f"e_f{l}": p.detach().cpu().numpy() for l, p in enumerate(octree.hier_features)})
    save.update({f"e_g{l}": g.detach().cpu().numpy() for l, g in enumerate(tr.table_grads)})
    for name, buf in (("m", tr.exp_avg), ("v", tr.exp_avg_sq)):
        save.update({f"e_{name}{l}": buf[tr._offs[l]:tr._offs[l] + tr._sizes[l]].view(tr.table_grads[l].shape).cpu().numpy()
                     for l in range(L)})
        dec0 = tr._offs[L]
        save[f"e_{name}_dec"] = buf[dec0:].cpu().numpy()
    save["e_dec_params"] = torch.cat([p.detach().reshape(-1) for p in decoder.fused_params() if p is not None]).cpu().numpy()
    save["folds"] = np.array([max(c) for c in spy.calls] or [1])
    save["timeouts"] = np.int64(p2p.timeouts())
    save["plan_dec_floats"] = np.int64(plan.dec_floats)
    np.savez(os.path.join(out_dir, f"bench_r{rank}.npz"), **save)
    dist.barrier()
    p2p.close()
    dist.destroy_process_group()


@pytest.mark.timeout(600)
@pytest.mark.parametrize("world", [2, 3])
def test_bench_partitioned_step_on_one_gpu(world, tmp_path, built_lib):
    """The step `bench.py --gpus N` times, with its ranks as processes on this GPU: the Morton-ordered grouped kernel and
    the peer-memory exchange captured in one CUDA graph.  Every replay graded against the fp64 step of the global batch
    (tables assembled by corner key) with the bound of a partitioned step, shared rows bitwise equal across ranks; then
    three eager steps with Adam, after which every shared corner's features, Adam moments and gradients are still
    bit-identical on every rank (the drift claim of DESIGN §6)."""
    import bench
    from shine_mapping_b200.partition import BoundaryPlan
    from tests.test_gpu_replicas import Ref
    _spawn(_bench_worker, world, str(tmp_path))
    if (tmp_path / "skip").exists():
        reason = (tmp_path / "skip").read_text()
        print(f"[bench step] {world} ranks: skipped, peer-memory exchange unavailable: {reason}")
        pytest.skip(f"peer-memory exchange could not be set up: {reason}")
    z = [dict(np.load(tmp_path / f"bench_r{r}.npz")) for r in range(world)]
    cfg = bench.workload_config("cpu")
    L = cfg.tree_level_feat
    keys = [[torch.from_numpy(zz[f"k{l}"]) for l in range(L)] for zz in z]
    plans = [BoundaryPlan(r, keys, cfg.feature_dim, int(z[0]["plan_dec_floats"])) for r in range(world)]
    check_plans(plans, keys, cfg.feature_dim, plans[0].dec_floats)
    dec_names = ["dec_" + k for k in DEC_KEYS if "dec_" + k in z[0]]
    for zz in z[1:]:
        assert all(np.array_equal(zz[k], z[0][k]) for k in dec_names), "the ranks start from different decoders"
    assert all(int(zz["timeouts"]) == 0 for zz in z), f"timeouts {[int(zz['timeouts']) for zz in z]}"
    assert all(int(zz["folds"].max()) == 1 for zz in z), "the grouped step ran a replica fold with R > 1"
    _shared_agree(plans, [[zz[f"f{l}"] for l in range(L)] for zz in z], f"{world} ranks: features after unify_values")
    # the global map: the oracle octree of every rank's surface samples, rows filled by corner key from the ranks' tables
    o = orc.OracleOctree(cfg.tree_level_world, L, cfg.feature_dim, cfg.feature_std, cfg.poly_int_on)
    o.update(torch.from_numpy(np.load(tmp_path / "surface.npy")))
    key_to_row = [o.corners_lookup_tables[o.free_level_num + k] for k in range(o.featured_level_num)]
    rank_rows = [[global_rows(keys[r][l], key_to_row[l]) for l in range(L)] for r in range(world)]
    tables = []
    for l in range(L):
        t = np.zeros((len(key_to_row[l]) + 1, cfg.feature_dim), dtype=np.float32)
        filled = np.zeros(t.shape[0], dtype=bool)
        for r in range(world):
            t[rank_rows[r][l]] = z[r][f"f{l}"][:-1]
            filled[rank_rows[r][l]] = True
        assert filled[:-1].all(), f"level {l}: a corner of the global map is on no rank"
        tables.append(t)
    o.hier_features = [torch.from_numpy(t) for t in tables]
    dec = {k[4:]: torch.from_numpy(z[0][k]) for k in dec_names}
    batch = (torch.from_numpy(np.concatenate([zz["coord"] for zz in z])),
             torch.from_numpy(np.concatenate([zz["label"] for zz in z])))
    case = global_case(cfg, o, batch, dec)
    ref = Ref(case).for_kernel(True)
    points = [np.arange(r * BENCH_BS, (r + 1) * BENCH_BS) for r in range(world)]      # each rank's batch as it ran
    pb = PartitionBound(ref, points, rank_rows, grouped=True)
    depth = pb.decoder_depth([BENCH_BS] * world, _sms())
    lref = pb.loss_ref(case)
    for k in range(4):
        what = f"{world} ranks bench step, replay {k}"
        loss = np.float32(0)
        for r in range(world):
            pb.grade_rank(r, [z[r][f"r{k}_g{l}"] for l in range(L)], f"{what} rank {r}")
            ref.dec.grade({n[len(f"r{k}_dec_"):]: v for n, v in z[r].items() if n.startswith(f"r{k}_dec_")}, depth,
                          f"{what} rank {r}")
            loss = loss + z[r][f"r{k}_loss"]
            if r:
                assert all(np.array_equal(z[r][n].view(np.uint32), z[0][n].view(np.uint32))
                           for n in z[r] if n.startswith(f"r{k}_dec_")), f"{what}: decoder gradients differ across ranks"
        lref.grade(loss, what)
        _shared_agree(plans, [[zz[f"r{k}_g{l}"] for l in range(L)] for zz in z], what)
        if k:
            diff = sum(int((z[r][f"r{k}_g{l}"].view(np.uint32) != z[r][f"r0_g{l}"].view(np.uint32)).sum())
                       for r in range(world) for l in range(L))
            print(f"[bench step] {what}: {diff} table-gradient floats differ in their last bits from replay 0 "
                  f"(fp32 atomics of the grouped scatter land in any order)")
    n = 0
    for name in ("f", "m", "v", "g"):
        n = _shared_agree(plans, [[zz[f"e_{name}{l}"] for l in range(L)] for zz in z],
                          f"{world} ranks after 3 Adam steps: {dict(f='features', m='exp_avg', v='exp_avg_sq', g='grads')[name]}")
    for name in ("e_dec_params", "e_m_dec", "e_v_dec"):
        assert all(np.array_equal(zz[name].view(np.uint32), z[0][name].view(np.uint32)) for zz in z[1:]), \
            f"{world} ranks after 3 Adam steps: {name} differs across ranks"
    print(f"[bench step] {world} ranks: ran; shared corners per level {plans[0].counts}, {n} shared floats bit-identical "
          f"on every holder after 3 Adam steps (features, moments, gradients); timeouts = 0")
