"""Spatial partition with the real kernels: (1) every rank of a 3-way partition run in turn on ONE GPU, the collective
replaced by a sum of the exchange buffers; (2) two ranks on two GPUs with the C-ABI NCCL all-reduce.  Reference in both:
the single-process oracle step on the same global batch (loss, decoder gradients, every table row by corner key)."""
import os
import socket

import numpy as np
import pytest
import torch

from tests.parity_utils import DEC_KEYS
from tests.partition_utils import check_rank_against_global, global_case, global_oracle_step, global_scene

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def _build_rank(cfg_cpu, part, dec, key_to_row, o_glob, device, rank, all_keys=None):
    """Package octree + decoder on `device` for one range; features copied from the global tables by corner key."""
    from shine_mapping_b200 import Decoder, FeatureOctree
    from shine_mapping_b200.partition import corner_keys_of
    from tests.parity_utils import make_config
    cfg = make_config(cfg_cpu.tree_level_feat, device=device, pc_radius=30.0)
    c, l, w = part
    octree = FeatureOctree(cfg)
    octree.update(c[w > 0].to(device))
    keys = [k.cpu() for k in corner_keys_of(octree)]
    with torch.no_grad():
        for lvl, (p, ks) in enumerate(zip(octree.hier_features, keys)):
            rows = torch.tensor([key_to_row[lvl][int(k)] for k in ks.tolist()], dtype=torch.long)
            p[:-1].copy_(o_glob.hier_features[lvl].detach()[rows])
    decoder = Decoder(cfg)
    sd = decoder.state_dict()
    for k in DEC_KEYS:
        sd[k] = dec[k].detach().to(device)
    decoder.load_state_dict(sd)
    return cfg, octree, decoder, keys


def _check_decoder_and_loss(trainer, loss, res_glob):
    want = torch.cat([torch.cat([res_glob["dec_grads"][k].reshape(-1), torch.zeros((-res_glob["dec_grads"][k].numel()) % 4)])
                      for k in DEC_KEYS])
    got = trainer.dec_flat.detach().cpu()[:want.numel()]
    assert float((got - want).abs().max()) <= 2e-4 * float(want.abs().max())
    assert abs(loss - float(res_glob["loss"])) <= 2e-5 * abs(float(res_glob["loss"]))


def _three_ranges_on_one_gpu(replicas_per_rank=None):
    """replicas_per_rank: a list that receives, per rank, the R per level of the step's replica fold (which runs inside
    forward_backward, before the boundary pack)."""
    from shine_mapping_b200 import SdfTrainer
    from shine_mapping_b200.partition import BoundaryPlan, coarse_keys, owner_of, partition_pool
    world = 3
    cfg0, pool, batch, dec = global_scene(levels=4, n_azimuth=128, n_frames=3, n_batch=20000)
    o_glob, key_to_row, res_glob = global_oracle_step(cfg0, pool, batch, dec)
    bounds, parts = partition_pool(*pool, cfg0, world)
    owner = owner_of(coarse_keys(batch[0], cfg0.tree_level_world - cfg0.tree_level_feat + 1), bounds)
    built = [_build_rank(cfg0, parts[r], dec, key_to_row, o_glob, DEV, r) for r in range(world)]
    plans = [BoundaryPlan(r, [b[3] for b in built], cfg0.feature_dim, 1380).to(DEV) for r in range(world)]
    assert plans[0].total_floats > 1380
    n_global = batch[0].shape[0]
    trainers = []
    for r, (cfg, octree, decoder, keys) in enumerate(built):
        tr = SdfTrainer(cfg, octree, decoder, shard_mode="spatial", boundary=plans[r])
        if replicas_per_rank is not None:
            fold = octree._reduce_replicas

            def spy(desc, device, fold=fold):
                replicas_per_rank.append([max(1, desc.lv[i].num_replicas) for i in range(desc.num_levels)])
                fold(desc, device)
            octree._reduce_replicas = spy
        tr.zero_grad()
        m = owner == r
        tr.forward_backward(batch[0][m].to(DEV), batch[1][m].to(DEV), None, n_norm=n_global)
        plans[r].pack(tr.table_grads, tr.exchange)
        trainers.append(tr)
    total = torch.stack([t.exchange for t in trainers]).sum(0)            # what the all-reduce leaves everywhere
    loss = sum(float(t.loss) for t in trainers)
    for r, tr in enumerate(trainers):
        tr.exchange.copy_(total)
        plans[r].unpack(tr.table_grads, tr.exchange)
        torch.cuda.synchronize()
        worst = check_rank_against_global([g.detach().cpu().numpy() for g in tr.table_grads], built[r][3], key_to_row,
                                          res_glob)
        _check_decoder_and_loss(tr, loss, res_glob)
    print("3 ranges on one GPU == single step; boundary rows per level:", plans[0].counts, "worst rel", worst)
    for tr in trainers:
        assert all(int(torch.count_nonzero(b)) == 0 for b in tr.octree._grad_scratch.values())


def test_three_ranges_on_one_gpu_equal_the_single_step(built_lib):
    _three_ranges_on_one_gpu()


def test_three_ranges_on_one_gpu_with_forced_replicas(built_lib, monkeypatch):
    """The same partition with gradient replicas on every rank's coarse levels."""
    from shine_mapping_b200 import FeatureOctree
    monkeypatch.setattr(FeatureOctree, "_REPLICA_TARGET", 1)
    monkeypatch.setattr(FeatureOctree, "_REPLICA_MAX", 64)
    seen = []
    _three_ranges_on_one_gpu(seen)
    assert len(seen) == 3 and all(max(r) > 1 for r in seen), f"R per level and rank: {seen}"
    print("R per level (leaf first) and rank:", seen)


def _free_port():
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        return s.getsockname()[1]


def _grade_exchanged(tr, plan, loss, pb, ref, case, sizes, what):
    """Every table element of this rank and the decoder gradients against the bound of a partitioned step
    (tests/boundary_oracle.py), the summed loss against its own, and the exchange's result bitwise equal on every rank:
    decoder segment and every shared corner's rows gathered from all ranks."""
    import torch.distributed as dist
    from tests.boundary_oracle import pack_host
    from tests.test_gpu_replicas import dec_grads
    torch.cuda.synchronize()
    tables = [g.detach().cpu().numpy() for g in tr.table_grads]
    pb.grade_rank(plan.rank, tables, what)
    ref.dec.grade(dec_grads(tr), pb.decoder_depth(sizes, torch.cuda.get_device_properties(0).multi_processor_count), what)
    pb.loss_ref(case).grade(loss, what)
    mine = pack_host(plan, tables)
    mine[:plan.dec_floats] = tr.dec_flat.detach().cpu().numpy()[:plan.dec_floats]
    held = np.zeros(plan.total_floats, dtype=bool)
    held[:plan.dec_floats] = True
    for lvl, n in enumerate(plan.counts):
        held[plan.offsets[lvl]:plan.offsets[lvl] + n * plan.feature_dim].reshape(-1, plan.feature_dim)[
            plan.slots[lvl].cpu().numpy()] = True
    everyone = [None] * dist.get_world_size()
    dist.all_gather_object(everyone, (mine, held))
    for r, (theirs, their_held) in enumerate(everyone):
        both = held & their_held
        bad = np.flatnonzero(mine[both].view(np.uint32) != theirs[both].view(np.uint32))
        assert bad.size == 0, f"{what}: {bad.size} exchanged floats differ from rank {r}'s"


def _nccl_worker(rank, world, port, out_dir):
    os.environ.update(RANK=str(rank), WORLD_SIZE=str(world), LOCAL_RANK=str(rank), MASTER_ADDR="127.0.0.1",
                      MASTER_PORT=str(port))
    import torch.distributed as dist
    from shine_mapping_b200 import SdfTrainer, dist as sdist
    from shine_mapping_b200.partition import BoundaryPlan, coarse_keys, gather_corner_keys, owner_of, partition_pool
    sdist.init_from_env("nccl")
    dev = f"cuda:{rank}"
    from tests.boundary_oracle import PartitionBound, global_rows
    from tests.test_gpu_replicas import Ref
    cfg0, pool, batch, dec = global_scene(levels=4, n_azimuth=128, n_frames=3, n_batch=20000)
    o_glob, key_to_row, res_glob = global_oracle_step(cfg0, pool, batch, dec)
    bounds, parts = partition_pool(*pool, cfg0, world)
    cfg, octree, decoder, keys = _build_rank(cfg0, parts[rank], dec, key_to_row, o_glob, dev, rank)
    comm = sdist.NcclComm(rank, world, torch.device(dev))
    all_keys = gather_corner_keys(octree)
    plan = BoundaryPlan(rank, all_keys, cfg0.feature_dim, 1380).to(dev)
    tr = SdfTrainer(cfg, octree, decoder, shard_mode="spatial", boundary=plan, comm=comm)
    tr.zero_grad()
    owner = owner_of(coarse_keys(batch[0], cfg0.tree_level_world - cfg0.tree_level_feat + 1), bounds)
    m = owner == rank
    # the fp64 step of the global batch and the bound of the per-point kernel on this split (kink points keep their
    # envelope bound: the batch is the one the fp32 checks use)
    case = global_case(cfg0, o_glob, batch, dec)
    ref = Ref(case)
    points = [np.flatnonzero(owner.numpy() == r) for r in range(world)]
    rank_rows = [[global_rows(k, key_to_row[kk]) for kk, k in enumerate(ks)] for ks in all_keys]
    pb = PartitionBound(ref, points, rank_rows, grouped=False)
    sizes = [p.size for p in points]
    loss = tr.forward_backward(batch[0][m].to(dev), batch[1][m].to(dev), None, n_norm=batch[0].shape[0]).clone()
    tr.all_reduce_grads()                       # pack -> shine_allreduce_decoder_grads (NCCL, C ABI) -> unpack
    comm.all_reduce(loss.view(1))
    torch.cuda.synchronize()
    check_rank_against_global([g.detach().cpu().numpy() for g in tr.table_grads], keys, key_to_row, res_glob)
    _check_decoder_and_loss(tr, float(loss), res_glob)
    _grade_exchanged(tr, plan, float(loss), pb, ref, case, sizes, f"NCCL rank {rank}")
    # second step through the pipelined host entry with the exchange inside
    h = tr.submit_host_step(batch[0][m].pin_memory(), batch[1][m].pin_memory(), n_norm=batch[0].shape[0], exchange=True)
    h.result()
    check_rank_against_global([g.detach().cpu().numpy() for g in tr.table_grads], keys, key_to_row, res_glob)
    pb.grade_rank(rank, [g.detach().cpu().numpy() for g in tr.table_grads], f"NCCL host step rank {rank}")
    # the same exchange as ONE NVLink peer-memory kernel (IPC buffers + flags, no NCCL) — three steps in a row so that both
    # buffer parities and the flag hand-over between consecutive steps are exercised
    p2p = sdist.P2PExchange(rank, world, torch.device(dev), plan.total_floats)
    tr2 = SdfTrainer(cfg, octree, decoder, shard_mode="spatial", boundary=plan, p2p=p2p)
    for _ in range(3):
        tr2.zero_grad()
        loss2 = tr2.forward_backward(batch[0][m].to(dev), batch[1][m].to(dev), None, n_norm=batch[0].shape[0]).clone()
        tr2.all_reduce_grads()
        comm.all_reduce(loss2.view(1))
        torch.cuda.synchronize()
        check_rank_against_global([g.detach().cpu().numpy() for g in tr2.table_grads], keys, key_to_row, res_glob)
        _check_decoder_and_loss(tr2, float(loss2), res_glob)
        _grade_exchanged(tr2, plan, float(loss2), pb, ref, case, sizes, f"peer memory rank {rank}")
    # the whole step {zero, fused kernel, peer-memory exchange} captured as a CUDA graph and replayed: the exchange keeps
    # its step number on the device, so replays keep the protocol going (four replays: both buffer parities twice)
    cd, ld = batch[0][m].to(dev), batch[1][m].to(dev)
    graph = tr2.capture_step(cd, ld, None, n_norm=batch[0].shape[0], exchange=True)
    for _ in range(4):
        graph.replay()
        torch.cuda.synchronize()
        check_rank_against_global([g.detach().cpu().numpy() for g in tr2.table_grads], keys, key_to_row, res_glob)
        loss3 = tr2.loss.detach().clone()
        comm.all_reduce(loss3.view(1))
        _check_decoder_and_loss(tr2, float(loss3), res_glob)
        _grade_exchanged(tr2, plan, float(loss3), pb, ref, case, sizes, f"graph replay rank {rank}")
    assert p2p.timeouts() == 0
    open(os.path.join(out_dir, f"ok{rank}"), "w").write("ok")
    dist.barrier()
    p2p.close()
    comm.close()
    dist.destroy_process_group()


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs 2 GPUs")
@pytest.mark.timeout(600)
def test_two_gpu_spatial_partition_matches_single_step(tmp_path, built_lib):
    import torch.multiprocessing as mp
    mp.spawn(_nccl_worker, args=(2, _free_port(), str(tmp_path)), nprocs=2, join=True)
    assert os.path.exists(tmp_path / "ok0") and os.path.exists(tmp_path / "ok1")
