"""The shine_batch.py-equivalent loop and the multi-GPU step on real devices."""
import os
import socket

import numpy as np
import pytest
import torch

from tests.parity_utils import build_cuda_models, make_case, make_config, run_oracle_step

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def test_batch_loop_trains_and_checkpoints(tmp_path, built_lib):
    from shine_mapping_b200 import Decoder, FeatureOctree, synth
    from shine_mapping_b200.batch_loop import check_supported, run_shine_mapping_batch
    cfg = make_config(4, device=DEV, bs=4096, lr=0.01, iters=300, weight_decay=1e-7, save_freq_iters=300)
    torch.manual_seed(42)
    octree, decoder = FeatureOctree(cfg), Decoder(cfg)
    pool = synth.build_scene_map(cfg, octree, n_azimuth=256, n_frames=2, seed=42, device=DEV)
    out = run_shine_mapping_batch(cfg, octree, decoder, pool, run_path=str(tmp_path))
    assert out["loss_last"] < 0.8 * out["loss_first"], out
    print("graphed loop (incl. checkpoint write):", out["iters_per_s"], "it/s")
    torch.manual_seed(42)
    octree2, decoder2 = FeatureOctree(cfg), Decoder(cfg)
    pool2 = synth.build_scene_map(cfg, octree2, n_azimuth=256, n_frames=2, seed=42, device=DEV)
    out2 = run_shine_mapping_batch(cfg, octree2, decoder2, pool2, use_cuda_graph=False)
    print("eager loop:", out2["iters_per_s"], "it/s")
    assert out2["loss_last"] < 0.8 * out2["loss_first"], out2
    assert abs(out["loss_last"] - out2["loss_last"]) < 0.1 * out2["loss_last"]   # same optimisation, different batches
    assert out["points_per_s"] > 1e6
    ck = torch.load(tmp_path / "model" / "model_iter_300.pth", weights_only=False)   # reference checkpoint layout
    assert set(ck) >= {"iters", "feature_octree", "geo_decoder", "optimizer"}
    restored = ck["feature_octree"]
    coord, _, _ = pool.get_batch(1000)
    assert torch.equal(restored.query_feature(coord), octree.query_feature(coord))    # hash rebuilt after unpickle
    cfg.normal_loss_on = True
    with pytest.raises(NotImplementedError):
        check_supported(cfg)
    cfg.normal_loss_on = False
    # the shipped KITTI batch config has ekional_loss_on: True (config/kitti/kitti_batch.yaml:46)
    cfg.ekional_loss_on, cfg.weight_e, cfg.iters, cfg.bs = True, 0.1, 60, 2048
    torch.manual_seed(42)
    octree3, decoder3 = FeatureOctree(cfg), Decoder(cfg)
    pool3 = synth.build_scene_map(cfg, octree3, n_azimuth=256, n_frames=1, seed=42, device=DEV)
    out3 = run_shine_mapping_batch(cfg, octree3, decoder3, pool3)
    assert np.isfinite(out3["loss_last"]) and out3["loss_last"] < out3["loss_first"], out3


def _free_port():
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        return s.getsockname()[1]


def _dp_worker(rank, world, port, out_dir):
    os.environ.update(RANK=str(rank), WORLD_SIZE=str(world), LOCAL_RANK=str(rank), MASTER_ADDR="127.0.0.1",
                      MASTER_PORT=str(port))
    from shine_mapping_b200 import SdfTrainer, dist as sdist
    sdist.init_from_env("nccl")
    dev = f"cuda:{rank}"
    case = make_case(n_points=2500, n_batch=6000, feat_levels=4, seed=51)
    cfg, octree, dec = build_cuda_models(case, dev)
    n = case["coord"].shape[0]
    b, e = sdist.shard_range(n, rank, world)
    coord = torch.from_numpy(case["coord"][b:e]).to(dev); label = torch.from_numpy(case["label"][b:e]).to(dev)
    tr = SdfTrainer(cfg, octree, dec, shard_mode="replicated")
    tr.zero_grad()
    loss = tr.forward_backward(coord, label, n_norm=n).clone()
    tr.all_reduce_grads()
    sdist.all_reduce_sum(loss)
    torch.cuda.synchronize()
    if rank == 0:
        np.save(os.path.join(out_dir, "flat.npy"), tr.flat_grad.cpu().numpy())
        np.save(os.path.join(out_dir, "loss.npy"), loss.cpu().numpy())
    torch.distributed.destroy_process_group()


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs 2 GPUs")
def test_two_gpu_data_parallel_matches_oracle(tmp_path, built_lib):
    """Point batch sharded over 2 GPUs + ONE NCCL all-reduce of the flat gradient == oracle gradient of the batch."""
    import torch.multiprocessing as mp
    mp.spawn(_dp_worker, args=(2, _free_port(), str(tmp_path)), nprocs=2, join=True)
    got = np.load(tmp_path / "flat.npy")
    case = make_case(n_points=2500, n_batch=6000, feat_levels=4, seed=51)
    want = run_oracle_step(case)
    off = 0
    for g in want["table_grads"]:
        seg = got[off:off + g.size].reshape(g.shape)
        assert np.abs(seg[:-1] - g[:-1]).max() <= 2e-4 * np.abs(g).max() + 1e-10
        off += (g.size + 3) & ~3
    for k in ["layers.0.weight", "layers.0.bias", "layers.1.weight", "layers.1.bias", "lout.weight", "lout.bias"]:
        g = want["dec_grads"][k]
        seg = got[off:off + g.size].reshape(g.shape)
        assert np.abs(seg - g).max() <= 2e-4 * np.abs(g).max() + 1e-10, k
        off += (g.size + 3) & ~3
    assert abs(float(np.load(tmp_path / "loss.npy")) - want["loss"]) <= 2e-5 * abs(want["loss"])


def _dp_eikonal_worker(rank, world, port, out_dir):
    os.environ.update(RANK=str(rank), WORLD_SIZE=str(world), LOCAL_RANK=str(rank), MASTER_ADDR="127.0.0.1",
                      MASTER_PORT=str(port))
    from shine_mapping_b200 import SdfTrainer, dist as sdist
    sdist.init_from_env("nccl")
    dev = f"cuda:{rank}"
    case = _eikonal_dp_case()
    cfg, octree, dec = build_cuda_models(case, dev)
    cfg.ekional_loss_on, cfg.weight_e = True, 1.0
    n = case["coord"].shape[0]
    b, e = sdist.shard_range(n, rank, world)
    coord = torch.from_numpy(case["coord"][b:e]).to(dev); label = torch.from_numpy(case["label"][b:e]).to(dev)
    weight = torch.from_numpy(case["weight"][b:e]).to(dev)
    tr = SdfTrainer(cfg, octree, dec, shard_mode="replicated")
    tr.zero_grad()
    bce, eik = tr.forward_backward_eikonal(coord, label, weight, n_norm=n)    # surface count summed over the ranks
    scalars = torch.stack([bce.clone(), eik.clone()])
    tr.all_reduce_grads()
    sdist.all_reduce_sum(scalars)
    torch.cuda.synchronize()
    if rank == 0:
        np.save(os.path.join(out_dir, "flat.npy"), tr.flat_grad.cpu().numpy())
        np.save(os.path.join(out_dir, "scalars.npy"), scalars.cpu().numpy())
    torch.distributed.destroy_process_group()


def _eikonal_dp_case():
    case = make_case(n_points=2500, n_batch=6000, feat_levels=4, seed=52)
    case["tables"] = [t * np.float32(300.0) for t in case["tables"]]       # surface |g| around 1
    return case


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs 2 GPUs")
def test_two_gpu_data_parallel_eikonal_matches_oracle(tmp_path, built_lib):
    """ekional_loss_on with the point batch sharded over 2 GPUs: the eikonal mean is over the surface samples of the
    GLOBAL batch, so the summed per-rank values and the all-reduced gradients equal the oracle's for the whole batch."""
    import torch.multiprocessing as mp
    from oracle import shine_oracle as orc
    from tests.parity_utils import DEC_KEYS, oracle_from_case
    mp.spawn(_dp_eikonal_worker, args=(2, _free_port(), str(tmp_path)), nprocs=2, join=True)
    got = np.load(tmp_path / "flat.npy")
    bce, eik = np.load(tmp_path / "scalars.npy")
    case = _eikonal_dp_case()
    o, odec = oracle_from_case(case)
    want = orc.train_step_eikonal(o, odec, torch.from_numpy(case["coord"]), torch.from_numpy(case["label"]),
                                  torch.from_numpy(case["weight"]), case["cfg"]["sigma"], 1.0)
    assert abs(float(eik) - float(want["eikonal"])) <= 1e-4 * float(want["eikonal"])
    assert abs(float(bce) + float(eik) - float(want["loss"])) <= 1e-4 * float(want["loss"])
    off = 0
    for g in want["table_grads"]:
        g = g.numpy()
        seg = got[off:off + g.size].reshape(g.shape)
        assert np.abs(seg[:-1] - g[:-1]).max() <= 1e-3 * np.abs(g).max() + 1e-10
        off += (g.size + 3) & ~3
    for k in DEC_KEYS:
        g = want["dec_grads"][k].numpy()
        seg = got[off:off + g.size].reshape(g.shape)
        assert np.abs(seg - g).max() <= 1e-3 * np.abs(g).max() + 1e-10, k
        off += (g.size + 3) & ~3


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs 2 GPUs")
def test_abi_launches_on_the_device_that_owns_the_tensors(built_lib):
    """ADVICE r01: model on cuda:1 while the current device is cuda:0 — every entry point must launch on cuda:1 (device
    looked up from the pointers, per-device function-attribute caches), and a batch on the wrong device is an argument error."""
    from shine_mapping_b200 import SdfTrainer, _abi
    from tests.parity_utils import compare_step, run_oracle_step
    assert torch.cuda.current_device() == 0
    case = make_case(n_points=2000, n_batch=2500, feat_levels=4, seed=77)
    cfg, octree, dec = build_cuda_models(case, "cuda:1")
    coord = torch.from_numpy(case["coord"]).to("cuda:1"); label = torch.from_numpy(case["label"]).to("cuda:1")
    tr = SdfTrainer(cfg, octree, dec)
    tr.zero_grad()
    pred = torch.empty(coord.shape[0], device="cuda:1")
    loss = tr.forward_backward(coord, label, None, pred_out=pred)
    torch.cuda.synchronize("cuda:1")
    assert torch.cuda.current_device() == 0
    want = run_oracle_step(case)
    assert abs(float(loss) - want["loss"]) <= 2e-5 * abs(want["loss"])
    assert np.abs(pred.cpu().numpy() - want["pred"]).max() <= 2e-5 + 1e-5 * np.abs(want["pred"]).max()
    with pytest.raises(_abi.ShineB200Error):
        tr.forward_backward(coord.to("cuda:0"), label.to("cuda:0"), None)


def test_step_from_host_matches_resident_step(built_lib):
    """The host-buffer entry (pinned memory, chunked H2D overlapped with compute) gives the same loss / gradients
    as one launch on resident inputs."""
    from shine_mapping_b200 import SdfTrainer
    case = make_case(n_points=3000, n_batch=300000, feat_levels=4, seed=61)
    cfg, octree, dec = build_cuda_models(case, DEV)
    coord_h = torch.from_numpy(case["coord"]).pin_memory(); label_h = torch.from_numpy(case["label"]).pin_memory()
    tr = SdfTrainer(cfg, octree, dec)
    loss_host = tr.step_from_host(coord_h, label_h, chunks=4)
    g_host = tr.flat_grad.clone()
    tr.zero_grad()
    loss_res = float(tr.forward_backward(coord_h.to(DEV), label_h.to(DEV)))
    assert abs(loss_host - loss_res) <= 2e-5 * abs(loss_res)      # fp32 atomic accumulation order differs
    assert (g_host - tr.flat_grad).abs().max() <= 1e-4 * tr.flat_grad.abs().max()


def test_incremental_loop_runs(built_lib):
    from shine_mapping_b200 import Decoder, FeatureOctree, synth
    from shine_mapping_b200.incre_loop import run_shine_mapping_incremental
    cfg = make_config(3, device=DEV, bs=2048, lr=0.01, iters=40, continual_learning_reg=True, lambda_forget=1e3,
                      freeze_after_frame=2)
    torch.manual_seed(1)
    octree, decoder = FeatureOctree(cfg), Decoder(cfg)
    dirs, boxes = synth.lidar_directions(128, device=DEV), synth.default_boxes(DEV)
    gen = torch.Generator(device=DEV).manual_seed(3)
    frames = []
    for f in range(3):
        origin = torch.tensor([2.0 * f, 0.0, 0.0], device=DEV)
        hits = synth.raycast_scene(origin, dirs, boxes, cfg.min_range, cfg.pc_radius)
        frames.append(synth.sample_rays(hits * cfg.scale, origin * cfg.scale, cfg, gen))
    hist = run_shine_mapping_incremental(cfg, octree, decoder, frames)
    assert len(hist) == 3 and all(h["bce_last"] < h["bce_first"] for h in hist), hist
    assert all(np.isfinite(h["loss_last"]) for h in hist)
    assert hist[2]["rows"][-1] > hist[0]["rows"][-1]                       # the map grew
    assert not any(p.requires_grad for p in decoder.parameters())          # frozen after frame 2
    assert all(w.abs().sum() > 0 for w in octree.importance_weight)


def test_incremental_loop_with_eikonal(built_lib, monkeypatch):
    """ekional_loss_on in the incremental loop (the reference's replay configs set it; shine_incre.py:159-165): every
    step is the fused BCE + eikonal launch, including after the decoder is frozen (the table-gradient-only kernel)."""
    from shine_mapping_b200 import Decoder, FeatureOctree, SdfTrainer, synth
    from shine_mapping_b200.incre_loop import run_shine_mapping_incremental
    calls = []
    step = SdfTrainer.forward_backward_eikonal

    def counted(self, *a, **kw):
        calls.append(self._dec_trainable)
        return step(self, *a, **kw)
    monkeypatch.setattr(SdfTrainer, "forward_backward_eikonal", counted)
    cfg = make_config(3, device=DEV, bs=2048, lr=0.01, iters=40, continual_learning_reg=True, lambda_forget=1e3,
                      freeze_after_frame=1, ekional_loss_on=True, weight_e=1.0)
    torch.manual_seed(1)
    octree, decoder = FeatureOctree(cfg), Decoder(cfg)
    dirs, boxes = synth.lidar_directions(128, device=DEV), synth.default_boxes(DEV)
    gen = torch.Generator(device=DEV).manual_seed(3)
    frames = []
    for f in range(2):
        origin = torch.tensor([2.0 * f, 0.0, 0.0], device=DEV)
        hits = synth.raycast_scene(origin, dirs, boxes, cfg.min_range, cfg.pc_radius)
        frames.append(synth.sample_rays(hits * cfg.scale, origin * cfg.scale, cfg, gen))
    hist = run_shine_mapping_incremental(cfg, octree, decoder, frames)
    assert len(hist) == 2, hist
    for h in hist:
        assert all(np.isfinite(h[k]) for k in ("loss_first", "loss_last", "eik_first", "eik_last")), h
        # first step of a frame: the regulariser is 0 (features == last frame's), total = bce + weight_e * eikonal
        assert abs(h["loss_first"] - (h["bce_first"] + h["eik_first"])) <= 1e-5 * abs(h["loss_first"]), h
    assert calls == [True] * 40 + [False] * 40                        # frame 1: frozen decoder
    assert not any(p.requires_grad for p in decoder.parameters())


def test_capture_step_replays_the_eager_step():
    """SdfTrainer.capture_step: the graph re-runs {zero, fused step} on whatever the captured tensors hold at replay time
    and gives what the eager calls give (same kernels: gradients equal up to atomics order)."""
    from shine_mapping_b200 import SdfTrainer
    case = make_case(n_points=2500, n_batch=4000, feat_levels=3, seed=31)
    cfg, octree, dec = build_cuda_models(case, DEV)
    tr = SdfTrainer(cfg, octree, dec)
    coord = torch.from_numpy(case["coord"]).to(DEV); label = torch.from_numpy(case["label"]).to(DEV)
    graph = tr.capture_step(coord, label, None, exchange=False)
    perm = torch.randperm(coord.shape[0], device=DEV)
    for data in ((coord.clone(), label.clone()), (coord[perm] * 0.999, label[perm])):
        coord.copy_(data[0]); label.copy_(data[1])
        graph.replay(); torch.cuda.synchronize()
        got_loss, got = float(tr.loss), [g.clone() for g in tr.table_grads] + [g.clone() for g in tr.dec_grads if g is not None]
        tr.zero_grad(); tr.forward_backward(coord, label, None); torch.cuda.synchronize()
        want = list(tr.table_grads) + [g for g in tr.dec_grads if g is not None]
        assert abs(got_loss - float(tr.loss)) <= 1e-6 * abs(float(tr.loss))
        for a, b in zip(got, want):
            assert float((a - b).abs().max()) <= 1e-5 * float(b.abs().max()) + 1e-12
