"""The batch-mode sample pool in pinned host memory (`synth.HostSamplePool`: `shine_host_pool_append` and
`shine_host_pool_gather`) against the reference's semantics — `torch.cat` of the frames, indexed with the drawn indices,
which is what a device `SamplePool` fed the same frames computes — bit for bit: across chunk boundaries, past 2^32 bytes,
inside a CUDA graph and inside the batch-mode loop."""
import ctypes as C
import gc

import numpy as np
import pytest
import torch

from tests.parity_utils import make_config

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def _frame(n, gen, tag=0.0):
    coord = torch.rand(n, 3, device=DEV, generator=gen) * 2 - 1
    label = torch.randn(n, device=DEV, generator=gen) + tag
    weight = torch.where(torch.rand(n, device=DEV, generator=gen) < 0.5, 1.0, -1.0)
    return coord, label, weight


def _equal(got, want):
    return all(torch.equal(g, w) for g, w in zip(got, want))


def _pools(frames, chunk_shift=10):
    from shine_mapping_b200 import synth
    host, dev = synth.HostSamplePool(DEV, chunk_shift=chunk_shift), synth.SamplePool(DEV)
    for f in frames:
        host.append(*f)
        dev.append(*f)
    return host, dev


def test_append_across_chunk_boundaries_equals_concatenation(built_lib):
    """Frames of 0, 1, 31, 32 and 33 samples and frames that straddle 1 to 3 boundaries of 1024-record chunks: after
    every frame, gathering arange(len) returns the concatenation."""
    from shine_mapping_b200 import synth
    gen = torch.Generator(device=DEV).manual_seed(1)
    chunk = 1 << 10
    host, dev = synth.HostSamplePool(DEV, chunk_shift=10), synth.SamplePool(DEV)
    sizes = [0, 1, 31, 32, 33, chunk - 97 - 1, 2, chunk + 5, 2 * chunk + 3, 3 * chunk - 1, 0, chunk, 1]
    crossings = []
    for k, n in enumerate(sizes):
        f = _frame(n, gen, tag=100.0 * k)
        before = len(host)
        host.append(*f)
        dev.append(*f)
        crossings.append((len(host) - 1) // chunk - before // chunk if n else 0)
        assert len(host) == len(dev) == before + n
        if len(host):
            idx = torch.arange(len(host), device=DEV)
            assert _equal(host.gather(idx), (dev.coord_pool, dev.sdf_label_pool, dev.weight_pool)), (k, n)
    assert {1, 2, 3} <= set(crossings), crossings
    assert host.capacity == len(host._chunks) * chunk >= len(host)


@pytest.mark.parametrize("bs", [1, 4096, 65536, 1048576])
def test_get_batch_equals_sample_pool(built_lib, bs):
    """Same frames, same generator seed: HostSamplePool.get_batch == SamplePool.get_batch bit for bit."""
    gen = torch.Generator(device=DEV).manual_seed(2)
    frames = [_frame(n, gen, tag=10.0 * i) for i, n in enumerate((300_001, 1, 777_777, 65_536))]
    host, dev = _pools(frames, chunk_shift=18)
    assert len(host._chunks) == 5
    for seed in (0, 7):
        g1 = torch.Generator(device=DEV).manual_seed(seed)
        g2 = torch.Generator(device=DEV).manual_seed(seed)
        for _ in range(2):
            got, want = host.get_batch(bs, g1), dev.get_batch(bs, g2)
            assert got[0].shape == (bs, 3) and got[1].shape == (bs,) and got[2].shape == (bs,)
            assert _equal(got, want)
    # ordered=False is the order drawn, as on an unsorted SamplePool
    g1, g2 = torch.Generator(device=DEV).manual_seed(3), torch.Generator(device=DEV).manual_seed(3)
    assert _equal(host.get_batch(bs, g1, ordered=False), dev.get_batch(bs, g2, ordered=False))


def test_gather_first_and_last_record_of_every_chunk_and_duplicates(built_lib):
    gen = torch.Generator(device=DEV).manual_seed(4)
    frames = [_frame(n, gen, tag=float(i)) for i, n in enumerate((5000, 1023, 1, 4097))]
    host, dev = _pools(frames, chunk_shift=10)
    n, chunk = len(host), 1 << 10
    first = torch.arange(0, n, chunk, device=DEV)
    last = torch.clamp(first + chunk - 1, max=n - 1)
    idx = torch.cat((first, last, last.flip(0), first, torch.full((33,), n - 1, device=DEV),
                     torch.randint(0, n, (10_000,), device=DEV, generator=gen)))
    idx = torch.cat((idx, idx[torch.randperm(idx.numel(), device=DEV, generator=gen)]))     # every index at least twice
    got = host.gather(idx)
    assert _equal(got, (dev.coord_pool[idx], dev.sdf_label_pool[idx], dev.weight_pool[idx]))


def test_pool_past_four_gigabytes(built_lib):
    """One pool whose records span more than 2^32 bytes (1.4e8 samples, 4.5 GB pinned): the first and last record of every
    chunk and 10^6 random records, against a numpy restatement of the record addressing over the chunks' bytes and
    against the values appended.  The pool is freed at the end."""
    from shine_mapping_b200 import synth
    n, step = 140_000_000, 1 << 24
    pool = synth.HostSamplePool(DEV)
    shift = pool.chunk_shift

    def values(i):                  # exact in fp32: i % 1000003 < 2^24, i // 1000003 <= 140
        coord = torch.stack(((i % 1000003).float(), (i // 1000003).float(), (i & 255).float()), 1)
        return coord, (i % 65521).float(), torch.where(i % 2 == 0, 1.0, -1.0)

    try:
        for b in range(0, n, step):
            pool.append(*values(torch.arange(b, min(n, b + step), device=DEV)))
        assert len(pool) == n and n * 32 > 2 ** 32
        torch.cuda.synchronize()
        starts = torch.arange(0, n, 1 << shift, device=DEV)
        gen = torch.Generator(device=DEV).manual_seed(5)
        idx = torch.cat((starts, torch.clamp(starts + (1 << shift) - 1, max=n - 1), torch.tensor([n - 1], device=DEV),
                         torch.randint(0, n, (1_000_000,), device=DEV, generator=gen)))
        got = pool.gather(idx)
        assert _equal(got, values(idx))
        # numpy: record i is floats [0:5] of row (i & (2^shift - 1)) of chunk i >> shift
        ih = idx.cpu().numpy()
        want = np.empty((ih.size, 5), np.float32)
        for c in np.unique(ih >> shift):
            sel = (ih >> shift) == c
            rows = pool._chunks[int(c)].numpy().reshape(-1, 8)
            want[sel] = rows[ih[sel] & ((1 << shift) - 1), :5]
        assert np.array_equal(got[0].cpu().numpy(), want[:, :3])
        assert np.array_equal(got[1].cpu().numpy(), want[:, 3]) and np.array_equal(got[2].cpu().numpy(), want[:, 4])
        assert (ih >= 2 ** 27).sum() > 10_000                         # records beyond byte 2^32
    finally:
        del pool
        gc.collect()
        torch.cuda.synchronize()
        torch._C._host_emptyCache()                                   # hand the pinned chunks back to the system


def test_get_batch_in_a_cuda_graph(built_lib):
    """A captured get_batch draws new indices at every replay; each batch equals the eager gather of the indices that
    replay drew (and the device pool's indexing)."""
    gen = torch.Generator(device=DEV).manual_seed(6)
    host, dev = _pools([_frame(n, gen) for n in (40_000, 12_345)], chunk_shift=12)
    bs = 4096
    side = torch.cuda.Stream(device=DEV)
    side.wait_stream(torch.cuda.current_stream(DEV))
    with torch.cuda.stream(side):
        host.get_batch(bs)
    torch.cuda.current_stream(DEV).wait_stream(side)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        out = host.get_batch(bs)
    idx = host.last_index
    seen = []
    for _ in range(2):
        graph.replay()
        torch.cuda.synchronize()
        i, batch = idx.clone(), [t.clone() for t in out]
        assert _equal(batch, host.gather(i))
        assert _equal(batch, (dev.coord_pool[i], dev.sdf_label_pool[i], dev.weight_pool[i]))
        seen.append(i)
    assert not torch.equal(seen[0], seen[1])


def _loop_run(cfg, frames, make_pool, monkeypatch, use_cuda_graph):
    from shine_mapping_b200 import Decoder, FeatureOctree, SdfTrainer
    from shine_mapping_b200.batch_loop import run_shine_mapping_batch
    torch.manual_seed(3)
    octree, decoder = FeatureOctree(cfg), Decoder(cfg)
    pool = make_pool()
    for coord, label, weight, _ in frames:
        octree.update(coord[weight > 0, :])
        pool.append(coord, label, weight)
    batches = []
    name = "forward_backward_eikonal" if cfg.ekional_loss_on else "forward_backward"
    step = getattr(SdfTrainer, name)

    def recorded_step(self, coord, sdf_label, weight, *a, **kw):
        batches.append(torch.cat((coord.reshape(-1), sdf_label, weight)))
        return step(self, coord, sdf_label, weight, *a, **kw)
    if not use_cuda_graph:          # a graph's replays do not call back into Python
        monkeypatch.setattr(SdfTrainer, name, recorded_step)
    out = run_shine_mapping_batch(cfg, octree, decoder, pool, log_every=1, use_cuda_graph=use_cuda_graph)
    monkeypatch.undo()
    return out, batches, pool, octree, decoder


def _step_grads(trainer, pool, eikonal, seed):
    """Table and decoder gradients and loss of one step on the batch `pool` draws with a generator seeded `seed`."""
    trainer.zero_grad()
    coord, label, weight = pool.get_batch(trainer.config.bs, torch.Generator(device=DEV).manual_seed(seed))
    if eikonal:
        loss = torch.stack(trainer.forward_backward_eikonal(coord, label, weight))
    else:
        loss = trainer.forward_backward(coord, label, weight).reshape(1)
    tables = trainer.flat_grad[:trainer.flat_grad.numel() - trainer.dec_flat.numel()]
    return tables.clone(), trainer.dec_flat.clone(), loss.clone()


@pytest.mark.parametrize("eikonal", [False, True])
@pytest.mark.parametrize("graphed", [False, True])
def test_batch_loop_on_host_pool_matches_device_pool(built_lib, monkeypatch, eikonal, graphed):
    """run_shine_mapping_batch for 50 iterations on a host pool and on a device pool with the same frames and seeds: the
    same batches (compared on the eager loop; a graph's replays do not call back into Python) and losses within the
    parity tolerance (relative 2e-5).  Then, from the map and decoder the host-pool run trained, the gradients of one more
    step on the batch each pool draws for the same generator state agree within 2e-4 * max|ref|.  The training kernels
    add with fp32 atomics in no fixed order, so two runs differ in the last bits even on identical batches, and 50 Adam
    steps carry that into the tables: the two runs' own last-step gradients are not compared, because they come from two
    slightly different maps."""
    from shine_mapping_b200 import SdfTrainer, synth
    cfg = make_config(3, device=DEV, bs=4096, lr=0.01, iters=50, ekional_loss_on=eikonal, weight_e=0.1,
                      continual_learning_reg=False, window_replay_on=False)
    frames = synth.generate_scans(cfg, 256, 2, seed=42, device=DEV)
    torch.manual_seed(11)
    a, ba, host, octree, decoder = _loop_run(cfg, frames, lambda: synth.HostSamplePool(DEV), monkeypatch, graphed)
    assert isinstance(host, synth.HostSamplePool)
    torch.manual_seed(11)
    b, bb, device_pool, _, _ = _loop_run(cfg, frames, lambda: synth.SamplePool(DEV), monkeypatch, graphed)
    la, lb = [a["losses"][i] for i in range(50)], [b["losses"][i] for i in range(50)]
    drift = max(abs(x - y) / abs(y) for x, y in zip(la, lb))
    print(f"eikonal={eikonal} graphed={graphed}: loss {la[0]:.6f} -> {la[-1]:.6f}, max relative difference {drift:.3e}")
    assert all(np.isfinite(la)) and la[-1] < la[0]
    assert drift <= 2e-5, (la, lb)
    if not graphed:
        assert len(ba) == len(bb) == 50
        assert all(torch.equal(x, y) for x, y in zip(ba, bb))
    trainer = SdfTrainer(cfg, octree, decoder)
    got, want = _step_grads(trainer, host, eikonal, 99), _step_grads(trainer, device_pool, eikonal, 99)
    for g, w in zip(got[:2], want[:2]):
        assert float(w.abs().max()) > 0
        assert float((g - w).abs().max()) <= 2e-4 * float(w.abs().max()) + 1e-10
    assert torch.allclose(got[2], want[2], rtol=2e-5, atol=0)


CLI_YAML = """
setting: {name: "synthetic_batch", begin_frame: 0, end_frame: 3, every_frame: 1, device: "cuda", gpu_id: "0"%s}
process: {min_range_m: 3.0, pc_radius_m: 30.0, min_z_m: -3.5, rand_downsample: False, vox_down_m: 0.05, rand_down_r: 0.2}
sampler: {surface_sample_range_m: 0.3, surface_sample_n: 3, free_sample_begin_ratio: 0.3, free_sample_end_dist_m: 0.8,
          free_sample_n: 3}
octree: {leaf_vox_size: 0.3, tree_level_world: 12, tree_level_feat: 3, feature_dim: 8, poly_int_on: True,
         octree_from_surface_samples: True}
decoder: {mlp_level: 2, mlp_hidden_dim: 32, freeze_after_frame: 0}
loss: {ray_loss: False, main_loss_type: sdf_bce, sigma_sigmoid_m: 0.1, loss_weight_on: False, behind_dropoff_on: False,
       ekional_loss_on: True, weight_e: 0.1}
continual: {continual_learning_reg: False, lambda_forget: 0, window_replay_on: False, window_radius_m: 0}
optimizer: {iters: 20, batch_size: 4096, learning_rate: 0.05, weight_decay: 1e-7}
"""


@pytest.mark.parametrize("limit", [2, None])
def test_command_line_picks_the_pool_by_the_reference_rule(built_lib, tmp_path, capsys, limit):
    from shine_mapping_b200.batch_loop import main
    y = tmp_path / "batch.yaml"
    y.write_text(CLI_YAML % (f", pc_count_gpu_limit: {limit}" if limit is not None else ""))
    main([str(y), "--synthetic-azimuth", "128", "--frames", "3", "--iters", "20"])
    out = capsys.readouterr().out
    if limit == 2:
        assert "Sample pool: HostSamplePool in pinned host memory" in out, out
    else:
        assert "Sample pool: SamplePool in device memory" in out, out
    assert "'loss_last':" in out


def test_host_pool_rejects_bad_input(built_lib):
    from shine_mapping_b200 import _abi, synth
    gen = torch.Generator(device=DEV).manual_seed(8)
    pool = synth.HostSamplePool(DEV, chunk_shift=10)
    with pytest.raises(ValueError):
        pool.get_batch(16)                                                     # empty pool
    coord, label, weight = _frame(100, gen)
    with pytest.raises(_abi.ShineB200Error):
        pool.append(coord.cpu(), label.cpu(), weight.cpu())                   # CPU frame
    with pytest.raises(ValueError):
        pool.append(coord, label[:99], weight)                                 # mismatched lengths
    assert len(pool) == 0
    pool.append(coord, label, weight)
    with pytest.raises(ValueError):
        pool.get_batch(16, ordered=True)
    with pytest.raises(NotImplementedError):
        pool.sort_morton()
    with pytest.raises(ValueError):
        synth.HostSamplePool(DEV, chunk_shift=4)
    # the ABI: negative codes, nothing launched
    lib = built_lib
    desc = pool._descriptor()
    idx = torch.zeros(4, dtype=torch.int64, device=DEV)
    outs = [torch.full((4, 3), 7.0, device=DEV), torch.full((4,), 7.0, device=DEV), torch.full((4,), 7.0, device=DEV)]
    st = _abi.stream_ptr(DEV)

    def gather(d=desc, i=idx.data_ptr(), n=4, c=outs[0].data_ptr()):
        return lib.shine_host_pool_gather(C.byref(d), i, n, c, outs[1].data_ptr(), outs[2].data_ptr(), st)
    assert gather(i=None) == gather(c=None) == gather(n=-1) == -1
    idx_host = idx.cpu()
    assert gather(i=idx_host.data_ptr()) == -1                                # indices in host memory
    for shift in (4, 32):
        assert gather(d=_abi.ShineHostPool(desc.chunks, shift, desc.num_chunks, desc.size)) == -1
    assert lib.shine_host_pool_append(C.byref(desc), 0, coord.data_ptr(), label.data_ptr(), weight.data_ptr(), -1,
                                      st) == -1
    assert lib.shine_host_pool_append(C.byref(desc), 1000, coord.data_ptr(), label.data_ptr(), weight.data_ptr(), 100,
                                      st) == -1                               # past the last chunk
    torch.cuda.synchronize()
    assert all(bool((t == 7.0).all()) for t in outs)
    assert gather() == 0
    torch.cuda.synchronize()
    assert torch.equal(outs[1], label[:1].expand(4))
