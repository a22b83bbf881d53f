"""The replay sample pool on the GPU: `synth.ReplayPool.add_frame` (one launch of `shine_pool_window_append`) against the
oracle of the reference's window filter and concatenation (dataset/lidar_dataset.py:235-271, tests/replay_oracle.py),
bit for bit, at every tile boundary, at scale, along a synthetic drive and inside the incremental loop."""
import ctypes as C

import numpy as np
import pytest
import torch

from tests.parity_utils import make_config
from tests.replay_oracle import OraclePool, replay_pool_update, window_mask

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
TILE = 2048                                   # samples per tile of the kernel
ORIGIN = (0.0371, -0.0113, 0.0042)


def _assert_pool_equals(pool, want):
    c, l, w = want
    assert len(pool) == l.shape[0]
    assert torch.equal(pool.coord_pool, c) and torch.equal(pool.sdf_label_pool, l) and torch.equal(pool.weight_pool, w)


def _runs(n, gen, nan_every=0):
    """n samples in runs of 1 to 3 tiles that lie alternately near the origin (distance < 0.5) and far (1 to 2), so that a
    0.75 window drops scattered runs across many tiles; labels are distinct tags, weights +-1."""
    o = torch.tensor(ORIGIN, device=DEV)
    lengths = torch.randint(1, 3 * TILE, (n // TILE + 2,), device=DEV, generator=gen).cpu().tolist()
    far = torch.zeros(n, dtype=torch.bool, device=DEV)
    pos, flip = 0, False
    for length in lengths:
        if pos >= n:
            break
        far[pos:pos + length] = flip
        pos, flip = pos + length, not flip
    d = torch.randn(n, 3, device=DEV, generator=gen)
    d = d / d.norm(dim=1, keepdim=True).clamp(min=1e-6)
    dist = torch.rand(n, device=DEV, generator=gen)
    dist = torch.where(far, 1.0 + dist, 0.5 * dist)
    coord = (o + d * dist[:, None]).contiguous()
    if nan_every and n:
        coord[::nan_every, 1] = float("nan")
    label = torch.arange(n, device=DEV, dtype=torch.float32) + float(torch.randint(0, 1 << 20, (1,), generator=gen, device=DEV))
    weight = torch.where(torch.rand(n, device=DEV, generator=gen) < 0.5, 1.0, -1.0)
    return coord, label, weight


def _radius(kind, coord):
    if kind == "all":
        return 1e30
    if kind == "none":
        return 0.0
    if kind == "runs":
        return 0.75
    if coord.shape[0] == 0:                    # "half"
        return 0.5
    o = torch.tensor(ORIGIN, device=DEV)
    return float((coord - o).norm(dim=1).nan_to_num(0.0).median())


@pytest.mark.parametrize("old", [0, 1, TILE - 1, TILE, TILE + 1, 100_003, 3_000_000])
def test_add_frame_equals_oracle(built_lib, old):
    """Every new-frame size, window (keep all, keep none, about half, scattered runs) and capacity (exact, with slack,
    too small: the pool grows first)."""
    from shine_mapping_b200 import synth
    gen = torch.Generator(device=DEV).manual_seed(old + 1)
    old_c, old_l, old_w = _runs(old, gen, nan_every=997)
    for n_new in (0, 1, 777, 200_000):
        new = _runs(n_new, gen)
        for kind in ("all", "none", "half", "runs"):
            r = _radius(kind, old_c)
            want = replay_pool_update(old_c, old_l, old_w, *new, ORIGIN, r)
            for capacity in (old + n_new, old + n_new + 12_345, old):
                pool = synth.ReplayPool(DEV, capacity=capacity)
                pool.add_frame(old_c, old_l, old_w)
                pool.add_frame(*new, ORIGIN, r)
                assert pool.capacity >= old + n_new
                _assert_pool_equals(pool, want)
            if kind == "half" and old > 100:
                assert 0.3 * old < len(want[1]) - n_new < 0.7 * old
            if kind == "runs" and old > 100_000:
                kept = window_mask(old_c, ORIGIN, r)
                runs = int((kept[1:] != kept[:-1]).sum())
                assert runs > old // (3 * TILE), runs                    # drops scattered over many tiles


def test_several_frames_compact_an_already_compacted_pool(built_lib):
    """Frames of various sizes with a moving origin: each launch compacts the output of the previous ones."""
    from shine_mapping_b200 import synth
    gen = torch.Generator(device=DEV).manual_seed(11)
    pool, oracle = synth.ReplayPool(DEV), OraclePool(DEV)
    sizes = []
    for f in range(20):
        n = int(torch.randint(1, 300_000, (1,), generator=gen, device=DEV))
        c, l, w = _runs(n, gen)
        c = c + torch.tensor([0.05 * f, 0.0, 0.0], device=DEV)
        origin = (ORIGIN[0] + 0.05 * f, ORIGIN[1], ORIGIN[2])
        r = 0.9 if f % 5 else 1e30
        pool.add_frame(c, l, w, origin, r)
        oracle.add_frame(c, l, w, origin, r)
        _assert_pool_equals(pool, (oracle._pool.coord_pool, oracle._pool.sdf_label_pool, oracle._pool.weight_pool))
        sizes.append(len(pool))
    assert min(sizes) > 0 and any(b < a for a, b in zip(sizes, sizes[1:]))       # some frames shrank the pool


def _fp32_distance(p, o):
    d = p - o
    return np.sqrt((d[:, 0] * d[:, 0] + d[:, 1] * d[:, 1]) + d[:, 2] * d[:, 2])


def test_window_boundary_is_strict(built_lib):
    """Samples whose fp32 distance is exactly r are dropped, those at nextafter(r, 0) are kept; against the reference's own
    `(coord - origin).norm(2, dim=-1) < r` the kernel differs only on samples within 2 ulp of r (distance in fp64)."""
    from shine_mapping_b200 import synth
    scale = 1.0 / (0.3 * 2 ** 11)                      # kitti_incre_replay: leaf 0.3 m, world level 12
    r_scaled = 50.0 * scale
    r32 = np.float32(r_scaled)
    below = np.nextafter(r32, np.float32(0))
    o = np.asarray(ORIGIN, dtype=np.float32)
    rng = np.random.default_rng(5)
    u = rng.normal(size=(2_000_000, 3))
    u /= np.linalg.norm(u, axis=1, keepdims=True)
    cand = (o.astype(np.float64) + u * float(r32)).astype(np.float32)
    dist = _fp32_distance(cand, o)
    at_r, at_below = cand[dist == r32], cand[dist == below]
    assert len(at_r) > 100 and len(at_below) > 100
    coord = torch.from_numpy(np.concatenate([at_r, at_below])).to(DEV)
    label = torch.arange(coord.shape[0], device=DEV, dtype=torch.float32)
    pool = synth.ReplayPool(DEV)
    pool.add_frame(coord, label, torch.ones_like(label))
    pool.add_frame(torch.empty(0, 3, device=DEV), torch.empty(0, device=DEV), torch.empty(0, device=DEV), ORIGIN, r_scaled)
    assert torch.equal(pool.sdf_label_pool, label[len(at_r):])

    # a pool around the window's edge: kernel == oracle exactly; against torch's norm only near-ties differ
    n = 3_000_000
    gen = torch.Generator(device=DEV).manual_seed(9)
    d = torch.randn(n, 3, device=DEV, generator=gen)
    d = d / d.norm(dim=1, keepdim=True)
    od = torch.tensor(ORIGIN, device=DEV)
    coord = (od + d * (float(r32) * (0.999 + 0.002 * torch.rand(n, 1, device=DEV, generator=gen)))).contiguous()
    label = torch.arange(n, device=DEV, dtype=torch.float32)
    pool = synth.ReplayPool(DEV)
    pool.add_frame(coord, label, torch.ones_like(label))
    pool.add_frame(torch.empty(0, 3, device=DEV), torch.empty(0, device=DEV), torch.empty(0, device=DEV), ORIGIN, r_scaled)
    kept = torch.zeros(n, dtype=torch.bool, device=DEV)
    kept[pool.sdf_label_pool.long()] = True
    assert torch.equal(kept, window_mask(coord, ORIGIN, r_scaled))
    ref = (coord - od).norm(2, dim=-1) < r_scaled                           # lidar_dataset.py:238-239 as written
    diff = (kept != ref).nonzero().flatten()
    d64 = (coord[diff].double() - od.double()).norm(dim=1)
    ulp = float(np.spacing(r32))
    assert bool(((d64 - float(r32)).abs() <= 2 * ulp).all()), (d64 - float(r32)) / ulp
    assert 0.3 * n < int(kept.sum()) < 0.7 * n


def _drive_config(**kw):
    # config/kitti/kitti_incre_replay.yaml: leaf 0.3 m, world level 12, 3 levels, range 3-30 m, window 50 m
    base = dict(world_level=12, leaf_vox=0.3, device=DEV, min_range=3.0, pc_radius=30.0, surface_sample_range_m=0.3,
                surface_sample_n=3, free_sample_begin_ratio=0.3, free_sample_end_dist_m=1.0, free_sample_n=3,
                continual_learning_reg=False, lambda_forget=0.0, window_replay_on=True, window_radius=50.0, bs=2048,
                lr=0.01, iters=40, freeze_after_frame=20)
    base.update(kw)
    return make_config(3, **base)


def _drive(cfg, n_frames, step_m, azimuth=256, seed=3):
    from shine_mapping_b200 import synth
    scans = synth.generate_scans(cfg, azimuth, n_frames, step_m, seed=seed, device=DEV)
    return [(c, l, w, torch.tensor([f * step_m, 0.0, 0.0]) * cfg.scale) for f, (c, l, w, _) in enumerate(scans)]


def test_synthetic_drive_pool_equals_oracle_and_plateaus(built_lib):
    """32 frames 5 m apart with a 50 m window and a 30 m scan radius: the first frames leave the window after a few
    frames; the pool equals the oracle's after every frame, grows, then stays about the same size."""
    from shine_mapping_b200 import synth
    cfg = _drive_config()
    frames = _drive(cfg, 32, 5.0)
    r = cfg.window_radius * cfg.scale
    pool, oracle = synth.ReplayPool(DEV), OraclePool(DEV)
    sizes, total = [], 0
    for c, l, w, origin in frames:
        pool.add_frame(c, l, w, origin, r)
        oracle.add_frame(c, l, w, origin, r)
        _assert_pool_equals(pool, (oracle._pool.coord_pool, oracle._pool.sdf_label_pool, oracle._pool.weight_pool))
        sizes.append(len(pool))
        total += c.shape[0]
    print("pool sizes:", sizes)
    assert sizes[3] > 3 * sizes[0]                                  # grows while every frame is inside the window
    tail = np.asarray(sizes[-10:], dtype=np.float64)
    assert tail.max() - tail.min() <= 0.1 * tail.mean(), sizes     # plateau
    assert sizes[-1] < 0.6 * total


@pytest.mark.parametrize("eikonal", [False, True])
def test_loop_with_replay_pool_matches_the_oracle_pool(built_lib, monkeypatch, eikonal):
    """run_shine_mapping_incremental with a ReplayPool and with the oracle's pool (same seed): identical pools and
    identical batches at every step.  The losses are not bit-identical: the training kernels sum the loss and the table
    gradients with fp32 atomics in no fixed order, so two runs of the same loop on the same batches differ in the last
    bits, and Adam carries that difference from step to step.  The first loss is compared closely, later ones loosely."""
    from shine_mapping_b200 import Decoder, FeatureOctree, SdfTrainer, synth
    from shine_mapping_b200.incre_loop import run_shine_mapping_incremental
    cfg = _drive_config(ekional_loss_on=eikonal, weight_e=0.1)
    frames = _drive(cfg, 8, 5.0, azimuth=128)
    name = "forward_backward_eikonal" if eikonal else "forward_backward"
    step = getattr(SdfTrainer, name)
    runs = []
    for make_pool in (lambda: synth.ReplayPool(DEV), lambda: OraclePool(DEV)):
        batches = []

        def recorded(self, coord, sdf_label, weight, *a, **kw):
            batches.append(torch.cat((coord.reshape(-1), sdf_label, weight)))
            return step(self, coord, sdf_label, weight, *a, **kw)
        monkeypatch.setattr(SdfTrainer, name, recorded)
        torch.manual_seed(1)
        octree, decoder = FeatureOctree(cfg), Decoder(cfg)
        hist = run_shine_mapping_incremental(cfg, octree, decoder, frames, pool=make_pool())
        runs.append((hist, batches))
    (h1, b1), (h2, b2) = runs
    assert len(b1) == len(b2) == 8 * cfg.iters
    assert all(torch.equal(x, y) for x, y in zip(b1, b2))
    assert [h["pool"] for h in h1] == [h["pool"] for h in h2]
    assert h1[0]["loss_first"] == pytest.approx(h2[0]["loss_first"], rel=1e-5)    # same batch, same initial state
    for x, y in zip(h1, h2):        # later frames: the two runs' tables drift apart through the atomics' order only
        assert x["rows"] == y["rows"]
        assert x["loss_first"] == pytest.approx(y["loss_first"], rel=5e-2)
        assert x["loss_last"] == pytest.approx(y["loss_last"], rel=5e-2)
        if eikonal:
            assert np.isfinite(x["eik_last"]) and np.isfinite(y["eik_last"])
    assert cfg.loss_reduction == "mean"
    assert all(h["bce_last"] < h["bce_first"] for h in h1), h1
    cfg.continual_learning_reg = True
    with pytest.raises(ValueError):
        run_shine_mapping_incremental(cfg, FeatureOctree(cfg), Decoder(cfg), frames, pool=synth.ReplayPool(DEV))


REPLAY_YAML = """
setting: {name: "synthetic_incre_replay", begin_frame: 0, end_frame: 100, every_frame: 1, device: "cuda", gpu_id: "0"}
process: {min_range_m: 3.0, pc_radius_m: 30.0, min_z_m: -3.5, rand_downsample: False, vox_down_m: 0.08, rand_down_r: 0.2}
sampler: {surface_sample_range_m: 0.3, surface_sample_n: 3, free_sample_begin_ratio: 0.3, free_sample_end_dist_m: 1.0,
          free_sample_n: 3}
octree: {leaf_vox_size: 0.3, tree_level_world: 12, tree_level_feat: 3, feature_dim: 8, poly_int_on: True,
         octree_from_surface_samples: True}
decoder: {mlp_level: 2, mlp_hidden_dim: 32, freeze_after_frame: 20}
loss: {ray_loss: False, main_loss_type: sdf_bce, sigma_sigmoid_m: 0.1, loss_weight_on: False, behind_dropoff_on: False,
       ekional_loss_on: True, weight_e: 0.1}
continual: {continual_learning_reg: False, lambda_forget: 0, window_replay_on: True, window_radius_m: 50.0}
optimizer: {iters: 100, batch_size: 8192, learning_rate: 0.01, weight_decay: 0}
"""


def test_command_line_runs_a_replay_config(built_lib, tmp_path, capsys):
    from shine_mapping_b200.incre_loop import main
    y = tmp_path / "incre_replay.yaml"
    y.write_text(REPLAY_YAML)
    hist = main([str(y), "--synthetic-azimuth", "128", "--frames", "30", "--frame-step-m", "5", "--iters", "5"])
    out = capsys.readouterr().out
    assert "replay (window 50.0 m)" in out and "'pool':" in out
    sizes = [h["pool"] for h in hist]
    assert len(sizes) == 30 and sizes[3] > 3 * sizes[0]
    tail = np.asarray(sizes[-10:], dtype=np.float64)
    assert tail.max() - tail.min() <= 0.1 * tail.mean(), sizes
    assert all(np.isfinite(h["loss_last"]) and np.isfinite(h["eik_last"]) for h in hist)


def test_thirty_million_sample_pool(built_lib):
    """A 30 M-sample pool and an 800 k-sample frame, a window that drops about 5 %: equal to the oracle."""
    from shine_mapping_b200 import synth
    n, n_new = 30_000_000, 800_000
    gen = torch.Generator(device=DEV).manual_seed(30)
    o = torch.tensor(ORIGIN, device=DEV)
    coord = (o + (torch.rand(n, 3, device=DEV, generator=gen) - 0.5) * 0.2).contiguous()
    label = torch.randn(n, device=DEV, generator=gen)
    weight = torch.where(torch.rand(n, device=DEV, generator=gen) < 0.5, 1.0, -1.0)
    new = (o + (torch.rand(n_new, 3, device=DEV, generator=gen) - 0.5) * 0.2, torch.randn(n_new, device=DEV, generator=gen),
           torch.ones(n_new, device=DEV))
    r = float((coord[::97] - o).norm(dim=1).quantile(0.95))
    want = replay_pool_update(coord, label, weight, *new, ORIGIN, r)
    pool = synth.ReplayPool(DEV, capacity=n + n_new)
    pool.add_frame(coord, label, weight)
    del coord, label, weight
    pool.add_frame(*new, ORIGIN, r)
    _assert_pool_equals(pool, want)
    assert 0.9 * n < len(pool) - n_new < 0.99 * n


def test_pool_window_append_rejects_bad_arguments(built_lib):
    from shine_mapping_b200 import _abi
    lib = built_lib
    cap, n_new = 4096, 100
    buf = [torch.zeros(cap, 3, device=DEV), torch.zeros(cap, device=DEV), torch.zeros(cap, device=DEV)]
    frame = [torch.zeros(n_new, 3, device=DEV), torch.zeros(n_new, device=DEV), torch.zeros(n_new, device=DEV)]
    size_out = torch.full((1,), -7, dtype=torch.int64, device=DEV)
    nbytes = int(lib.shine_pool_scratch_bytes(cap))
    scratch = torch.zeros(nbytes, dtype=torch.uint8, device=DEV)
    host = np.zeros((n_new, 3), dtype=np.float32)                    # pageable host memory: the kernel cannot read it
    assert lib.shine_pool_scratch_bytes(-1) == -1 and lib.shine_pool_scratch_bytes(0) > 0

    def call(size=10, capacity=cap, pool=True, pool_coord=None, coord=None, label=None, n=n_new, out=True, scr=True,
             scr_bytes=nbytes):
        d = _abi.ShineSamplePool(pool_coord if pool_coord is not None else buf[0].data_ptr(), buf[1].data_ptr(),
                                 buf[2].data_ptr(), size, capacity)
        return lib.shine_pool_window_append(
            C.byref(d) if pool else None, coord if coord is not None else frame[0].data_ptr(),
            label if label is not None else frame[1].data_ptr(), frame[2].data_ptr(), n, 0.0, 0.0, 0.0, 1.0,
            size_out.data_ptr() if out else None, scratch.data_ptr() if scr else None, scr_bytes,
            _abi.stream_ptr(DEV))

    assert call() == 0
    torch.cuda.synchronize()
    assert int(size_out) == 10 + n_new
    bad = {
        "no pool": dict(pool=False), "null pool buffer": dict(pool_coord=0), "null frame coord": dict(coord=0),
        "null size_out": dict(out=False), "null scratch": dict(scr=False), "negative size": dict(size=-1),
        "negative capacity": dict(capacity=-1), "negative n_new": dict(n=-1), "size above capacity": dict(size=cap + 1),
        "size + n_new above capacity": dict(size=cap - n_new + 1), "scratch too small": dict(scr_bytes=int(lib.shine_pool_scratch_bytes(10 + n_new)) - 1),
        "frame in pageable host memory": dict(coord=host.ctypes.data), "pool in pageable host memory":
            dict(pool_coord=np.zeros((cap, 3), np.float32).ctypes.data),
    }
    if torch.cuda.device_count() > 1:
        other = torch.zeros(n_new, device="cuda:1")
        bad["frame on another device"] = dict(label=other.data_ptr())
    for what, kw in bad.items():
        assert call(**kw) == -1, what
    torch.cuda.synchronize()
    assert int(size_out) == 10 + n_new                                # nothing was launched
