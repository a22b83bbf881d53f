"""Saved maps on the GPU: the reference-written fixture through the kernels, checkpoints of both mapping loops loaded again
(`load_model`, `python -m shine_mapping_b200.mesher`), and the `save_map` export kernel (`shine_mesh_export_points`) against
a torch restatement on the same chunk buffers."""
import ctypes as C
import json
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = os.path.join(ROOT, "tests", "golden")

YAML = """setting:
  name: "test"
  device: "{dev}"
  load_model: {load_model}
  model_path: "{model_path}"
octree:
  leaf_vox_size: 0.3
  tree_level_world: 12
  tree_level_feat: 3
sampler:
  surface_sample_range_m: 0.3
  free_sample_end_dist_m: 1.0
process:
  min_range_m: 2.0
  pc_radius_m: 25.0
continual:
  continual_learning_reg: {reg}
optimizer:
  iters: {iters}
  batch_size: 8192
eval:
  vis_freq_iters: {freq}
  save_freq_iters: {freq}
  mesh_freq_frame: 3
  mc_res_m: 0.2
  mc_with_octree: {octree_mode}
  save_map: {save_map}
"""


@pytest.fixture(scope="module", autouse=True)
def _lib(built_lib):
    assert torch.cuda.is_available()
    return built_lib


def _config_file(tmp_path, name="config.yaml", **kw):
    args = dict(dev=DEV, load_model=False, model_path="/", reg=True, iters=300, freq=300, octree_mode=True, save_map=False)
    args.update(kw)
    path = str(tmp_path / name)
    with open(path, "w") as fh:
        fh.write(YAML.format(**args))
    return path


def _config(path):
    from shine_mapping_b200.config import SHINEConfig
    cfg = SHINEConfig()
    cfg.load(path)
    return cfg


def _fixed_points(n=100_000):
    g = torch.Generator().manual_seed(11)
    return ((torch.rand(n, 3, generator=g) - 0.5) * torch.tensor([0.06, 0.03, 0.006])).to(DEV)


@pytest.fixture(scope="module")
def batch_run(tmp_path_factory):
    """300 iterations of the batch loop's command line on a synthetic map, with --run-path: checkpoint, mesh, SDF map."""
    from shine_mapping_b200 import batch_loop, sdf_infer
    tmp = tmp_path_factory.mktemp("batch_run")
    cfg_path = _config_file(tmp, save_map=True)
    run = str(tmp / "run")
    captured = {}
    real = batch_loop.run_shine_mapping_batch

    def spy(config, octree, decoder, *a, **kw):
        out = real(config, octree, decoder, *a, **kw)
        captured.update(octree=octree, decoder=decoder, pred=sdf_infer(octree, decoder, _fixed_points()).cpu())
        return out
    batch_loop.run_shine_mapping_batch = spy
    try:
        batch_loop.main([cfg_path, "--synthetic-azimuth", "512", "--frames", "6", "--run-path", run])
    finally:
        batch_loop.run_shine_mapping_batch = real
    return dict(captured, config=cfg_path, run=run, tmp=tmp, checkpoint=os.path.join(run, "model", "model_iter_300.pth"),
                mesh=os.path.join(run, "mesh", "mesh_iter_300.ply"), sdf_map=os.path.join(run, "map", "sdf_map_iter_300.ply"))


# ---- the reference's checkpoint through the kernels ------------------------------------------------------------------

def test_reference_fixture_on_the_gpu():
    from shine_mapping_b200 import Decoder, checkpoint, sdf_infer
    from shine_mapping_b200.config import SHINEConfig
    g = np.load(os.path.join(GOLD, "ref_checkpoint_l3.npz"))
    cfg = SHINEConfig(device=DEV, **json.loads(str(g["cfg_json"])))
    state, octree = checkpoint.load_checkpoint(os.path.join(GOLD, "ref_checkpoint_l3.pt"), cfg, DEV)
    dec = Decoder(cfg)
    dec.load_state_dict(state)
    coord = torch.from_numpy(g["coord"]).to(DEV)
    idx = octree.get_indices(coord)
    assert len(idx) == cfg.tree_level_feat
    for i, got in enumerate(idx):
        assert np.array_equal(got.cpu().numpy(), g[f"exp_indices_{i}"].astype(np.int64))
    assert (g["exp_indices_0"][:, 0] < 0).any() and (g["exp_indices_0"][:, 0] >= 0).sum() > 1000
    feat = octree.query_feature(coord).detach().cpu().numpy()
    assert np.abs(feat - g["exp_feature"]).max() <= 1e-6
    pred = sdf_infer(octree, dec, coord).cpu().numpy()
    assert np.all(np.abs(pred - g["exp_pred"]) <= 2e-5 + 1e-5 * np.abs(g["exp_pred"]))     # parity_utils.compare_step's bound
    # a frame added to the loaded map: append-only, like on a map grown here
    rows = [p.shape[0] for p in octree.hier_features]
    old = [p.data[:-1].clone() for p in octree.hier_features]
    octree.update(coord[:500] + 0.01)
    assert all(p.shape[0] > r for p, r in zip(octree.hier_features, rows))
    assert all(torch.equal(p.data[:o.shape[0]], o) for p, o in zip(octree.hier_features, old))
    for i, got in enumerate(octree.get_indices(coord)):
        want = g[f"exp_indices_{i}"].astype(np.int64)
        hit = want[:, 0] >= 0
        assert np.array_equal(got.cpu().numpy()[hit], want[hit])


# ---- round trip ------------------------------------------------------------------------------------------------------

_FRESH = """
import sys, torch
sys.path.insert(0, {root!r})
from shine_mapping_b200 import Decoder, checkpoint, sdf_infer
from shine_mapping_b200.config import SHINEConfig
cfg = SHINEConfig(); cfg.load({config!r})
state, octree = checkpoint.load_checkpoint({ckpt!r}, cfg, {dev!r})
dec = Decoder(cfg); dec.load_state_dict(state)
g = torch.Generator().manual_seed(11)
pts = ((torch.rand(100000, 3, generator=g) - 0.5) * torch.tensor([0.06, 0.03, 0.006])).to({dev!r})
torch.save(sdf_infer(octree, dec, pts).cpu(), {out!r})
"""


def test_round_trip_in_a_fresh_process(batch_run):
    from shine_mapping_b200.mesher import read_ply
    out = str(batch_run["tmp"] / "pred.pt")
    script = _FRESH.format(root=ROOT, config=batch_run["config"], ckpt=batch_run["checkpoint"], dev=DEV, out=out)
    subprocess.run([sys.executable, "-c", script], check=True, cwd=ROOT)
    pred = torch.load(out)
    assert batch_run["pred"].unique().numel() > 10_000                  # the points see the map
    assert torch.equal(pred, batch_run["pred"])                         # bit-identical
    mesh = str(batch_run["tmp"] / "again.ply")
    env = dict(os.environ, PYTHONPATH=ROOT + os.pathsep + os.environ.get("PYTHONPATH", ""))
    subprocess.run([sys.executable, "-m", "shine_mapping_b200.mesher", batch_run["config"], batch_run["checkpoint"], "--out",
                    mesh], check=True, cwd=ROOT, env=env)
    v0, f0, _ = read_ply(batch_run["mesh"])
    v1, f1, _ = read_ply(mesh)
    assert f0.shape[0] > 100 and f1.shape == f0.shape
    key = lambda v: v[np.lexsort(v.T[::-1])]
    assert np.array_equal(key(v0), key(v1))
    # another resolution, and a checkpoint without a map
    subprocess.run([sys.executable, "-m", "shine_mapping_b200.mesher", batch_run["config"], batch_run["checkpoint"], "--out",
                    mesh, "--mc-res-m", "0.4"], check=True, cwd=ROOT, env=env)
    assert 0 < read_ply(mesh)[1].shape[0] < f0.shape[0]
    only = str(batch_run["tmp"] / "decoder_only.pth")
    torch.save({"geo_decoder": batch_run["decoder"].state_dict()}, only)
    r = subprocess.run([sys.executable, "-m", "shine_mapping_b200.mesher", batch_run["config"], only, "--out", mesh],
                       cwd=ROOT, env=env, capture_output=True, text=True)
    assert r.returncode != 0 and "no map" in r.stderr


# ---- load_model in the command lines -----------------------------------------------------------------------------------

def _spy_trainer(monkeypatch, seen):
    """Record the octree / decoder a loop trains, and the tables before its first step."""
    from shine_mapping_b200 import trainer as tr
    real = tr.SdfTrainer.__init__

    def init(self, config, octree, decoder, *a, **kw):
        if "octree" not in seen:
            seen.update(octree=octree, decoder=decoder, tables=[p.data.clone() for p in octree.hier_features],
                        frozen=not any(p.requires_grad for p in decoder.parameters()))
        return real(self, config, octree, decoder, *a, **kw)
    monkeypatch.setattr(tr.SdfTrainer, "__init__", init)


def test_batch_loop_loads_a_decoder_only_file(tmp_path, monkeypatch, batch_run):
    from shine_mapping_b200 import batch_loop
    only = str(tmp_path / "geo_decoder.pth")
    want = {k: v.clone() for k, v in batch_run["decoder"].state_dict().items()}
    torch.save({"geo_decoder": want, "sem_decoder": {}}, only)
    seen = {}
    _spy_trainer(monkeypatch, seen)
    batch_loop.main([_config_file(tmp_path, load_model=True, model_path=only, iters=30, freq=1000), "--synthetic-azimuth",
                     "512", "--frames", "3"])
    assert seen["frozen"]
    assert all(torch.equal(v, want[k]) for k, v in seen["decoder"].state_dict().items())        # unchanged at the end
    assert any(not torch.equal(p.data, t) for p, t in zip(seen["octree"].hier_features, seen["tables"]))   # tables moved


def test_batch_loop_continues_a_full_checkpoint(tmp_path, monkeypatch, batch_run):
    from shine_mapping_b200 import batch_loop
    saved = batch_run["octree"]
    seen = {}
    _spy_trainer(monkeypatch, seen)
    cfg = _config_file(tmp_path, load_model=True, model_path=batch_run["checkpoint"], iters=10, freq=1000)
    batch_loop.main([cfg, "--synthetic-azimuth", "512", "--frames", "12"])     # six frames more than the saved map saw
    for p, q, t in zip(saved.hier_features, seen["octree"].hier_features, seen["tables"]):
        assert q.shape[0] > p.shape[0]
        assert torch.equal(t[:p.shape[0] - 1], p.data[:-1])                      # saved rows: same numbering, same values
    for a, b in zip(saved._levels, seen["octree"]._levels):
        n = a.node_keys.numel()
        assert torch.equal(b.node_keys[:n], a.node_keys) and torch.equal(b.node_ids[:n], a.node_ids)


def test_incremental_loop_continues_from_its_checkpoint(tmp_path):
    from shine_mapping_b200 import incre_loop
    run = str(tmp_path / "run")
    cfg = _config_file(tmp_path, iters=40)
    full = incre_loop.main([cfg, "--synthetic-azimuth", "512", "--frames", "6", "--run-path", run])
    assert sorted(os.listdir(os.path.join(run, "model"))) == ["model_frame_1.pth", "model_frame_3.pth", "model_frame_6.pth"]
    assert not os.path.exists(os.path.join(run, "map"))                         # save_map is off
    cont = _config_file(tmp_path, "cont.yaml", iters=40, load_model=True,
                        model_path=os.path.join(run, "model", "model_frame_3.pth"))
    # the same drive; the second run maps frames 3..5 on top of the saved map
    from shine_mapping_b200 import synth
    real = synth.generate_scans
    synth.generate_scans = lambda *a, **kw: real(*a, **kw)[3:]
    try:
        rest = incre_loop.main([cont, "--synthetic-azimuth", "512", "--frames", "6"])
    finally:
        synth.generate_scans = real
    assert len(rest) == 3
    assert all(r >= f for r, f in zip(rest[0]["rows"], full[2]["rows"])) and rest[0]["rows"] != full[2]["rows"]
    assert rest[-1]["rows"] == full[-1]["rows"]                                  # the same nodes in the end
    assert 0.2 < rest[-1]["bce_last"] / full[-1]["bce_last"] < 5.0


# ---- the export kernel -------------------------------------------------------------------------------------------------

def _restate(mesher, grid, bricks, sdf, mask, masked_only):
    """The records shine_mesh_export_points must write for one chunk, in torch on the same buffers."""
    from shine_mapping_b200.mesher import SDF_MAP_RECORD
    n = grid["n"]
    l = torch.arange(n + 1, device=DEV)
    loc = torch.stack(torch.meshgrid(l, l, l, indexing="ij"), -1).reshape(-1, 3)
    G = bricks.long()[:, None, :] * n + loc[None]
    hi = torch.tensor(grid["hi"], device=DEV)
    lo = torch.tensor(grid["lo"], device=DEV)
    owned = (loc < n).all(1)[None] & (G < hi).all(-1)
    m = mask != 0
    take = owned & (m if masked_only else torch.ones_like(m))
    x = torch.tensor(grid["origin_m"], dtype=torch.float64, device=DEV) + grid["voxel_m"] * (G[take] - lo).double()
    T = torch.tensor(mesher.global_transform, dtype=torch.float64, device=DEV)
    pos = [(((T[a, 0] * x[:, 0] + T[a, 1] * x[:, 1]) + T[a, 2] * x[:, 2]) + T[a, 3]).float() for a in range(3)]
    factor = torch.tensor(mesher.config.logistic_gaussian_ratio * mesher.config.sigma_sigmoid_m).float().to(DEV)
    rec = np.empty(int(take.sum()), dtype=SDF_MAP_RECORD)
    for a, name in enumerate("xyz"):
        rec[name] = pos[a].cpu().numpy()
    rec["intensities"] = (sdf[take] * factor).cpu().numpy()
    rec["labels"] = m[take].int().cpu().numpy()
    return rec, int((m & owned).sum())


def _sorted(rec):
    return np.sort(rec, order=["x", "y", "z", "intensities", "labels"])


@pytest.mark.parametrize("octree_mode", [True, False])
def test_export_matches_a_torch_restatement(tmp_path, monkeypatch, batch_run, octree_mode):
    from shine_mapping_b200 import Mesher, mesher as mm
    cfg = _config(batch_run["config"])
    octree, dec = batch_run["octree"], batch_run["decoder"]
    m = Mesher(cfg, octree, dec)
    ang = 0.3
    m.global_transform = np.array([[np.cos(ang), -np.sin(ang), 0, 1.5], [np.sin(ang), np.cos(ang), 0, -2.25],
                                   [0, 0, 1, 0.125], [0, 0, 0, 1]])
    lo_m, hi_m = np.array([-12.0, -6.0, -2.0]), np.array([14.0, 6.0, 3.0])
    make = (lambda: m.octree_grid(octree.free_level_num, 0.2)) if octree_mode else (lambda: m.bbx_grid(lo_m, hi_m, 0.2))
    monkeypatch.setattr(mm, "CHUNK_POINTS", 1 << 15)
    grid = make()
    want, masked_total, chunks = [], 0, 0
    for bricks, sdf, mask, _ in m.chunks(grid):
        rec, masked = _restate(m, grid, bricks, sdf, mask, octree_mode)
        want.append(rec); masked_total += masked; chunks += 1
    want = np.concatenate(want)
    assert chunks > 3 and masked_total > 1000
    # through an edge-table restart: the file still holds each point once
    calls = []
    real_restart = mm.SdfMapWriter.restart
    monkeypatch.setattr(mm.SdfMapWriter, "restart", lambda self: (calls.append(1), real_restart(self))[1])
    monkeypatch.setattr(mm.Mesher, "edge_capacity", staticmethod(lambda g: 1 << 8))
    path = str(tmp_path / "map.ply")
    mesh = str(tmp_path / "mesh.ply")
    if octree_mode:
        m.recon_octree_mesh(octree.free_level_num, 0.2, mesh, path)
    else:
        m.recon_bbx_mesh(lo_m, hi_m, 0.2, mesh, path)
    assert len(calls) > 1
    got = mm.read_point_ply(path)
    assert got.shape[0] == want.shape[0] and (got["labels"] == 1).sum() == masked_total
    if octree_mode:
        assert got.shape[0] == masked_total
    else:
        assert got.shape[0] > masked_total and set(np.unique(got["labels"]).tolist()) == {0, 1}
    assert _sorted(got).tobytes() == _sorted(want).tobytes()                                    # bit for bit
    pos = np.stack([got["x"], got["y"], got["z"]], 1)
    assert np.unique(pos, axis=0).shape[0] == pos.shape[0]                                      # no point twice
    # the same file without the mesh
    assert m.save_sdf_map(make(), str(tmp_path / "alone.ply"), octree_mode) == got.shape[0]
    assert _sorted(mm.read_point_ply(str(tmp_path / "alone.ply"))).tobytes() == _sorted(want).tobytes()


def test_written_sdf_map(batch_run):
    from shine_mapping_b200 import sdf_infer
    from shine_mapping_b200.mesher import read_point_ply
    cfg = _config(batch_run["config"])
    with open(batch_run["sdf_map"], "rb") as fh:
        head = fh.read(200).split(b"end_header")[0].decode()
    count = int(head.split("element vertex ")[1].split("\n")[0])
    pts = read_point_ply(batch_run["sdf_map"])
    assert pts.shape[0] == count > 1000
    assert os.path.getsize(batch_run["sdf_map"]) == len(head) + len("end_header\n") + 20 * count
    assert np.isfinite(pts["intensities"]).all() and set(np.unique(pts["labels"]).tolist()) <= {0, 1}
    assert (pts["labels"] == 1).all()                                  # octree mode: masked points only
    # sign and factor: the synthetic loop writes in the map frame (identity transform)
    xyz = torch.from_numpy(np.stack([pts["x"], pts["y"], pts["z"]], 1)).to(DEV)
    pred = sdf_infer(batch_run["octree"], batch_run["decoder"], xyz * cfg.scale)
    want = (-pred * (cfg.logistic_gaussian_ratio * cfg.sigma_sigmoid_m)).cpu().numpy()
    assert np.abs(want).max() > 0.01 and np.abs(pts["intensities"] - want).max() <= 0.01 * np.abs(want).max()


def test_no_map_directory_without_save_map(tmp_path):
    from shine_mapping_b200 import batch_loop
    run = str(tmp_path / "run")
    batch_loop.main([_config_file(tmp_path, iters=20, freq=20), "--synthetic-azimuth", "256", "--frames", "2", "--run-path", run])
    assert sorted(os.listdir(run)) == ["mesh", "model"]


# ---- the ABI entry's argument checks -----------------------------------------------------------------------------------

def _chunk(nb=3, n=4):
    from shine_mapping_b200 import _abi
    r = torch.arange(nb, device=DEV)
    bricks = torch.stack((r, r * 0, r * 0), -1).to(torch.int32).contiguous()
    per = (n + 1) ** 3
    sdf = torch.arange(nb * per, device=DEV, dtype=torch.float32) / 7
    mask = (torch.arange(nb * per, device=DEV) % 3 == 0).to(torch.uint8)
    g = _abi.ShineBrickGrid()
    g.bricks, g.sdf, g.mask, g.num_bricks, g.n = bricks.data_ptr(), sdf.data_ptr(), mask.data_ptr(), nb, n
    for a in range(3):
        g.lo[a], g.hi[a] = 0, nb * n
    return g, (bricks, sdf, mask)


def _export(g, records, capacity, counter, masked_only=0, origin=True, transform=True):
    from shine_mapping_b200 import _abi
    o = (C.c_double * 3)(0.0, 0.0, 0.0) if origin else None
    t = (C.c_double * 12)(1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1, 0) if transform else None
    n = C.c_int64(-1)
    rc = _abi.lib().shine_mesh_export_points(C.byref(g) if g is not None else None, o, 0.5, t, 2.0, masked_only,
                                              _abi.ptr(records), capacity, _abi.ptr(counter), C.byref(n),
                                              _abi.stream_ptr(DEV))
    return rc, n.value


def test_export_capacity_and_argument_errors():
    from shine_mapping_b200 import _abi
    g, keep = _chunk()
    owned = 3 * 4 ** 3
    counter = torch.zeros(1, dtype=torch.int64, device=DEV)
    buf = torch.full((owned * 20 + 64,), 0xAB, dtype=torch.uint8, device=DEV)
    rc, n = _export(g, buf, owned, counter)
    assert rc == 0 and n == owned and int(counter) == owned
    assert (buf[owned * 20:] == 0xAB).all()
    rec = np.frombuffer(buf[:owned * 20].cpu().numpy().tobytes(), dtype=[("p", "<f4", (3,)), ("i", "<f4"), ("l", "<i4")])
    assert np.unique(rec["p"], axis=0).shape[0] == owned and rec["p"].max() == 0.5 * 11
    # too small: counted, not written, the guard region untouched
    cap = 50
    counter.zero_()
    small = torch.full((cap * 20 + 64,), 0xAB, dtype=torch.uint8, device=DEV)
    rc, n = _export(g, small, cap, counter)
    assert rc == _abi.ERR_CAPACITY == -3 and n == owned
    assert (small[cap * 20:] == 0xAB).all() and not (small[:cap * 20] == 0xAB).all()
    assert b"too small" in _abi.lib().shine_error_string(rc)
    # masked only, appended after what the counter already holds
    counter.fill_(5)
    buf.fill_(0xAB)
    rc, n = _export(g, buf, owned, counter, masked_only=1)
    masked = int(keep[2].view(3, 5, 5, 5)[:, :4, :4, :4].sum())
    assert rc == 0 and n == 5 + masked and (buf[:100] == 0xAB).all() and (buf[(5 + masked) * 20:] == 0xAB).all()
    # arguments
    counter.zero_()
    INVALID = -1
    assert _export(None, buf, owned, counter)[0] == INVALID
    assert _export(g, None, owned, counter)[0] == INVALID
    assert _export(g, buf, owned, None)[0] == INVALID
    assert _export(g, buf, -1, counter)[0] == INVALID
    assert _export(g, buf, owned, counter, origin=False)[0] == INVALID
    assert _export(g, buf, owned, counter, transform=False)[0] == INVALID
    assert _export(g, buf[1:], owned, counter)[0] == INVALID                                   # records not 4-byte aligned
    assert _export(g, buf, owned, torch.zeros(1, dtype=torch.int64))[0] == INVALID               # counter on the host
    assert _export(g, torch.zeros(owned * 20, dtype=torch.uint8), owned, counter)[0] == INVALID  # records on the host
    if torch.cuda.device_count() > 1:
        other = torch.zeros(owned * 20, dtype=torch.uint8, device="cuda:1")
        assert _export(g, other, owned, counter)[0] == INVALID
    assert int(counter) == 0
