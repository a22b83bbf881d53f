"""csrc/shine_scan.cu against tests/scan_oracle.py: filter and voxel grid bit-exact in fp64, scaled fp32 points and
samples bit-exact on the same uniforms, a written sequence end to end (pool, octree tables, surfaces), the command lines
with --scans, and the one host read of a frame."""
import ast
import math
import os
import warnings

import numpy as np
import pytest
import torch

from shine_mapping_b200 import scans, synth
from tests import scan_oracle
from tests.parity_utils import make_config, orc
from tests.test_scans_host import check_against_reference_sampler, _golden_cfg

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _cfg(**kw):
    base = dict(device=DEV, rand_downsample=False, vox_down_m=0.1, min_range=2.75, pc_radius=20.0, min_z=-10.0,
                max_z=30.0)
    base.update(kw)
    return make_config(3, **base)


def _pose(seed=3):
    a, b = 0.4 + seed * 0.1, 0.05
    Rz = np.array([[math.cos(a), -math.sin(a), 0], [math.sin(a), math.cos(a), 0], [0, 0, 1]])
    Rx = np.array([[1, 0, 0], [0, math.cos(b), -math.sin(b)], [0, math.sin(b), math.cos(b)]])
    T = np.eye(4)
    T[:3, :3] = Rz @ Rx
    T[:3, 3] = (1.25, -3.5, 0.3)
    return T


def _cases():
    rng = np.random.default_rng(0)
    cloud = rng.uniform(-25, 25, (20000, 3)) * np.array([1, 1, 0.4])
    edge = np.array([[5.0, 0.0, -10.0], [2.75, 0.0, 0.0], [0.0, 2.75, 0.0], [20.0, 1.0, 1.0], [-20.0, 1.0, 1.0],
                     [3.0, 20.0, 1.0], [3.0, -20.0, 1.0], [5.0, 5.0, 30.0], [3.0, 3.0, -9.5],
                     [np.nan, 4.0, 1.0], [4.0, 4.0, np.nan], [np.inf, 4.0, 1.0], [4.0, -np.inf, 1.0],
                     [4.0, 4.0, np.inf], [20.0 + 1e-9, 1.0, 1.0]])
    grid = np.stack(np.meshgrid(*[np.arange(-2.0, 2.01, 0.1)] * 3), -1).reshape(-1, 3) + np.array([6.0, 0.0, 0.0])
    return {
        "edges": np.concatenate((edge, cloud[:2000])),
        "voxel_boundaries": np.concatenate((grid, [[-20.0, -20.0, -9.95]])),
        "copies": np.repeat([[7.3, -4.1, 0.2]], 10000, 0),
        "one_voxel": np.array([8.01, 3.02, 1.03]) + rng.uniform(0, 0.04, (100000, 3)),   # within v/2 of the minimum
        "empty": np.zeros((0, 3)),
        "single": np.array([[10.0, 1.0, 1.0]]),
        "dropped_only": np.array([[0.1, 0.1, 0.1]]),
        "cloud": cloud,
        "two_million": rng.uniform(-22, 22, (2_000_000, 3)) * np.array([1, 1, 0.5]),
    }


def _records(points, fp64):
    """float32 x y z i (16-byte KITTI records) or float64 x y z (24-byte records), pinned."""
    if fp64:
        return scans._records_from_xyz(points.astype(np.float64), True)
    raw = np.concatenate((points.astype(np.float32), np.ones((points.shape[0], 1), np.float32)), 1)
    buf = torch.empty(raw.nbytes, dtype=torch.uint8, pin_memory=True)
    buf.numpy()[:] = raw.reshape(-1).view(np.uint8)
    return scans.ScanRecords(buf, points.shape[0], 16, False)


@pytest.mark.parametrize("fp64", [False, True])
@pytest.mark.parametrize("case", list(_cases()))
def test_filter_voxel_transform_bit_exact(case, fp64):
    if case == "two_million" and fp64:
        pytest.skip("one record format is enough for the grid-stride and sort-tail size")
    cfg = _cfg()
    pts = _cases()[case]
    rec = _records(pts, fp64)
    pose = _pose()
    got_pts, got_vox = scans.ScanProcessor(cfg, DEV).points(rec, pose, voxels_out=True)
    want_pts, want_vox = scan_oracle.frame_points(rec.points(), pose, cfg, voxels=True)
    assert got_vox.shape[0] == want_vox.shape[0]
    np.testing.assert_array_equal(got_vox.cpu().numpy().view(np.int64), want_vox.view(np.int64))
    np.testing.assert_array_equal(got_pts.cpu().numpy().view(np.int32), want_pts.view(np.int32))
    if case == "edges":                      # z == min_z dropped; range == min_range and every crop face kept
        kept = scan_oracle.crop(scan_oracle.preprocess(rec.points(), cfg.min_z, cfg.min_range), cfg.pc_radius,
                                cfg.min_z, cfg.max_z)
        assert {tuple(p) for p in kept[:8]} == {tuple(p) for p in pts[1:9]}
    if case == "one_voxel":
        assert want_vox.shape[0] == 1


def test_sampler_kernel_against_oracle_and_reference():
    g = np.load(os.path.join(ROOT, "tests", "golden", "ref_sampler.npz"))
    cfg = _golden_cfg(g)
    cfg.scale = float(g["scale"])
    proc = scans.ScanProcessor(cfg, DEV)
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(DEV)
    coord, label, weight = proc.sample(t(g["points"]), g["origin"], t(g["u_surface"]), t(g["u_free"]))
    coord, label, weight = coord.cpu().numpy(), label.cpu().numpy(), weight.cpu().numpy()
    want = scan_oracle.sample(g["points"], g["origin"], g["u_surface"], g["u_free"], cfg)
    for a, b in zip((coord, label, weight), want):
        np.testing.assert_array_equal(a.view(np.int32), b.view(np.int32))
    check_against_reference_sampler(coord, label, weight, g)


# ----------------------------------------------------------------------------------------------- written sequence

def _surface_distance(p):
    """Distance (m) from world points to the analytic scene of synth.raycast_scene (ground, walls, boxes)."""
    d = np.abs(p[:, 2] + 1.7)
    wall = np.where(p[:, 2] <= 4.3, np.abs(np.abs(p[:, 1]) - 8.0), np.inf)
    d = np.minimum(d, wall)
    for b in synth.default_boxes().numpy().astype(np.float64):
        q = np.maximum(b[:3] - p, 0) + np.maximum(p - b[3:], 0)
        outside = np.linalg.norm(q, axis=1)
        inside = np.min(np.minimum(p - b[:3], b[3:] - p), axis=1)
        d = np.minimum(d, np.where(outside > 0, outside, np.maximum(-inside, 0) + np.abs(inside)))
    return d


def write_sequence(root, fmt, n_frames=10, n_azimuth=512):
    """Ten frames of the analytic street seen from a drive that turns, written as KITTI poses + calib and scans."""
    os.makedirs(os.path.join(root, "scans"), exist_ok=True)
    Tr = np.eye(4)
    Tr[:3, :3] = np.array([[0, -1, 0], [0, 0, -1], [1, 0, 0]], dtype=np.float64)
    Tr[:3, 3] = (-0.01, -0.05, -0.27)
    dirs = synth.lidar_directions(n_azimuth).double()
    lines = []
    for f in range(n_frames):
        yaw = 0.08 * f * (1 if f < 6 else -1)
        W = np.eye(4)
        W[:3, :3] = [[math.cos(yaw), -math.sin(yaw), 0], [math.sin(yaw), math.cos(yaw), 0], [0, 0, 1]]
        W[:3, 3] = (1.5 * f, 0.2 * math.sin(f), 0.0)
        hits = synth.raycast_scene(torch.tensor(W[:3, 3]), (torch.tensor(W[:3, :3]) @ dirs.T).T.float(),
                                   synth.default_boxes(), min_range=1.0, max_range=40.0).double().numpy()
        local = (hits - W[:3, 3]) @ W[:3, :3]
        P = Tr @ W @ np.linalg.inv(Tr)                  # camera pose: the reader recovers W = Tr^-1 P Tr
        lines.append(" ".join(repr(float(v)) for v in P[:3].reshape(-1)))
        path = os.path.join(root, "scans", f"{f}.{fmt}")
        if fmt == "bin":
            np.concatenate((local.astype(np.float32), np.ones((len(local), 1), np.float32)), 1).tofile(path)
        elif fmt == "ply":
            with open(path, "wb") as fh:
                fh.write(f"ply\nformat binary_little_endian 1.0\nelement vertex {len(local)}\nproperty double x\n"
                         f"property double y\nproperty double z\nproperty uchar label\nend_header\n".encode())
                rec = np.zeros(len(local), np.dtype([("p", "<f8", 3), ("l", "u1")]))
                rec["p"] = local
                fh.write(rec.tobytes())
        else:
            with open(path, "wb") as fh:
                fh.write(f"VERSION 0.7\nFIELDS intensity x y z\nSIZE 4 4 4 4\nTYPE F F F F\nCOUNT 1 1 1 1\n"
                         f"WIDTH {len(local)}\nHEIGHT 1\nPOINTS {len(local)}\nDATA binary\n".encode())
                rec = np.zeros((len(local), 4), np.float32)
                rec[:, 1:] = local
                fh.write(rec.tobytes())
    with open(os.path.join(root, "poses.txt"), "w") as fh:
        fh.write("\n".join(lines) + "\n")
    with open(os.path.join(root, "calib.txt"), "w") as fh:
        fh.write("P0: " + " ".join(["1", "0", "0", "0", "0", "1", "0", "0", "0", "0", "1", "0"]) + "\n")
        fh.write("Tr: " + " ".join(repr(float(v)) for v in Tr[:3].reshape(-1)) + "\n")
    return dict(pc_path=os.path.join(root, "scans"), pose_path=os.path.join(root, "poses.txt"),
                calib_path=os.path.join(root, "calib.txt"))


@pytest.mark.parametrize("fmt", ["bin", "ply", "pcd"])
def test_sequence_end_to_end(tmp_path, fmt):
    from shine_mapping_b200 import FeatureOctree
    paths = write_sequence(str(tmp_path), fmt)
    cfg = _cfg(window_replay_on=False, continual_learning_reg=False, end_frame=100, **paths)
    octree = FeatureOctree(cfg)
    ds = scans.LiDARDataset(cfg, octree)
    assert ds.total_pc_count == 10 and ds.used_pc_count == 10 and isinstance(ds.pool, synth.SamplePool)
    o = orc.OracleOctree(cfg.tree_level_world, cfg.tree_level_feat, cfg.feature_dim, cfg.feature_std, cfg.poly_int_on)
    from tests.test_gpu_octree_build import assert_tables_match
    want = []
    for f in ds.used_frames:
        torch.manual_seed(100 + f)
        ds.process_frame(f)
        rec = scans.read_scan(os.path.join(cfg.pc_path, ds.pc_filenames[f]), pinned=False)
        pts = scan_oracle.frame_points(rec.points(), ds.poses_ref[f], cfg)
        origin = (ds.poses_ref[f][:3, 3] * cfg.scale).astype(np.float32)
        torch.manual_seed(100 + f)
        R, ns, nf = pts.shape[0], cfg.surface_sample_n, cfg.free_sample_n
        us = torch.rand(R * ns, 1, device=DEV)
        torch.rand(0, 1, device=DEV)
        uf = torch.rand(R * nf, 1, device=DEV)
        coord, label, weight = scan_oracle.sample(pts, origin, us.cpu().numpy(), uf.cpu().numpy(), cfg)
        want.append((coord, label, weight))
        o.update(coord[weight > 0])
        assert_tables_match(octree, o)
        Wf = np.linalg.inv(ds.begin_pose_inv)
        pw = (pts.astype(np.float64) / cfg.scale) @ Wf[:3, :3].T + Wf[:3, 3]
        assert _surface_distance(pw).max() < cfg.vox_down_m * 1.8
    for got, w in zip((ds.pool.coord_pool, ds.pool.sdf_label_pool, ds.pool.weight_pool), zip(*want)):
        np.testing.assert_array_equal(got.cpu().numpy().view(np.int32), np.concatenate(w).view(np.int32))


def test_one_host_read_per_frame(tmp_path):
    paths = write_sequence(str(tmp_path), "bin", n_frames=2)
    ds = scans.LiDARDataset(_cfg(**paths))
    ds.frame_samples(0)
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("warn")
    try:
        with warnings.catch_warnings(record=True) as caught:
            warnings.simplefilter("always")
            ds.frame_samples(1)
    finally:
        torch.cuda.set_sync_debug_mode("default")
    syncs = [w for w in caught if "synchroniz" in str(w.message)]
    assert len(syncs) == 1, [str(w.message) for w in syncs]


# ---------------------------------------------------------------------------------------------------- command lines

def _yaml(tmp_path, paths, **over):
    import yaml
    doc = {"setting": dict(paths, begin_frame=0, end_frame=100, every_frame=1, first_frame_ref=True, device=DEV),
           "process": {"min_range_m": 2.75, "pc_radius_m": 20.0, "min_z_m": -10.0, "rand_downsample": False,
                       "vox_down_m": 0.1},
           "sampler": {"surface_sample_range_m": 0.3, "surface_sample_n": 3, "free_sample_begin_ratio": 0.3,
                       "free_sample_end_dist_m": 0.8, "free_sample_n": 3},
           "octree": {"tree_level_world": 12, "tree_level_feat": 3, "leaf_vox_size": 0.2, "feature_dim": 8},
           "continual": {"continual_learning_reg": False, "window_replay_on": False},
           "optimizer": {"batch_size": 4096, "learning_rate": 0.01}}
    for k, v in over.items():
        sec, key = k.split("__")
        doc.setdefault(sec, {})[key] = v
    p = tmp_path / "cfg.yaml"
    p.write_text(yaml.safe_dump(doc))
    return str(p)


def _printed(out: str):
    return ast.literal_eval([l for l in out.splitlines() if l.startswith("{'loss_first'")][-1])


@pytest.mark.parametrize("mode", ["device", "host", "eikonal"])
def test_batch_loop_scans(tmp_path, capsys, mode):
    from shine_mapping_b200 import batch_loop
    paths = write_sequence(str(tmp_path), "bin", n_frames=4)
    over = {"setting__pc_count_gpu_limit": 2} if mode == "host" else {}
    if mode == "eikonal":
        over["loss__ekional_loss_on"] = True
    batch_loop.main([_yaml(tmp_path, paths, **over), "--scans", "--iters", "300"])
    out = capsys.readouterr().out
    assert ("HostSamplePool" in out) == (mode == "host")
    res = _printed(out)
    assert res["loss_last"] < res["loss_first"]


@pytest.mark.parametrize("replay", [False, True])
def test_incre_loop_scans(tmp_path, replay):
    from shine_mapping_b200 import incre_loop
    paths = write_sequence(str(tmp_path), "pcd", n_frames=4)
    over = {"continual__continual_learning_reg": not replay, "continual__window_replay_on": replay,
            "continual__window_radius_m": 30.0}
    history = incre_loop.main([_yaml(tmp_path, paths, **over), "--scans", "--iters", "40"])
    assert len(history) == 4
    assert all(math.isfinite(h["loss_last"]) for h in history)
    assert history[0]["bce_last"] < history[0]["bce_first"]
    assert ("pool" in history[-1]) == replay
