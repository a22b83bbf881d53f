"""Host side of the pose-free mapping mode (odometry.py): SE(3) maps, the Gauss-Newton loop on an analytic street
restated in numpy with the kernel's 29-value layout, the KITTI pose file round trip and the argument
checks of shine_register_normal_eq."""
import ctypes as C
import math

import numpy as np
import pytest
import torch

from shine_mapping_b200 import odometry, scans, synth
from tests.parity_utils import make_config


def _rot(yaw, pitch=0.0, roll=0.0):
    cz, sz, cy, sy, cx, sx = math.cos(yaw), math.sin(yaw), math.cos(pitch), math.sin(pitch), math.cos(roll), math.sin(roll)
    return (np.array([[cz, -sz, 0], [sz, cz, 0], [0, 0, 1]]) @ np.array([[cy, 0, sy], [0, 1, 0], [-sy, 0, cy]]) @
            np.array([[1, 0, 0], [0, cx, -sx], [0, sx, cx]]))


def _pose(t, yaw, pitch=0.0, roll=0.0):
    T = np.eye(4)
    T[:3, :3] = _rot(yaw, pitch, roll)
    T[:3, 3] = t
    return T


@pytest.mark.parametrize("xi", [[0.3, -1.2, 0.05, 0.01, -0.02, 0.4], [1e-9, 0, 0, 1e-8, -2e-8, 3e-9], [0, 0, 0, 0, 0, 0],
                                [2.0, 1.0, -0.5, 0.0, 0.0, 3.0], [0.1, 0.2, 0.3, 1.5, -1.0, 0.5]])
def test_se3_exp_log_round_trip(xi):
    T = odometry.se3_exp(xi)
    np.testing.assert_allclose(T[:3, :3] @ T[:3, :3].T, np.eye(3), atol=1e-14)
    assert abs(np.linalg.det(T[:3, :3]) - 1) < 1e-14
    np.testing.assert_allclose(odometry.se3_log(T), xi, atol=1e-12)
    np.testing.assert_allclose(odometry.se3_exp(odometry.se3_log(T)), T, atol=1e-12)


def test_se3_exp_matches_the_series():
    """exp of the 4x4 twist matrix by its power series."""
    xi = np.array([0.4, -0.3, 0.2, 0.3, 0.5, -0.7])
    M = np.zeros((4, 4))
    M[:3, :3] = odometry.hat(xi[3:])
    M[:3, 3] = xi[:3]
    want, term = np.eye(4), np.eye(4)
    for k in range(1, 40):
        term = term @ M / k
        want = want + term
    np.testing.assert_allclose(odometry.se3_exp(xi), want, atol=1e-13)


# ---- the Gauss-Newton loop on an analytic street ---------------------------------------------------------------------------

BOXES = synth.default_boxes().numpy().astype(np.float64)


def street_sdf(p):
    """Signed distance (m) to synth.raycast_scene's street, positive in free space: ground z = -1.7, walls |y| = 8, boxes."""
    d = np.minimum(p[:, 2] + 1.7, 8.0 - np.abs(p[:, 1]))
    for b in BOXES:
        q = np.maximum(b[:3] - p, p - b[3:])
        outside = np.linalg.norm(np.maximum(q, 0), axis=1)
        d = np.minimum(d, outside + np.minimum(q.max(1), 0))
    return d


def street_normal_equations(points, pose_scaled, scale, kappa_scaled, band_m=0.3):
    """The 29 values of shine_register_normal_eq for the analytic street (fp64, central differences for g).  Like the
    map's finest level, the field exists only within band_m of a surface: farther points are masked."""
    q = np.asarray(points, dtype=np.float64) @ pose_scaled[:3, :3].T + pose_scaled[:3, 3]
    qm = q / scale
    near = np.abs(street_sdf(qm)) < band_m
    q, qm = q[near], qm[near]
    r = street_sdf(qm) * scale
    h = 1e-6
    g = np.stack([(street_sdf(qm + h * e) - street_sdf(qm - h * e)) / (2 * h) for e in np.eye(3)], 1)
    J = np.concatenate((g, np.cross(q, g)), 1)
    w = (kappa_scaled ** 2 / (kappa_scaled ** 2 + r ** 2)) ** 2
    H = (w[:, None, None] * J[:, :, None] * J[:, None, :]).sum(0)
    out = np.concatenate((H[np.triu_indices(6)], (w[:, None] * J * r[:, None]).sum(0), [(w * r * r).sum(), len(r)]))
    return out


class StreetRegistration(odometry.ScanToMapRegistration):
    """The registration loop with the kernel replaced by the numpy street (a grid of every other candidate, to keep the
    numpy field affordable)."""

    GRID_X = odometry.ScanToMapRegistration.GRID_X[::2]
    GRID_YAW = odometry.ScanToMapRegistration.GRID_YAW[::2]

    def launch(self, points, pose_scaled, kappa_scaled, out=None):
        (self.out if out is None else out).copy_(
            torch.from_numpy(street_normal_equations(points.numpy(), pose_scaled, self.scale, kappa_scaled)))


def _street_scan(pose_w):
    dirs = synth.lidar_directions(96).double()
    hits = synth.raycast_scene(torch.tensor(pose_w[:3, 3]), (torch.tensor(pose_w[:3, :3]) @ dirs.T).T.float(),
                               synth.default_boxes(), min_range=2.0, max_range=30.0).double().numpy()
    return (hits - pose_w[:3, 3]) @ pose_w[:3, :3]          # sensor frame, metres


@pytest.mark.parametrize("dt, dyaw", [((0.5, 0.0, 0.0), 0.0), ((0.3, -0.3, 0.1), math.radians(5)),
                                      ((-0.4, 0.2, 0.0), math.radians(-4)), ((0.0, 0.0, 0.0), 0.0),
                                      ((-1.5, -0.3, 0.0), math.radians(-2.5)), ((1.8, 0.0, 0.0), 0.0)])
def test_gauss_newton_recovers_known_perturbations(dt, dyaw):
    cfg = make_config(3)
    truth = _pose((10.0, 0.5, 0.0), 0.1)
    local = torch.from_numpy(_street_scan(truth) * cfg.scale).float()
    init = _pose(truth[:3, 3] + np.array(dt), 0.1 + dyaw)
    reg = StreetRegistration(cfg, None, None, kappa_m=0.1, max_iters=40, tol=1e-6)
    pose, info = reg.register(local, init)
    assert info["ok"] and info["converged"] and info["valid"] > 0.95 * local.shape[0]
    assert np.linalg.norm(pose[:3, 3] - truth[:3, 3]) < 2e-3, (pose[:3, 3], truth[:3, 3], info)
    assert np.linalg.norm(odometry.se3_log(np.linalg.inv(truth) @ pose)[3:]) < 1e-4
    assert info["rmse_m"] < 2e-3


def test_search_along_the_weak_direction():
    """From a pose 1.2 m along the street, the search alone lands within one step of the truth along the street (the
    other directions are Gauss-Newton's)."""
    cfg = make_config(3)
    truth = _pose((10.0, 0.5, 0.0), 0.1)
    local = torch.from_numpy(_street_scan(truth) * cfg.scale).float()
    start = truth.copy()
    start[:3, 3] += (1.2 * math.cos(0.1), 1.2 * math.sin(0.1), 0.0)
    reg = StreetRegistration(cfg, None, None)
    pose, moved = reg.search_weak_direction(local, start)
    along = np.array([math.cos(0.1), math.sin(0.1), 0.0])
    assert moved and abs(np.dot(pose[:3, 3] - truth[:3, 3], along)) < 0.06, pose[:3, 3]
    # at the truth nothing beats the current pose
    pose, moved = reg.search_weak_direction(local, truth)
    assert not moved and np.array_equal(pose, truth)


def test_registration_flags_non_convergence():
    cfg = make_config(3)
    truth = _pose((10.0, 0.5, 0.0), 0.1)
    local = torch.from_numpy(_street_scan(truth) * cfg.scale).float()
    pose, info = StreetRegistration(cfg, None, None, max_iters=4, tol=1e-12).register(
        local, _pose(truth[:3, 3] + np.array([0.2, 0.2, 0.0]), 0.15))
    assert info["ok"] and not info["converged"]


def test_registration_refuses_too_few_points_and_singular_systems():
    cfg = make_config(3)
    init = _pose((1.0, 2.0, 0.0), 0.3)

    class Few(StreetRegistration):
        def launch(self, points, pose_scaled, kappa_scaled, out=None):
            super().launch(points, pose_scaled, kappa_scaled, out)
            (self.out if out is None else out)[28] = 3.0

    pose, info = Few(cfg, None, None).register(torch.zeros(10, 3), init)
    assert not info["ok"] and np.array_equal(pose, init) and "points on the map" in info["reason"]
    # ground points only: x, y and yaw are free
    flat = torch.from_numpy(np.stack([np.linspace(-5, 5, 400), np.linspace(-3, 3, 400)[::-1], np.full(400, -1.7)], 1)
                            * cfg.scale).float()
    pose, info = StreetRegistration(cfg, None, None).register(flat, np.eye(4))
    assert not info["ok"] and np.array_equal(pose, np.eye(4)) and info["reason"] == "singular normal equations"


def test_unpack_normal_equations_layout():
    out = np.arange(29, dtype=np.float64)
    H, b, cost, count = odometry.unpack_normal_equations(out)
    assert H[0, 0] == 0 and H[0, 5] == H[5, 0] == 5 and H[1, 1] == 6 and H[5, 5] == 20
    assert np.array_equal(H, H.T) and list(b) == list(range(21, 27)) and cost == 27 and count == 28


# ---- the pose file, the frame source, the command line ------------------------------------------------------------------------

def test_write_kitti_poses_round_trip_is_bit_exact(tmp_path):
    scans_dir = tmp_path / "scans"
    scans_dir.mkdir()
    for f in range(6):
        (scans_dir / f"{f}.bin").write_bytes(b"")
    cfg = make_config(3, rand_downsample=False, pc_path=str(scans_dir), begin_frame=1, end_frame=100, every_frame=2, pose_path="",
                      calib_path="")
    ds = odometry.OdometryScans(cfg, None, None)
    assert ds.used_frames == [2, 4] and ds.total_pc_count == 6
    rng = np.random.default_rng(1)
    for f in ds.used_frames:
        ds.poses_ref[f] = _pose(rng.normal(size=3) * 10 / 3, rng.normal(), rng.normal() * 0.1, rng.normal() * 0.1)
        ds.reg_info[f] = {"iters": 3, "valid": 10, "rmse_m": 0.01, "ok": True}
    path = str(tmp_path / "out" / "poses.txt")
    ds.write_kitti_poses(path)
    back = scans.read_poses_file(path, {"Tr": np.eye(4)})
    assert len(back) == 6
    want = [np.eye(4), np.eye(4), ds.poses_ref[2], ds.poses_ref[2], ds.poses_ref[4], ds.poses_ref[4]]
    for got, w in zip(back, want):
        assert np.array_equal(got.view(np.int64), w.view(np.int64))
    # the remap's reference poses are the estimated ones, bit for bit, with first_frame_ref
    poses_ref, begin_inv, used = scans.reference_poses(cfg, back, 6)
    assert used == [2, 4] and np.array_equal(begin_inv, np.linalg.inv(back[2]))
    cfg.begin_frame = 0
    ds.poses_ref[0] = np.eye(4)
    ds.reg_info[0] = ds.reg_info[2]
    ds.write_kitti_poses(path)
    poses_ref, begin_inv, used = scans.reference_poses(cfg, scans.read_poses_file(path, {"Tr": np.eye(4)}), 6)
    for f in (2, 4):
        assert np.array_equal(poses_ref[f].view(np.int64), ds.poses_ref[f].view(np.int64))
    assert ds.frame_info(2)["reg_ok"] and ds.frame_info(2)["pose"] == ds.poses_ref[2][:3].tolist()


def test_odometry_scans_reads_no_pose_or_calib_file(tmp_path):
    (tmp_path / "0.bin").write_bytes(b"")
    cfg = make_config(3, rand_downsample=False, pc_path=str(tmp_path), pose_path=str(tmp_path / "missing.txt"),
                      calib_path=str(tmp_path / "missing_calib.txt"), end_frame=10)
    ds = odometry.OdometryScans(cfg, None, None)
    assert ds.used_frames == [0] and np.array_equal(ds.begin_pose_inv, np.eye(4))
    cfg.behind_dropoff_on = True
    with pytest.raises(NotImplementedError, match="behind_dropoff_on"):
        odometry.OdometryScans(cfg, None, None)


def test_odometry_scans_refuses_shifted_frames_and_loaded_maps(tmp_path):
    from shine_mapping_b200 import FeatureOctree
    (tmp_path / "0.bin").write_bytes(b"")
    cfg = make_config(3, rand_downsample=False, pc_path=str(tmp_path), end_frame=10, first_frame_ref=False)
    with pytest.raises(ValueError, match="first_frame_ref"):
        odometry.OdometryScans(cfg, None, None)
    cfg.first_frame_ref = True
    octree = FeatureOctree(cfg)
    odometry.OdometryScans(cfg, octree, None)                      # an empty map is fine
    octree.update(torch.tensor([[0.01, 0.02, 0.0], [0.0, -0.01, 0.005]]))
    with pytest.raises(ValueError, match="load_model"):
        odometry.OdometryScans(cfg, octree, None)


def test_register_entry_argument_checks_need_no_gpu(built_lib):
    from shine_mapping_b200 import _abi
    lib = built_lib
    slots = (C.c_uint8 * 64)()
    feats = (C.c_float * 8)()
    oct_ = _abi.ShineOctree()
    oct_.num_levels, oct_.feature_dim = 1, 8
    lv = oct_.lv[0]
    lv.hash_slots, lv.features, lv.hash_capacity, lv.rows, lv.level = C.addressof(slots), C.addressof(feats), 1, 1, 12
    w = (C.c_float * 1024)()
    dec = _abi.ShineDecoder()
    dec.w1 = dec.w2 = dec.w3 = C.addressof(w)
    dec.in_dim, dec.hidden, dec.mlp_level = 8, 32, 2
    pose = (C.c_double * 16)(*np.eye(4).reshape(-1).tolist())
    out = (C.c_double * 29)()
    scratch = C.addressof((C.c_double * 8)())
    big = _abi.REGISTER_SCRATCH_BYTES
    pts = C.addressof((C.c_float * 3)())

    def call(o=oct_, d=dec, points=pts, n=1, p=pose, sigma=1.0, kappa=0.1, o_ut=out, s=scratch, sb=big):
        return lib.shine_register_normal_eq(C.byref(o) if o is not None else None, C.byref(d) if d is not None else None,
                                            points, n, p, sigma, kappa, C.addressof(o_ut) if o_ut is not None else None,
                                            s, sb, None)

    assert call(o=None) == -1 and call(d=None) == -1 and call(p=None) == -1 and call(o_ut=None) == -1
    assert call(points=None) == -1 and call(n=-1) == -1 and call(s=None) == -1 and call(sb=big - 8) == -1
    assert call(s=scratch + 4) == -1                                                   # scratch not 8-byte aligned
    for bad in (0.0, -1.0, float("nan"), float("inf")):
        assert call(kappa=bad) == -1 and call(sigma=bad) == -1
    for i in (0, 3, 11):
        for bad in (float("nan"), float("inf")):
            p = (C.c_double * 16)(*np.eye(4).reshape(-1).tolist())
            p[i] = bad
            assert call(p=p) == -1
    p = (C.c_double * 16)(*np.eye(4).reshape(-1).tolist())
    p[15] = float("nan")                                                               # row 3 is not read
    assert call(p=p, o=_abi.ShineOctree()) == -1                                       # ... but an empty octree is refused
    dec.hidden = 64
    assert call() == -2                                                                # decoder shape
    dec.hidden, oct_.feature_dim = 32, 6
    assert call() == -2                                                                # feature_dim not a multiple of 4
