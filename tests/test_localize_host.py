"""Host side of localization in a saved map (localize.py, odometry.register_scans): the argument checks of
shine_register_normal_eq_scans and its scratch size, the command's argument and pose-file refusals, the pose-file round
trip, and the lock-step scheduler on the analytic street equal to per-scan `register` bit for bit."""
import ctypes as C
import math

import numpy as np
import pytest
import torch

from shine_mapping_b200 import localize, scans
from tests.parity_utils import make_config
from tests.test_odometry_host import StreetRegistration, _pose, _street_scan


def test_scans_entry_argument_checks_need_no_gpu(built_lib):
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
    K, N = 3, 300
    poses = (C.c_double * (16 * K))(*np.tile(np.eye(4).reshape(-1), K).tolist())
    begin = (C.c_int64 * K)(0, 0, 257)
    count = (C.c_int64 * K)(257, 0, 43)
    out = (C.c_double * (29 * K))()
    scratch = C.addressof((C.c_double * 8)())
    pts = C.addressof((C.c_float * 3)())
    need = lib.shine_register_scans_scratch_bytes(count, K)
    assert need == (2 + 0 + 1) * 29 * 8

    def call(o=oct_, d=dec, points=pts, n=N, b=begin, c=count, p=poses, k=K, sigma=1.0, kappa=0.1, o_ut=out, s=scratch,
             sb=need):
        return lib.shine_register_normal_eq_scans(C.byref(o) if o is not None else None,
                                                  C.byref(d) if d is not None else None, points, n, b, c, p, k, sigma,
                                                  kappa, C.addressof(o_ut) if o_ut is not None else None, s, sb, None)

    # what shine_register_normal_eq_poses refuses
    assert call(k=0) == -1 and call(k=-2) == -1 and call(k=2 ** 31) == -1
    assert call(p=None) == -1 and call(o_ut=None) == -1
    assert call(o=None) == -1 and call(d=None) == -1 and call(points=None) == -1 and call(n=-1) == -1
    assert call(s=None) == -1 and call(sb=need - 8) == -1 and call(s=scratch + 4) == -1
    for bad in (0.0, -1.0, float("nan"), float("inf")):
        assert call(kappa=bad) == -1 and call(sigma=bad) == -1
    for k in range(K):
        for i in (0, 3, 11):
            p = (C.c_double * (16 * K))(*poses)
            p[16 * k + i] = float("nan")
            assert call(p=p) == -1
    assert call(o=_abi.ShineOctree()) == -1
    dec.hidden = 64
    assert call() == -2
    dec.hidden = 32
    # the segment table
    assert call(b=None) == -1 and call(c=None) == -1
    assert call(c=(C.c_int64 * K)(257, -1, 43)) == -1                                 # a negative n
    assert call(b=(C.c_int64 * K)(0, -1, 257)) == -1                                  # a negative begin
    assert call(b=(C.c_int64 * K)(0, 0, 258)) == -1                                   # past the points array
    assert call(n=299) == -1 and call(c=(C.c_int64 * K)(301, 0, 43)) == -1
    # the scratch size: each item's min(ceil(n / 256), 1024) blocks of 29 doubles
    f = lib.shine_register_scans_scratch_bytes
    assert f((C.c_int64 * 4)(0, 1, 256, 257), 4) == (0 + 1 + 1 + 2) * 29 * 8
    assert f((C.c_int64 * 2)(10 ** 6, 262145), 2) == 2048 * 29 * 8
    assert f(None, 1) == -1 and f((C.c_int64 * 1)(5), 0) == -1 and f((C.c_int64 * 1)(-1), 1) == -1
    assert _abi.REGISTER_ITEMS_PER_LAUNCH == 384


# ---- the command's arguments and pose files --------------------------------------------------------------------------

def _rows(poses):
    return "\n".join(" ".join(repr(float(v)) for v in P[:3].reshape(-1)) for P in poses) + "\n"


def test_command_refuses_bad_arguments(tmp_path, capsys):
    init = tmp_path / "init.txt"
    init.write_text(_rows([np.eye(4)]))
    base = ["cfg.yaml", "map.pth", "--init-poses", str(init)]
    for bad in ([], ["cfg.yaml", "map.pth"], base + ["--frames", "3:1"], base + ["--frames", "a:b"],
                base + ["--scan-dir", str(tmp_path / "missing")], base + ["--truth-poses", str(tmp_path / "none.txt")],
                ["cfg.yaml", "map.pth", "--init-poses", str(tmp_path / "none.txt")], base + ["--rgbd", "DIR"]):
        with pytest.raises(SystemExit) as e:
            localize.parse_args(bad)
        assert e.value.code == 2, bad
    args = localize.parse_args(base + ["--frames", "1:9:2", "--scan-dir", str(tmp_path)])
    assert list(args.frames) == [1, 3, 5, 7] and args.scan_dir == str(tmp_path)


def test_pose_file_refusals(tmp_path):
    rng = np.random.default_rng(0)
    poses = [_pose(rng.normal(size=3), rng.normal()) for _ in range(4)]
    path = tmp_path / "p.txt"
    path.write_text(_rows(poses))
    assert len(localize.read_init_poses(str(path), {"Tr": np.eye(4)}, 4)) == 4
    assert len(localize.read_init_poses(str(path), {"Tr": np.eye(4)}, 2)) == 2
    with pytest.raises(ValueError, match="holds 4 poses for 5 scans"):
        localize.read_init_poses(str(path), {"Tr": np.eye(4)}, 5)
    for i, bad in [(1, "nan"), (2, "inf"), (0, "-inf")]:
        text = _rows(poses).splitlines()
        vals = text[i].split()
        vals[5] = bad
        text[i] = " ".join(vals)
        path.write_text("\n".join(text) + "\n")
        with pytest.raises(ValueError, match=f"row {i}: a non-finite value"):
            localize.read_init_poses(str(path), {"Tr": np.eye(4)}, 4)
    path.write_text(_rows(poses[:1]) + "1 2 3\n")
    with pytest.raises(ValueError, match="row 1: 3 values"):
        localize.read_init_poses(str(path), {"Tr": np.eye(4)}, 2)
    path.write_text(_rows(poses) + "\n")                                      # a blank row, as read_poses_file
    with pytest.raises(ValueError, match="row 4: 0 values"):
        localize.read_init_poses(str(path), {"Tr": np.eye(4)}, 4)
    path.write_text(_rows(poses[:1]) + "1 2 x 4 5 6 7 8 9 10 11 12\n")
    with pytest.raises(ValueError, match="row 1: not a list of numbers"):
        localize.read_init_poses(str(path), {"Tr": np.eye(4)}, 2)


def _calib_file(tmp_path):
    T = _pose((0.27, -0.08, -0.12), 0.01, 0.02, -1.57)
    path = tmp_path / "calib.txt"
    path.write_text("P0: " + " ".join(["0"] * 12) + "\nTr: " + " ".join(repr(float(v)) for v in T[:3].reshape(-1)) + "\n")
    return scans.read_calib_file(str(path))


@pytest.mark.parametrize("with_calib", [False, True])
def test_pose_file_round_trip(tmp_path, with_calib):
    """--out: the estimate of each localized frame, the input row of every other frame as it was.  With calib_path ""
    the estimates read back bit for bit; with a calib to 1e-12."""
    calib = _calib_file(tmp_path) if with_calib else {"Tr": np.eye(4)}
    rng = np.random.default_rng(3)
    init = tmp_path / "init.txt"
    lines = [" ".join(f"{v:.9e}" for v in _pose(rng.normal(size=3) * 20, rng.normal())[:3].reshape(-1))
             for _ in range(6)]
    init.write_text("\n".join(lines) + "\n")
    want = localize.read_init_poses(str(init), calib, 6)
    estimates = {f: _pose(rng.normal(size=3) * 20, rng.normal(), rng.normal() * 0.1, rng.normal() * 0.1)
                 for f in (1, 4)}
    out = tmp_path / "sub" / "out.txt"
    localize.write_poses(str(out), str(init), 6, estimates, calib)
    back = scans.read_poses_file(str(out), calib)
    assert len(back) == 6
    text = out.read_text().splitlines()
    for f in range(6):
        if f in estimates:
            if with_calib:
                np.testing.assert_allclose(back[f], estimates[f], rtol=0, atol=1e-12)
            else:
                assert np.array_equal(back[f].view(np.int64), estimates[f].view(np.int64))
        else:
            assert text[f] == lines[f]
            assert np.array_equal(back[f].view(np.int64), want[f].view(np.int64))


def test_pose_errors():
    truth = _pose((1.0, 2.0, 0.5), 0.3)
    est = truth @ _pose((0.03, -0.04, 0.0), math.radians(0.5))
    t, r = localize.pose_errors(est, truth)
    assert abs(t - 0.05) < 1e-12 and abs(r - 0.5) < 1e-9


# ---- the lock-step scheduler on the analytic street ---------------------------------------------------------------------

@pytest.mark.parametrize("max_iters", [6, 3])
def test_lock_step_equals_per_scan_register_on_the_street(max_iters):
    """Two scans from poses along the street, each started off its own, and one that fails (no point on the map):
    register_scans equals register scan by scan, poses and info, bit for bit.  With max_iters = 3 (the widened
    iterations only) every scan stops at max_iters without converging."""
    cfg = make_config(3)
    scans_, inits = [], []
    for t, yaw, dt, dyaw in [((10.0, 0.5, 0.0), 0.1, (0.4, 0.0, 0.0), 0.0),
                             ((14.0, -0.5, 0.0), 0.05, (0.2, -0.3, 0.0), math.radians(4))]:
        truth = _pose(t, yaw)
        scans_.append(torch.from_numpy(_street_scan(truth) * cfg.scale).float())
        inits.append(_pose(truth[:3, 3] + np.array(dt), yaw + dyaw))
    scans_.insert(1, torch.zeros(10, 3))                              # far from every surface: no point on the map
    inits.insert(1, _pose((1.0, 2.0, 0.0), 0.3))
    reg = StreetRegistration(cfg, None, None, max_iters=max_iters, tol=1e-6)
    got = reg.register_scans(scans_, inits)
    for s, (pose, info) in enumerate(got):
        want_pose, want_info = reg.register(scans_[s], inits[s])
        assert np.array_equal(pose.view(np.int64), want_pose.view(np.int64)), s
        assert info.keys() == want_info.keys() and all(
            info[k] == want_info[k] or (info[k] != info[k] and want_info[k] != want_info[k]) for k in info), (info, want_info)
    assert not got[1][1]["ok"] and "points on the map" in got[1][1]["reason"] and np.array_equal(got[1][0], inits[1])
    assert got[0][1]["ok"] and got[2][1]["ok"]
    assert got[0][1]["converged"] == got[2][1]["converged"] == (max_iters == 6), [g[1] for g in got]


def test_register_scans_edge_cases():
    cfg = make_config(3)
    reg = StreetRegistration(cfg, None, None)
    assert reg.register_scans([], []) == []
    with pytest.raises(ValueError, match="2 scans, 1 initial poses"):
        reg.register_scans([torch.zeros(1, 3)] * 2, [np.eye(4)])
