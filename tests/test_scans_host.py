"""Host side of real-scan input: readers, natural order, frame selection, poses, the sampler oracle against the
reference's own sampler (tests/golden/ref_sampler.npz) and the settings that are rejected."""
import os
import sys

import numpy as np
import pytest

from shine_mapping_b200 import scans
from shine_mapping_b200.config import SHINEConfig
from oracle.make_golden import REF as REFERENCE   # the reference checkout, where one is mounted
from tests import scan_oracle

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _points(n=50, seed=0):
    p = np.random.default_rng(seed).normal(size=(n, 3)) * 10
    p[0] = (np.nan, 1.0, 2.0)
    p[1] = (np.inf, 0.0, 0.0)
    return p


def _write_ply(path, p, fmt, t):
    extra = np.arange(p.shape[0], dtype=np.float32)
    with open(path, "wb") as fh:
        fh.write(f"ply\nformat {fmt} 1.0\ncomment test\nelement vertex {p.shape[0]}\nproperty uchar tag\n"
                 f"property {t} x\nproperty {t} y\nproperty {t} z\nproperty float intensity\n"
                 f"element face 0\nproperty list uchar int vertex_indices\nend_header\n".encode())
        if fmt == "ascii":
            for i, q in enumerate(p):
                fh.write(f"7 {float(q[0])!r} {float(q[1])!r} {float(q[2])!r} {float(extra[i])!r}\n".encode())
        else:
            dt = np.dtype([("tag", "u1"), ("x", t[0] == "f" and "<f4" or "<f8"), ("y", t[0] == "f" and "<f4" or "<f8"),
                           ("z", t[0] == "f" and "<f4" or "<f8"), ("i", "<f4")])
            rec = np.zeros(p.shape[0], dt)
            rec["tag"], rec["x"], rec["y"], rec["z"], rec["i"] = 7, p[:, 0], p[:, 1], p[:, 2], extra
            fh.write(rec.tobytes())


def _write_pcd(path, p, data, xyz_last=False):
    n = p.shape[0]
    if xyz_last:
        fields, size, typ, count = "intensity rgb x y z", "4 1 8 8 8", "F U F F F", "1 3 1 1 1"
        dt = np.dtype([("i", "<f4"), ("c", "u1", 3), ("x", "<f8"), ("y", "<f8"), ("z", "<f8")])
    else:
        fields, size, typ, count = "x y z intensity", "4 4 4 4", "F F F F", "1 1 1 1"
        dt = np.dtype([("x", "<f4"), ("y", "<f4"), ("z", "<f4"), ("i", "<f4")])
    rec = np.zeros(n, dt)
    rec["x"], rec["y"], rec["z"] = p[:, 0], p[:, 1], p[:, 2]
    with open(path, "wb") as fh:
        fh.write(f"# .PCD v0.7\nVERSION 0.7\nFIELDS {fields}\nSIZE {size}\nTYPE {typ}\nCOUNT {count}\nWIDTH {n}\n"
                 f"HEIGHT 1\nVIEWPOINT 0 0 0 1 0 0 0\nPOINTS {n}\nDATA {data}\n".encode())
        if data == "ascii":
            for r in rec:
                vals = [r[name] for name in dt.names]
                flat = []
                for v in vals:
                    flat.extend(np.atleast_1d(v).tolist())
                fh.write((" ".join(repr(float(v)) if not isinstance(v, int) else str(v) for v in flat) + "\n").encode())
        else:
            fh.write(rec.tobytes())
    return rec


def _same(a, b):
    np.testing.assert_array_equal(np.isnan(a), np.isnan(b))
    np.testing.assert_array_equal(np.nan_to_num(a), np.nan_to_num(b))


def test_bin_round_trip(tmp_path):
    p = _points().astype(np.float32)
    raw = np.concatenate((p, np.ones((p.shape[0], 1), np.float32)), 1)
    raw.tofile(tmp_path / "000.bin")
    rec = scans.read_scan(str(tmp_path / "000.bin"), pinned=False)
    assert (rec.n, rec.stride, rec.fp64, rec.offset) == (p.shape[0], 16, False, 0)
    _same(rec.points(), np.fromfile(tmp_path / "000.bin", dtype=np.float32).reshape(-1, 4)[:, :3].astype(np.float64))
    (tmp_path / "bad.bin").write_bytes(b"\0" * 20)
    with pytest.raises(ValueError, match="bad.bin"):
        scans.read_scan(str(tmp_path / "bad.bin"), pinned=False)


@pytest.mark.parametrize("fmt", ["ascii", "binary_little_endian"])
@pytest.mark.parametrize("t", ["float", "double"])
def test_ply_round_trip(tmp_path, fmt, t):
    p = _points()
    want = p.astype(np.float32).astype(np.float64) if t == "float" else p
    path = str(tmp_path / "a.ply")
    _write_ply(path, want, fmt, t)
    rec = scans.read_scan(path, pinned=False)
    assert rec.n == p.shape[0] and rec.fp64 == (t == "double")
    _same(rec.points(), want)


@pytest.mark.parametrize("data", ["ascii", "binary"])
@pytest.mark.parametrize("xyz_last", [False, True])
def test_pcd_round_trip(tmp_path, data, xyz_last):
    p = _points()
    path = str(tmp_path / "a.pcd")
    rec = _write_pcd(path, p, data, xyz_last)
    got = scans.read_scan(path, pinned=False)
    want = np.stack([rec["x"], rec["y"], rec["z"]], 1).astype(np.float64)
    assert got.n == p.shape[0] and got.fp64 == xyz_last
    _same(got.points(), want)


def test_rejected_files(tmp_path):
    p = _points(5)
    _write_ply(str(tmp_path / "be.ply"), p, "binary_big_endian", "float")
    with pytest.raises(ValueError, match="be.ply.*big-endian"):
        scans.read_scan(str(tmp_path / "be.ply"), pinned=False)
    (tmp_path / "list.ply").write_bytes(b"ply\nformat ascii 1.0\nelement vertex 1\nproperty float x\nproperty float y\n"
                                        b"property float z\nproperty list uchar int idx\nend_header\n1 2 3 1 4\n")
    with pytest.raises(ValueError, match="list.ply.*list property"):
        scans.read_scan(str(tmp_path / "list.ply"), pinned=False)
    (tmp_path / "nohead.ply").write_bytes(b"ply\nformat ascii 1.0\nelement vertex 1\nproperty float x\n1 2 3\n")
    with pytest.raises(ValueError, match="nohead.ply.*malformed header"):
        scans.read_scan(str(tmp_path / "nohead.ply"), pinned=False)
    _write_pcd(str(tmp_path / "c.pcd"), p, "binary_compressed")
    with pytest.raises(ValueError, match="c.pcd.*binary_compressed"):
        scans.read_scan(str(tmp_path / "c.pcd"), pinned=False)
    (tmp_path / "m.pcd").write_bytes(b"VERSION 0.7\nFIELDS x y z\nSIZE 4 4\nTYPE F F F\nPOINTS 1\nDATA ascii\n1 2 3\n")
    with pytest.raises(ValueError, match="m.pcd.*malformed"):
        scans.read_scan(str(tmp_path / "m.pcd"), pinned=False)
    (tmp_path / "noz.pcd").write_bytes(b"FIELDS x y\nSIZE 4 4\nTYPE F F\nPOINTS 1\nDATA ascii\n1 2\n")
    with pytest.raises(ValueError, match="noz.pcd.*'z'"):
        scans.read_scan(str(tmp_path / "noz.pcd"), pinned=False)
    with pytest.raises(ValueError, match="x.txt"):
        scans.read_scan(str(tmp_path / "x.txt"), pinned=False)


def test_natural_order_and_selection():
    assert scans.natural_sorted(["10.bin", "2.bin", "1.bin", "a10", "a9"]) == ["1.bin", "2.bin", "10.bin", "a9", "a10"]
    cfg = SHINEConfig(begin_frame=2, end_frame=9, every_frame=3)
    assert [f for f in range(12) if scans.used_frame(cfg, f)] == [3, 6, 9]


def _pose_files(tmp_path, n=6, seed=1):
    rng = np.random.default_rng(seed)
    lines = []
    for k in range(n):
        a = 0.3 * k
        R = np.array([[np.cos(a), -np.sin(a), 0], [np.sin(a), np.cos(a), 0], [0, 0, 1]])
        t = rng.normal(size=3) * 5
        lines.append(" ".join(repr(float(v)) for v in np.concatenate((R, t[:, None]), 1).reshape(-1)))
    (tmp_path / "poses.txt").write_text("\n".join(lines) + "\n")
    tr = "0.0004276 -0.9999 -0.0080 -0.0119 -0.0072 0.0080 -0.9999 -0.0540 0.9999 0.0004 -0.0072 -0.2921"
    (tmp_path / "calib.txt").write_text(f"P0: 1 0 0 0 0 1 0 0 0 0 1 0\nTr: {tr}\n")


def _restated_poses(tmp_path, calib_path, first_frame_ref, shift, frames):
    calib = {}
    if calib_path:
        for line in open(calib_path):
            key, content = line.strip().split(":")
            v = [float(x) for x in content.split()]
            m = np.zeros((4, 4)); m[0, :4], m[1, :4], m[2, :4] = v[0:4], v[4:8], v[8:12]; m[3, 3] = 1.0
            calib[key] = m
    else:
        calib["Tr"] = np.eye(4)
    poses = []
    for line in open(tmp_path / "poses.txt"):
        v = [float(x) for x in line.split()]
        m = np.zeros((4, 4)); m[0, :4], m[1, :4], m[2, :4] = v[0:4], v[4:8], v[8:12]; m[3, 3] = 1.0
        poses.append(np.matmul(np.linalg.inv(calib["Tr"]), np.matmul(m, calib["Tr"])))
    inv0 = np.linalg.inv(poses[frames[0]]) if first_frame_ref else np.eye(4)
    if not first_frame_ref:
        inv0[2, 3] += shift
    return [np.matmul(inv0, poses[f]) if f in frames else poses[f] for f in range(len(poses))]


@pytest.mark.parametrize("first_frame_ref", [True, False])
@pytest.mark.parametrize("with_calib", [True, False])
def test_poses_bit_identical(tmp_path, first_frame_ref, with_calib):
    _pose_files(tmp_path)
    calib = str(tmp_path / "calib.txt") if with_calib else ""
    cfg = SHINEConfig(pose_path=str(tmp_path / "poses.txt"), calib_path=calib, first_frame_ref=first_frame_ref,
                      global_shift_default=0.17241, begin_frame=1, end_frame=4, every_frame=1)
    c = scans.read_calib_file(calib) if calib else {"Tr": np.eye(4)}
    got, _, used = scans.reference_poses(cfg, scans.read_poses_file(cfg.pose_path, c), 6)
    assert used == [1, 2, 3, 4]
    want = _restated_poses(tmp_path, calib, first_frame_ref, 0.17241, used)
    for g, w in zip(got, want):
        assert np.array_equal(g, w)
    if os.path.isfile(os.path.join(REFERENCE, "utils", "pose.py")):
        import types
        sys.modules.setdefault("pyquaternion", types.SimpleNamespace(Quaternion=object))
        sys.path.insert(0, REFERENCE)
        try:
            from utils import pose as ref_pose
            ref_calib = ref_pose.read_calib_file(calib) if calib else {"Tr": np.eye(4)}
            for g, w in zip(scans.read_poses_file(cfg.pose_path, c), ref_pose.read_poses_file(cfg.pose_path, ref_calib)):
                assert np.array_equal(g, w)
        finally:
            sys.path.remove(REFERENCE)


def test_fewer_poses_than_scans(tmp_path):
    _pose_files(tmp_path, n=3)
    cfg = SHINEConfig(pose_path=str(tmp_path / "poses.txt"))
    with pytest.raises(ValueError, match="3 poses for 5 scans"):
        scans.reference_poses(cfg, scans.read_poses_file(cfg.pose_path, {"Tr": np.eye(4)}), 5)


def _golden_cfg(g):
    return SHINEConfig(surface_sample_n=int(g["surface_sample_n"]), free_sample_n=int(g["free_sample_n"]),
                       surface_sample_range_m=float(g["surface_sample_range_m"]),
                       free_sample_end_dist_m=float(g["free_sample_end_dist_m"]),
                       free_sample_begin_ratio=float(g["free_sample_begin_ratio"]))


def check_against_reference_sampler(coord, label, weight, g):
    """Bit for bit on rays whose fp32 distance agrees with the reference's CPU torch.linalg.norm.  Elsewhere the norm's
    reduction order moved the distance by one ulp, which the ratio carries on: coordinates within 2 ulp of the ray's
    distance, labels (a difference of ratios near 1, times the distance) within 3."""
    ns_nf = int(g["surface_sample_n"]) + int(g["free_sample_n"])
    s = (g["points"] - g["origin"]).astype(np.float32)
    d = np.sqrt((s[:, 0] * s[:, 0] + s[:, 1] * s[:, 1]) + s[:, 2] * s[:, 2])
    import torch
    agree = np.repeat(torch.linalg.norm(torch.tensor(s), dim=1).numpy() == d, ns_nf)
    assert agree.mean() > 0.8
    np.testing.assert_array_equal(coord[agree], g["coord"][agree])
    np.testing.assert_array_equal(label[agree], g["label"][agree])
    np.testing.assert_array_equal(weight, g["weight"])
    tol = 2 * np.repeat(np.spacing(d), ns_nf)
    assert (np.abs(coord - g["coord"]).max(1) <= tol).all()
    assert (np.abs(label - g["label"]) <= 1.5 * tol).all()


def test_sampler_oracle_matches_reference():
    g = np.load(os.path.join(ROOT, "tests", "golden", "ref_sampler.npz"))
    cfg = _golden_cfg(g)
    cfg.scale = float(g["scale"])
    coord, label, weight = scan_oracle.sample(g["points"], g["origin"], g["u_surface"], g["u_free"], cfg)
    check_against_reference_sampler(coord, label, weight, g)


@pytest.mark.parametrize("key,value", [("rand_downsample", True), ("filter_noise", True), ("estimate_normal", True),
                                       ("behind_dropoff_on", True), ("clearance_sample_n", 2), ("semantic_on", True),
                                       ("pose_path", "odom.csv")])
def test_rejected_settings(key, value):
    cfg = SHINEConfig(rand_downsample=False, pose_path="poses.txt")
    setattr(cfg, key, value)
    with pytest.raises(NotImplementedError, match=key):
        scans.check_scan_config(cfg)
