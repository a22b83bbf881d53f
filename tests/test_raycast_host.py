"""Host side of held-out scan evaluation: the argument checks of shine_raycast, the `evaluate scans` command line, the
held-out frame selection, `--frames` parsing and the metric assembly.  No GPU needed."""
import ctypes as C
import math

import numpy as np
import pytest
import torch

from shine_mapping_b200 import evaluate, raycast
from tests.parity_utils import make_config


def test_raycast_entry_argument_checks_need_no_gpu(built_lib):
    from shine_mapping_b200 import _abi
    lib = built_lib
    slots = (C.c_uint8 * 64)()
    feats = (C.c_float * 8)()
    oct_ = _abi.ShineOctree()
    oct_.num_levels, oct_.feature_dim = 2, 8
    for i in range(2):
        lv = oct_.lv[i]
        lv.hash_slots, lv.features, lv.hash_capacity, lv.rows, lv.level = C.addressof(slots), C.addressof(feats), 1, 1, 12 - i
    w = (C.c_float * 1024)()
    dec = _abi.ShineDecoder()
    dec.w1 = dec.w2 = dec.w3 = C.addressof(w)
    dec.in_dim, dec.hidden, dec.mlp_level = 8, 32, 2
    origin = (C.c_float * 3)(0.0, 0.0, 0.0)
    pts = C.addressof((C.c_float * 3)())
    out_t = C.addressof((C.c_float * 1)())
    out_s = C.addressof((C.c_uint8 * 1)())

    def call(o=oct_, d=dec, org=origin, points=pts, n=1, h=1e-3, t_min=0.0, beyond=0.01, t_max=float("inf"), it=8, ml=0,
             ot=out_t, os_=out_s):
        return lib.shine_raycast(C.byref(o) if o is not None else None, C.byref(d) if d is not None else None, org, points,
                                 n, h, t_min, beyond, t_max, it, ml, ot, os_, None)

    assert call(n=0, points=None, ot=None, os_=None) == 0                # nothing to cast: no launch, no device
    assert call(n=-1) == -1
    assert call(points=None) == -1 and call(ot=None) == -1 and call(os_=None) == -1
    assert call(o=None) == -1 and call(d=None) == -1 and call(org=None) == -1
    for bad in (0.0, -1e-3, float("nan"), float("inf")):
        assert call(h=bad, n=0) == -1
    for bad in (float("nan"), float("inf"), -float("inf")):
        assert call(t_min=bad, n=0) == -1
        assert call(org=(C.c_float * 3)(0.0, bad, 0.0), n=0) == -1
    assert call(t_max=0.0, n=0) == -1 and call(t_min=1.0, t_max=0.5, n=0) == -1 and call(t_max=float("nan"), n=0) == -1
    for bad in (-1e-6, float("nan"), float("inf")):
        assert call(beyond=bad, n=0) == -1
    assert call(it=-1, n=0) == -1 and call(it=_abi.RAYCAST_MAX_REFINE + 1, n=0) == -1
    assert call(it=0, n=0) == 0 and call(it=_abi.RAYCAST_MAX_REFINE, n=0) == 0
    assert call(ml=-1, n=0) == -1 and call(ml=2, n=0) == -1 and call(ml=1, n=0) == 0
    assert call(o=_abi.ShineOctree(), n=0) == -1
    dec.hidden = 64
    assert call(n=0) == -2
    dec.hidden, oct_.feature_dim = 32, 6
    assert call(n=0) == -2


def _parse(argv):
    return evaluate.parse_args(["scans", "cfg.yaml", "model.pth", *argv])


def test_scans_command_line():
    mode, a = _parse([])
    assert mode == "scans" and a.config == "cfg.yaml" and a.checkpoint == "model.pth"
    assert a.frames is None and a.step_m is None and a.beyond_m == 1.0 and a.threshold == 0.1
    assert a.refine_iters == raycast.REFINE_ITERS and a.csv is None and a.points_dir is None and a.rgbd is None
    _, a = _parse(["--frames", "3:11:2", "--step-m", "0.05", "--beyond-m", "0", "--threshold", "0.2", "--csv", "o.csv",
                   "--points-dir", "pts", "--refine-iters", "0"])
    assert list(a.frames) == [3, 5, 7, 9] and a.step_m == 0.05 and a.beyond_m == 0.0 and a.threshold == 0.2
    assert a.csv == "o.csv" and a.points_dir == "pts" and a.refine_iters == 0
    _, a = _parse(["--rgbd", "depth", "--pose-file", "poses.txt", "--intrinsic-file", "focal.txt"])
    assert a.rgbd == "depth" and a.pose_file == "poses.txt" and a.intrinsic_file == "focal.txt"
    # the crop and mesh forms are unchanged
    assert evaluate.parse_args(["crop", "gt.ply", "a.ply", "--out", "o.ply"])[0] == "crop"
    assert evaluate.parse_args(["pred.ply", "gt.ply"])[0] == "eval"


@pytest.mark.parametrize("argv,message", [
    (["--frames", "5"], "START:STOP"), (["--frames", "a:b"], "START:STOP"), (["--frames", "4:4"], "START < STOP"),
    (["--frames", "0:4:0"], "STEP >= 1"), (["--frames=-2:4"], "START < STOP"),
    (["--step-m", "0"], "--step-m must be > 0"), (["--step-m", "nan"], "--step-m must be > 0"),
    (["--threshold", "-1"], "--threshold must be > 0"), (["--beyond-m", "-0.1"], "--beyond-m must be >= 0"),
    (["--refine-iters", "33"], "--refine-iters must be in [0, 32]"), (["--rgbd", "depth"], "--rgbd needs --pose-file"),
])
def test_scans_command_line_errors(capsys, argv, message):
    with pytest.raises(SystemExit):
        _parse(argv)
    assert message in capsys.readouterr().err


def test_parse_frames():
    assert list(raycast.parse_frames("0:3")) == [0, 1, 2]
    assert list(raycast.parse_frames("1:10:4")) == [1, 5, 9]
    for bad in ("", "3", "1:2:3:4", "x:2", "2:1", "0:5:-1", "1.5:3"):
        with pytest.raises(ValueError):
            raycast.parse_frames(bad)


def test_held_out_frames():
    cfg = make_config(begin_frame=0, end_frame=100, every_frame=2)
    assert raycast.held_out_frames(cfg, 20) == list(range(1, 20, 2))
    cfg = make_config(begin_frame=3, end_frame=10, every_frame=3)
    assert raycast.held_out_frames(cfg, 50) == [4, 5, 7, 8, 10]
    cfg = make_config(begin_frame=0, end_frame=100, every_frame=1)
    assert raycast.held_out_frames(cfg, 20) == []                # every frame mapped: the command asks for --frames


def test_map_pose_of_held_out_frames():
    """poses_ref keeps world poses for the frames mapping skips; map_pose puts every frame into the map frame."""
    W = [np.eye(4) for _ in range(4)]
    for f, T in enumerate(W):
        T[:3, 3] = [2.0 * f + 1.0, 0.5 * f, 0.0]

    class DS:
        used_frames = [0, 2]
        begin_pose_inv = np.linalg.inv(W[0])
        poses_ref = [np.linalg.inv(W[0]) @ W[0], W[1], np.linalg.inv(W[0]) @ W[2], W[3]]

    for f in range(4):
        np.testing.assert_allclose(raycast.map_pose(DS, f), np.linalg.inv(W[0]) @ W[f], atol=1e-12)


def test_ray_metrics():
    rng = torch.tensor([10.0, 5.05, float("nan"), 2.0, 8.3], dtype=torch.float64)
    hit = torch.tensor([True, True, False, True, True])
    meas = torch.tensor([10.02, 5.0, 7.0, 2.5, 8.3], dtype=torch.float64)
    m = raycast.ray_metrics(rng, hit, meas, 0.1)
    err = np.array([-0.02, 0.05, -0.5, 0.0])
    assert m["rays"] == 5 and m["hits"] == 4 and m["hit_ratio"] == 0.8
    assert m["mean_abs_err_m"] == pytest.approx(np.abs(err).mean())
    assert m["median_abs_err_m"] == pytest.approx(np.median(np.abs(err)))
    assert m["rmse_m"] == pytest.approx(np.sqrt((err ** 2).mean()))
    assert m["bias_m"] == pytest.approx(err.mean())
    assert m["within_threshold"] == pytest.approx(3 / 5)              # the miss counts as outside
    assert list(m) == raycast.METRIC_COLUMNS
    miss = raycast.ray_metrics(torch.full((3,), float("nan")), torch.zeros(3, dtype=torch.bool), torch.ones(3), 0.1)
    assert miss["rays"] == 3 and miss["hits"] == 0 and miss["hit_ratio"] == 0.0 and miss["within_threshold"] == 0.0
    assert all(math.isnan(miss[k]) for k in ("mean_abs_err_m", "median_abs_err_m", "rmse_m", "bias_m"))
    empty = raycast.ray_metrics(torch.zeros(0), torch.zeros(0, dtype=torch.bool), torch.zeros(0), 0.1)
    assert empty["rays"] == 0 and empty["hits"] == 0
    assert all(math.isnan(empty[k]) for k in raycast.METRIC_COLUMNS[2:])
    with pytest.raises(ValueError):
        raycast.ray_metrics(torch.zeros(2), torch.zeros(3, dtype=torch.bool), torch.zeros(2), 0.1)


def test_scans_csv(tmp_path):
    import csv
    rows = [{"frame": 1, **raycast.ray_metrics(torch.tensor([1.0]), torch.tensor([True]), torch.tensor([1.05]), 0.1)},
            {"frame": 3, **raycast.ray_metrics(torch.zeros(0), torch.zeros(0, dtype=torch.bool), torch.zeros(0), 0.1)}]
    total = raycast.ray_metrics(torch.tensor([1.0]), torch.tensor([True]), torch.tensor([1.05]), 0.1)
    path = tmp_path / "out" / "scans.csv"
    evaluate.write_scans_csv(str(path), {"frames": rows, "total": total})
    with open(path) as fh:
        got = list(csv.DictReader(fh))
    assert [r["frame"] for r in got] == ["1", "3", "total"]
    assert list(got[0]) == ["frame"] + raycast.METRIC_COLUMNS
    assert float(got[0]["median_abs_err_m"]) == pytest.approx(0.05) and got[1]["rays"] == "0"
