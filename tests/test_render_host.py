"""Host-side parts of rendering (render.py, DESIGN §14): `depth_metrics` against goldens recorded from the reference's
own `eval_depth` (oracle/make_depth_golden.py), the camera-ray formulas against fp64, the PNG writer through rgbd's
decoder, the command lines and frame selection.  No GPU needed."""
import math
import os
import types

import numpy as np
import pytest
import torch

from shine_mapping_b200 import render
from tests import render_rays as rr

GOLDEN = os.path.join(os.path.dirname(__file__), "golden", "ref_eval_depth.npz")


def test_depth_metrics_match_reference_goldens():
    z = np.load(GOLDEN)
    assert list(z["keys"]) == render.DEPTH_METRICS
    for i in range(int(z["count"])):
        got = render.depth_metrics(torch.from_numpy(z[f"pred_{i}"]), torch.from_numpy(z[f"target_{i}"]))
        want = z[f"metrics_{i}"]
        assert list(got) == render.DEPTH_METRICS
        # fp64 sums in another order than numpy's pairwise sum: a few units in the last place
        np.testing.assert_allclose([got[k] for k in render.DEPTH_METRICS], want, rtol=1e-12, atol=0, err_msg=f"case {i}")


def test_depth_metrics_empty_mask_and_shapes():
    m = render.depth_metrics(torch.zeros(3, 4, dtype=torch.float64), torch.ones(3, 4, dtype=torch.float64))
    assert m["complete"] == 0.0 and all(math.isnan(m[k]) for k in render.DEPTH_METRICS if k != "complete")
    with pytest.raises(ValueError, match="differ in shape"):
        render.depth_metrics(torch.zeros(3, 4), torch.zeros(4, 3))


def test_pinhole_rays_against_fp64():
    W, H, fx, fy, cx, cy = 64, 48, 52.5, 49.0, 31.5, 23.5
    c, cz = rr.pinhole_dirs(W, H, fx, fy, cx, cy)
    u, v = rr.pixel_grid(W, H)
    want = np.stack([(u - cx) / fx, (v - cy) / fy, np.ones(u.shape)], 1)
    want /= np.linalg.norm(want, axis=1, keepdims=True)
    # four roundings before the square root, one after, and the division: well inside 8 u per component
    assert np.abs(c.astype(np.float64) - want).max() <= 8 * 2.0 ** -24
    assert np.array_equal(cz, c[:, 2])
    centre = (v == 23) & (u == 31)
    assert c[centre, 0] < 0 and c[centre, 1] < 0                        # left of and above the principal point


def test_range_image_rays_against_fp64():
    W, H, up, down = 1024, 64, 2.0, -24.8
    c, ones = rr.range_image_dirs(W, H, up, down)
    assert (ones == 1).all()
    u, v = rr.pixel_grid(W, H)
    el = np.deg2rad(up) - v * np.deg2rad(up - down) / (H - 1)
    az = np.pi - 2 * np.pi * u / W
    want = np.stack([np.cos(el) * np.cos(az), np.cos(el) * np.sin(az), np.sin(el)], 1)
    # el and az rounded to fp32 (|el| <= 0.44, |az| <= pi), then rounded sines and cosines and one product
    assert np.abs(c.astype(np.float64) - want).max() <= 8 * 2.0 ** -24 * math.pi
    assert np.allclose(np.rad2deg(np.arcsin(c[v == 0, 2])), up, atol=1e-5)
    assert np.allclose(np.rad2deg(np.arcsin(c[v == H - 1, 2])), down, atol=1e-5)
    first = c[(u == 0) & (v == H // 2)][0]
    assert first[0] < 0 and abs(first[1]) < 1e-6                     # column 0 looks along -x (azimuth +pi)
    quarter = c[(u == W // 4) & (v == H // 2)][0]
    assert quarter[1] > 0.9                                           # azimuth falls with the column: +pi/2 at W/4
    one_row = rr.range_image_dirs(8, 1, 10.0, -10.0)[0]
    assert np.allclose(np.rad2deg(np.arcsin(one_row[:, 2])), 10.0, atol=1e-5)


def test_map_rays_rotate_per_row():
    c, _ = rr.pinhole_dirs(5, 4, 3.0, 3.0, 2.0, 1.5)
    P = np.array([[0, 0, 1, 0.25], [1, 0, 0, -0.5], [0, 1, 0, 0.125]], np.float32)
    o, d = rr.map_rays(c, P)
    assert np.array_equal(o, P[:, 3])
    assert np.array_equal(d, c[:, [2, 0, 1]])                         # a permutation is exact


def test_range_image_camera_from_points():
    pts = torch.tensor([[10.0, 0.0, 1.0], [0.0, -5.0, -5.0], [3.0, 4.0, 0.0]])
    cam = render.RangeImageCamera.from_points(pts)
    assert (cam.width, cam.height) == render.RANGE_IMAGE_SIZE
    assert cam.fov_up == pytest.approx(math.degrees(math.atan2(1.0, 10.0)))
    assert cam.fov_down == pytest.approx(-45.0)
    for bad in [(0, 64, 2.0, -24.0), (1024, -1, 2.0, -24.0), (8, 8, -1.0, -1.0), (8, 8, float("nan"), 0.0)]:
        with pytest.raises(ValueError):
            render.RangeImageCamera(*bad)
    with pytest.raises(ValueError, match="no points"):
        render.RangeImageCamera.from_points(torch.zeros(0, 3))


def test_sensor_to_map_folds_the_extrinsic():
    from shine_mapping_b200.rgbd import FLIP_YZ, RGBDCamera
    pose = np.eye(4)
    pose[:3, 3] = (1.0, 2.0, 3.0)
    cam = RGBDCamera(64, 48, 50.0, 50.0, 31.5, 23.5, extrinsic=FLIP_YZ)
    assert np.array_equal(render.sensor_to_map(pose, cam), pose @ np.linalg.inv(FLIP_YZ))
    assert np.array_equal(render.sensor_to_map(pose, render.RangeImageCamera(8, 4, 1.0, -1.0)), pose)


# ---- PNG -----------------------------------------------------------------------------------------------------------------

def test_png_round_trip_through_rgbd_decoder(tmp_path):
    from shine_mapping_b200 import rgbd
    rng = np.random.default_rng(3)
    depth = rng.uniform(0.1, 70.0, (37, 53))
    depth[0, :5] = 0.0
    depth[1, :3] = np.nan
    depth[2, 0] = 65.535                                               # the largest value that fits at 1000 / m
    depth[2, 1] = 65.5355                                              # rounds to 65536: does not fit
    raw, over = render.depth_png(depth, 1000.0)
    fits = np.isfinite(depth) & (depth > 0) & (np.floor(depth * 1000.0 + 0.5) <= 65535)
    assert over == int((np.isfinite(depth) & (depth > 0) & ~fits).sum()) and over > 0
    assert raw[2, 0] == 65535 and raw[2, 1] == 0 and (raw[0, :5] == 0).all() and (raw[1, :3] == 0).all()
    assert np.array_equal(raw[fits], np.floor(depth[fits] * 1000.0 + 0.5).astype(np.uint16))
    p = str(tmp_path / "d" / "depth.png")
    render.write_png(p, raw)
    assert np.array_equal(rgbd.read_depth(p, pinned=False).numpy(), raw)

    n = rng.normal(size=(37, 53, 3))
    n /= np.linalg.norm(n, axis=2, keepdims=True)
    n[3, 4] = np.nan
    img = render.normal_png(torch.from_numpy(n))
    assert img.dtype == np.uint8 and (img[3, 4] == 0).all()
    assert np.array_equal(img[0, 0], np.rint((n[0, 0] + 1) * 0.5 * 255).astype(np.uint8))
    q = str(tmp_path / "n.png")
    render.write_png(q, img)
    assert np.array_equal(rgbd.read_color(q, pinned=False).numpy(), img)
    for bad in [np.zeros((4, 4), np.float32), np.zeros((4, 4, 3), np.uint16), np.zeros((0, 4), np.uint16)]:
        with pytest.raises(ValueError):
            render.write_png(str(tmp_path / "x.png"), bad)


# ---- command lines and frames ----------------------------------------------------------------------------------------

def _usage_error(capsys, fn, argv, text):
    with pytest.raises(SystemExit) as e:
        fn(argv)
    assert e.value.code == 2
    assert text in capsys.readouterr().err


def test_render_command_line(capsys):
    with pytest.raises(SystemExit) as e:
        render.parse_args(["--help"])
    assert e.value.code == 0 and "--range-image" in capsys.readouterr().out
    a = render.parse_args(["c.yaml", "m.pth", "--out", "o", "--frames", "2:9:3", "--range-image", "512", "32", "3", "-25",
                           "--npz"])
    assert list(a.frames) == [2, 5, 8] and a.npz and isinstance(a.range_image, render.RangeImageCamera)
    assert (a.range_image.width, a.range_image.height, a.range_image.fov_up, a.range_image.fov_down) == (512, 32, 3, -25)
    _usage_error(capsys, render.parse_args, ["c.yaml", "m.pth"], "--out")
    _usage_error(capsys, render.parse_args, ["c", "m", "--out", "o", "--frames", "5:2"], "START < STOP")
    _usage_error(capsys, render.parse_args, ["c", "m", "--out", "o", "--step-m", "0"], "--step-m must be > 0")
    _usage_error(capsys, render.parse_args, ["c", "m", "--out", "o", "--max-range-m", "inf"], "--max-range-m must be > 0")
    _usage_error(capsys, render.parse_args, ["c", "m", "--out", "o", "--range-image", "0", "64", "2", "-24"],
                 "--range-image")
    _usage_error(capsys, render.parse_args, ["c", "m", "--out", "o", "--range-image", "8", "8", "-3", "2"],
                 "--range-image")
    _usage_error(capsys, render.parse_args, ["c", "m", "--out", "o", "--rgbd", "d"], "--pose-file")
    _usage_error(capsys, render.parse_args, ["c", "m", "--out", "o", "--rgbd", "d", "--pose-file", "p",
                                             "--range-image", "8", "8", "2", "-2"], "pinhole")


def test_evaluate_depth_command_line(capsys):
    from shine_mapping_b200 import evaluate
    with pytest.raises(SystemExit) as e:
        evaluate.parse_args(["depth", "--help"])
    assert e.value.code == 0 and "eval_depth" in capsys.readouterr().out
    mode, a = evaluate.parse_args(["depth", "c", "m", "--rgbd", "d", "--pose-file", "p", "--frames", "1:4", "--csv",
                                   "x.csv", "--out", "o"])
    assert mode == "depth" and list(a.frames) == [1, 2, 3] and a.max_range_m == 10.0 and a.csv == "x.csv"
    _usage_error(capsys, evaluate.parse_args, ["depth", "c", "m"], "needs RGB-D frames")
    _usage_error(capsys, evaluate.parse_args, ["depth", "c", "m", "--rgbd", "d"], "--pose-file")
    _usage_error(capsys, evaluate.parse_args, ["depth", "c", "m", "--rgbd", "d", "--pose-file", "p", "--frames", "x"],
                 "--frames")
    _usage_error(capsys, evaluate.parse_args, ["depth", "c", "m", "--rgbd", "d", "--pose-file", "p", "--max-range-m",
                                               "-1"], "--max-range-m must be > 0")


def test_frame_selection():
    from shine_mapping_b200 import evaluate
    cfg = types.SimpleNamespace(begin_frame=2, end_frame=30, every_frame=3)
    assert render.all_frames(cfg, 10) == list(range(2, 10))
    assert render.all_frames(types.SimpleNamespace(begin_frame=0, end_frame=4, every_frame=1), 10) == [0, 1, 2, 3, 4]
    ds = types.SimpleNamespace(total_pc_count=10)
    assert evaluate.selected_frames(cfg, ds, None) == [2, 4, 5, 7, 8]      # ids with id % every_frame != 0
    assert evaluate.selected_frames(cfg, ds, range(0, 4)) == [0, 1, 2, 3]
    with pytest.raises(SystemExit, match="no held-out frames"):
        evaluate.selected_frames(types.SimpleNamespace(begin_frame=0, end_frame=5, every_frame=1), ds, None)
