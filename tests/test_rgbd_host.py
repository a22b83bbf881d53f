"""shine_mapping_b200.rgbd on the host: the converter's camera cases, readers, pose round trip, argument names and
defaults, image decoding of PNG fixtures written here, and the rejections."""
import json
import struct
import sys
import zlib

import numpy as np
import pytest
import torch

from shine_mapping_b200 import rgbd, scans


def png_bytes(a: np.ndarray) -> bytes:
    """A minimal PNG: [H,W] uint8 / uint16 greyscale or [H,W,3|4] uint8 RGB / RGBA, filter 0, one IDAT chunk."""
    a = np.asarray(a)
    H, W = a.shape[:2]
    channels = 1 if a.ndim == 2 else a.shape[2]
    colour_type = {1: 0, 3: 2, 4: 6}[channels]
    depth = 16 if a.dtype == np.uint16 else 8
    rows = a.reshape(H, W * channels).astype(">u2" if depth == 16 else "u1")
    body = b"".join(b"\x00" + r.tobytes() for r in rows)

    def chunk(tag, data):
        return struct.pack(">I", len(data)) + tag + data + struct.pack(">I", zlib.crc32(tag + data) & 0xFFFFFFFF)
    ihdr = struct.pack(">IIBBBBB", W, H, depth, colour_type, 0, 0, 0)
    return b"\x89PNG\r\n\x1a\n" + chunk(b"IHDR", ihdr) + chunk(b"IDAT", zlib.compress(body)) + chunk(b"IEND", b"")


def write_png(path, a) -> None:
    with open(path, "wb") as fh:
        fh.write(png_bytes(a))


def rigid(seed: int) -> np.ndarray:
    """A rotation (no zero entries) and a translation as a 4x4 fp64 matrix."""
    rng = np.random.default_rng(seed)
    q, _ = np.linalg.qr(rng.normal(size=(3, 3)))
    T = np.eye(4)
    T[:3, :3] = q * np.sign(np.linalg.det(q))
    T[:3, 3] = rng.uniform(-3, 3, 3)
    return T


# ----------------------------------------------------------------------------------------------------------- cameras


def test_primesense_default(tmp_path):
    cam = rgbd.RGBDCamera.from_converter_args("", True, (100, 200))
    assert (cam.width, cam.height, cam.fx, cam.fy, cam.cx, cam.cy) == (640, 480, 525.0, 525.0, 319.5, 239.5)
    assert cam.depth_scale == 1000.0
    np.testing.assert_array_equal(cam.extrinsic, np.diag([1.0, -1.0, -1.0, 1.0]))
    np.testing.assert_array_equal(cam.camera_pose, np.diag([1.0, -1.0, -1.0, 1.0]))


def test_neural_rgbd_focal_file(tmp_path):
    (tmp_path / "focal.txt").write_text("554.2562584220408\n")
    assert rgbd.load_focal_length(str(tmp_path / "focal.txt")) == 554.2562584220408
    cam = rgbd.RGBDCamera.from_converter_args(str(tmp_path / "focal.txt"), True, (480, 640))
    assert (cam.width, cam.height, cam.fx, cam.fy) == (640, 480, 554.2562584220408, 554.2562584220408)
    assert (cam.cx, cam.cy, cam.depth_scale) == (319.5, 239.5, 1000.0)
    np.testing.assert_array_equal(cam.extrinsic, np.diag([1.0, -1.0, -1.0, 1.0]))
    odd = rgbd.RGBDCamera.from_converter_args(str(tmp_path / "focal.txt"), True, (7, 12))
    assert (odd.cx, odd.cy) == (5.5, 3.0)


def test_replica_json(tmp_path):
    doc = {"camera": {"w": 1200, "h": 680, "fx": 600.0, "fy": 601.5, "cx": 599.5, "cy": 339.5, "scale": 6553.5}}
    (tmp_path / "cam.json").write_text(json.dumps(doc))
    cam = rgbd.RGBDCamera.from_converter_args(str(tmp_path / "cam.json"), False, (1, 1))
    assert (cam.width, cam.height, cam.fx, cam.fy, cam.cx, cam.cy) == (1200, 680, 600.0, 601.5, 599.5, 339.5)
    assert cam.depth_scale == 6553.5
    np.testing.assert_array_equal(cam.extrinsic, np.eye(4))
    np.testing.assert_array_equal(cam.camera_pose, np.eye(4))
    del doc["camera"]["scale"]
    (tmp_path / "bad.json").write_text(json.dumps(doc))
    with pytest.raises(ValueError, match="bad.json.*scale"):
        rgbd.load_replica_intrinsic(str(tmp_path / "bad.json"))


def test_camera_pose_is_the_fp64_inverse_of_the_extrinsic():
    E = rigid(4)
    cam = rgbd.RGBDCamera(4, 3, 1.0, 1.0, 1.5, 1.0, 1000.0, E)
    np.testing.assert_array_equal(cam.camera_pose, np.linalg.inv(E))


# ------------------------------------------------------------------------------------------------------------- poses


def _write_matrices(path, mats, blank_between=False):
    with open(path, "w") as fh:
        for m in mats:
            fh.write("\n".join(" ".join(repr(float(v)) for v in row) for row in m) + "\n")
            if blank_between:
                fh.write("\n")


def test_four_line_poses_and_kitti_round_trip_bit_for_bit(tmp_path):
    mats = [rigid(s) for s in range(12)]
    _write_matrices(tmp_path / "poses.txt", mats)
    got = rgbd.load_poses(str(tmp_path / "poses.txt"))
    assert len(got) == 12
    for g, m in zip(got, mats):
        np.testing.assert_array_equal(g, m)
    out = tmp_path / "kitti.txt"
    rgbd.write_poses_kitti_format(got, str(out))
    assert all(len(line.split()) == 12 and "e" in line for line in out.read_text().splitlines())
    back = scans.read_poses_file(str(out), {"Tr": np.eye(4)})
    direct = rgbd.read_pose_file(str(tmp_path / "poses.txt"))
    kitti = rgbd.read_pose_file(str(out), kitti_format_pose=True)
    for b, d, k, m in zip(back, direct, kitti, mats):
        assert b[:3].tobytes() == m[:3].tobytes()
        assert d.tobytes() == b.tobytes() and k.tobytes() == b.tobytes()
        np.testing.assert_array_equal(b[3], [0, 0, 0, 1])


def test_pose_reader_rejects_missing_rows(tmp_path):
    mats = [rigid(s) for s in range(2)]
    _write_matrices(tmp_path / "poses.txt", mats, blank_between=True)
    assert len(rgbd.load_poses(str(tmp_path / "poses.txt"))) == 2
    (tmp_path / "short.txt").write_text("1 0 0 0\n" * 7)          # the second matrix lacks its last row
    with pytest.raises(ValueError, match="short.txt"):
        rgbd.load_poses(str(tmp_path / "short.txt"))
    (tmp_path / "narrow.txt").write_text("1 0 0\n0 1 0\n0 0 1\n0 0 0\n")
    with pytest.raises(ValueError, match="narrow.txt"):
        rgbd.load_poses(str(tmp_path / "narrow.txt"))


def test_natural_order(tmp_path):
    names = ["depth10.png", "depth2.png", "depth1.png", "depth100.png", "depth20.png"]
    for n in names:
        (tmp_path / n).write_bytes(b"")
    assert rgbd.image_files(str(tmp_path)) == ["depth1.png", "depth2.png", "depth10.png", "depth20.png", "depth100.png"]


# ------------------------------------------------------------------------------------------------- converter arguments

REFERENCE_ARGUMENTS = {            # dataset/rgbd_to_kitti_format.py's argparse: name -> default
    "depth_img_folder": None, "rgb_img_folder": None, "intrinsic_file": "", "pose_file": None, "output_root": None,
    "max_depth_m": 5.0, "is_focal_file": True, "already_kitti_format_pose": False, "vis_on": False,
}


def test_converter_argument_names_and_defaults():
    args = vars(rgbd.converter_parser().parse_args([]))
    assert args == REFERENCE_ARGUMENTS
    # the command of scripts/convert_rgbd_to_kitti_format.sh, module swapped
    cmd = ("--output_root out --depth_img_folder d/depth_filtered/ --rgb_img_folder d/images/ --intrinsic_file "
           "d/focal.txt --pose_file d/poses.txt --is_focal_file True --already_kitti_format_pose False --vis_on False")
    a = rgbd.converter_parser().parse_args(cmd.split())
    assert (a.output_root, a.depth_img_folder, a.rgb_img_folder) == ("out", "d/depth_filtered/", "d/images/")
    assert a.is_focal_file is True and a.already_kitti_format_pose is False and a.vis_on is False
    a = rgbd.converter_parser().parse_args(["--is_focal_file", "no", "--already_kitti_format_pose", "1",
                                            "--max_depth_m", "3.5"])
    assert a.is_focal_file is False and a.already_kitti_format_pose is True and a.max_depth_m == 3.5
    with pytest.raises(SystemExit):
        rgbd.converter_parser().parse_args(["--is_focal_file", "maybe"])
    assert rgbd.main([]) == 2
    with pytest.raises(SystemExit):
        rgbd.main(["convert", "--depth_img_folder", "d"])


@pytest.mark.parametrize("module", ["batch_loop", "incre_loop"])
def test_loop_argument_errors(module, capsys):
    import importlib
    main = importlib.import_module(f"shine_mapping_b200.{module}").main
    with pytest.raises(SystemExit):
        main(["cfg.yaml", "--rgbd", "depth", "--pose-file", "p.txt", "--scans"])
    assert "--scans" in capsys.readouterr().err
    with pytest.raises(SystemExit):
        main(["cfg.yaml", "--rgbd", "depth"])
    assert "--pose-file" in capsys.readouterr().err
    with pytest.raises(SystemExit):
        main(["cfg.yaml", "--rgbd", "depth", "--pose-file", "p.txt", "--focal-file", "--json-intrinsic"])


# ----------------------------------------------------------------------------------------------------------- decoding

@pytest.fixture(params=["torchvision", "PIL"])
def decoder(request, monkeypatch):
    if request.param == "PIL":
        monkeypatch.setitem(sys.modules, "torchvision.io", None)
    monkeypatch.setattr(rgbd, "_DECODE", None)
    return request.param


def _fixtures(tmp_path):
    rng = np.random.default_rng(1)
    d16 = rng.integers(0, 65536, (13, 17), dtype=np.uint16)
    d16[0, :3] = (0, 1, 65535)
    rgb = rng.integers(0, 256, (13, 17, 3), dtype=np.uint8)
    rgba = rng.integers(0, 256, (13, 17, 4), dtype=np.uint8)
    g8 = rng.integers(0, 256, (13, 17), dtype=np.uint8)
    for name, a in (("d16", d16), ("rgb", rgb), ("rgba", rgba), ("g8", g8), ("small", rgb[:12]),
                    ("rgb16", rng.integers(0, 65536, (13, 17), dtype=np.uint16))):
        write_png(tmp_path / f"{name}.png", a)
    return d16, rgb, rgba


def test_decode_fixtures(tmp_path, decoder):
    d16, rgb, rgba = _fixtures(tmp_path)
    d = rgbd.read_depth(str(tmp_path / "d16.png"), pinned=False)
    assert d.dtype == torch.uint16 and tuple(d.shape) == (13, 17)
    np.testing.assert_array_equal(d.numpy(), d16)
    c = rgbd.read_color(str(tmp_path / "rgb.png"), pinned=False)
    assert c.dtype == torch.uint8 and tuple(c.shape) == (13, 17, 3) and c.is_contiguous()
    np.testing.assert_array_equal(c.numpy(), rgb)
    np.testing.assert_array_equal(rgbd.read_color(str(tmp_path / "rgba.png"), pinned=False).numpy(), rgba[..., :3])


def test_decode_rejections(tmp_path, decoder):
    _fixtures(tmp_path)
    for name in ("g8", "rgb"):
        with pytest.raises(ValueError, match=f"{name}.png.*16-bit single-channel"):
            rgbd.read_depth(str(tmp_path / f"{name}.png"), pinned=False)
    for name in ("d16", "g8"):
        with pytest.raises(ValueError, match=f"{name}.png.*8-bit RGB"):
            rgbd.read_color(str(tmp_path / f"{name}.png"), pinned=False)


def test_no_decoder_names_both(monkeypatch):
    monkeypatch.setitem(sys.modules, "torchvision.io", None)
    monkeypatch.setitem(sys.modules, "PIL", None)
    with pytest.raises(ImportError, match="torchvision.*PIL"):
        rgbd._decode_fn()


def test_converter_rejects_size_mismatch_and_short_pose_file(tmp_path):
    """Both are found on the host, before the first frame reaches the GPU."""
    _fixtures(tmp_path)
    for d in ("depth", "color"):
        (tmp_path / d).mkdir()
    (tmp_path / "depth" / "0.png").write_bytes((tmp_path / "d16.png").read_bytes())
    (tmp_path / "color" / "0.png").write_bytes((tmp_path / "small.png").read_bytes())
    (tmp_path / "focal.txt").write_text("20.0\n")
    _write_matrices(tmp_path / "poses.txt", [rigid(0)])
    with pytest.raises(ValueError, match="color/0.png.*differ"):
        rgbd.convert(str(tmp_path / "depth"), str(tmp_path / "color"), str(tmp_path / "poses.txt"),
                     str(tmp_path / "out"), str(tmp_path / "focal.txt"), log=lambda *a: None)
    (tmp_path / "depth" / "1.png").write_bytes((tmp_path / "d16.png").read_bytes())
    cam = rgbd.RGBDCamera.from_converter_args(str(tmp_path / "focal.txt"), True, (13, 17))
    from tests.parity_utils import make_config
    with pytest.raises(ValueError, match="1 poses for 2 depth images"):
        rgbd.RGBDDataset(make_config(2, rand_downsample=False), str(tmp_path / "depth"), str(tmp_path / "poses.txt"), cam)
