"""RGB-D sequences: depth images back-projected on the GPU, mapped directly or written in the reference's KITTI layout.

The reference maps RGB-D data only after `dataset/rgbd_to_kitti_format.py` has turned every depth image into a PLY point
cloud with open3d.  Here both steps share one kernel, `shine_rgbd_backproject` (csrc/shine_rgbd.cu):

* `RGBDCamera` — intrinsics, depth scale and extrinsic of the converter's three cases (`from_converter_args`).
* `load_focal_length`, `load_replica_intrinsic`, `load_poses`, `write_poses_kitti_format`, `read_pose_file` — the
  converter's readers and writer; `read_depth` / `read_color` decode PNG (or any format torchvision / PIL reads) on the
  host into pinned memory.
* `RGBDDataset` — `scans.LiDARDataset` whose frames come from depth images: decode, one H2D copy, one back-projection
  launch, then the scan pipeline as it is.  Invalid pixels are NaN records, which its filter drops, so the frame's one
  host read is still the voxel count.
* `python -m shine_mapping_b200.rgbd convert ...` — the converter, with the reference's argument names and defaults:
  `output_root/poses.txt` and `output_root/rgbd_ply/%06d.ply` (binary, double x y z, uchar red green blue).
"""
from __future__ import annotations

import argparse
import ctypes as C
import json
import os
import shutil
import sys

import numpy as np
import torch

from . import scans
from .config import SHINEConfig

# the PrimeSense default of open3d's PinholeCameraIntrinsicParameters, and the extrinsic the converter pairs with it and
# with Neural RGB-D focal files (those frames are captured upside down)
PRIMESENSE = dict(width=640, height=480, fx=525.0, fy=525.0, cx=319.5, cy=239.5)
FLIP_YZ = np.diag([1.0, -1.0, -1.0, 1.0])


class RGBDCamera:
    """A pinhole camera: image size, focal lengths and principal point in pixels, raw depth units per metre, and the
    extrinsic of the converter.  Points are camera_pose · (x, y, z, 1) with camera_pose = inv(extrinsic) in fp64."""

    def __init__(self, width: int, height: int, fx: float, fy: float, cx: float, cy: float, depth_scale: float = 1000.0,
                 extrinsic=None):
        self.width, self.height = int(width), int(height)
        self.fx, self.fy, self.cx, self.cy = float(fx), float(fy), float(cx), float(cy)
        self.depth_scale = float(depth_scale)
        self.extrinsic = np.eye(4) if extrinsic is None else np.asarray(extrinsic, dtype=np.float64).reshape(4, 4)
        self.camera_pose = np.linalg.inv(self.extrinsic)

    @classmethod
    def from_converter_args(cls, intrinsic_file: str, is_focal_file: bool, first_depth_image_shape) -> "RGBDCamera":
        """The converter's cases: no intrinsic file -> PrimeSense default; a focal file (Neural RGB-D) -> fx = fy = focal
        and the centre of the first depth image; otherwise a Replica JSON with its own depth scale and no flip."""
        H, W = (int(v) for v in first_depth_image_shape[:2])
        if intrinsic_file == "":
            return cls(**PRIMESENSE, depth_scale=1000.0, extrinsic=FLIP_YZ)
        if is_focal_file:
            focal = load_focal_length(intrinsic_file)
            return cls(W, H, focal, focal, (W - 1.0) / 2.0, (H - 1.0) / 2.0, depth_scale=1000.0, extrinsic=FLIP_YZ)
        cam = load_replica_intrinsic(intrinsic_file)
        return cls(cam["w"], cam["h"], cam["fx"], cam["fy"], cam["cx"], cam["cy"], depth_scale=cam["scale"])


# ---------------------------------------------------------------------------------------------------------- host input


def load_focal_length(path: str) -> float:
    """Neural RGB-D `focal.txt`: the float on its first line."""
    with open(path) as fh:
        return float(fh.readline())


def load_replica_intrinsic(path: str) -> dict:
    """Replica `cam_params.json`: its "camera" object, which must hold w h fx fy cx cy scale."""
    with open(path) as fh:
        cam = json.load(fh).get("camera")
    missing = [k for k in ("w", "h", "fx", "fy", "cx", "cy", "scale") if not isinstance(cam, dict) or k not in cam]
    if missing:
        raise ValueError(f"{path}: the \"camera\" object has no {', '.join(missing)}")
    return cam


def load_poses(path: str) -> list:
    """4x4 pose matrices, four lines of four values each, no header -> list of fp64 [4,4].  Blank lines are skipped."""
    with open(path) as fh:
        rows = [line.split() for line in fh if line.strip()]
    if len(rows) % 4 or any(len(r) != 4 for r in rows):
        raise ValueError(f"{path}: expected 4x4 matrices as four lines of four values each ({len(rows)} rows)")
    return [np.array([[float(v) for v in r] for r in rows[i:i + 4]]) for i in range(0, len(rows), 4)]


def write_poses_kitti_format(poses: list, path: str) -> None:
    """The first three rows of every pose on one line, as np.savetxt's %.18e (values round-trip exactly)."""
    np.savetxt(path, [np.asarray(p).flatten()[0:12] for p in poses], delimiter=" ")


def kitti_poses(poses: list) -> list:
    """What scans.read_poses_file(write_poses_kitti_format(poses), {"Tr": I}) returns, without the file."""
    eye = np.eye(4)
    eye_inv = np.linalg.inv(eye)
    out = []
    for p in poses:
        pose = np.zeros((4, 4))
        pose[0:3, 0:4] = np.asarray(p, dtype=np.float64).flatten()[0:12].reshape(3, 4)
        pose[3, 3] = 1.0
        out.append(np.matmul(eye_inv, np.matmul(pose, eye)))
    return out


def read_pose_file(path: str, kitti_format_pose: bool = False) -> list:
    """The camera poses as the converted sequence's poses.txt yields them through scans.read_poses_file with Tr = I."""
    if kitti_format_pose:
        return scans.read_poses_file(path, {"Tr": np.eye(4)})
    return kitti_poses(load_poses(path))


def image_files(folder: str) -> list:
    return scans.natural_sorted(os.listdir(folder))


def _decode_fn():
    """path -> [C,H,W] tensor of the image as stored: torchvision, else PIL."""
    try:
        from torchvision.io import ImageReadMode, decode_image, read_file
        return lambda path: decode_image(read_file(path), mode=ImageReadMode.UNCHANGED)
    except ImportError:
        pass
    try:
        from PIL import Image
    except ImportError:
        raise ImportError("decoding RGB-D images needs torchvision or PIL (Pillow); neither can be imported") from None

    def decode(path):
        with Image.open(path) as im:
            a = np.array(im)
        a = a[None] if a.ndim == 2 else a.transpose(2, 0, 1)
        return torch.from_numpy(np.ascontiguousarray(a))
    return decode


_DECODE = None


def decode(path: str) -> torch.Tensor:
    global _DECODE
    if _DECODE is None:
        _DECODE = _decode_fn()
    return _DECODE(path)


def read_depth(path: str, pinned: bool = True) -> torch.Tensor:
    """A 16-bit single-channel depth image -> uint16 [H,W] (pinned for an asynchronous H2D copy)."""
    img = decode(path)
    if img.dim() != 3 or img.shape[0] != 1 or img.dtype != torch.uint16:
        raise ValueError(f"{path}: depth must be a 16-bit single-channel image, not {tuple(img.shape)} {img.dtype}")
    out = torch.empty(tuple(img.shape[1:]), dtype=torch.uint16, pin_memory=pinned)
    out.copy_(img[0])
    return out


def read_color(path: str, pinned: bool = True) -> torch.Tensor:
    """An 8-bit RGB or RGBA image -> uint8 [H,W,3] RGB (pinned)."""
    img = decode(path)
    if img.dim() != 3 or img.shape[0] not in (3, 4) or img.dtype != torch.uint8:
        raise ValueError(f"{path}: colour must be an 8-bit RGB or RGBA image, not {tuple(img.shape)} {img.dtype}")
    out = torch.empty((img.shape[1], img.shape[2], 3), dtype=torch.uint8, pin_memory=pinned)
    out.copy_(img[:3].permute(1, 2, 0))
    return out


# ----------------------------------------------------------------------------------------------------------- GPU frame


def backproject(depth: torch.Tensor, camera: RGBDCamera, max_depth_m: float = 5.0, device="cuda",
                color: torch.Tensor | None = None):
    """One shine_rgbd_backproject launch.  depth: uint16 [H,W] (host or device); color: uint8 [H,W,3] or None.
    -> fp64 [H*W,3] device points in row-major pixel order, NaN for invalid pixels (and uint8 [H*W,3] colours)."""
    from . import _abi
    dev = torch.device(device)
    H, W = depth.shape
    if color is not None and tuple(color.shape) != (H, W, 3):
        raise ValueError(f"colour image {tuple(color.shape)} does not match depth image {(H, W)}")
    d = depth.contiguous().view(torch.uint8).to(dev, non_blocking=True)
    xyz = torch.empty(H * W, 3, dtype=torch.float64, device=dev)
    rgb_in = color.contiguous().to(dev, non_blocking=True) if color is not None else None
    rgb = torch.empty(H * W, 3, dtype=torch.uint8, device=dev) if color is not None else None
    pose = (C.c_double * 16)(*np.ascontiguousarray(camera.camera_pose, dtype=np.float64).reshape(16).tolist())
    _abi.check(_abi.lib().shine_rgbd_backproject(
        _abi.ptr(d), H, W, W, camera.fx, camera.fy, camera.cx, camera.cy, camera.depth_scale, float(max_depth_m), pose,
        _abi.ptr(xyz), _abi.ptr(rgb), _abi.ptr(rgb_in), _abi.stream_ptr(dev)), "shine_rgbd_backproject")
    return xyz if color is None else (xyz, rgb)


class RGBDDataset(scans.LiDARDataset):
    """`LiDARDataset` over a folder of depth images: the same frame selection, reference poses, pool and scan pipeline,
    with each frame back-projected on the GPU instead of read from a point-cloud file.  The config's pc_path, pose_path
    and calib_path are not read; pose_file is a Neural RGB-D 4x4 pose file, or KITTI poses with kitti_format_pose."""

    def __init__(self, config: SHINEConfig, depth_dir: str, pose_file: str, camera: RGBDCamera,
                 kitti_format_pose: bool = False, max_depth_m: float = 5.0, octree=None, pool=None):
        scans.check_process_config(config)
        self.depth_dir, self.camera, self.max_depth_m = depth_dir, camera, float(max_depth_m)
        self.depth_filenames = image_files(depth_dir)
        poses_w = read_pose_file(pose_file, kitti_format_pose)
        if len(poses_w) < len(self.depth_filenames):
            raise ValueError(f"{pose_file} holds {len(poses_w)} poses for {len(self.depth_filenames)} depth images in "
                             f"{depth_dir}")
        self._init_frames(config, poses_w, len(self.depth_filenames), octree, pool)

    def read_frame(self, frame_id: int) -> scans.ScanRecords:
        depth = read_depth(os.path.join(self.depth_dir, self.depth_filenames[frame_id]))
        xyz = backproject(depth, self.camera, self.max_depth_m, self.device)
        return scans.ScanRecords(xyz.view(torch.uint8).reshape(-1), xyz.shape[0], 24, True)


# -------------------------------------------------------------------------------------------------------- command lines


def add_loop_arguments(ap: argparse.ArgumentParser) -> None:
    """The mapping loops' flags for a folder of depth images."""
    ap.add_argument("--rgbd", default=None, metavar="DEPTH_DIR",
                    help="map the 16-bit depth images of DEPTH_DIR directly (with --pose-file); the config's pc_path, "
                         "pose_path and calib_path are not read")
    ap.add_argument("--intrinsic-file", default="", metavar="FILE",
                    help="focal.txt (Neural RGB-D) or, with --json-intrinsic, a Replica JSON; default: PrimeSense")
    kind = ap.add_mutually_exclusive_group()
    kind.add_argument("--focal-file", dest="is_focal_file", action="store_const", const=True, default=True,
                      help="the intrinsic file holds one focal length (default)")
    kind.add_argument("--json-intrinsic", dest="is_focal_file", action="store_const", const=False,
                      help="the intrinsic file is a JSON file with a \"camera\" object")
    ap.add_argument("--pose-file", default=None, metavar="FILE", help="camera poses: 4x4 matrices, four lines each")
    ap.add_argument("--kitti-format-pose", action="store_true", help="the pose file holds KITTI poses (Replica)")
    ap.add_argument("--max-depth-m", type=float, default=5.0, help="depth at or beyond this is dropped (default 5.0)")


def check_loop_arguments(ap: argparse.ArgumentParser, args) -> None:
    if args.rgbd is None:
        return
    if args.scans:
        ap.error("--rgbd and --scans select two different inputs: give one of them")
    if args.pose_file is None:
        ap.error("--rgbd needs --pose-file")


def dataset_from_args(config: SHINEConfig, args, octree=None) -> RGBDDataset:
    files = image_files(args.rgbd)
    if not files:
        raise ValueError(f"{args.rgbd}: no depth images")
    shape = read_depth(os.path.join(args.rgbd, files[0]), pinned=False).shape
    camera = RGBDCamera.from_converter_args(args.intrinsic_file, args.is_focal_file, shape)
    return RGBDDataset(config, args.rgbd, args.pose_file, camera, args.kitti_format_pose, args.max_depth_m, octree)


_PLY_POINT = np.dtype([("x", "<f8"), ("y", "<f8"), ("z", "<f8"), ("red", "u1"), ("green", "u1"), ("blue", "u1")])


def write_color_ply(path: str, xyz: np.ndarray, rgb: np.ndarray) -> None:
    """Binary little-endian PLY: double x y z, uchar red green blue."""
    rec = np.empty(xyz.shape[0], dtype=_PLY_POINT)
    for i, k in enumerate("xyz"):
        rec[k] = xyz[:, i]
    for i, k in enumerate(("red", "green", "blue")):
        rec[k] = rgb[:, i]
    header = (f"ply\nformat binary_little_endian 1.0\nelement vertex {xyz.shape[0]}\nproperty double x\n"
              "property double y\nproperty double z\nproperty uchar red\nproperty uchar green\nproperty uchar blue\n"
              "end_header\n")
    with open(path, "wb") as fh:
        fh.write(header.encode("ascii"))
        fh.write(rec.tobytes())


def convert(depth_img_folder: str, rgb_img_folder: str, pose_file: str, output_root: str, intrinsic_file: str = "",
            max_depth_m: float = 5.0, is_focal_file: bool = True, already_kitti_format_pose: bool = False,
            device="cuda", log=print) -> int:
    """dataset/rgbd_to_kitti_format.py: output_root/poses.txt and output_root/rgbd_ply/{k:06d}.ply for the k-th
    (colour, depth) pair in natural order.  Each PLY holds the frame's valid points in row-major pixel order.
    -> the number of frames written."""
    ply_dir = os.path.join(output_root, "rgbd_ply")
    os.makedirs(ply_dir, exist_ok=True)
    pose_out = os.path.join(output_root, "poses.txt")
    if already_kitti_format_pose:
        shutil.copyfile(pose_file, pose_out)
    else:
        write_poses_kitti_format(load_poses(pose_file), pose_out)
    depth_files, rgb_files = image_files(depth_img_folder), image_files(rgb_img_folder)
    if not depth_files:
        raise ValueError(f"{depth_img_folder}: no depth images")
    first = read_depth(os.path.join(depth_img_folder, depth_files[0]), pinned=False)
    camera = RGBDCamera.from_converter_args(intrinsic_file, is_focal_file, first.shape)
    log(f"Image size: {first.shape[0]} x {first.shape[1]}; fx {camera.fx} fy {camera.fy} cx {camera.cx} cy {camera.cy}, "
        f"depth scale {camera.depth_scale}")
    count = 0
    for rgb_name, depth_name in zip(rgb_files, depth_files):
        # each frame ends with a download, so the uploads gain nothing from pinned buffers here
        depth = read_depth(os.path.join(depth_img_folder, depth_name), pinned=False)
        color_path = os.path.join(rgb_img_folder, rgb_name)
        color = read_color(color_path, pinned=False)
        if tuple(color.shape[:2]) != tuple(depth.shape):
            raise ValueError(f"{color_path}: colour image {tuple(color.shape[:2])} and depth image "
                             f"{depth_name} {tuple(depth.shape)} differ in size")
        xyz, rgb = backproject(depth, camera, max_depth_m, device, color)
        xyz, rgb = xyz.cpu().numpy(), rgb.cpu().numpy()
        keep = np.isfinite(xyz[:, 0])
        write_color_ply(os.path.join(ply_dir, f"{count:06d}.ply"), xyz[keep], rgb[keep])
        count += 1
    log(f"{count} frames in KITTI format under {output_root}")
    return count


def _bool(text) -> bool:
    if isinstance(text, bool):
        return text
    word = text.strip().lower()
    if word in ("yes", "true", "t", "y", "1"):
        return True
    if word in ("no", "false", "f", "n", "0"):
        return False
    raise argparse.ArgumentTypeError(f"expected a boolean, not {text!r}")


def converter_parser() -> argparse.ArgumentParser:
    """The arguments of dataset/rgbd_to_kitti_format.py, with its names and defaults (a bare boolean flag means True)."""
    ap = argparse.ArgumentParser(prog="python -m shine_mapping_b200.rgbd convert",
                                 description="Convert an RGB-D sequence to the KITTI layout the --scans loops read")
    ap.add_argument("--depth_img_folder", help="folder of 16-bit depth images")
    ap.add_argument("--rgb_img_folder", help="folder of the colour images")
    ap.add_argument("--intrinsic_file", default="", help="focal.txt or a Replica JSON (default: PrimeSense intrinsics)")
    ap.add_argument("--pose_file", help="camera poses, 4x4 matrices (or KITTI lines with --already_kitti_format_pose)")
    ap.add_argument("--output_root", help="where poses.txt and rgbd_ply/ are written")
    ap.add_argument("--max_depth_m", type=float, default=5.0, help="depth at or beyond this is dropped")
    ap.add_argument("--is_focal_file", type=_bool, nargs="?", const=True, default=True,
                    help="the intrinsic file holds one focal length (Neural RGB-D) rather than a Replica JSON")
    ap.add_argument("--already_kitti_format_pose", type=_bool, nargs="?", const=True, default=False,
                    help="the pose file is already in KITTI format (Replica); it is copied")
    ap.add_argument("--vis_on", type=_bool, nargs="?", const=True, default=False, help="accepted and ignored")
    return ap


def main(argv=None):
    argv = sys.argv[1:] if argv is None else list(argv)
    if not argv or argv[0] != "convert":
        print("usage: python -m shine_mapping_b200.rgbd convert --depth_img_folder DIR --rgb_img_folder DIR "
              "--pose_file FILE --output_root DIR [--intrinsic_file FILE] [--is_focal_file B] "
              "[--already_kitti_format_pose B] [--max_depth_m M]", file=sys.stderr)
        return 2
    ap = converter_parser()
    args = ap.parse_args(argv[1:])
    missing = [k for k in ("depth_img_folder", "rgb_img_folder", "pose_file", "output_root") if getattr(args, k) is None]
    if missing:
        ap.error("missing " + ", ".join("--" + k for k in missing))
    convert(args.depth_img_folder, args.rgb_img_folder, args.pose_file, args.output_root, args.intrinsic_file,
            args.max_depth_m, args.is_focal_file, args.already_kitti_format_pose)
    return 0


if __name__ == "__main__":
    sys.exit(main())
