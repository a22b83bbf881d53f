"""Look at a map from a sensor pose: depth, range and normal images rendered on the GPU, and depth images scored with
the reference's depth metrics.

* `render_view`       — `shine_render` (csrc/shine_raycast.cu): one ray per pixel of a pinhole (`rgbd.RGBDCamera`) or
                        spherical range image (`RangeImageCamera`) view, marched as `raycast.cast_rays` marches -> depth,
                        range, unit normal and hit images in metres.
* `depth_metrics`     — eval/eval_utils.py `eval_depth` (AbsRel, AbsDiff, SqRel, RMSE, LogRMSE, r1-r3, complete) in fp64 on
                        the images' device.
* `depth_png`, `normal_png`, `write_png` — 16-bit depth and 8-bit RGB normal PNGs (zlib and struct only); `rgbd.read_depth`
                        and `rgbd.read_color` read them back.
* `python -m shine_mapping_b200.render CONFIG CHECKPOINT --out DIR [...]` — every selected frame rendered from its pose.

DESIGN.md §14 states the camera models, the march and how they are tested.
"""
from __future__ import annotations

import argparse
import ctypes as C
import math
import os
import struct
import sys
import zlib

import numpy as np
import torch

from . import _abi
from .raycast import REFINE_ITERS, mask_level

DEPTH_METRICS = ["AbsRel", "AbsDiff", "SqRel", "RMSE", "LogRMSE", "r1", "r2", "r3", "complete"]
RANGE_IMAGE_SIZE = (1024, 64)          # width, height of a LiDAR frame's range image when none is given
RANGE_DEPTH_SCALE = 256.0              # range image PNG units per metre (the KITTI depth-map convention, up to 256 m)


class RangeImageCamera:
    """A spherical range image: row 0 looks at fov_up_deg, row height - 1 at fov_down_deg, column 0 at azimuth +pi and
    the azimuth falls by 2 pi / width per column (include/shine_b200.h, SHINE_CAMERA_RANGE_IMAGE).  The sensor frame is
    the pose's: x forward at azimuth 0, z up.  depth_scale: PNG units per metre."""

    def __init__(self, width: int, height: int, fov_up_deg: float, fov_down_deg: float,
                 depth_scale: float = RANGE_DEPTH_SCALE):
        self.width, self.height = int(width), int(height)
        self.fov_up, self.fov_down = float(fov_up_deg), float(fov_down_deg)
        self.depth_scale = float(depth_scale)
        if self.width <= 0 or self.height <= 0:
            raise ValueError(f"range image {self.width} x {self.height}: both sides must be > 0")
        if not (math.isfinite(self.fov_up) and math.isfinite(self.fov_down) and self.fov_up > self.fov_down):
            raise ValueError(f"range image FOV up {self.fov_up} down {self.fov_down}: need finite values, up > down")

    @classmethod
    def from_points(cls, points_sensor: torch.Tensor, width: int = RANGE_IMAGE_SIZE[0],
                    height: int = RANGE_IMAGE_SIZE[1]) -> "RangeImageCamera":
        """The FOV from the elevation extremes of a scan's points in its sensor frame ([n,3], any unit)."""
        p = points_sensor.reshape(-1, 3).double()
        if p.shape[0] == 0:
            raise ValueError("the frame has no points to take a range image's FOV from")
        el = torch.rad2deg(torch.atan2(p[:, 2], torch.hypot(p[:, 0], p[:, 1])))
        return cls(width, height, float(el.max()), float(el.min()))


def _camera_struct(camera) -> _abi.ShineCamera:
    if isinstance(camera, RangeImageCamera):
        return _abi.ShineCamera(_abi.CAMERA_RANGE_IMAGE, camera.width, camera.height, 0.0, 0.0, 0.0, 0.0, camera.fov_up,
                                camera.fov_down)
    return _abi.ShineCamera(_abi.CAMERA_PINHOLE, camera.width, camera.height, camera.fx, camera.fy, camera.cx, camera.cy,
                            0.0, 0.0)


def sensor_to_map(pose_map, camera) -> np.ndarray:
    """The camera-to-map transform the kernel gets, in metres: pose_map with a pinhole camera's extrinsic folded in
    (`RGBDCamera.camera_pose`, as `rgbd.backproject` applies it)."""
    T = np.asarray(pose_map, dtype=np.float64).reshape(4, 4)
    return T if isinstance(camera, RangeImageCamera) else T @ camera.camera_pose


def render_view(config, octree, decoder, pose_map, camera, max_range_m: float, step_m: float | None = None,
                refine_iters: int = REFINE_ITERS) -> dict:
    """One `shine_render` launch.  pose_map: the sensor's 4x4 pose in the map frame, metres; camera: `rgbd.RGBDCamera`
    or `RangeImageCamera`; rays are sampled every step_m (default mc_res_m) up to max_range_m, with the mesher's mask
    level.  -> CUDA tensors, metres: depth fp64 [H,W] (0 where no hit), range fp64 [H,W] (NaN where no hit), normal
    fp32 [H,W,3] (unit, map frame, facing free space; NaN where no hit) and hit bool [H,W]."""
    scale = float(config.scale)
    step = float(config.mc_res_m if step_m is None else step_m)
    if not (max_range_m > 0 and math.isfinite(max_range_m)):
        raise ValueError(f"max_range_m {max_range_m}: must be finite and > 0")
    T = sensor_to_map(pose_map, camera)
    pose = np.array(T[:3, :4], dtype=np.float64)
    pose[:, 3] *= scale
    pose32 = (C.c_float * 12)(*pose.astype(np.float32).reshape(12).tolist())
    cam = _camera_struct(camera)
    dev = octree.hier_features[0].device
    H, W = camera.height, camera.width
    rng = torch.empty(H, W, dtype=torch.float32, device=dev)
    depth = torch.empty(H, W, dtype=torch.float32, device=dev)
    normal = torch.empty(H, W, 3, dtype=torch.float32, device=dev)
    status = torch.empty(H, W, dtype=torch.uint8, device=dev)
    od, dd = octree._descriptor(None, None), decoder.c_descriptor(None)
    _abi.check(_abi.lib().shine_render(C.byref(od), C.byref(dd), C.byref(cam), pose32, float(np.float32(step * scale)),
                                       0.0, float(np.float32(max_range_m * scale)), int(refine_iters),
                                       mask_level(config, octree), _abi.ptr(rng), _abi.ptr(depth), _abi.ptr(normal),
                                       _abi.ptr(status), _abi.stream_ptr(dev)), "shine_render")
    hit = status.bool()
    depth_m = torch.where(hit, depth.double() / scale, torch.zeros((), dtype=torch.float64, device=dev))
    return {"depth": depth_m, "range": rng.double() / scale, "normal": normal, "hit": hit}


# ---- metrics -----------------------------------------------------------------------------------------------------------

def depth_metrics(pred, target) -> dict:
    """eval/eval_utils.py `eval_depth` in fp64 on the images' device: over the pixels with 0 < target < 10 and pred > 0,
    AbsRel, AbsDiff, SqRel, RMSE, LogRMSE and the fractions r1, r2, r3 of max(target / pred, pred / target) below
    1.25, 1.25^2, 1.25^3; `complete` is the fraction of all pixels with pred > 0.  An empty mask gives NaN (numpy's mean
    of nothing)."""
    p = torch.as_tensor(pred).double()
    t = torch.as_tensor(target).double().to(p.device)
    if p.shape != t.shape:
        raise ValueError(f"depth_metrics: prediction {tuple(p.shape)} and target {tuple(t.shape)} differ in shape")
    mask1 = p > 0
    mask = (t < 10) & (t > 0) & mask1
    p, t = p[mask], t[mask]
    n = p.numel()
    mean = (lambda x: x.sum() / n) if n else (lambda x: torch.tensor(float("nan"), dtype=torch.float64))
    abs_diff = (p - t).abs()
    sq_diff = abs_diff * abs_diff
    thresh = torch.maximum(t / p, p / t)
    vals = [mean(abs_diff / t), mean(abs_diff), mean(sq_diff / t), mean(sq_diff).sqrt(),
            mean((p.log() - t.log()) ** 2).sqrt(), mean((thresh < 1.25).double()), mean((thresh < 1.25 ** 2).double()),
            mean((thresh < 1.25 ** 3).double()), mask1.double().sum() / mask1.numel()]
    return dict(zip(DEPTH_METRICS, torch.stack([v.to(p.device) for v in vals]).tolist()))


# ---- PNG ---------------------------------------------------------------------------------------------------------------

def write_png(path: str, image) -> None:
    """A uint16 [H,W] array as a 16-bit greyscale PNG, or a uint8 [H,W,3] array as an 8-bit RGB PNG."""
    a = np.asarray(image)
    if a.dtype == np.uint16 and a.ndim == 2:
        bit_depth, colour, rows = 16, 0, a.astype(">u2").view(np.uint8).reshape(a.shape[0], -1)
    elif a.dtype == np.uint8 and a.ndim == 3 and a.shape[2] == 3:
        bit_depth, colour, rows = 8, 2, a.reshape(a.shape[0], -1)
    else:
        raise ValueError(f"write_png: a uint16 [H,W] or uint8 [H,W,3] array, not {a.dtype} {a.shape}")
    H, W = a.shape[:2]
    if H == 0 or W == 0:
        raise ValueError("write_png: an empty image")
    raw = np.concatenate([np.zeros((H, 1), np.uint8), rows], 1).tobytes()     # filter type 0 on every row

    def chunk(tag: bytes, data: bytes) -> bytes:
        return struct.pack(">I", len(data)) + tag + data + struct.pack(">I", zlib.crc32(tag + data) & 0xFFFFFFFF)

    os.makedirs(os.path.dirname(os.path.abspath(path)), exist_ok=True)
    with open(path, "wb") as fh:
        fh.write(b"\x89PNG\r\n\x1a\n" + chunk(b"IHDR", struct.pack(">IIBBBBB", W, H, bit_depth, colour, 0, 0, 0)) +
                 chunk(b"IDAT", zlib.compress(raw, 6)) + chunk(b"IEND", b""))


def depth_png(depth_m, depth_scale: float):
    """Depth in metres (0 or NaN: none) -> (uint16 [H,W] in depth_scale units per metre, rounded half up; the number of
    depths that do not fit in 16 bits and are written as 0)."""
    d = np.asarray(torch.as_tensor(depth_m).detach().cpu(), dtype=np.float64)
    with np.errstate(invalid="ignore"):
        raw = np.floor(d * float(depth_scale) + 0.5)
        ok = np.isfinite(raw) & (d > 0)
        over = ok & (raw > 65535)
    return np.where(ok & ~over, raw, 0).astype(np.uint16), int(over.sum())


def normal_png(normal) -> np.ndarray:
    """Unit normals [H,W,3] -> uint8 RGB (n + 1) / 2 * 255, rounded; NaN (no hit) -> 0."""
    n = np.asarray(torch.as_tensor(normal).detach().cpu(), dtype=np.float64)
    v = np.rint(np.clip((np.nan_to_num(n, nan=-1.0) + 1.0) * 0.5 * 255.0, 0.0, 255.0))
    return v.astype(np.uint8)


def write_view(out_dir: str, name, view: dict, depth_scale: float, npz: bool = False) -> int:
    """out_dir/depth/{name}.png and out_dir/normal/{name}.png (and out_dir/npz/{name}.npz with the fp32 depth, range,
    normal and hit arrays).  -> the number of depths that did not fit in 16 bits."""
    raw, over = depth_png(view["depth"], depth_scale)
    write_png(os.path.join(out_dir, "depth", f"{name}.png"), raw)
    write_png(os.path.join(out_dir, "normal", f"{name}.png"), normal_png(view["normal"]))
    if npz:
        os.makedirs(os.path.join(out_dir, "npz"), exist_ok=True)
        np.savez(os.path.join(out_dir, "npz", f"{name}.npz"),
                 **{k: view[k].cpu().numpy().astype(np.float32 if k != "hit" else bool) for k in view})
    return over


# ---- command line ------------------------------------------------------------------------------------------------------

def _parser():
    from .rgbd import add_loop_arguments
    ap = argparse.ArgumentParser(prog="python -m shine_mapping_b200.render",
                                 description="Render depth and normal images of a saved map from each frame's pose. "
                                             "The checkpoint is unpickled: load only files you trust.")
    ap.add_argument("config")
    ap.add_argument("checkpoint")
    ap.add_argument("--out", required=True, metavar="DIR", help="write DIR/depth/{frame}.png and DIR/normal/{frame}.png")
    add_loop_arguments(ap)
    ap.set_defaults(scans=False)
    ap.add_argument("--frames", default=None, metavar="START:STOP[:STEP]",
                    help="frames to render (default: every frame in [begin_frame, end_frame])")
    ap.add_argument("--max-range-m", type=float, default=None,
                    help="ray length, m (default: the config's pc_radius_m; with --rgbd, --max-depth-m)")
    ap.add_argument("--step-m", type=float, default=None, help="ray sample spacing, m (default: the config's mc_res_m)")
    ap.add_argument("--range-image", nargs=4, default=None, metavar=("W", "H", "FOV_UP", "FOV_DOWN"),
                    help="LiDAR range image size and vertical FOV in degrees (default: 1024 x 64, the FOV from the "
                         "elevation extremes of each frame's points)")
    ap.add_argument("--npz", action="store_true", help="also write DIR/npz/{frame}.npz with the fp32 images")
    return ap


def check_view_arguments(ap, args) -> None:
    """--step-m and --max-range-m: finite and > 0 when given."""
    for name in ("step_m", "max_range_m"):
        v = getattr(args, name)
        if v is not None and not (v > 0 and math.isfinite(v)):
            ap.error(f"--{name.replace('_', '-')} must be > 0")


def parse_args(argv):
    from .raycast import parse_frames
    from .rgbd import check_loop_arguments
    ap = _parser()
    args = ap.parse_args(argv)
    check_loop_arguments(ap, args)
    check_view_arguments(ap, args)
    if args.frames is not None:
        try:
            args.frames = parse_frames(args.frames)
        except ValueError as e:
            ap.error(str(e))
    if args.range_image is not None:
        if args.rgbd:
            ap.error("--range-image is the LiDAR camera; --rgbd frames render through their pinhole camera")
        try:
            w, h, up, down = args.range_image
            args.range_image = RangeImageCamera(int(w), int(h), float(up), float(down))
        except ValueError as e:
            ap.error(f"--range-image: {e}")
    return args


def all_frames(config, total_frames: int) -> list:
    """The frame ids in [begin_frame, end_frame] below total_frames."""
    return list(range(max(0, int(config.begin_frame)), min(int(config.end_frame), int(total_frames) - 1) + 1))


def lidar_camera(dataset, frame_id: int, pose_map) -> RangeImageCamera:
    """The default range image of a LiDAR frame: 1024 x 64, the FOV from its preprocessed points' elevations."""
    scale = float(dataset.config.scale)
    T = torch.as_tensor(np.asarray(pose_map, dtype=np.float64))
    pts = dataset.processor.points(dataset.read_frame(frame_id), pose_map).double()
    local = (pts / scale - T[:3, 3].to(pts.device)) @ T[:3, :3].to(pts.device)
    return RangeImageCamera.from_points(local)


def main(argv=None) -> int:
    from .evaluate import load_map_and_dataset
    from .raycast import map_pose
    args = parse_args(sys.argv[1:] if argv is None else argv)
    config, octree, decoder, dataset = load_map_and_dataset(args)
    frames = list(args.frames) if args.frames is not None else all_frames(config, dataset.total_pc_count)
    for f in frames:
        if not 0 <= f < dataset.total_pc_count:
            raise SystemExit(f"frame {f}: the sequence has frames 0 .. {dataset.total_pc_count - 1}")
    max_range = args.max_range_m
    if max_range is None:
        max_range = args.max_depth_m if args.rgbd else float(config.pc_radius)
    for f in frames:
        pose = map_pose(dataset, f)
        camera = dataset.camera if args.rgbd else (args.range_image or lidar_camera(dataset, f, pose))
        view = render_view(config, octree, decoder, pose, camera, max_range, args.step_m)
        over = write_view(args.out, f, view, camera.depth_scale, args.npz)
        print(f"frame {f}: {camera.width} x {camera.height}, hit ratio {float(view['hit'].double().mean()):.4f}"
              + (f", {over} depths beyond 16 bits written as 0" if over else ""))
    return 0


if __name__ == "__main__":
    sys.exit(main())
