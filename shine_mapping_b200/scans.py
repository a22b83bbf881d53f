"""Real LiDAR sequences: the scan list, poses and point-cloud readers of the reference's `LiDARDataset`
(dataset/lidar_dataset.py:22-113, utils/pose.py:7-58), and `process_frame` (:115-218) on the GPU.

* `natural_sorted`, `read_calib_file`, `read_poses_file`, `reference_poses` — host input, numpy fp64 with the reference's
  calls, so the 4x4 poses are bit-identical to the reference's.
* `read_scan` — `.bin` (KITTI, float32 x y z i), `.ply` (ascii / binary_little_endian) and `.pcd` (ascii / binary) into
  a pinned host buffer: the file's records as they are, x y z first in each record.  Binary files whose x y z are
  adjacent, aligned and of one type are read straight into the pinned buffer; other layouts, and ascii files, are parsed into
  [n,3] records of their declared type.  NaN and inf points are kept (the filters drop them), as open3d does.
* `LiDARDataset` — the reference class's surface.  `frame_samples` is one H2D copy and four launches of
  csrc/shine_scan.cu (filter + keys, sort, average + transform, sample); its one host read is the voxel count.
"""
from __future__ import annotations

import ctypes as C
import os
import re

import numpy as np
import torch

from .config import SHINEConfig

# -------------------------------------------------------------------------------------------------------- host input


def natural_key(name: str):
    """natsort's order for file names: digit runs compare as integers (1, 2, 10), the rest as text."""
    return [(0, int(t), "") if t.isdigit() else (1, 0, t) for t in re.split(r"(\d+)", name) if t != ""]


def natural_sorted(names):
    return sorted(names, key=natural_key)


def read_calib_file(filename: str) -> dict:
    """utils/pose.py:7-30: every `key: 12 values` line as a 4x4 fp64 matrix."""
    calib = {}
    with open(filename) as fh:
        for line in fh:
            key, content = line.strip().split(":")
            values = [float(v) for v in content.strip().split()]
            pose = np.zeros((4, 4))
            pose[0, 0:4] = values[0:4]
            pose[1, 0:4] = values[4:8]
            pose[2, 0:4] = values[8:12]
            pose[3, 3] = 1.0
            calib[key] = pose
    return calib


def read_poses_file(filename: str, calibration: dict) -> list:
    """utils/pose.py:33-58: KITTI poses, each as Tr^-1 · P · Tr (the LiDAR pose in the world frame)."""
    Tr = calibration["Tr"]
    Tr_inv = np.linalg.inv(Tr)
    poses = []
    with open(filename) as fh:
        for line in fh:
            values = [float(v) for v in line.strip().split()]
            pose = np.zeros((4, 4))
            pose[0, 0:4] = values[0:4]
            pose[1, 0:4] = values[4:8]
            pose[2, 0:4] = values[8:12]
            pose[3, 3] = 1.0
            poses.append(np.matmul(Tr_inv, np.matmul(pose, Tr)))
    return poses


def used_frame(config: SHINEConfig, frame_id: int) -> bool:
    """dataset/lidar_dataset.py:73-78."""
    return not (frame_id < config.begin_frame or frame_id > config.end_frame or frame_id % config.every_frame != 0)


def reference_poses(config: SHINEConfig, poses_w: list, total_pc_count: int):
    """dataset/lidar_dataset.py:67-91 -> (poses_ref, begin_pose_inv, used frame ids).  poses_ref[f] is
    begin_pose_inv @ poses_w[f] for used frames and poses_w[f] for the others."""
    if len(poses_w) < total_pc_count:
        raise ValueError(f"{config.pose_path} holds {len(poses_w)} poses for {total_pc_count} scans in {config.pc_path}")
    poses_ref = list(poses_w)
    begin_pose_inv = np.eye(4)
    used = []
    for frame_id in range(total_pc_count):
        if not used_frame(config, frame_id):
            continue
        if not used:
            if config.first_frame_ref:
                begin_pose_inv = np.linalg.inv(poses_w[frame_id])
            else:
                begin_pose_inv[2, 3] += config.global_shift_default
        poses_ref[frame_id] = np.matmul(begin_pose_inv, poses_w[frame_id])
        used.append(frame_id)
    return poses_ref, begin_pose_inv, used


def check_process_config(config: SHINEConfig) -> None:
    """Settings of process_frame that are not implemented raise, naming their key."""
    for key in ("rand_downsample", "filter_noise", "estimate_normal", "behind_dropoff_on", "semantic_on"):
        if getattr(config, key):
            raise NotImplementedError(f"{key}: True is not implemented for real scans")
    if config.clearance_sample_n > 0:
        raise NotImplementedError("clearance_sample_n > 0 is not implemented for real scans")


def check_scan_config(config: SHINEConfig) -> None:
    """check_process_config, and the config's pose file must be a KITTI *.txt file."""
    check_process_config(config)
    if config.pose_path.endswith("csv"):
        raise NotImplementedError("pose_path: CSV odometry poses are not implemented; use KITTI poses.txt")
    if not config.pose_path.endswith("txt"):
        raise ValueError(f"pose_path {config.pose_path!r}: expected a KITTI *.txt pose file")


# ------------------------------------------------------------------------------------------------------------ readers


class ScanRecords:
    """A scan as records: `data` is a uint8 tensor (pinned when read for the GPU); record i starts at byte
    offset + i * stride and holds x y z as float32 (fp64 False) or float64 (fp64 True)."""

    def __init__(self, data: torch.Tensor, n: int, stride: int, fp64: bool, offset: int = 0):
        self.data, self.n, self.stride, self.fp64, self.offset = data, n, stride, fp64, offset

    def points(self) -> np.ndarray:
        """[n,3] float64: what the reference's reader hands on (`.astype(np.float64)`)."""
        t = np.float64 if self.fp64 else np.float32
        w = np.dtype(t).itemsize
        raw = self.data.numpy()[self.offset:self.offset + self.n * self.stride]
        if self.n == 0:
            return np.zeros((0, 3))
        rec = np.lib.stride_tricks.as_strided(raw.view(np.uint8), (self.n, 3 * w), (self.stride, 1))
        return np.ascontiguousarray(rec).view(t).reshape(self.n, 3).astype(np.float64)


def _host_buffer(nbytes: int, pinned: bool) -> torch.Tensor:
    return torch.empty(nbytes, dtype=torch.uint8, pin_memory=pinned)


def _read_body(fh, nbytes: int, pinned: bool, filename: str) -> torch.Tensor:
    buf = _host_buffer(nbytes, pinned)
    if nbytes and fh.readinto(memoryview(buf.numpy())) != nbytes:
        raise ValueError(f"{filename}: file ends before the {nbytes} bytes of points its header declares")
    return buf


def _records_from_xyz(xyz: np.ndarray, pinned: bool) -> ScanRecords:
    xyz = np.ascontiguousarray(xyz)
    buf = _host_buffer(xyz.nbytes, pinned)
    buf.numpy()[:] = xyz.reshape(-1).view(np.uint8)
    return ScanRecords(buf, xyz.shape[0], 3 * xyz.itemsize, xyz.dtype == np.float64)


def read_bin(filename: str, pinned: bool = True) -> ScanRecords:
    """KITTI velodyne: float32 x y z intensity, 16-byte records, read whole into the buffer."""
    nbytes = os.path.getsize(filename)
    if nbytes % 16:
        raise ValueError(f"{filename}: {nbytes} bytes is not a whole number of 16-byte x y z i records")
    with open(filename, "rb") as fh:
        return ScanRecords(_read_body(fh, nbytes, pinned, filename), nbytes // 16, 16, False)


def _read_header(fh, filename: str, end: bytes, limit: int = 256) -> list:
    lines = []
    for _ in range(limit):
        line = fh.readline()
        if not line:
            break
        text = line.strip()
        lines.append(text.decode("ascii", "replace"))
        if text.startswith(end):
            return lines
    raise ValueError(f"{filename}: malformed header (no {end.decode()} line)")


def _xyz_layout(filename: str, fields: list):
    """fields: (name, numpy dtype, count) in record order -> (stride, offset of x, xyz dtype or None when x y z are not
    three adjacent fields of one type, offsets of x y z)."""
    offsets, off = {}, 0
    for name, dt, count in fields:
        offsets.setdefault(name, (off, dt, count))
        off += dt.itemsize * count
    for axis in "xyz":
        if axis not in offsets:
            raise ValueError(f"{filename}: no '{axis}' field")
        o, dt, count = offsets[axis]
        if dt not in (np.dtype("<f4"), np.dtype("<f8")) or count != 1:
            raise ValueError(f"{filename}: field '{axis}' must be one float or double, not {count} x {dt}")
    (ox, tx, _), (oy, ty, _), (oz, tz, _) = offsets["x"], offsets["y"], offsets["z"]
    adjacent = tx == ty == tz and oy == ox + tx.itemsize and oz == oy + tx.itemsize
    return off, ox, (tx if adjacent else None), (ox, oy, oz), (tx, ty, tz)


def _binary_records(fh, filename, n, fields, pinned) -> ScanRecords:
    stride, ox, xyz_t, offs, types = _xyz_layout(filename, fields)
    if xyz_t is not None and stride % xyz_t.itemsize == 0 and ox % xyz_t.itemsize == 0:      # aligned for the kernel
        return ScanRecords(_read_body(fh, n * stride, pinned, filename), n, stride, xyz_t == np.float64, ox)
    raw = _read_body(fh, n * stride, False, filename).numpy().reshape(n, stride)
    cols = [np.ascontiguousarray(raw[:, o:o + t.itemsize]).view(t).reshape(n) for o, t in zip(offs, types)]
    return _records_from_xyz(np.stack(cols, 1).astype(np.result_type(*types)), pinned)


def _ascii_records(fh, filename, n, fields, pinned) -> ScanRecords:
    _xyz_layout(filename, fields)
    cols, col = {}, 0
    for name, dt, count in fields:
        cols.setdefault(name, (col, dt))
        col += count
    text = fh.read().split()
    if len(text) < n * col:
        raise ValueError(f"{filename}: {len(text)} values for {n} points of {col} values")
    vals = np.array(text[:n * col], dtype=np.float64).reshape(n, col)
    t = np.result_type(*(cols[a][1] for a in "xyz"))
    return _records_from_xyz(np.stack([vals[:, cols[a][0]].astype(cols[a][1]) for a in "xyz"], 1).astype(t), pinned)


_PLY_TYPES = {"char": "i1", "int8": "i1", "uchar": "u1", "uint8": "u1", "short": "<i2", "int16": "<i2",
              "ushort": "<u2", "uint16": "<u2", "int": "<i4", "int32": "<i4", "uint": "<u4", "uint32": "<u4",
              "float": "<f4", "float32": "<f4", "double": "<f8", "float64": "<f8"}


def read_ply_header(fh, filename: str):
    """Read a PLY header from `fh` (left at the first byte of the body) -> (format, elements): each element is
    (name, count, [(property, numpy dtype, 1)]); a list property is (property, (count dtype, item dtype), 0), with None
    for the types when they are not PLY scalar types.
    Big-endian files and list properties of the vertex element raise."""
    head = _read_header(fh, filename, b"end_header")
    if head[0] != "ply":
        raise ValueError(f"{filename}: malformed header (no 'ply' magic)")
    fmt, elements = None, []
    for line in head[1:-1]:
        tok = line.split()
        if not tok or tok[0] in ("comment", "obj_info"):
            continue
        if tok[0] == "format" and len(tok) >= 2:
            fmt = tok[1]
        elif tok[0] == "element" and len(tok) == 3 and tok[2].isdigit():
            elements.append((tok[1], int(tok[2]), []))
        elif tok[0] == "property" and elements and len(tok) >= 3:
            if tok[1] == "list":
                if elements[-1][0] == "vertex":
                    raise ValueError(f"{filename}: list property {tok[-1]!r} in the vertex element")
                types = None
                if len(tok) == 5 and tok[2] in _PLY_TYPES and tok[3] in _PLY_TYPES:
                    types = (np.dtype(_PLY_TYPES[tok[2]]), np.dtype(_PLY_TYPES[tok[3]]))
                elements[-1][2].append((tok[-1], types, 0))
                continue
            if tok[1] not in _PLY_TYPES:
                raise ValueError(f"{filename}: malformed header (property type {tok[1]!r})")
            elements[-1][2].append((tok[2], np.dtype(_PLY_TYPES[tok[1]]), 1))
        else:
            raise ValueError(f"{filename}: malformed header line {line!r}")
    if fmt == "binary_big_endian":
        raise ValueError(f"{filename}: big-endian PLY is not supported")
    if fmt not in ("ascii", "binary_little_endian"):
        raise ValueError(f"{filename}: malformed header (format {fmt!r})")
    return fmt, elements


def read_ply(filename: str, pinned: bool = True) -> ScanRecords:
    """PLY, ascii or binary_little_endian; x y z are float or double properties of the `vertex` element, which must
    come first; other scalar properties are skipped by size."""
    with open(filename, "rb") as fh:
        fmt, elements = read_ply_header(fh, filename)
        if not elements or elements[0][0] != "vertex":
            raise ValueError(f"{filename}: the vertex element must come first")
        _, n, fields = elements[0]
        return (_ascii_records if fmt == "ascii" else _binary_records)(fh, filename, n, fields, pinned)


_PCD_TYPES = {("F", 4): "<f4", ("F", 8): "<f8", ("I", 1): "i1", ("I", 2): "<i2", ("I", 4): "<i4", ("I", 8): "<i8",
              ("U", 1): "u1", ("U", 2): "<u2", ("U", 4): "<u4", ("U", 8): "<u8"}


def read_pcd(filename: str, pinned: bool = True) -> ScanRecords:
    """PCD with DATA ascii or binary and any FIELDS / SIZE / TYPE / COUNT layout; x y z are located by name."""
    with open(filename, "rb") as fh:
        head = [line for line in _read_header(fh, filename, b"DATA") if line and not line.startswith("#")]
        kv = {}
        for line in head:
            tok = line.split()
            kv[tok[0].upper()] = tok[1:]
        try:
            names, sizes, types = kv["FIELDS"], [int(s) for s in kv["SIZE"]], kv["TYPE"]
            counts = [int(c) for c in kv.get("COUNT", ["1"] * len(names))]
            n = int(kv["POINTS"][0]) if "POINTS" in kv else int(kv["WIDTH"][0]) * int(kv["HEIGHT"][0])
            data = kv["DATA"][0]
            if not len(names) == len(sizes) == len(types) == len(counts):
                raise ValueError
            fields = [(nm, np.dtype(_PCD_TYPES[(t, s)]), c) for nm, s, t, c in zip(names, sizes, types, counts)]
        except (KeyError, ValueError, IndexError):
            raise ValueError(f"{filename}: malformed PCD header") from None
        if data == "binary_compressed":
            raise ValueError(f"{filename}: DATA binary_compressed is not supported")
        if data not in ("ascii", "binary"):
            raise ValueError(f"{filename}: malformed header (DATA {data!r})")
        return (_ascii_records if data == "ascii" else _binary_records)(fh, filename, n, fields, pinned)


def read_scan(filename: str, pinned: bool = True) -> ScanRecords:
    """dataset/lidar_dataset.py:283-293: the format follows the file name."""
    if ".bin" in filename:
        return read_bin(filename, pinned)
    if ".ply" in filename:
        return read_ply(filename, pinned)
    if ".pcd" in filename:
        return read_pcd(filename, pinned)
    raise ValueError(f"{filename}: point clouds are read from *.bin, *.ply or *.pcd files")


# ---------------------------------------------------------------------------------------------------------- GPU frame


class ScanProcessor:
    """Caller-owned device scratch of csrc/shine_scan.cu, grown to the largest frame seen."""

    def __init__(self, config: SHINEConfig, device):
        self.config = config
        self.device = torch.device(device)
        self._scratch = torch.empty(0, dtype=torch.uint8, device=self.device)
        self.count = torch.zeros(1, dtype=torch.int64, device=self.device)

    def _scratch_for(self, n: int):
        from . import _abi
        need = int(_abi.lib().shine_scan_scratch_bytes(n))
        if need < 0:
            raise _abi.ShineB200Error(f"a frame of {n} points is too large")
        if self._scratch.numel() < need:
            self._scratch = torch.empty(need, dtype=torch.uint8, device=self.device)
        return self._scratch

    def points(self, rec: ScanRecords, pose_ref: np.ndarray, voxels_out: bool = False):
        """Filter, crop, voxel down-sample, transform by pose_ref and scale one scan on the GPU.
        -> fp32 [m,3] points in scaled reference coordinates (and the fp64 [m,3] voxel averages with voxels_out)."""
        from . import _abi
        cfg = self.config
        lib, st = _abi.lib(), _abi.stream_ptr(self.device)
        data = rec.data.to(self.device, non_blocking=True)
        inp = _abi.ShineScanInput(data.data_ptr() + rec.offset, rec.n, rec.stride, int(rec.fp64))
        scratch = self._scratch_for(rec.n)
        _abi.check(lib.shine_scan_filter_keys(C.byref(inp), float(cfg.min_z), float(cfg.max_z), float(cfg.min_range),
                                              float(cfg.pc_radius), float(cfg.vox_down_m), _abi.ptr(scratch),
                                              scratch.numel(), st), "shine_scan_filter_keys")
        _abi.check(lib.shine_scan_sort_voxels(rec.n, _abi.ptr(self.count), _abi.ptr(scratch), scratch.numel(), st),
                   "shine_scan_sort_voxels")
        m = int(self.count.item())                           # the frame's one host read: it sizes every later buffer
        pts = torch.empty(m, 3, device=self.device)
        vox = torch.empty(m, 3, dtype=torch.float64, device=self.device) if voxels_out else None
        pose = (C.c_double * 16)(*np.ascontiguousarray(pose_ref, dtype=np.float64).reshape(16).tolist())
        _abi.check(lib.shine_scan_average_transform(C.byref(inp), pose, float(cfg.scale), m, _abi.ptr(vox), _abi.ptr(pts),
                                                    _abi.ptr(scratch), scratch.numel(), st),
                   "shine_scan_average_transform")
        return (pts, vox) if voxels_out else pts

    def sample(self, points: torch.Tensor, origin32: np.ndarray, u_surface=None, u_free=None):
        """dataSampler.sample (utils/data_sampler.py:18-139) for fp32 points and the fp32 origin.  The uniforms default to
        the reference's own draws: torch.rand(R*ns, 1), torch.rand(R*clearance_n, 1), torch.rand(R*nf, 1).
        -> coord [R(ns+nf),3], sdf_label, weight in ray-wise order."""
        from . import _abi
        cfg = self.config
        R, ns, nf = points.shape[0], cfg.surface_sample_n, cfg.free_sample_n
        if u_surface is None:
            u_surface = torch.rand(R * ns, 1, device=self.device)
            torch.rand(R * cfg.clearance_sample_n, 1, device=self.device)
            u_free = torch.rand(R * nf, 1, device=self.device)
        coord = torch.empty(R * (ns + nf), 3, device=self.device)
        label = torch.empty(R * (ns + nf), device=self.device)
        weight = torch.empty(R * (ns + nf), device=self.device)
        o = np.asarray(origin32, dtype=np.float32).reshape(3)
        _abi.check(_abi.lib().shine_scan_sample(
            _abi.ptr(points.contiguous()), R, float(o[0]), float(o[1]), float(o[2]), _abi.ptr(u_surface.contiguous()), ns,
            _abi.ptr(u_free.contiguous()), nf, float(np.float32(cfg.surface_sample_range_m * cfg.scale)),
            float(np.float32(cfg.free_sample_end_dist_m * cfg.scale)), float(np.float32(cfg.free_sample_begin_ratio)),
            _abi.ptr(coord), _abi.ptr(label), _abi.ptr(weight), _abi.stream_ptr(self.device)), "shine_scan_sample")
        return coord, label, weight


class LiDARDataset:
    """dataset/lidar_dataset.py:22-281 for KITTI *.bin, *.ply and *.pcd sequences with KITTI poses.

    The pool follows the existing rules: `synth.use_host_pool` -> HostSamplePool; `continual_learning_reg` -> the
    current frame's samples only (`process_frame(f, incremental_on=True)`); `window_replay_on` -> ReplayPool and its
    window; otherwise a device SamplePool.  The map cloud (`map_down_pc`) is not kept: it only feeds meshing."""

    def __init__(self, config: SHINEConfig, octree=None, pool=None):
        check_scan_config(config)
        calib = read_calib_file(config.calib_path) if config.calib_path != "" else {"Tr": np.eye(4)}
        poses_w = read_poses_file(config.pose_path, calib)
        self.pc_filenames = natural_sorted(os.listdir(config.pc_path))
        self._init_frames(config, poses_w, len(self.pc_filenames), octree, pool)

    def _init_frames(self, config: SHINEConfig, poses_w: list, total_pc_count: int, octree, pool):
        """Frame selection, reference poses, the pool and the GPU scratch: what every frame source shares."""
        from . import synth
        self.config = config
        self.device = torch.device(config.device)
        self.total_pc_count = total_pc_count
        self.poses_ref, self.begin_pose_inv, self.used_frames = reference_poses(config, poses_w, self.total_pc_count)
        self.used_pc_count = len(self.used_frames)
        self.octree = octree
        if pool is None:
            if synth.use_host_pool(config, self.used_pc_count):
                pool = synth.HostSamplePool(self.device)
            elif config.window_replay_on and not config.continual_learning_reg:
                pool = synth.ReplayPool(self.device)
            else:
                pool = synth.SamplePool(self.device)
        self.pool = pool
        self.processor = ScanProcessor(config, self.device)
        self._bbx = None

    def origin_scaled(self, frame_id: int) -> np.ndarray:
        """dataset/lidar_dataset.py:175: the frame's sensor origin in scaled coordinates, numpy fp64."""
        return self.poses_ref[frame_id][:3, 3] * self.config.scale

    def read_frame(self, frame_id: int) -> ScanRecords:
        """The frame's point records, in pinned host or device memory."""
        return read_scan(os.path.join(self.config.pc_path, self.pc_filenames[frame_id]))

    def frame_samples(self, frame_id: int):
        """Read, preprocess and sample one scan -> (coord, sdf_label, weight, origin_scaled fp32 tensor, points)."""
        rec = self.read_frame(frame_id)
        points = self.processor.points(rec, self.poses_ref[frame_id])
        origin = torch.tensor(self.origin_scaled(frame_id), dtype=torch.float32)
        coord, label, weight = self.processor.sample(points, origin.numpy())
        if points.shape[0]:       # map_bbx of dataset/lidar_dataset.py:196-203, kept on the device (no host read here)
            lo, hi = points.amin(0), points.amax(0)
            self._bbx = (lo, hi) if self._bbx is None else (torch.minimum(self._bbx[0], lo), torch.maximum(self._bbx[1], hi))
        return coord, label, weight, origin, points

    def surface_samples(self, coord: torch.Tensor) -> torch.Tensor:
        """coord[weight > 0] without a compaction: the first surface_sample_n samples of every ray."""
        per_ray = self.config.surface_sample_n + self.config.free_sample_n
        return coord.view(-1, per_ray, 3)[:, :self.config.surface_sample_n]

    def process_frame(self, frame_id: int, incremental_on: bool = False):
        """dataset/lidar_dataset.py:115-281: sample the scan, grow the octree, fill the pool."""
        coord, label, weight, origin, points = self.frame_samples(frame_id)
        if self.octree is not None:                                              # :211-218
            src = self.surface_samples(coord) if self.config.octree_from_surface_samples else points
            self.octree.update(src.reshape(-1, 3), incremental_on)
        from . import synth
        if incremental_on:                                                       # :223-233
            self.pool = synth.SamplePool(self.device)
            self.pool.append(coord, label, weight)
        elif isinstance(self.pool, synth.ReplayPool) and self.config.window_replay_on:     # :237-270
            self.pool.add_frame(coord, label, weight, origin, self.config.window_radius * self.config.scale)
        else:
            self.pool.append(coord, label, weight)
        return coord, label, weight

    @property
    def map_bbx(self):
        """(min, max) metres in the map frame of the points of the frames read so far (None before the first)."""
        if self._bbx is None:
            return None
        return tuple((t.double() / self.config.scale).cpu().numpy() for t in self._bbx)

    def frames(self):
        """(coord, sdf_label, weight, origin_scaled) per used frame, for `run_shine_mapping_incremental`."""
        for frame_id in self.used_frames:
            yield self.frame_samples(frame_id)[:4]

    def get_batch(self, bs: int, **kw):
        return self.pool.get_batch(bs, **kw)

    def __len__(self):
        return len(self.pool)
