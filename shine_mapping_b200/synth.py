"""Synthetic LiDAR data for the hot path (there is no dataset on the GPU box; SURVEY.md §8d).

* `raycast_scene`   — analytic scene (ground plane, two walls, axis-aligned boxes) hit by an HDL-64-like
                      scan pattern from a sensor origin -> hit points in metres.
* `scene_surface_points` — lattice points on the hittable surfaces of that scene: the ground truth of mesh evaluation.
* `sample_rays`     — the training-sample contract of the reference's `dataSampler.sample`
                      (utils/data_sampler.py:18-139): per hit, `surface_sample_n` samples uniformly within
                      +-surface_sample_range of the hit and `free_sample_n` samples in free space; label = signed
                      displacement along the ray in scaled units (positive behind the surface, :109-111); weight
                      +1 for surface samples, -1 for free-space samples (:104); ray-wise output order (:123-134).
* `SamplePool`      — the device sample pools and `get_batch()` of `LiDARDataset`
                      (dataset/lidar_dataset.py:104-113,431-448): `torch.randint` gather.
* `ReplayPool`      — the pool of incremental mapping with replay: earlier frames' samples kept, those outside the
                      sliding window dropped on the GPU before the frame is appended (dataset/lidar_dataset.py:235-271).
* `HostSamplePool`  — the batch-mode pool in pinned host memory past `pc_count_gpu_limit` scans (dataset/lidar_dataset.py:
                      94-101), gathered on the GPU; `use_host_pool` states the reference's rule.
* `build_scene_map` — scans -> samples -> `octree.update(surface samples)` (dataset/lidar_dataset.py:204-218).
"""
from __future__ import annotations

import ctypes as C
import math

import numpy as np
import torch

from .config import SHINEConfig


def lidar_directions(n_azimuth: int, n_elev: int = 64, elev_min_deg: float = -24.8, elev_max_deg: float = 2.0,
                     device="cpu") -> torch.Tensor:
    """Unit ray directions [n_elev * n_azimuth, 3] of an HDL-64-like spinning LiDAR."""
    el = torch.linspace(math.radians(elev_min_deg), math.radians(elev_max_deg), n_elev, device=device)
    az = torch.arange(n_azimuth, device=device, dtype=torch.float32) * (2 * math.pi / n_azimuth)
    el, az = torch.meshgrid(el, az, indexing="ij")
    d = torch.stack((torch.cos(el) * torch.cos(az), torch.cos(el) * torch.sin(az), torch.sin(el)), -1)
    return d.reshape(-1, 3)


def default_boxes(device="cpu") -> torch.Tensor:
    """[K, 6] axis-aligned boxes (xmin, ymin, zmin, xmax, ymax, zmax) in metres: parked-car / kiosk sized."""
    return torch.tensor([
        [6.0, -5.5, -1.7, 10.0, -3.7, -0.2], [14.0, 3.5, -1.7, 18.5, 5.4, -0.1], [-9.0, -6.0, -1.7, -5.0, -4.2, 0.0],
        [24.0, -6.5, -1.7, 27.0, -4.0, 1.0], [-20.0, 4.0, -1.7, -16.0, 6.0, -0.2], [35.0, 2.0, -1.7, 38.0, 6.5, 1.5],
        [48.0, -6.0, -1.7, 52.0, -3.8, -0.3], [62.0, 3.0, -1.7, 66.0, 5.0, 0.2], [77.0, -6.8, -1.7, 80.0, -4.4, 0.8],
        [91.0, 3.6, -1.7, 95.0, 5.6, -0.2]], dtype=torch.float32, device=device)


def _lattice(lo, hi, spacing: float):
    """Points lo + spacing * i per axis with i = 0 .. floor((hi - lo) / spacing), fp64, all combinations."""
    axes = [lo[a] + spacing * np.arange(int(np.floor((hi[a] - lo[a]) / spacing + 1e-9)) + 1) for a in range(len(lo))]
    return np.stack(np.meshgrid(*axes, indexing="ij"), -1).reshape(-1, len(lo))


def scene_surface_points(x_min: float, x_max: float, spacing: float, ground_z: float = -1.7, wall_y: float = 8.0,
                         wall_top: float = 4.3, boxes: torch.Tensor | None = None) -> torch.Tensor:
    """Deterministic lattice points (fp64 [M,3], metres) on the surfaces of `raycast_scene` that a ray can hit, over
    x in [x_min, x_max]: the ground between the walls outside the boxes' footprints, the inner faces of both walls, and
    the four sides and the top of every box (`default_boxes()` unless given), clipped to the x range."""
    if not spacing > 0 or not x_max >= x_min:
        raise ValueError("scene_surface_points needs spacing > 0 and x_max >= x_min")
    bx = (default_boxes() if boxes is None else boxes).double().cpu().numpy()
    parts = []
    g = _lattice((x_min, -wall_y), (x_max, wall_y), spacing)
    inside = np.zeros(g.shape[0], dtype=bool)
    for b in bx:
        inside |= (g[:, 0] > b[0]) & (g[:, 0] < b[3]) & (g[:, 1] > b[1]) & (g[:, 1] < b[4])
    g = g[~inside]
    parts.append(np.column_stack((g, np.full(g.shape[0], ground_z))))
    for y in (-wall_y, wall_y):
        w = _lattice((x_min, ground_z), (x_max, wall_top), spacing)
        parts.append(np.column_stack((w[:, 0], np.full(w.shape[0], y), w[:, 1])))
    for b in bx:
        lo_x, hi_x = max(b[0], x_min), min(b[3], x_max)
        if lo_x > hi_x:
            continue
        top = _lattice((lo_x, b[1]), (hi_x, b[4]), spacing)
        parts.append(np.column_stack((top, np.full(top.shape[0], b[5]))))
        for y in (b[1], b[4]):
            s = _lattice((lo_x, b[2]), (hi_x, b[5]), spacing)
            parts.append(np.column_stack((s[:, 0], np.full(s.shape[0], y), s[:, 1])))
        for x in (b[0], b[3]):
            if x_min <= x <= x_max:
                s = _lattice((b[1], b[2]), (b[4], b[5]), spacing)
                parts.append(np.column_stack((np.full(s.shape[0], x), s)))
    return torch.from_numpy(np.concatenate(parts))


def raycast_scene(origin: torch.Tensor, dirs: torch.Tensor, boxes: torch.Tensor | None = None,
                  min_range: float = 3.0, max_range: float = 50.0, ground_z: float = -1.7,
                  wall_y: float = 8.0, wall_top: float = 4.3) -> torch.Tensor:
    """First hit of every ray with {ground plane, walls y=+-wall_y, boxes}; returns the hit points [M,3] (metres)
    whose range lies in [min_range, max_range]."""
    o = origin.reshape(1, 3).to(dirs)
    inf = torch.full((dirs.shape[0],), float("inf"), device=dirs.device)
    dz = dirs[:, 2]
    t_best = torch.where(dz < -1e-6, (ground_z - o[0, 2]) / dz.clamp(max=-1e-6), inf)
    for sign in (1.0, -1.0):
        dy = dirs[:, 1] * sign
        t = torch.where(dy > 1e-6, (wall_y - sign * o[0, 1]) / dy.clamp(min=1e-6), inf)
        z_hit = o[0, 2] + t * dz
        t = torch.where((z_hit >= ground_z) & (z_hit <= wall_top), t, inf)
        t_best = torch.minimum(t_best, t)
    if boxes is not None and boxes.numel():
        safe = torch.where(dirs.abs() < 1e-9, torch.full_like(dirs, 1e-9), dirs)
        inv = (1.0 / safe).unsqueeze(1)                                   # [R,1,3]
        t0 = (boxes[None, :, :3] - o[:, None, :]) * inv
        t1 = (boxes[None, :, 3:] - o[:, None, :]) * inv
        t_near = torch.minimum(t0, t1).amax(-1)
        t_far = torch.maximum(t0, t1).amin(-1)
        hit = (t_far >= t_near) & (t_near > 0)
        t_box = torch.where(hit, t_near, torch.full_like(t_near, float("inf"))).amin(1)
        t_best = torch.minimum(t_best, t_box)
    keep = (t_best >= min_range) & (t_best <= max_range)
    return o + dirs[keep] * t_best[keep].unsqueeze(1)


def sample_rays(points_scaled: torch.Tensor, origin_scaled: torch.Tensor, config: SHINEConfig,
                generator: torch.Generator | None = None):
    """-> coord [M,3] (scaled, in [-1,1]), sdf_label [M] (scaled), weight [M] (+1 surface / -1 free), ray-wise
    ordered: for every ray its surface samples then its free-space samples."""
    dev = points_scaled.device
    shift = points_scaled - origin_scaled
    dist = torch.linalg.norm(shift, dim=1, keepdim=True)                              # [R,1]
    R = shift.shape[0]
    ns, nf = config.surface_sample_n, config.free_sample_n
    rng = config.surface_sample_range_m * config.scale

    def rand(*shape):
        return torch.rand(*shape, device=dev, generator=generator)

    surf_disp = (rand(R, ns) - 0.5) * 2.0 * rng                                       # [R,ns]
    surf_ratio = surf_disp / dist + 1.0
    free_max = config.free_sample_end_dist_m * config.scale / dist + 1.0
    free_ratio = rand(R, nf) * (free_max - config.free_sample_begin_ratio) + config.free_sample_begin_ratio
    free_disp = (free_ratio - 1.0) * dist
    ratio = torch.cat((surf_ratio, free_ratio), 1)                                    # [R, ns+nf]
    disp = torch.cat((surf_disp, free_disp), 1)
    coord = (shift.unsqueeze(1) * ratio.unsqueeze(2) + origin_scaled.reshape(1, 1, 3)).reshape(-1, 3)
    weight = torch.ones(R, ns + nf, device=dev)
    weight[:, ns:] = -1.0
    return coord.contiguous(), disp.reshape(-1).contiguous(), weight.reshape(-1).contiguous()


class SamplePool:
    """coord / sdf_label / weight pools + `get_batch()` (dataset/lidar_dataset.py:431-448).

    `sort_morton()` puts the pool in Morton order of the sample coordinates (once, when the map is built).  From then on
    `get_batch()` draws the SAME random index multiset as the reference (`torch.randint`, with replacement) and hands the
    samples out in ascending index order, i.e. in Morton order: neighbouring points of a batch then touch the same octree
    nodes, which is what the gather (L1 hits) and the voxel-grouped scatter of the training kernel feed on
    (`SdfTrainer.forward_backward(..., morton_ordered=pool.ordered)`).  The loss of a batch does not depend on its order."""

    def __init__(self, device):
        self.device = device
        self.coord_pool = torch.empty(0, 3, device=device)
        self.sdf_label_pool = torch.empty(0, device=device)
        self.weight_pool = torch.empty(0, device=device)
        self.ordered = False

    def append(self, coord, label, weight):
        self.coord_pool = torch.cat((self.coord_pool, coord.to(self.device)))
        self.sdf_label_pool = torch.cat((self.sdf_label_pool, label.to(self.device)))
        self.weight_pool = torch.cat((self.weight_pool, weight.to(self.device)))
        self.ordered = False

    def __len__(self):
        return self.sdf_label_pool.shape[0]

    def sort_morton(self, level: int = 16, octree=None):
        """Reorder the pool along the Z-order curve of a 2^level grid over [-1, 1]^3 (16: kaolin's int16 coordinates).
        With `octree` (the map the pool belongs to) the samples that see no node on any level — free space: their features
        are 0 whatever the tables hold — go behind all others, each part in Z-order: the tiles of a batch that take the
        step kernel's zero-tile shortcut then sit at the end of the batch, where the kernel's strided tile schedule hands
        every warp the same share of them."""
        from .feature_octree import points_to_morton, quantize_points
        if len(self):
            key = points_to_morton(quantize_points(self.coord_pool, level))
            if octree is not None:
                key = key | ((~octree.sees_a_node(self.coord_pool)).long() << 62)      # Morton keys use 48 bits
            order = torch.argsort(key)
            self.coord_pool = self.coord_pool[order].contiguous()
            self.sdf_label_pool = self.sdf_label_pool[order].contiguous()
            self.weight_pool = self.weight_pool[order].contiguous()
        self.ordered = True
        return self

    def get_batch(self, bs: int, generator: torch.Generator | None = None, ordered: bool | None = None):
        """ordered: None = Morton order iff the pool is sorted; False = the reference's order (as drawn)."""
        index = torch.randint(0, len(self), (bs,), device=self.device, generator=generator)
        if self.ordered and ordered is not False:
            index = torch.sort(index).values
        elif ordered:
            raise ValueError("ordered batches need a pool in Morton order: call sort_morton() first")
        return self.coord_pool[index, :], self.sdf_label_pool[index], self.weight_pool[index]


class ReplayPool(SamplePool):
    """The pool of incremental mapping with replay (`continual_learning_reg: False`, dataset/lidar_dataset.py:235-271):
    every earlier frame's samples stay; with a window (`window_replay_on`) the ones `window_radius * scale` or more from
    the new sensor origin are dropped before the new frame is appended behind the survivors, in the reference's order.

    The samples live in capacity buffers that grow by about 1.5x; `coord_pool` / `sdf_label_pool` / `weight_pool` are
    views `[:size]` of them, so `get_batch` is SamplePool's: the reference's `torch.randint` draw, in the order drawn.
    With a window, `add_frame` is one launch of `shine_pool_window_append` (filter and append in place) and reading the
    new size back is its only host synchronisation; without one, the frame is copied behind the old samples."""

    GROWTH = 1.5

    def __init__(self, device, capacity: int = 0):
        super().__init__(device)
        self._coord = torch.empty(capacity, 3, device=device)
        self._label = torch.empty(capacity, device=device)
        self._weight = torch.empty(capacity, device=device)
        self._scratch = None
        self._size_out = None
        self._set_size(0)

    @property
    def capacity(self) -> int:
        return self._label.shape[0]

    def _set_size(self, n: int) -> None:
        self.size = n
        self.coord_pool, self.sdf_label_pool, self.weight_pool = self._coord[:n], self._label[:n], self._weight[:n]

    def _reserve(self, need: int) -> None:
        if need <= self.capacity:
            return
        cap = max(need, int(self.capacity * self.GROWTH))
        n = self.size
        self.coord_pool = self.sdf_label_pool = self.weight_pool = None     # the views would keep the old buffers alive
        for name, shape in (("_coord", (cap, 3)), ("_label", (cap,)), ("_weight", (cap,))):
            old = getattr(self, name)
            new = torch.empty(shape, device=self.device)
            new[:n] = old[:n]
            setattr(self, name, new)
            del old                  # one array at a time: the pool is never held twice
        self._set_size(n)

    def add_frame(self, coord, label, weight, origin_scaled=None, window_radius_scaled: float | None = None):
        """Append one frame's samples.  window_radius_scaled (`window_radius * scale`, a Python float): first drop the
        samples whose distance to origin_scaled (the frame's sensor origin in scaled coordinates, 3 values on the host)
        is not below it; None: keep every earlier sample (`window_replay_on: False`)."""
        coord = coord.to(self.device, torch.float32).reshape(-1, 3).contiguous()
        label = label.to(self.device, torch.float32).reshape(-1).contiguous()
        weight = weight.to(self.device, torch.float32).reshape(-1).contiguous()
        n_new = coord.shape[0]
        if label.shape[0] != n_new or weight.shape[0] != n_new:
            raise ValueError("coord, label and weight of a frame must have the same number of samples")
        self._reserve(self.size + n_new)
        self.ordered = False
        if window_radius_scaled is None:                 # lidar_dataset.py:260-270: simply keep all previous samples
            self._coord[self.size:self.size + n_new] = coord
            self._label[self.size:self.size + n_new] = label
            self._weight[self.size:self.size + n_new] = weight
            self._set_size(self.size + n_new)
            return self
        from . import _abi
        _abi.require_cuda(self._coord, "ReplayPool.add_frame")
        o = torch.as_tensor(origin_scaled, dtype=torch.float32).reshape(3).tolist()
        lib = _abi.lib()
        need = int(lib.shine_pool_scratch_bytes(self.size + n_new))
        if self._scratch is None or self._scratch.numel() < need:
            self._scratch = torch.empty(need, dtype=torch.uint8, device=self.device)
            self._size_out = torch.empty(1, dtype=torch.int64, device=self.device)
        desc = _abi.ShineSamplePool(self._coord.data_ptr(), self._label.data_ptr(), self._weight.data_ptr(), self.size,
                                    self.capacity)
        _abi.check(lib.shine_pool_window_append(C.byref(desc), _abi.ptr(coord), _abi.ptr(label), _abi.ptr(weight), n_new,
                                                o[0], o[1], o[2], float(window_radius_scaled), _abi.ptr(self._size_out),
                                                _abi.ptr(self._scratch), self._scratch.numel(),
                                                _abi.stream_ptr(self._coord.device)), "shine_pool_window_append")
        self._set_size(int(self._size_out.item()))      # randint needs the size on the host
        return self

    def append(self, coord, label, weight):
        return self.add_frame(coord, label, weight)

    def sort_morton(self, level: int = 16, octree=None):
        raise NotImplementedError("ReplayPool keeps the reference's sample order (the window filter preserves it)")


class HostSamplePool:
    """The batch-mode pool in pinned host memory, for maps of more scans than `pc_count_gpu_limit`
    (dataset/lidar_dataset.py:94-101: the reference then keeps its pools in CPU memory).  Same contract as SamplePool:
    `append`, `len`, `get_batch(bs, generator=None, ordered=None)`, `ordered = False`.

    Samples are 32-byte records {x, y, z, label, weight, pad x3} in pinned chunks of 2^chunk_shift records (a power of two
    in bytes, which is what torch's pinned allocator hands out); the pool grows by adding chunks, never by copying.
    `append` is one launch of `shine_host_pool_append` that packs a frame's device samples straight into the chunks.
    `get_batch` draws the indices exactly like SamplePool (`torch.randint` on the device, same generator calls), then one
    launch of `shine_host_pool_gather` reads the drawn records over PCIe: a host pool and a device pool filled with the same
    frames give bit-identical batches for the same generator state.  The reference instead draws and indexes on the CPU and
    copies the batch (:431-448); the distribution is the same (uniform, with replacement) and here the draw stays on the
    device, so `get_batch` has no host synchronisation and can be captured in a CUDA graph (capture it after the last
    append: a captured batch draws from the pool size at capture time)."""

    RECORD_FLOATS = 8
    DEFAULT_CHUNK_SHIFT = 22          # 4 Mi records = 128 MiB per chunk

    def __init__(self, device, chunk_shift: int = DEFAULT_CHUNK_SHIFT):
        if not 5 <= chunk_shift <= 31:
            raise ValueError("chunk_shift must lie in [5, 31]")
        self.device = torch.device(device)
        if self.device.type != "cuda":
            raise ValueError("HostSamplePool feeds a GPU: device must be a CUDA device")
        if self.device.index is None:
            self.device = torch.device("cuda", torch.cuda.current_device())
        self.chunk_shift = chunk_shift
        self.size = 0
        self.ordered = False
        self.last_index = None        # the indices of the last get_batch (a graph's static tensor when captured)
        self._chunks: list[torch.Tensor] = []
        self._table = torch.empty(0, dtype=torch.int64, device=self.device)   # device array of the chunks' addresses

    @property
    def chunk_records(self) -> int:
        return 1 << self.chunk_shift

    @property
    def capacity(self) -> int:
        return len(self._chunks) << self.chunk_shift

    def __len__(self):
        return self.size

    def _descriptor(self):
        from . import _abi
        return _abi.ShineHostPool(self._table.data_ptr() if self._chunks else None, self.chunk_shift, len(self._chunks),
                                  self.size)

    def _reserve(self, need: int) -> None:
        if self.capacity >= need:
            return
        while self.capacity < need:
            self._chunks.append(torch.empty(self.chunk_records * self.RECORD_FLOATS, dtype=torch.float32, pin_memory=True))
        self._table = torch.tensor([c.data_ptr() for c in self._chunks], dtype=torch.int64, device=self.device)

    def append(self, coord, label, weight):
        from . import _abi
        for t in (coord, label, weight):
            _abi.require_cuda(t, "HostSamplePool.append")
            if t.device != self.device:
                raise ValueError(f"HostSamplePool.append: frame on {t.device}, pool fed to {self.device}")
        coord = coord.to(torch.float32).reshape(-1, 3).contiguous()
        label = label.to(torch.float32).reshape(-1).contiguous()
        weight = weight.to(torch.float32).reshape(-1).contiguous()
        n = coord.shape[0]
        if label.shape[0] != n or weight.shape[0] != n:
            raise ValueError("coord, label and weight of a frame must have the same number of samples")
        if n == 0:
            return self
        self._reserve(self.size + n)
        desc = self._descriptor()
        _abi.check(_abi.lib().shine_host_pool_append(C.byref(desc), self.size, _abi.ptr(coord), _abi.ptr(label),
                                                     _abi.ptr(weight), n, _abi.stream_ptr(self.device)),
                   "shine_host_pool_append")
        self.size += n
        return self

    def gather(self, index: torch.Tensor):
        """-> coord [n,3], sdf_label [n], weight [n] on the device: the samples at `index` (int64 device tensor)."""
        from . import _abi
        _abi.require_cuda(index, "HostSamplePool.gather")
        index = index.to(torch.int64).reshape(-1).contiguous()
        n = index.shape[0]
        coord = torch.empty(n, 3, device=self.device)
        label = torch.empty(n, device=self.device)
        weight = torch.empty(n, device=self.device)
        if n:
            desc = self._descriptor()
            _abi.check(_abi.lib().shine_host_pool_gather(C.byref(desc), _abi.ptr(index), n, _abi.ptr(coord),
                                                         _abi.ptr(label), _abi.ptr(weight),
                                                         _abi.stream_ptr(self.device)), "shine_host_pool_gather")
        return coord, label, weight

    def get_batch(self, bs: int, generator: torch.Generator | None = None, ordered: bool | None = None):
        """ordered: None or False = the order drawn; True raises (the host pool is never in Morton order)."""
        if ordered:
            raise ValueError("HostSamplePool hands batches out in the order drawn; it has no Morton order")
        if self.size == 0:
            raise ValueError("get_batch on an empty HostSamplePool")
        index = torch.randint(0, self.size, (bs,), device=self.device, generator=generator)
        self.last_index = index
        return self.gather(index)

    def sort_morton(self, level: int = 16, octree=None):
        raise NotImplementedError("HostSamplePool keeps the samples in the order appended")


def use_host_pool(config: SHINEConfig, n_frames: int) -> bool:
    """The reference's rule for the pool's place in batch mode (dataset/lidar_dataset.py:94): pinned host memory iff the
    run uses more than `pc_count_gpu_limit` scans and neither continual-learning mode is on."""
    return n_frames > config.pc_count_gpu_limit and not config.continual_learning_reg and not config.window_replay_on


def generate_scans(config: SHINEConfig, n_azimuth: int, n_frames: int = 1, frame_step_m: float = 1.0, seed: int = 42,
                   device=None, origin_x0: float = 0.0):
    """Scan the analytic scene from `n_frames` poses along +x and sample every scan like the reference's sampler.
    -> list of (coord, sdf_label, weight, hits_scaled) per frame."""
    device = device or config.device
    gen = torch.Generator(device=device)
    gen.manual_seed(seed)
    dirs = lidar_directions(n_azimuth, device=device)
    boxes = default_boxes(device)
    boxes[:, 0] += origin_x0
    boxes[:, 3] += origin_x0
    frames = []
    for f in range(n_frames):
        origin = torch.tensor([origin_x0 + f * frame_step_m, 0.0, 0.0], device=device)
        hits = raycast_scene(origin, dirs, boxes, min_range=config.min_range, max_range=config.pc_radius)
        coord, label, weight = sample_rays(hits * config.scale, origin * config.scale, config, gen)
        frames.append((coord, label, weight, hits * config.scale))
    return frames


def build_scene_map(config: SHINEConfig, octree, n_azimuth: int, n_frames: int = 1, frame_step_m: float = 1.0,
                    seed: int = 42, device=None, origin_x0: float = 0.0, pool=None):
    """Scan the analytic scene from `n_frames` poses along +x, sample every scan, grow the octree from the
    surface samples (weight > 0; dataset/lidar_dataset.py:212-218) and return the pool, with `map_bbx` set to the
    (min, max) metres of the surface samples.
    pool: None = a new SamplePool; "auto" = a new HostSamplePool if `use_host_pool(config, n_frames)`, else a new
    SamplePool; or the (Host)SamplePool to fill."""
    from . import mesher as _mesher
    device = device or config.device
    if pool is None:
        pool = SamplePool(device)
    elif isinstance(pool, str):
        if pool != "auto":
            raise ValueError(f"pool must be None, 'auto' or a pool object, not {pool!r}")
        pool = HostSamplePool(device) if use_host_pool(config, n_frames) else SamplePool(device)
    for coord, label, weight, hits in generate_scans(config, n_azimuth, n_frames, frame_step_m, seed, device, origin_x0):
        if config.octree_from_surface_samples:
            octree.update(coord[weight > 0, :])
        else:
            octree.update(hits)
        pool.append(coord, label, weight)
        pool.map_bbx = _mesher.surface_bbx(coord, weight, config.scale, getattr(pool, "map_bbx", None))   # for bbx meshing
    return pool
