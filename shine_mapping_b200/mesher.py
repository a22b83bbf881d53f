"""Mesh reconstruction from the map, after reference utils/mesher.py (`recon_octree_mesh`, `recon_bbx_mesh`).

The SDF grid is block-sparse: bricks of n^3 marching-cubes cells, each stored with its +1 faces so that a chunk of bricks
is queried (`shine_mesh_grid`, shine_sdf_infer's kernel over generated coordinates) and meshed (`shine_marching_cubes`)
without the others.  Peak device memory of the grid is 5 (n+1)^3 bytes per brick of a chunk: CHUNK_POINTS points,
80 MiB, whatever the size of the map.  Vertices are welded across bricks and chunks through an edge table (16 bytes per
slot, kept at most half full).  Normals and the cluster filter follow on the GPU (`shine_mesh_clusters`), the compaction and
`global_transform` are tensor indexing and one 4x4 product.

DESIGN.md §8 states the grid rules and where this differs from the reference.
"""
from __future__ import annotations

import ctypes as C
import os

import numpy as np
import torch

from . import _abi
from .config import SHINEConfig
from .decoder import Decoder
from .feature_octree import FeatureOctree, morton_to_points

CHUNK_POINTS = 1 << 24      # grid points per chunk (sdf fp32 + mask byte: 80 MiB)
BBX_TILE = 16               # cubes per brick side in bbx mode
MAX_EDGE_SLOTS = 1 << 31   # edge-table capacity is a uint32 power of two (32 GiB of 16-byte slots)
OCTREE_MIN_CLUSTER = 300    # filter_isolated_vertices' default (utils/mesher.py:240), used by recon_octree_mesh


def _next_pow2(n: int) -> int:
    return 1 << max(0, int(n) - 1).bit_length()


def _brick_keys(bricks: torch.Tensor) -> torch.Tensor:
    b = bricks.long()
    return (b[:, 0] << 42) | (b[:, 1] << 21) | b[:, 2]


class Mesher:
    def __init__(self, config: SHINEConfig, octree: FeatureOctree, decoder: Decoder):
        if config.mc_local:
            raise NotImplementedError("mc_local (a mesh of the current frame's bounding box only) is not implemented")
        if config.semantic_on:
            raise NotImplementedError("semantic meshing is not implemented")
        self.config = config
        self.octree = octree
        self.decoder = decoder
        self.world_scale = config.scale
        self.global_transform = np.eye(4)

    # ---- the reference's surface ---------------------------------------------------------------------------------

    @torch.no_grad()
    def recon_octree_mesh(self, query_level: int, mc_res_m: float, mesh_path: str | None = None,
                          map_path: str | None = None):
        """utils/mesher.py:296-368: one n^3 block per octree node at `query_level`.  map_path: also write the SDF map, the
        masked grid points only (the mode the reference leaves commented out, utils/mesher.py:341)."""
        grid = self.octree_grid(query_level, mc_res_m)
        return self._mesh(grid, OCTREE_MIN_CLUSTER, mesh_path, map_path, True)

    @torch.no_grad()
    def recon_bbx_mesh(self, bbx_min_m, bbx_max_m, mc_res_m: float, mesh_path: str | None = None,
                       map_path: str | None = None):
        """utils/mesher.py:253-290 with get_query_from_bbx (:110-150): a dense grid over the padded box, of which only
        the tiles that overlap a node at the coarsest featured level are queried (the others are masked everywhere).
        map_path: also write the SDF map (utils/mesher.py:263-264), every grid point of the queried tiles."""
        grid = self.bbx_grid(bbx_min_m, bbx_max_m, mc_res_m)
        return self._mesh(grid, self.config.min_cluster_vertices, mesh_path, map_path, False)

    @torch.no_grad()
    def save_sdf_map(self, grid: dict, map_path: str, masked_only: bool) -> int:
        """Write the SDF map of `grid` (`octree_grid` / `bbx_grid`) on its own, without a mesh -> number of points."""
        with SdfMapWriter(self, grid, map_path, masked_only) as out:
            out.restart()
            for *_, g in self.chunks(grid):
                out.add(g)
        return out.count

    # ---- grids -------------------------------------------------------------------------------------------------

    def _mask_level(self) -> int:
        return min(self.octree.featured_level_num, self.config.mc_vis_level) - 1       # utils/mesher.py:47

    def octree_grid(self, query_level: int, mc_res_m: float) -> dict:
        dev = self.octree.hier_features[0].device
        nodes = morton_to_points(self.octree._levels[query_level].node_keys.to(dev)).to(torch.int32)
        node_res = 2.0 ** (1 - query_level)
        n = int(np.ceil(node_res / self.world_scale / mc_res_m))
        h = node_res / n
        if nodes.shape[0] == 0:
            lo = hi = [0, 0, 0]
        else:
            lo = (nodes.amin(0).long() * n).tolist()
            hi = ((nodes.amax(0).long() + 1) * n).tolist()
        origin = np.full(3, -1.0 + 0.5 * h)
        return dict(bricks=nodes.contiguous(), n=n, origin_scaled=origin, spacing=h, lo=lo, hi=hi,
                    all_keys=torch.sort(_brick_keys(nodes)).values, voxel_m=h / self.world_scale,
                    origin_m=(origin + h * np.asarray(lo, dtype=np.float64)) / self.world_scale)

    def bbx_grid(self, bbx_min_m, bbx_max_m, mc_res_m: float) -> dict:
        cfg = self.config
        lo_m, hi_m = np.asarray(bbx_min_m, dtype=np.float64), np.asarray(bbx_max_m, dtype=np.float64)
        dims = (np.ceil((hi_m - lo_m) / mc_res_m) + cfg.pad_voxel * 2).astype(np.int64)    # utils/mesher.py:126-130
        origin_m = lo_m - cfg.pad_voxel * mc_res_m
        origin_m[2] -= mc_res_m
        dims[2] += 1
        n = BBX_TILE
        dev = self.octree.hier_features[0].device
        q = self.octree.free_level_num
        nodes = morton_to_points(self.octree._levels[q].node_keys.to(dev)).double()
        node_res = 2.0 ** (1 - q)
        o = torch.tensor(origin_m * self.world_scale, dtype=torch.float64, device=dev)
        s = mc_res_m * self.world_scale
        d = torch.tensor(dims, device=dev)
        # tiles that a node (closed box, widened by one grid step) overlaps; tiles without a node are masked everywhere
        gmin = torch.floor((nodes * node_res - 1.0 - o) / s).long() - 1
        gmax = torch.ceil(((nodes + 1) * node_res - 1.0 - o) / s).long() + 1
        ok = ((gmax >= 0) & (gmin <= d - 1)).all(1)
        tmin = (gmin[ok].clamp(min=0) // n)
        tmax = (torch.minimum(gmax[ok], d - 1) // n)
        if tmin.shape[0]:
            span = int((tmax - tmin).max()) + 1
            r = torch.arange(span, device=dev)
            off = torch.stack(torch.meshgrid(r, r, r, indexing="ij"), -1).reshape(-1, 3)
            cand = tmin[:, None, :] + off[None]
            cand = cand[(cand <= tmax[:, None, :]).all(-1)]
            bricks = torch.unique(cand, dim=0).to(torch.int32)
        else:
            bricks = torch.zeros(0, 3, dtype=torch.int32, device=dev)
        return dict(bricks=bricks.contiguous(), n=n, origin_scaled=origin_m * self.world_scale, spacing=s, lo=[0, 0, 0],
                    hi=dims.tolist(), all_keys=None, voxel_m=mc_res_m, origin_m=origin_m)

    # ---- queries -------------------------------------------------------------------------------------------------

    def _desc(self, grid: dict, bricks, sdf, mask) -> _abi.ShineBrickGrid:
        g = _abi.ShineBrickGrid()
        g.bricks, g.sdf, g.mask = bricks.data_ptr(), sdf.data_ptr(), mask.data_ptr()
        keys = grid["all_keys"]
        g.all_keys, g.num_all = (keys.data_ptr(), keys.numel()) if keys is not None else (None, 0)
        g.num_bricks = bricks.shape[0]
        for a in range(3):
            g.origin[a] = float(np.float32(grid["origin_scaled"][a]))
            g.lo[a], g.hi[a] = int(grid["lo"][a]), int(grid["hi"][a])
        g.spacing = float(np.float32(grid["spacing"]))
        g.n = grid["n"]
        g.missing_sdf = 0.0
        return g

    def chunks(self, grid: dict):
        """-> (bricks, sdf [b, (n+1)^3], mask) per chunk, filled by shine_mesh_grid.  The buffers are reused."""
        n1 = grid["n"] + 1
        per = n1 ** 3
        step = max(1, CHUNK_POINTS // per)
        bricks = grid["bricks"]
        dev = bricks.device
        nb = min(step, bricks.shape[0])
        sdf = torch.empty(nb * per, dtype=torch.float32, device=dev)
        mask = torch.empty(nb * per, dtype=torch.uint8, device=dev)
        od = self.octree._descriptor(None, None)
        dd = self.decoder.c_descriptor(None)
        for s in range(0, bricks.shape[0], step):
            b = bricks[s:s + step]
            g = self._desc(grid, b, sdf, mask)
            _abi.check(_abi.lib().shine_mesh_grid(C.byref(od), C.byref(dd), C.byref(g), self._mask_level(), 0,
                                                  _abi.stream_ptr(dev)), "shine_mesh_grid")
            yield b, sdf[:b.shape[0] * per].view(b.shape[0], per), mask[:b.shape[0] * per].view(b.shape[0], per), g

    @staticmethod
    def edge_capacity(grid: dict) -> int:
        """First size of the edge table: room for about one vertex per cube on two faces of every brick, at load 1/2."""
        return min(MAX_EDGE_SLOTS, _next_pow2(max(1 << 16, 4 * grid["n"] ** 2 * grid["bricks"].shape[0])))

    def marching_cubes(self, grid: dict, sdf_map: "SdfMapWriter | None" = None):
        """-> (verts [V,3] fp32 in grid units relative to grid['lo'], faces [T,3] int32), welded, on the device.
        The edge table is kept at most half full (checked after every chunk); past that, or when an insert finds no free
        slot, the mesh starts over with a table 4x larger.  sdf_map receives every chunk in the same pass (the grid is
        queried once), and starts over with the mesh."""
        dev = grid["bricks"].device
        cap = self.edge_capacity(grid)
        lib, st = _abi.lib(), _abi.stream_ptr(dev)
        while True:
            slots = torch.full((cap * 16,), 0xFF, dtype=torch.uint8, device=dev)
            counters = torch.zeros(4, dtype=torch.int32, device=dev)
            verts = torch.empty(0, 3, dtype=torch.float32, device=dev)
            faces, full = [], False
            if sdf_map is not None:
                sdf_map.restart()
            for _, _, _, g in self.chunks(grid):
                if sdf_map is not None:
                    sdf_map.add(g)
                counters[1:3].zero_()
                _abi.check(lib.shine_marching_cubes(C.byref(g), _abi.ptr(slots), cap, _abi.ptr(counters), None, 0, None, 0,
                                                    st), "shine_marching_cubes")
                nv, nt, _, lost = counters.tolist()                # the chunk's one read-back: output sizes
                if lost or 2 * nv > cap:
                    full = True
                    break
                if nv > verts.shape[0]:
                    grown = torch.empty(max(nv, 2 * verts.shape[0]), 3, dtype=torch.float32, device=dev)
                    grown[:verts.shape[0]] = verts
                    verts = grown
                f = torch.empty(nt, 3, dtype=torch.int32, device=dev)
                _abi.check(lib.shine_marching_cubes(C.byref(g), _abi.ptr(slots), cap, _abi.ptr(counters), _abi.ptr(verts),
                                                    verts.shape[0], _abi.ptr(f), nt, st), "shine_marching_cubes")
                faces.append(f)
            if not full:
                nv = int(counters[0])
                return verts[:nv], (torch.cat(faces) if faces else torch.zeros(0, 3, dtype=torch.int32, device=dev))
            if cap >= MAX_EDGE_SLOTS:
                raise _abi.ShineB200Error(f"the mesh has more than {MAX_EDGE_SLOTS // 2} vertices (edge table limit)")
            cap = min(MAX_EDGE_SLOTS, cap * 4)

    def _mesh(self, grid: dict, min_tris: int, mesh_path, map_path=None, masked_only=False):
        if map_path:
            with SdfMapWriter(self, grid, map_path, masked_only) as out:
                verts, faces = self.marching_cubes(grid, out)
        else:
            verts, faces = self.marching_cubes(grid)
        verts_m = (torch.tensor(grid["origin_m"], dtype=torch.float64, device=verts.device)
                   + verts.double() * grid["voxel_m"])
        normals, keep = normals_and_clusters(verts_m.float(), faces, min_tris)
        verts_m, faces, normals = compact(verts_m, faces, normals, keep)
        T = torch.tensor(self.global_transform, dtype=torch.float64, device=verts.device)     # mesh.transform (:284,:362)
        verts_out = (verts_m @ T[:3, :3].T + T[:3, 3]).float()
        normals = normals.double() @ T[:3, :3].T
        normals = (normals / normals.norm(dim=1, keepdim=True).clamp_min(1e-300)).float()
        if mesh_path:
            write_ply(mesh_path, verts_out, faces, normals)
        return verts_out, faces, normals


_SDF_MAP_HEADER = ("ply\nformat binary_little_endian 1.0\nelement vertex {:012d}\nproperty float x\nproperty float y\n"
                   "property float z\nproperty float intensities\nproperty int labels\nend_header\n")
SDF_MAP_RECORD = np.dtype([("x", "<f4"), ("y", "<f4"), ("z", "<f4"), ("intensities", "<f4"), ("labels", "<i4")])


class SdfMapWriter:
    """`save_map` (utils/mesher.py:152-173 generate_sdf_map): the grid points as a binary little-endian PLY point cloud,
    `intensities` = the SDF in metres (positive in free space, the sign of the reference's sdf_pred), `labels` = the
    marching-cubes mask, positions transformed by the mesher's global_transform.  `shine_mesh_export_points` compacts each
    chunk on the device into the file's records; one device-to-host copy per chunk, appended as it is.  The vertex count is
    a fixed-width header field, patched when the file is closed.  The order of the points is unspecified."""

    def __init__(self, mesher: Mesher, grid: dict, path: str, masked_only: bool):
        self.grid, self.path, self.masked_only = grid, path, bool(masked_only)
        cfg = mesher.config
        self.factor = float(np.float32(cfg.logistic_gaussian_ratio * cfg.sigma_sigmoid_m))     # utils/mesher.py:161
        self.origin = (C.c_double * 3)(*np.asarray(grid["origin_m"], dtype=np.float64))
        self.transform = (C.c_double * 12)(*np.asarray(mesher.global_transform, dtype=np.float64)[:3, :4].reshape(-1))
        self.count, self.fh, self.records = 0, None, None
        self.counter = torch.zeros(1, dtype=torch.int64, device=grid["bricks"].device)

    def __enter__(self):
        os.makedirs(os.path.dirname(os.path.abspath(self.path)), exist_ok=True)
        self.fh = open(self.path, "wb")
        return self

    def restart(self):
        self.fh.seek(0)
        self.fh.truncate()
        self.fh.write(_SDF_MAP_HEADER.format(0).encode("ascii"))
        self.count = 0

    def add(self, g: _abi.ShineBrickGrid):
        owned = g.num_bricks * g.n ** 3
        if self.records is None or self.records.numel() < owned * SDF_MAP_RECORD.itemsize:
            self.records = torch.empty(owned * SDF_MAP_RECORD.itemsize, dtype=torch.uint8, device=self.counter.device)
        self.counter.zero_()
        n = C.c_int64(0)
        _abi.check(_abi.lib().shine_mesh_export_points(
            C.byref(g), self.origin, float(self.grid["voxel_m"]), self.transform, self.factor, int(self.masked_only),
            _abi.ptr(self.records), owned, _abi.ptr(self.counter), C.byref(n), _abi.stream_ptr(self.counter.device)),
            "shine_mesh_export_points")
        self.fh.write(memoryview(self.records[:n.value * SDF_MAP_RECORD.itemsize].cpu().numpy()))
        self.count += n.value

    def __exit__(self, exc_type, exc, tb):
        if exc_type is None:
            self.fh.seek(0)
            self.fh.write(_SDF_MAP_HEADER.format(self.count).encode("ascii"))
        self.fh.close()
        return False


def normals_and_clusters(verts: torch.Tensor, faces: torch.Tensor, min_tris: int):
    """-> (normals [V,3], keep [T] bool): compute_vertex_normals and the cluster filter's triangle mask."""
    dev = verts.device
    nv, nt = verts.shape[0], faces.shape[0]
    cap = _next_pow2(max(16, 6 * nt))
    if cap > MAX_EDGE_SLOTS:
        raise _abi.ShineB200Error(f"{nt} triangles: more than the cluster filter's edge table holds")
    slots = torch.full((cap * 16,), 0xFF, dtype=torch.uint8, device=dev)
    scratch = torch.empty(max(1, 2 * nt), dtype=torch.int32, device=dev)
    keep = torch.empty(max(1, nt), dtype=torch.uint8, device=dev)
    normals = torch.empty(nv, 3, dtype=torch.float32, device=dev)
    _abi.check(_abi.lib().shine_mesh_clusters(_abi.ptr(verts.contiguous()), nv, _abi.ptr(faces.contiguous()), nt,
                                              int(min_tris), _abi.ptr(slots), cap, _abi.ptr(scratch), _abi.ptr(keep),
                                              _abi.ptr(normals), _abi.stream_ptr(dev)), "shine_mesh_clusters")
    return normals, keep[:nt].bool()


def compact(verts, faces, normals, keep):
    """Drop the triangles with keep False and then every vertex no triangle uses (Open3D's remove_triangles_by_mask
    keeps those vertices); vertex ids are renumbered in order."""
    faces = faces[keep]
    used = torch.zeros(verts.shape[0], dtype=torch.bool, device=verts.device)
    used[faces.reshape(-1).long()] = True
    remap = torch.cumsum(used.int(), 0, dtype=torch.int32) - 1
    return verts[used], remap[faces.long()], normals[used]


def reconstruct(config: SHINEConfig, mesher: Mesher, mesh_path: str, map_bbx=None, map_path: str | None = None):
    """The mesh call of the mapping loops (shine_batch.py:240-245, shine_incre.py:203-211): octree or bbx mode as
    `mc_with_octree` selects.  map_bbx: (min, max) metres in the map frame, needed by bbx mode.  map_path: the SDF map file
    of `save_map`, written in the same pass over the grid."""
    if config.mc_with_octree:      # mc_query_level = tree_level_world - tree_level_feat + 1 (utils/config.py:366)
        return mesher.recon_octree_mesh(mesher.octree.free_level_num, config.mc_res_m, mesh_path, map_path)
    if map_bbx is None:
        raise ValueError("mc_with_octree: False meshes the map's bounding box: pass map_bbx")
    return mesher.recon_bbx_mesh(map_bbx[0], map_bbx[1], config.mc_res_m, mesh_path, map_path)


def sdf_map_path(config: SHINEConfig, run_path: str, name: str) -> str | None:
    """RUN/map/sdf_map_{name}.ply (shine_batch.py:240, shine_incre.py:204) when `save_map` is on, else None."""
    return os.path.join(run_path, "map", f"sdf_map_{name}.ply") if config.save_map else None


def surface_bbx(coord: torch.Tensor, weight: torch.Tensor, scale: float, bbx=None):
    """(min, max) metres of the surface samples (weight > 0) of scaled coordinates, merged with `bbx` (None: nothing yet):
    the synthetic map's map_bbx.  A frame without surface samples leaves `bbx` as it is."""
    s = coord[weight > 0].double() / scale
    if s.shape[0] == 0:
        return bbx
    lo, hi = s.amin(0).cpu().numpy(), s.amax(0).cpu().numpy()
    return (lo, hi) if bbx is None else (np.minimum(bbx[0], lo), np.maximum(bbx[1], hi))


# ---- PLY -------------------------------------------------------------------------------------------------------------

_VERTEX = np.dtype([("x", "<f4"), ("y", "<f4"), ("z", "<f4"), ("nx", "<f4"), ("ny", "<f4"), ("nz", "<f4")])
_FACE = np.dtype([("n", "u1"), ("v", "<i4", (3,))])


def write_ply(path: str, verts, faces, normals) -> None:
    """Binary little-endian PLY: float32 x y z nx ny nz per vertex, `uchar int` vertex_indices per face."""
    v = np.asarray(torch.as_tensor(verts).detach().cpu(), dtype=np.float32).reshape(-1, 3)
    nrm = np.asarray(torch.as_tensor(normals).detach().cpu(), dtype=np.float32).reshape(-1, 3)
    f = np.asarray(torch.as_tensor(faces).detach().cpu(), dtype=np.int32).reshape(-1, 3)
    vert = np.empty(v.shape[0], dtype=_VERTEX)
    for i, k in enumerate("xyz"):
        vert[k] = v[:, i]
        vert["n" + k] = nrm[:, i]
    face = np.empty(f.shape[0], dtype=_FACE)
    face["n"] = 3
    face["v"] = f
    header = ("ply\nformat binary_little_endian 1.0\n"
              f"element vertex {v.shape[0]}\nproperty float x\nproperty float y\nproperty float z\n"
              "property float nx\nproperty float ny\nproperty float nz\n"
              f"element face {f.shape[0]}\nproperty list uchar int vertex_indices\nend_header\n")
    os.makedirs(os.path.dirname(os.path.abspath(path)), exist_ok=True)
    with open(path, "wb") as fh:
        fh.write(header.encode("ascii"))
        fh.write(vert.tobytes())
        fh.write(face.tobytes())


def read_point_ply(path: str) -> np.ndarray:
    """The vertex element of a binary little-endian PLY whose first element it is (an SDF map) -> structured array with
    one field per scalar property (`x`, `y`, `z`, `intensities`, `labels`, ...)."""
    from .scans import read_ply_header
    with open(path, "rb") as fh:
        fmt, elements = read_ply_header(fh, path)
        if fmt != "binary_little_endian" or not elements or elements[0][0] != "vertex":
            raise ValueError(f"{path}: expected a binary little-endian PLY that starts with its vertex element")
        _, n, fields = elements[0]
        dt = np.dtype([(name, t) for name, t, _ in fields])
        body = fh.read(n * dt.itemsize)
    if len(body) != n * dt.itemsize:
        raise ValueError(f"{path}: file ends inside the vertex element")
    return np.frombuffer(body, dtype=dt, count=n)


def read_ply(path: str):
    """A triangle mesh PLY, ascii or binary little-endian -> (verts [V,3], faces [T,3] int32, normals [V,3] or None)
    numpy arrays.  Vertex x y z (and nx ny nz, when present) are float or double and keep their type; other scalar
    properties are skipped.  The face element has one list property `vertex_indices` or `vertex_index` of any integer
    count and index types.  Polygons, big-endian files and a missing face element raise ValueError."""
    from .scans import _xyz_layout, read_ply_header
    with open(path, "rb") as fh:
        fmt, elements = read_ply_header(fh, path)
        body = fh.read()
    names = [e[0] for e in elements]
    if "vertex" not in names:
        raise ValueError(f"{path}: no vertex element")
    if "face" not in names:
        raise ValueError(f"{path}: no face element (not a triangle mesh)")
    vertex, face = elements[names.index("vertex")], elements[names.index("face")]
    _xyz_layout(path, vertex[2])
    props = face[2]
    if len(props) != 1 or props[0][2] != 0 or props[0][0] not in ("vertex_indices", "vertex_index"):
        raise ValueError(f"{path}: the face element must hold one list property vertex_indices / vertex_index")
    count_t, index_t = props[0][1] or (None, None)
    if count_t is None or count_t.kind not in "iu" or index_t.kind not in "iu":
        raise ValueError(f"{path}: face indices must be a list of integers")
    # elements before the face element are read; those after it are ignored
    order = names.index("face")
    for name, _, fields in elements[:order]:
        if any(c == 0 for _, _, c in fields):
            raise ValueError(f"{path}: element {name!r} before the faces has a list property")
    if fmt == "ascii":
        tok, pos = body.split(), 0
        arrays = {}
        for name, n, fields in elements[:order + 1]:
            width = len(fields) if name != "face" else 4
            if pos + n * width > len(tok):
                raise ValueError(f"{path}: file ends inside element {name!r}")
            arrays[name] = np.array(tok[pos:pos + n * width], dtype=np.float64).reshape(n, width)
            pos += n * width
        vals = arrays["vertex"]
        col = {nm: i for i, (nm, _, _) in reversed(list(enumerate(vertex[2])))}
        types = {nm: dt for nm, dt, _ in reversed(vertex[2])}
        v = np.stack([vals[:, col[a]].astype(types[a]) for a in "xyz"], 1)
        nrm = (np.stack([vals[:, col[a]].astype(types[a]) for a in ("nx", "ny", "nz")], 1)
               if all(a in col for a in ("nx", "ny", "nz")) else None)
        counts, idx = arrays["face"][:, 0], arrays["face"][:, 1:]
    else:
        off, recs = 0, {}
        for name, n, fields in elements[:order + 1]:
            if name == "face":
                dt = np.dtype([("n", count_t), ("v", index_t, (3,))])
            else:
                dt = np.dtype([(f"p{i}", f[1]) for i, f in enumerate(fields)])
            if off + n * dt.itemsize > len(body):
                raise ValueError(f"{path}: file ends inside element {name!r}")
            recs[name] = (np.frombuffer(body, dtype=dt, count=n, offset=off), fields)
            off += n * dt.itemsize
        vert, fields = recs["vertex"]
        col = {nm: f"p{i}" for i, (nm, _, _) in reversed(list(enumerate(fields)))}
        v = np.stack([vert[col[a]] for a in "xyz"], 1)
        nrm = (np.stack([vert[col[a]] for a in ("nx", "ny", "nz")], 1)
               if all(a in col for a in ("nx", "ny", "nz")) else None)
        counts, idx = recs["face"][0]["n"], recs["face"][0]["v"]
    if counts.shape[0] and not (counts == 3).all():
        raise ValueError(f"{path}: faces that are not triangles (polygons are not supported)")
    idx = np.asarray(idx)
    if idx.shape[0] and (idx.min() < 0 or idx.max() >= v.shape[0]):
        raise ValueError(f"{path}: face indices outside [0, {v.shape[0]})")
    return v, idx.astype(np.int32).reshape(-1, 3), nrm


def main(argv=None):
    """python -m shine_mapping_b200.mesher CONFIG CHECKPOINT --out MESH.ply: mesh a saved map without the scans."""
    import argparse
    from .checkpoint import load_checkpoint
    ap = argparse.ArgumentParser(description="Mesh a saved map (a checkpoint of either mapping loop, or of the reference). "
                                             "The checkpoint is unpickled: load only files you trust.")
    ap.add_argument("config")
    ap.add_argument("checkpoint")
    ap.add_argument("--out", required=True, metavar="MESH.ply")
    ap.add_argument("--mc-res-m", type=float, default=None, help="marching-cubes resolution (default: the config's mc_res_m)")
    ap.add_argument("--bbx", type=float, nargs=6, default=None, metavar=("X0", "Y0", "Z0", "X1", "Y1", "Z1"),
                    help="mesh this box (metres, map frame) in bbx mode instead of the octree's nodes")
    ap.add_argument("--sdf-map", default=None, metavar="MAP.ply", help="also write the SDF map as a point cloud")
    args = ap.parse_args(argv)
    config = SHINEConfig()
    config.load(args.config)
    state, octree = load_checkpoint(args.checkpoint, config, config.device)
    if octree is None or octree.is_empty():
        raise SystemExit(f"{args.checkpoint}: the checkpoint holds a decoder but no map (feature_octree): nothing to mesh")
    decoder = Decoder(config)
    decoder.load_state_dict(state)
    mesher = Mesher(config, octree, decoder)
    res = config.mc_res_m if args.mc_res_m is None else args.mc_res_m
    if args.bbx is not None:
        verts, faces, _ = mesher.recon_bbx_mesh(args.bbx[:3], args.bbx[3:], res, args.out, args.sdf_map)
    else:
        verts, faces, _ = mesher.recon_octree_mesh(octree.free_level_num, res, args.out, args.sdf_map)
    print(f"{args.out}: {verts.shape[0]} vertices, {faces.shape[0]} triangles")


if __name__ == "__main__":
    main()
