"""CPU restatement of the mesher's grid (reference utils/mesher.py recon_octree_mesh / query_points) and of the set of
vertices masked marching cubes must produce, for tests/test_gpu_mesh.py.  Independent of any triangle table."""
from __future__ import annotations

import numpy as np
import torch

from oracle import shine_oracle as orc


def octree_grid_rule(o: "orc.OracleOctree", query_level: int, scale: float, mc_res_m: float):
    """-> (node points [N,3] int, n, h): the level-q nodes, points per node side and grid spacing of recon_octree_mesh."""
    nodes = orc.morton_to_points(np.array(sorted(o.nodes_lookup_tables[query_level].keys()), dtype=np.int64))
    node_res = 2.0 ** (1 - query_level)
    n = int(np.ceil(node_res / scale / mc_res_m))
    return nodes.astype(np.int64), n, node_res / n


def bbx_grid_rule(bbx_min_m, bbx_max_m, voxel_size: float, pad_voxel: int):
    """get_query_from_bbx (utils/mesher.py:122-130) -> (voxel_num_xyz [3] int, voxel_origin [3] metres): the box padded by
    pad_voxel voxels on every side and by one more voxel below in z."""
    min_bound, max_bound = np.asarray(bbx_min_m, dtype=np.float64), np.asarray(bbx_max_m, dtype=np.float64)
    voxel_num_xyz = (np.ceil((max_bound - min_bound) / voxel_size) + pad_voxel * 2).astype(np.int64)
    voxel_origin = min_bound - pad_voxel * voxel_size
    voxel_origin[2] -= voxel_size
    voxel_num_xyz[2] += 1
    return voxel_num_xyz, voxel_origin


def dense_indices(dims) -> np.ndarray:
    """Every grid index of a dense [dims] grid, x-major like the reference's meshgrid(indexing='ij') -> [N,3]."""
    return np.stack(np.meshgrid(*[np.arange(int(d)) for d in dims], indexing="ij"), -1).reshape(-1, 3)


def grid_coords(G: np.ndarray, origin: float, h: float) -> np.ndarray:
    """Coordinates of grid indices G as the kernel forms them: fp32 origin + fp32 h * G, each rounded once (origin a
    scalar or one value per axis).  The reference forms bbx points as ((G * voxel) + origin) * scale in fp32; the two
    differ in the last bits only."""
    o = np.asarray(origin, dtype=np.float32)
    return (o + (np.float32(h) * G.astype(np.float32)).astype(np.float32)).astype(np.float32)


def query(o: "orc.OracleOctree", dec: dict, coord: np.ndarray, check_level: int):
    """query_points: sdf = -Decoder.sdf(query_feature(p)), mask = all(hierarchical_indices[check_level] >= 0)."""
    with torch.no_grad():
        c = torch.from_numpy(coord)
        sdf = -orc.decoder_sdf(o.query_feature(c), dec)
        mask = (o.hierarchical_indices[check_level] >= 0).all(1)
    return sdf.numpy(), mask.numpy()


def crossing_vertices(sdf: dict, mask: dict, hi):
    """Vertices of masked marching cubes on a sparse grid {G (tuple): value}: the cube at lowest corner G is processed
    iff mask[G] and G + 1 < hi; every edge of a processed cube with one corner < 0 and the other >= 0 has the vertex
    G0 + t e_a, t = v0 / (v0 - v1) (fp32).  A point missing from the dicts has sdf 0.  -> {(G0, axis): position}."""
    out = {}
    for g, m in mask.items():
        if not m or any(g[a] + 1 >= hi[a] for a in range(3)):
            continue
        for dx in (0, 1):
            for dy in (0, 1):
                for dz in (0, 1):
                    c0 = (g[0] + dx, g[1] + dy, g[2] + dz)
                    for a in range(3):
                        if (dx, dy, dz)[a]:
                            continue
                        c1 = list(c0); c1[a] += 1; c1 = tuple(c1)
                        v0, v1 = np.float32(sdf.get(c0, 0.0)), np.float32(sdf.get(c1, 0.0))
                        if (v0 < 0) == (v1 < 0):
                            continue
                        t = np.float32(v0 / np.float32(v0 - v1))
                        p = np.array(c0, dtype=np.float32)
                        p[a] = np.float32(p[a] + t)
                        out[(c0, a)] = p
    return out
