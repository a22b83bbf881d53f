"""CPU restatement of the mesher's grid (reference utils/mesher.py recon_octree_mesh / query_points), of the set of
vertices masked marching cubes must produce, and of the mesh post-processing (Open3D's cluster_connected_triangles and
compute_vertex_normals as DESIGN §8 states them), for tests/test_gpu_mesh.py and tests/test_gpu_mesh_oracle.py.
Independent of any triangle table."""
from __future__ import annotations

import numpy as np
import scipy.sparse
import scipy.sparse.csgraph
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


def triangle_clusters(faces, nv: int):
    """Open3D cluster_connected_triangles: two triangles are in one cluster iff a chain of shared undirected edges joins
    them (a shared vertex alone does not).  -> (label [T] int64: each triangle's cluster, sizes [clusters] int64: each
    cluster's triangle count); clusters are numbered in order of their first triangle."""
    f = np.asarray(faces, dtype=np.int64).reshape(-1, 3)
    nt = f.shape[0]
    if nt == 0:
        return np.zeros(0, dtype=np.int64), np.zeros(0, dtype=np.int64)
    e = np.sort(np.concatenate([f[:, [0, 1]], f[:, [1, 2]], f[:, [2, 0]]]), axis=1)
    _, edge_id = np.unique(e[:, 0] * np.int64(nv) + e[:, 1], return_inverse=True)
    tri = np.tile(np.arange(nt), 3)
    # triangle-edge incidence B [T, E]; B B^T joins triangles that share an edge
    B = scipy.sparse.csr_matrix((np.ones(3 * nt, dtype=np.int8), (tri, edge_id.reshape(-1))), shape=(nt, edge_id.max() + 1))
    _, raw = scipy.sparse.csgraph.connected_components(B @ B.T, directed=False)
    _, first, label = np.unique(raw, return_index=True, return_inverse=True)
    order = np.argsort(np.argsort(first))                  # renumber clusters by their first triangle
    label = order[label.reshape(-1)]
    return label.astype(np.int64), np.bincount(label).astype(np.int64)


def vertex_normals(verts64, faces):
    """DESIGN §8's normals in fp64: per vertex the sum of the unit normals of its adjacent non-degenerate triangles,
    normalised; a vertex whose sum is zero (or that no such triangle uses) gets the zero vector."""
    v = np.asarray(verts64, dtype=np.float64).reshape(-1, 3)
    f = np.asarray(faces, dtype=np.int64).reshape(-1, 3)
    out = np.zeros_like(v)
    if f.shape[0]:
        n = np.cross(v[f[:, 1]] - v[f[:, 0]], v[f[:, 2]] - v[f[:, 0]])
        ln = np.linalg.norm(n, axis=1)
        ok = ln > 0
        n = n[ok] / ln[ok, None]
        for k in range(3):
            np.add.at(out, f[ok, k], n)
    ln = np.linalg.norm(out, axis=1)
    nz = ln > 0
    out[nz] /= ln[nz, None]
    out[~nz] = 0.0
    return out


def canonical_mesh(verts, faces):
    """A key of a mesh that does not depend on vertex numbering or triangle order: (sorted vertex positions as fp32 bits,
    sorted triangles as position triples, each rotated to start at its smallest position so that winding is kept).  Two
    meshes with equal keys have the same vertex multiset and the same oriented triangles."""
    v = np.ascontiguousarray(np.asarray(verts, dtype=np.float32).reshape(-1, 3)).view(np.uint32)
    f = np.asarray(faces, dtype=np.int64).reshape(-1, 3)
    vkey = v[np.lexsort(v.T[::-1])]
    if f.shape[0] == 0:
        return vkey.tobytes(), b""
    p = v[f]                                               # [T, 3 corners, 3 coords] uint32 bits
    # the corner whose position (as a bit triple) is smallest starts the triangle
    rank = np.zeros((f.shape[0], 3), dtype=np.int64)
    for a in range(3):
        for b in range(3):
            if a == b:
                continue
            less = (p[:, b, 0] < p[:, a, 0]) | ((p[:, b, 0] == p[:, a, 0]) & ((p[:, b, 1] < p[:, a, 1]) |
                                                ((p[:, b, 1] == p[:, a, 1]) & (p[:, b, 2] < p[:, a, 2]))))
            rank[:, a] += less
    start = np.argmin(rank, axis=1)
    idx = (start[:, None] + np.arange(3)[None]) % 3
    rot = np.take_along_axis(p, idx[:, :, None], axis=1).reshape(-1, 9)
    tkey = rot[np.lexsort(rot.T[::-1])]
    return vkey.tobytes(), tkey.tobytes()


def enclosed_volume_bounds(sdf, mask, hi):
    """On a dense grid sdf [hi] (inside: < 0) with mask [hi]: (volume of the processed cubes whose 8 corners are all
    inside, volume of the processed cubes with at least one inside corner), in cubes.  A cube is processed iff the mask
    is set at its lowest corner (every cube of the array lies inside hi).  The signed volume of the closed, outward-wound
    mesh of masked marching cubes lies between the two."""
    s = np.asarray(sdf)
    hi = tuple(int(h) for h in hi)
    assert s.shape == hi
    inside = s < 0
    c = [inside[dx:hi[0] - 1 + dx, dy:hi[1] - 1 + dy, dz:hi[2] - 1 + dz]
         for dx in (0, 1) for dy in (0, 1) for dz in (0, 1)]
    proc = np.asarray(mask, dtype=bool)[:-1, :-1, :-1]
    all_in = np.logical_and.reduce(c) & proc
    any_in = np.logical_or.reduce(c) & proc
    return float(all_in.sum()), float(any_in.sum())
