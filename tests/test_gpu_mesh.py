"""The mesher (shine_mapping_b200/mesher.py, csrc/shine_mesh.cu): the block-sparse grid against a CPU restatement of the
reference's grid, masked marching cubes against the crossing points it must produce (whatever the triangle table),
analytic fields injected straight into the brick buffers, the cluster filter, and both mapping loops writing PLYs."""
import ctypes as C
import itertools
import math
import os
from collections import Counter

import numpy as np
import pytest
import torch

from tests import mesh_oracle as mo
from tests.parity_utils import build_cuda_models, make_case, oracle_from_case

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


@pytest.fixture(scope="module", autouse=True)
def _lib(built_lib):
    assert torch.cuda.is_available()
    return built_lib


def _mc(bricks, sdf, mask, n, hi, lo=(0, 0, 0), cap=1 << 16):
    """shine_marching_cubes over one chunk given as tensors -> (verts [V,3] grid units relative to lo, faces [T,3])."""
    from shine_mapping_b200 import _abi
    g = _abi.ShineBrickGrid()
    g.bricks, g.sdf, g.mask = bricks.data_ptr(), sdf.data_ptr(), mask.data_ptr()
    g.all_keys, g.num_all, g.num_bricks, g.n = None, 0, bricks.shape[0], n
    for a in range(3):
        g.lo[a], g.hi[a] = lo[a], hi[a]
    lib, st = _abi.lib(), _abi.stream_ptr(DEV)
    slots = torch.full((cap * 16,), 0xFF, dtype=torch.uint8, device=DEV)
    counters = torch.zeros(4, dtype=torch.int32, device=DEV)
    _abi.check(lib.shine_marching_cubes(C.byref(g), _abi.ptr(slots), cap, _abi.ptr(counters), None, 0, None, 0, st), "count")
    nv, nt, _, lost = counters.tolist()
    assert lost == 0
    verts = torch.empty(nv, 3, dtype=torch.float32, device=DEV)
    faces = torch.empty(nt, 3, dtype=torch.int32, device=DEV)
    _abi.check(lib.shine_marching_cubes(C.byref(g), _abi.ptr(slots), cap, _abi.ptr(counters), _abi.ptr(verts), nv,
                                        _abi.ptr(faces), nt, st), "emit")
    assert int(counters[2]) == nt
    return verts, faces


def _field(fn, nb=4, n=8, mask_fn=None):
    """Bricks [0, nb)^3 of n^3 cubes with sdf = fn(G) at every stored point (grid index G, float64)."""
    r = torch.arange(nb, device=DEV)
    bricks = torch.stack(torch.meshgrid(r, r, r, indexing="ij"), -1).reshape(-1, 3).to(torch.int32).contiguous()
    l = torch.arange(n + 1, device=DEV)
    loc = torch.stack(torch.meshgrid(l, l, l, indexing="ij"), -1).reshape(-1, 3)
    G = (bricks.long()[:, None, :] * n + loc[None]).double()
    sdf = fn(G).float().reshape(-1).contiguous()
    mask = (mask_fn(G) if mask_fn else torch.ones_like(G[..., 0], dtype=torch.bool)).to(torch.uint8).reshape(-1).contiguous()
    return bricks, sdf, mask, [nb * n] * 3


def _topology(faces):
    f = faces.cpu().numpy().astype(np.int64)
    e = np.sort(np.concatenate([f[:, [0, 1]], f[:, [1, 2]], f[:, [2, 0]]]), axis=1)
    _, counts = np.unique(e, axis=0, return_counts=True)
    nv = len(np.unique(f))
    return nv, len(counts), len(f), counts


def _signed_volume(verts, faces):
    v = verts.double().cpu().numpy()[faces.cpu().numpy().astype(np.int64)]
    return float(np.einsum("ij,ij->i", v[:, 0], np.cross(v[:, 1], v[:, 2])).sum() / 6.0)


def _mesher_for(cfg, octree, dec):
    from shine_mapping_b200 import Mesher
    return Mesher(cfg, octree, dec)


# ---- grid against the reference semantics ----------------------------------------------------------------------------

@pytest.mark.parametrize("levels,poly", [(2, True), (2, False), (3, True), (3, False)])
def test_octree_grid_matches_oracle(levels, poly):
    case = make_case(n_points=1500, n_batch=16, feat_levels=levels, seed=60 + levels, poly=poly)
    cfg, octree, dec = build_cuda_models(case, DEV)
    o, odec = oracle_from_case(case)
    q = cfg.tree_level_world - cfg.tree_level_feat + 1          # mc_query_level, derived (utils/config.py:366)
    mesher = _mesher_for(cfg, octree, dec)
    grid = mesher.octree_grid(q, 0.1)
    nodes, n, h = mo.octree_grid_rule(o, q, cfg.scale, 0.1)
    assert grid["n"] == n and abs(grid["spacing"] - h) == 0 and nodes.shape[0] > 24
    assert sorted(map(tuple, grid["bricks"].cpu().numpy().tolist())) == sorted(map(tuple, nodes.tolist()))
    # a sample of bricks, chosen so that some of their +1 faces lie in bricks that do not exist
    rng = np.random.default_rng(levels)
    pick = torch.from_numpy(rng.choice(grid["bricks"].shape[0], size=min(24, grid["bricks"].shape[0]), replace=False)).to(DEV)
    sub = dict(grid, bricks=grid["bricks"][pick].contiguous())
    keyset = set(map(tuple, nodes.tolist()))
    check = min(levels, cfg.mc_vis_level) - 1
    chunks = 0
    for bricks, sdf, mask, _ in mesher.chunks(sub):
        chunks += 1
        b = bricks.cpu().numpy().astype(np.int64)
        l = np.arange(n + 1)
        loc = np.stack(np.meshgrid(l, l, l, indexing="ij"), -1).reshape(-1, 3)
        G = (b[:, None, :] * n + loc[None]).reshape(-1, 3)
        coord = mo.grid_coords(G, grid["origin_scaled"][0], h)
        want_sdf, want_mask = mo.query(o, odec, coord, check)
        # +1 face points in a brick that is not a node: the reference's zero-initialised global grid
        owner = G // n
        missing = np.array([tuple(x) not in keyset for x in owner.tolist()])
        want_sdf[missing], want_mask[missing] = 0.0, False
        got_sdf, got_mask = sdf.cpu().numpy().reshape(-1), mask.cpu().numpy().reshape(-1).astype(bool)
        assert np.array_equal(got_mask, want_mask)
        assert np.abs(got_sdf - want_sdf).max() <= 2e-5
        assert missing.any() and np.all(got_sdf[missing] == 0) and not got_mask[missing].any()
        # the same chunk through marching cubes: its vertices are exactly the crossing points of processed cubes
        verts, faces = _mc(bricks, sdf, mask, n, [grid["hi"][a] for a in range(3)])
        sdf_d = {tuple(g): v for g, v in zip(G.tolist(), got_sdf.tolist())}
        own = np.tile((loc < n).all(1), b.shape[0])            # the chunk's own cubes, not its +1 faces
        mask_d = {tuple(g): m for g, m, w in zip(G.tolist(), got_mask.tolist(), own.tolist()) if w}
        want = mo.crossing_vertices(sdf_d, mask_d, grid["hi"])
        got = verts.cpu().numpy()       # lo = 0 here: grid units are grid indices
        # vertices matched through their edges: both sides compute t = v0 / (v0 - v1) and G0 + t in fp32, so an edge's
        # vertex has the same bits on both; edges that end on the same zero corner share a position, hence a multiset
        assert Counter(map(_bits, got)) == Counter(map(_bits, want.values()))
        # every triangle lies in one processed cube (lowest corner masked in, inside hi)
        for tri in got[faces.cpu().numpy().astype(np.int64)]:
            cands = itertools.product(*[{int(np.floor(tri[:, a].min())), int(np.ceil(tri[:, a].max())) - 1} for a in range(3)])
            assert any(mask_d.get(c, False) and all(c[a] + 1 < grid["hi"][a] and tri[:, a].min() >= c[a]
                                                    and tri[:, a].max() <= c[a] + 1 for a in range(3)) for c in cands)
    assert chunks == 1


def _bits(p):
    return np.asarray(p, dtype=np.float32).tobytes()


@pytest.mark.parametrize("levels,poly", [(2, True), (2, False), (3, True), (3, False)])
def test_bbx_grid_matches_oracle(levels, poly):
    """recon_bbx_mesh's grid: get_query_from_bbx's dense padded box (restated in numpy) against the GPU's 16^3 tiles
    scattered into it.  Queried points match the oracle (mask exact, sdf within 2e-5); every point of a tile that was not
    queried has mask false in the oracle, so skipping it is exact."""
    case = make_case(n_points=1500, n_batch=16, feat_levels=levels, seed=70 + levels, poly=poly)
    cfg, octree, dec = build_cuda_models(case, DEV)
    o, odec = oracle_from_case(case)
    mesher = _mesher_for(cfg, octree, dec)
    surf = np.concatenate(case["frames"]) / cfg.scale
    # a part of the map around a surface point, reaching 6 m above the scene: the top tiles hold no node
    centre = surf[len(surf) // 2]
    lo_m, hi_m = np.maximum(surf.min(0), centre - 4.5), np.minimum(surf.max(0), centre + 4.5)
    hi_m[2] = surf[:, 2].max() + 6.0
    res = 0.2
    grid = mesher.bbx_grid(lo_m, hi_m, res)
    dims, origin_m = mo.bbx_grid_rule(lo_m, hi_m, res, cfg.pad_voxel)
    assert grid["hi"] == dims.tolist() and np.array_equal(grid["origin_m"], origin_m) and grid["lo"] == [0, 0, 0]
    G = mo.dense_indices(dims)
    coord = mo.grid_coords(G, np.float32(origin_m * cfg.scale), np.float32(res * cfg.scale))
    want_sdf, want_mask = mo.query(o, odec, coord, min(levels, cfg.mc_vis_level) - 1)
    assert want_mask.any() and not want_mask.all()
    got_sdf = np.full(int(np.prod(dims)), np.nan, dtype=np.float32)
    got_mask = np.zeros(int(np.prod(dims)), dtype=bool)
    n = grid["n"]
    l = np.arange(n + 1)
    loc = np.stack(np.meshgrid(l, l, l, indexing="ij"), -1).reshape(-1, 3)
    for bricks, sdf, mask, _ in mesher.chunks(grid):
        Gb = (bricks.cpu().numpy().astype(np.int64)[:, None, :] * n + loc[None]).reshape(-1, 3)
        inside = (Gb < dims).all(1)
        flat = np.ravel_multi_index(Gb[inside].T, dims)
        got_sdf[flat] = sdf.cpu().numpy().reshape(-1)[inside]
        got_mask[flat] = mask.cpu().numpy().reshape(-1)[inside].astype(bool)
    queried = ~np.isnan(got_sdf)
    assert queried.any() and not queried.all()
    assert np.array_equal(got_mask[queried], want_mask[queried])
    assert np.abs(got_sdf[queried] - want_sdf[queried]).max() <= 2e-5
    assert not want_mask[~queried].any() and not got_mask[~queried].any()


# ---- analytic fields -------------------------------------------------------------------------------------------------

# radii avoid grid points exactly on the surface: a zero corner makes coincident vertices, whose triangles are dropped
def test_sphere_is_closed_outward_and_accurate():
    c, r = 16.0, 10.3
    bricks, sdf, mask, hi = _field(lambda G: (G - c).norm(dim=-1) - r)
    verts, faces = _mc(bricks, sdf, mask, 8, hi)
    nv, ne, nf, counts = _topology(faces)
    assert (counts == 2).all() and nv == verts.shape[0]
    assert nv - ne + nf == 2
    vol = _signed_volume(verts - c, faces)
    assert abs(vol / (4.0 / 3.0 * math.pi * r ** 3) - 1.0) < 0.01
    from shine_mapping_b200.mesher import normals_and_clusters
    normals, keep = normals_and_clusters(verts, faces, 1)
    grad = torch.nn.functional.normalize(verts.double() - c, dim=1)
    cos = (normals.double() * grad).sum(1)
    assert bool(keep.all()) and float(cos.min()) >= math.cos(math.radians(5.0))


def test_torus_has_euler_characteristic_zero():
    R, r, c = 10.2, 4.3, 16.0
    def torus(G):
        x, y, z = (G - c).unbind(-1)
        return torch.sqrt((torch.sqrt(x * x + y * y) - R) ** 2 + z * z) - r
    verts, faces = _mc(*_field(torus)[:3], 8, _field(torus)[3])
    nv, ne, nf, counts = _topology(faces)
    assert (counts == 2).all() and nv - ne + nf == 0


def test_plane_across_brick_faces_is_welded():
    bricks, sdf, mask, hi = _field(lambda G: G[..., 0] + 0.5 * G[..., 1] - 13.3)
    verts, faces = _mc(bricks, sdf, mask, 8, hi)
    v = verts.double().cpu().numpy()
    assert np.abs(v[:, 0] + 0.5 * v[:, 1] - 13.3).max() < 1e-4                   # on the plane
    assert len(np.unique(v, axis=0)) == len(v)                                   # no vertex twice
    assert len(np.unique(faces.cpu().numpy())) == len(v)
    nv, ne, nf, counts = _topology(faces)
    assert set(counts.tolist()) <= {1, 2} and nv - ne + nf == 1                  # one open sheet, no cracks


def test_mask_cut_follows_the_lowest_corner_rule():
    c, r, cut = 16.0, 10.3, 16
    bricks, sdf, mask, hi = _field(lambda G: (G - c).norm(dim=-1) - r, mask_fn=lambda G: G[..., 2] < cut)
    verts, faces = _mc(bricks, sdf, mask, 8, hi)
    v = verts.cpu().numpy()
    assert v[:, 2].max() <= cut + 1e-6 and v[:, 2].max() > cut - 0.5   # cubes with lowest z <= cut - 1 reach z = cut
    nv, ne, nf, counts = _topology(faces)
    assert (counts == 1).any() and set(counts.tolist()) <= {1, 2}


def test_cluster_filter_keeps_the_large_component_only():
    from shine_mapping_b200.mesher import compact, normals_and_clusters
    big, small = (14.0, 14.0, 14.0, 9.3), (27.0, 27.0, 27.0, 1.6)
    f = lambda G: torch.minimum((G - torch.tensor(big[:3], device=DEV, dtype=G.dtype)).norm(dim=-1) - big[3],
                                (G - torch.tensor(small[:3], device=DEV, dtype=G.dtype)).norm(dim=-1) - small[3])
    bricks, sdf, mask, hi = _field(f)
    verts, faces = _mc(bricks, sdf, mask, 8, hi)
    normals, keep = normals_and_clusters(verts, faces, 200)
    v, fk, nk = compact(verts, faces, normals, keep)
    assert 0 < fk.shape[0] < faces.shape[0]
    d = (v.double() - torch.tensor(big[:3], device=DEV, dtype=torch.float64)).norm(dim=1)
    assert float((d - big[3]).abs().max()) < 1.0
    assert len(torch.unique(fk)) == v.shape[0]                                   # no unreferenced vertex


# ---- the loops -------------------------------------------------------------------------------------------------------

def _street_config(**kw):
    from shine_mapping_b200.config import SHINEConfig
    base = dict(tree_level_world=12, tree_level_feat=3, leaf_vox_size=0.3, device=DEV, bs=8192, iters=400,
                vis_freq_iters=200, mc_res_m=0.15, surface_sample_range_m=0.3, free_sample_end_dist_m=1.0,
                min_range=2.0, pc_radius=25.0)
    base.update(kw)
    return SHINEConfig(**base)


@pytest.mark.parametrize("octree_mode", [True, False])
def test_batch_loop_writes_meshes(tmp_path, octree_mode):
    from shine_mapping_b200 import Decoder, FeatureOctree, Mesher, sdf_infer, synth
    from shine_mapping_b200.batch_loop import run_shine_mapping_batch
    from shine_mapping_b200.mesher import read_ply, reconstruct
    torch.manual_seed(0)
    cfg = _street_config(mc_with_octree=octree_mode)
    octree, dec = FeatureOctree(cfg), Decoder(cfg)
    pool = synth.build_scene_map(cfg, octree, 512, 20, frame_step_m=1.0, seed=3)
    out = run_shine_mapping_batch(cfg, octree, dec, pool, run_path=str(tmp_path), map_bbx=pool.map_bbx)
    assert [os.path.basename(p) for p in out["meshes"]] == ["mesh_iter_200.ply", "mesh_iter_400.ply"]
    v, f, nrm = read_ply(out["meshes"][-1])
    m = Mesher(cfg, octree, dec)
    grid = m.octree_grid(octree.free_level_num, cfg.mc_res_m) if octree_mode else m.bbx_grid(*pool.map_bbx, cfg.mc_res_m)
    raw_v, raw_f = m.marching_cubes(grid)
    print("bricks", grid["bricks"].shape[0], "n", grid["n"], "raw", raw_v.shape[0], raw_f.shape[0], "written", len(v), len(f),
          "loss", out["loss_first"], out["loss_last"])
    verts, faces, normals = reconstruct(cfg, Mesher(cfg, octree, dec), str(tmp_path / "again.ply"), pool.map_bbx)
    assert f.shape[0] > 100 and v.shape == tuple(verts.shape) and f.shape == tuple(faces.shape)
    order = lambda a: a[np.lexsort(a.T[::-1])]
    assert np.array_equal(order(v), order(verts.cpu().numpy()))
    assert np.allclose(np.linalg.norm(nrm, axis=1), 1.0, atol=1e-5)
    # the trained SDF is zero between an edge's two corners: at the vertex it is within a voxel of zero, except on edges
    # that cross the boundary of a node whose neighbour is missing, where the features (and the field) jump; those are few
    pred = sdf_infer(octree, dec, verts * cfg.scale) * cfg.sigma_sigmoid      # the decoder predicts sdf / sigma
    near = float((pred.abs() <= cfg.mc_res_m * cfg.scale).float().mean())
    print("vertices within mc_res_m of the zero level:", near)
    assert near >= 0.95


def test_incremental_loop_meshes_every_mesh_freq_frame(tmp_path):
    from shine_mapping_b200 import Decoder, FeatureOctree, synth
    from shine_mapping_b200.incre_loop import run_shine_mapping_incremental
    from shine_mapping_b200.mesher import read_ply
    torch.manual_seed(0)
    cfg = _street_config(iters=20, mesh_freq_frame=2, continual_learning_reg=True)
    octree, dec = FeatureOctree(cfg), Decoder(cfg)
    scans = synth.generate_scans(cfg, 512, 5, 1.0, seed=4, device=DEV)
    frames = [(c, l, w) for c, l, w, _ in scans]
    hist = run_shine_mapping_incremental(cfg, octree, dec, frames, run_path=str(tmp_path))
    written = [h["frame"] for h in hist if "mesh" in h]
    assert written == [0, 1, 3]
    for h in hist:
        if "mesh" in h:
            assert os.path.basename(h["mesh"]) == f"mesh_frame_{h['frame'] + 1}.ply"
            read_ply(h["mesh"])
