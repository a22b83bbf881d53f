"""The mesher's kernels graded against exact oracles (tests/mesh_oracle.py):
  A. `shine_mesh_grid` on every decoder-kernel instantiation (1 to 8 levels), poly and linear interpolation, with and
     without decoder biases, every mask level and brick sizes n = 1 .. 64, against the CPU oracle's query;
  B. the mesh does not depend on how the bricks are cut into chunks or on edge-table restarts;
  C. the triangle table through `shine_marching_cubes` on random fields: every cube configuration, a closed oriented
     surface whose volume lies between the grid's inner and outer cube counts;
  D. the cluster filter of `shine_mesh_clusters` against an exact edge-connected partition;
  E. the vertex normals against fp64, at the ABI and through the mesher at large map offsets.
Every test prints its worst deviation."""
import ctypes as C

import numpy as np
import pytest
import torch

from tests import mesh_oracle as mo
from tests.parity_utils import build_cuda_models, make_case, oracle_from_case

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
ANG = 0.3
TRANSFORM = np.array([[np.cos(ANG), -np.sin(ANG), 0, 1.5], [np.sin(ANG), np.cos(ANG), 0, -2.25], [0, 0, 1, 0.125],
                      [0, 0, 0, 1]])


@pytest.fixture(scope="module", autouse=True)
def _lib(built_lib):
    assert torch.cuda.is_available()
    return built_lib


def _angle(a, b):
    a, b = np.asarray(a, dtype=np.float64), np.asarray(b, dtype=np.float64)
    return np.arctan2(np.linalg.norm(np.cross(a, b), axis=1), (a * b).sum(1))


def _brick_grid(bricks, sdf, mask, n, origin=0.0, spacing=1.0, all_keys=None, lo=(0, 0, 0), hi=(1 << 20,) * 3,
                missing=0.0):
    from shine_mapping_b200 import _abi
    g = _abi.ShineBrickGrid()
    g.bricks, g.sdf, g.mask = [None if t is None else t.data_ptr() for t in (bricks, sdf, mask)]
    g.all_keys, g.num_all = (all_keys.data_ptr(), all_keys.numel()) if all_keys is not None else (None, 0)
    g.num_bricks = 0 if bricks is None else bricks.shape[0]
    g.n, g.spacing, g.missing_sdf = n, float(np.float32(spacing)), missing
    for a in range(3):
        g.origin[a] = float(np.float32(origin))
        g.lo[a], g.hi[a] = lo[a], hi[a]
    return g


def _local(n):
    l = np.arange(n + 1)
    return np.stack(np.meshgrid(l, l, l, indexing="ij"), -1).reshape(-1, 3)


# ---- A. the grid query -------------------------------------------------------------------------------------------------

def _oracle_levels(o, dec, coord):
    """-> (sdf, [mask at check level k for every level k]) of the oracle's query_points."""
    sdf, _ = mo.query(o, dec, coord, 0)
    return sdf, [(h >= 0).all(1).numpy() for h in o.hierarchical_indices]


GRID_SIZES = [(1, 64), (2, 48), (7, 12), (16, 4)]         # (n, bricks of the chunk)


@pytest.mark.parametrize("levels", [1, 3, 4, 5, 8])
@pytest.mark.parametrize("poly,bias", [(True, True), (False, False), (True, False), (False, True)])
def test_grid_query_matches_oracle(levels, poly, bias):
    from shine_mapping_b200 import _abi
    from shine_mapping_b200.feature_octree import morton_to_points
    from shine_mapping_b200.mesher import _brick_keys
    case = make_case(n_points=1500, n_batch=16, feat_levels=levels, seed=400 + 10 * levels + 2 * poly + bias, poly=poly,
                     bias=bias)
    cfg, octree, dec = build_cuda_models(case, DEV)
    o, odec = oracle_from_case(case)
    q = cfg.tree_level_world - cfg.tree_level_feat + 1
    nodes = morton_to_points(octree._levels[q].node_keys.to(DEV)).to(torch.int32)
    all_keys = torch.sort(_brick_keys(nodes)).values
    keyset = set(map(tuple, nodes.cpu().numpy().tolist()))
    node_res = 2.0 ** (1 - q)
    od, dd = octree._descriptor(None, None), dec.c_descriptor(None)
    lib, st = _abi.lib(), _abi.stream_ptr(DEV)
    rng = np.random.default_rng(levels)
    sizes = GRID_SIZES + ([(64, 1)] if poly == bias else [])
    worst, halo_elsewhere, halo_missing, shared = 0.0, 0, 0, 0
    for n, nb in sizes:
        # a compact set of bricks around a random node: many share faces, some neighbours are in the map but not here
        P = nodes.cpu().numpy().astype(np.int64)
        centre = P[rng.integers(P.shape[0])]
        pick = np.argsort(np.abs(P - centre).max(1), kind="stable")[:min(nb, P.shape[0])]
        bricks = torch.from_numpy(P[pick].astype(np.int32)).to(DEV).contiguous()
        h = node_res / n
        per = (n + 1) ** 3
        sdf = torch.full((bricks.shape[0] * per,), np.nan, dtype=torch.float32, device=DEV)
        mask = torch.full((bricks.shape[0] * per,), 7, dtype=torch.uint8, device=DEV)
        g = _brick_grid(bricks, sdf, mask, n, -1.0 + 0.5 * h, h, all_keys, missing=1234.5)
        G = (P[pick][:, None, :] * n + _local(n)[None]).reshape(-1, 3)
        want_sdf, want_masks = _oracle_levels(o, odec, mo.grid_coords(G, np.float32(-1.0 + 0.5 * h), h))
        owner = G // n
        missing = np.array([tuple(x) not in keyset for x in owner.tolist()])
        mine = set(map(tuple, P[pick].tolist()))
        halo_elsewhere += int(np.array([tuple(x) in keyset and tuple(x) not in mine for x in owner.tolist()]).sum())
        halo_missing += int(missing.sum())
        first = None
        for level in range(levels):
            _abi.check(lib.shine_mesh_grid(C.byref(od), C.byref(dd), C.byref(g), level, 0, st), "shine_mesh_grid")
            got_sdf = sdf.cpu().numpy()
            got_mask = mask.cpu().numpy()
            assert set(np.unique(got_mask).tolist()) <= {0, 1}
            want_mask = want_masks[level] & ~missing
            assert np.array_equal(got_mask.astype(bool), want_mask), (n, level)
            if first is None:
                first = got_sdf.copy()
            assert np.array_equal(got_sdf.view(np.uint32), first.view(np.uint32))   # the mask level leaves sdf alone
        assert np.all(first[missing] == np.float32(1234.5))
        d = np.abs(first[~missing].astype(np.float64) - want_sdf[~missing])
        worst = max(worst, float(d.max()))
        assert d.max() <= 2e-5, (n, float(d.max()))
        # copies of one grid point in several bricks of the chunk: the same bits
        flat = np.ravel_multi_index((G + 1).T, (P.max() * n + n + 3,) * 3)
        _, first_copy, inv = np.unique(flat, return_index=True, return_inverse=True)
        inv = inv.reshape(-1)
        shared += int(flat.shape[0] - first_copy.shape[0])
        assert np.array_equal(first.view(np.uint32), first.view(np.uint32)[first_copy][inv])
        assert np.array_equal(got_mask, got_mask[first_copy][inv])
    print(f"levels {levels} poly {poly} bias {bias}: max|dsdf| {worst:.2e}, halo points queried in other chunks "
          f"{halo_elsewhere}, zeroed {halo_missing}, shared copies {shared}")
    assert halo_elsewhere > 0 and halo_missing > 0 and shared > 0


def test_grid_refuses_n_above_64_and_ignores_zero_bricks():
    from shine_mapping_b200 import Mesher, _abi
    case = make_case(n_points=1500, n_batch=16, feat_levels=2, seed=450)
    cfg, octree, dec = build_cuda_models(case, DEV)
    od, dd = octree._descriptor(None, None), dec.c_descriptor(None)
    lib, st = _abi.lib(), _abi.stream_ptr(DEV)
    bricks = torch.zeros(1, 3, dtype=torch.int32, device=DEV)
    sdf = torch.full((66 ** 3,), 5.0, dtype=torch.float32, device=DEV)
    mask = torch.full((66 ** 3,), 3, dtype=torch.uint8, device=DEV)
    assert lib.shine_mesh_grid(C.byref(od), C.byref(dd), C.byref(_brick_grid(bricks, sdf, mask, 65)), 0, 0, st) == -1
    assert lib.shine_mesh_grid(C.byref(od), C.byref(dd), C.byref(_brick_grid(bricks, sdf, mask, 0)), 0, 0, st) == -1
    # zero bricks: nothing is written, with or without buffers
    empty = bricks[:0]
    assert lib.shine_mesh_grid(C.byref(od), C.byref(dd), C.byref(_brick_grid(empty, sdf, mask, 8)), 0, 0, st) == 0
    assert lib.shine_mesh_grid(C.byref(od), C.byref(dd), C.byref(_brick_grid(None, None, None, 8)), 0, 0, st) == 0
    torch.cuda.synchronize()
    assert bool((sdf == 5.0).all()) and bool((mask == 3).all())
    m = Mesher(cfg, octree, dec)
    grid = m.octree_grid(octree.free_level_num, 0.1)
    with pytest.raises(_abi.ShineB200Error, match="invalid argument"):
        list(m.chunks(dict(grid, n=65)))
    with pytest.raises(_abi.ShineB200Error, match="invalid argument"):
        m.marching_cubes(dict(grid, n=65))
    none = dict(grid, bricks=grid["bricks"][:0])
    v, f = m.marching_cubes(none)
    assert v.shape == (0, 3) and f.shape == (0, 3)
    v, f, nrm = m._mesh(none, 1, None)
    assert v.shape == (0, 3) and f.shape == (0, 3) and nrm.shape == (0, 3)
    print("n = 65 and n = 0 refused; zero bricks wrote nothing")


# ---- maps for B, D and E -----------------------------------------------------------------------------------------------

@pytest.fixture(scope="module")
def street():
    """A street map trained 300 iterations by the batch loop (6 frames)."""
    from shine_mapping_b200 import Decoder, FeatureOctree, synth
    from shine_mapping_b200.batch_loop import run_shine_mapping_batch
    from shine_mapping_b200.config import SHINEConfig
    torch.manual_seed(0)
    cfg = SHINEConfig(tree_level_world=12, tree_level_feat=3, leaf_vox_size=0.3, device=DEV, bs=8192, iters=300,
                      vis_freq_iters=1000, mc_res_m=0.15, surface_sample_range_m=0.3, free_sample_end_dist_m=1.0,
                      min_range=2.0, pc_radius=25.0)
    octree, dec = FeatureOctree(cfg), Decoder(cfg)
    pool = synth.build_scene_map(cfg, octree, 512, 6, frame_step_m=1.0, seed=3)
    run_shine_mapping_batch(cfg, octree, dec, pool)
    return cfg, octree, dec, pool.map_bbx


@pytest.fixture(scope="module")
def random_map():
    """A map of random features (make_case): its zero level set falls apart into many small components.  The decoder's
    output bias is moved so that the field changes sign among the surface points (a random decoder is of one sign
    there, and bbx mode would have no surface)."""
    from shine_mapping_b200 import sdf_infer
    case = make_case(n_points=1500, n_batch=16, feat_levels=3, seed=460)
    cfg, octree, dec = build_cuda_models(case, DEV)
    surf = np.concatenate(case["frames"])
    with torch.no_grad():
        dec.lout.bias -= sdf_infer(octree, dec, torch.from_numpy(surf).to(DEV)).median()
    surf = surf / cfg.scale
    return cfg, octree, dec, (surf.min(0) - 0.5, surf.max(0) + 0.5)


def _setup(which, octree_mode, request):
    from shine_mapping_b200 import Mesher
    from shine_mapping_b200.mesher import OCTREE_MIN_CLUSTER
    cfg, octree, dec, bbx = request.getfixturevalue(which)
    m = Mesher(cfg, octree, dec)
    res = 0.15 if which == "street" else 0.05
    grid = m.octree_grid(octree.free_level_num, res) if octree_mode else m.bbx_grid(*bbx, res)
    return m, grid, (OCTREE_MIN_CLUSTER if octree_mode else cfg.min_cluster_vertices)


def _keep_oracle(faces, nv, min_tris):
    label, sizes = mo.triangle_clusters(faces, nv)
    return sizes[label] >= min_tris, sizes


def _sorted_normals(verts, normals):
    v, nrm = np.asarray(verts, dtype=np.float64), np.asarray(normals, dtype=np.float64)
    order = np.lexsort(np.concatenate([v, nrm], 1).T[::-1])
    return v[order], nrm[order]


MAPS = [("random_map", True), ("random_map", False), ("street", True), ("street", False)]


# ---- B. chunks and restarts --------------------------------------------------------------------------------------------

@pytest.mark.parametrize("which,octree_mode", MAPS)
def test_chunking_and_restarts_do_not_change_the_mesh(which, octree_mode, request, monkeypatch):
    from shine_mapping_b200 import mesher as mm
    m, grid, min_tris = _setup(which, octree_mode, request)
    per = (grid["n"] + 1) ** 3
    v0, f0 = m.marching_cubes(grid)
    want = mo.canonical_mesh(v0.cpu().numpy(), f0.cpu().numpy())
    rv, rf, rn = m._mesh(grid, min_tris, None)
    want_out = mo.canonical_mesh(rv.cpu().numpy(), rf.cpu().numpy())
    want_n = _sorted_normals(rv.cpu().numpy(), rn.cpu().numpy())
    assert grid["bricks"].shape[0] > 17 and f0.shape[0] > 1000 and 0 < rf.shape[0]
    attempts = []
    real_chunks = mm.Mesher.chunks
    monkeypatch.setattr(mm.Mesher, "chunks", lambda self, g: (attempts.append(1), real_chunks(self, g))[1])
    worst = 0.0
    for k, small_table in ((1, False), (3, False), (17, False), (3, True)):
        monkeypatch.setattr(mm, "CHUNK_POINTS", k * per)
        if small_table:
            monkeypatch.setattr(mm.Mesher, "edge_capacity", staticmethod(lambda g: 1 << 8))
        attempts.clear()
        v, f = m.marching_cubes(grid)
        assert mo.canonical_mesh(v.cpu().numpy(), f.cpu().numpy()) == want, (k, small_table)
        assert len(attempts) >= (3 if small_table else 1)                    # 2^8 slots: at least two restarts
        kv, kf, kn = m._mesh(grid, min_tris, None)
        assert mo.canonical_mesh(kv.cpu().numpy(), kf.cpu().numpy()) == want_out
        pos, nrm = _sorted_normals(kv.cpu().numpy(), kn.cpu().numpy())
        assert np.array_equal(pos, want_n[0])
        worst = max(worst, float(np.abs(nrm - want_n[1]).max()))
        assert worst <= 1e-6
    print(f"{which} octree={octree_mode}: bricks {grid['bricks'].shape[0]} n {grid['n']}, {v0.shape[0]} vertices "
          f"{f0.shape[0]} triangles, {rf.shape[0]} kept; meshes bit-identical, max|dnormal| {worst:.1e}")


# ---- C. the triangle table on random fields ----------------------------------------------------------------------------

def _mc_chunks(bricks, sdf, mask, n, hi, per_chunk):
    """shine_marching_cubes over the bricks in chunks of per_chunk, one edge table, as Mesher.marching_cubes does."""
    from shine_mapping_b200 import _abi
    lib, st = _abi.lib(), _abi.stream_ptr(DEV)
    per = (n + 1) ** 3
    cap = 1 << 20
    slots = torch.full((cap * 16,), 0xFF, dtype=torch.uint8, device=DEV)
    counters = torch.zeros(4, dtype=torch.int32, device=DEV)
    verts = torch.empty(cap // 2, 3, dtype=torch.float32, device=DEV)
    faces = []
    for s in range(0, bricks.shape[0], per_chunk):
        b = bricks[s:s + per_chunk].contiguous()
        g = _brick_grid(b, sdf[s * per:(s + b.shape[0]) * per], mask[s * per:(s + b.shape[0]) * per], n, hi=hi)
        counters[1:3].zero_()
        _abi.check(lib.shine_marching_cubes(C.byref(g), _abi.ptr(slots), cap, _abi.ptr(counters), None, 0, None, 0, st), "count")
        nv, nt, _, lost = counters.tolist()
        assert lost == 0 and 2 * nv <= cap
        f = torch.empty(nt, 3, dtype=torch.int32, device=DEV)
        _abi.check(lib.shine_marching_cubes(C.byref(g), _abi.ptr(slots), cap, _abi.ptr(counters), _abi.ptr(verts),
                                            verts.shape[0], _abi.ptr(f), nt, st), "emit")
        assert int(counters[2]) == nt
        faces.append(f)
    return verts[:int(counters[0])], torch.cat(faces)


def _random_field(seed, nb=4, n=8, masked=False):
    """Dense random field on (nb n + 1)^3 points: random signs, |v| in [0.05, 1], the outer layer positive; the bricks
    [0, nb)^3 in shuffled order with their (n+1)^3 points gathered from it."""
    rng = np.random.default_rng(seed)
    N = nb * n + 1
    field = (rng.uniform(0.05, 1.0, (N, N, N)) * rng.choice([-1.0, 1.0], (N, N, N))).astype(np.float32)
    field[[0, -1], :, :] = np.abs(field[[0, -1], :, :])
    field[:, [0, -1], :] = np.abs(field[:, [0, -1], :])
    field[:, :, [0, -1]] = np.abs(field[:, :, [0, -1]])
    dmask = rng.random((N, N, N)) < 0.8 if masked else np.ones((N, N, N), dtype=bool)
    B = np.stack(np.meshgrid(*[np.arange(nb)] * 3, indexing="ij"), -1).reshape(-1, 3)[rng.permutation(nb ** 3)]
    G = (B[:, None, :] * n + _local(n)[None]).reshape(-1, 3)
    sdf = torch.from_numpy(field[G[:, 0], G[:, 1], G[:, 2]].copy()).to(DEV)
    mask = torch.from_numpy(dmask[G[:, 0], G[:, 1], G[:, 2]].astype(np.uint8)).to(DEV)
    return field, dmask, torch.from_numpy(B.astype(np.int32)).to(DEV).contiguous(), sdf, mask, (N, N, N)


def _configurations(field, dmask):
    inside = field < 0
    N = field.shape
    cls = np.zeros((N[0] - 1, N[1] - 1, N[2] - 1), dtype=np.int64)
    for cc in range(8):
        dx, dy, dz = cc & 1, (cc >> 1) & 1, (cc >> 2) & 1
        cls |= inside[dx:N[0] - 1 + dx, dy:N[1] - 1 + dy, dz:N[2] - 1 + dz].astype(np.int64) << cc
    return np.unique(cls[dmask[:-1, :-1, :-1]])


def _edges(faces):
    f = np.asarray(faces, dtype=np.int64)
    return np.concatenate([f[:, [0, 1]], f[:, [1, 2]], f[:, [2, 0]]])


def test_random_fields_give_closed_oriented_surfaces():
    field, dmask, bricks, sdf, mask, hi = _random_field(470)
    assert _configurations(field, dmask).shape[0] == 256
    verts, faces = _mc_chunks(bricks, sdf, mask, 8, hi, 5)
    v, f = verts.cpu().numpy(), faces.cpu().numpy().astype(np.int64)
    d = _edges(f)
    nv = v.shape[0]
    key = d[:, 0] * nv + d[:, 1]
    assert np.unique(key).shape[0] == key.shape[0]                    # each directed edge once ...
    assert np.isin(d[:, 1] * nv + d[:, 0], key).all()                 # ... and its reverse too: two triangles per edge
    assert np.array_equal(np.unique(f), np.arange(nv))                # every vertex used
    p = v.astype(np.float64)[f]
    vol = float(np.einsum("ij,ij->i", p[:, 0], np.cross(p[:, 1], p[:, 2])).sum() / 6.0)
    lo, up = mo.enclosed_volume_bounds(field, dmask, hi)
    assert lo < vol < up
    print(f"random field: {nv} vertices {f.shape[0]} triangles, 256 configurations, closed and oriented; "
          f"volume {vol:.1f} in [{lo:.0f}, {up:.0f}]")


def test_random_masked_field_is_open_on_the_processed_boundary_only():
    field, dmask, bricks, sdf, mask, hi = _random_field(471, masked=True)
    verts, faces = _mc_chunks(bricks, sdf, mask, 8, hi, 7)
    v, f = verts.cpu().numpy(), faces.cpu().numpy().astype(np.int64)
    d = _edges(f)
    nv = v.shape[0]
    key = d[:, 0] * nv + d[:, 1]
    assert np.unique(key).shape[0] == key.shape[0]
    once = ~np.isin(d[:, 1] * nv + d[:, 0], key)
    assert np.array_equal(np.unique(f), np.arange(nv)) and once.any()
    proc = dmask[:-1, :-1, :-1]
    N = np.array(hi)
    for a, b in d[once]:
        pa, pb = v[a].astype(np.float64), v[b].astype(np.float64)
        # a segment on a grid plane: one axis where both ends sit on the same integer coordinate
        ax = [k for k in range(3) if pa[k] == pb[k] and pa[k] == np.floor(pa[k])]
        assert len(ax) == 1, (pa, pb)
        k = ax[0]
        c = np.floor(np.minimum(pa, pb)).astype(np.int64)
        c[k] = int(pa[k])
        below, above = c.copy(), c.copy()
        below[k] -= 1
        inside = lambda q: bool((q >= 0).all() and (q < N - 1).all() and proc[tuple(q)])
        assert inside(below) != inside(above), (pa, pb)
    print(f"masked random field: {nv} vertices {f.shape[0]} triangles, {int(once.sum())} boundary edges, all on the "
          "processed region's boundary")


# ---- D. the cluster filter ---------------------------------------------------------------------------------------------

def _clusters(verts, faces, min_tris):
    from shine_mapping_b200.mesher import normals_and_clusters
    v = torch.as_tensor(np.asarray(verts, dtype=np.float32)).to(DEV)
    f = torch.as_tensor(np.asarray(faces, dtype=np.int32)).to(DEV)
    normals, keep = normals_and_clusters(v, f, min_tris)
    return normals.cpu().numpy(), keep.cpu().numpy()


@pytest.mark.parametrize("which,octree_mode", MAPS)
def test_cluster_filter_matches_partition_on_maps(which, octree_mode, request):
    m, grid, min_tris = _setup(which, octree_mode, request)
    verts, faces = m.marching_cubes(grid)
    v, f = verts.cpu().numpy(), faces.cpu().numpy()
    label, sizes = mo.triangle_clusters(f, v.shape[0])
    mid = int(np.sort(sizes)[len(sizes) // 2])
    for t in sorted({1, min_tris, mid, mid + 1, int(sizes.max()), int(sizes.max()) + 1}):
        _, keep = _clusters(v, f, t)
        assert np.array_equal(keep, sizes[label] >= t), t
    print(f"{which} octree={octree_mode}: {f.shape[0]} triangles in {sizes.shape[0]} clusters (largest {sizes.max()}); "
          "keep masks equal at every threshold")


def _strip(k, base, y0=0.0):
    """k triangles in a strip: vertices base .. base + k + 1 zig-zagging along x, consistently wound."""
    j = np.arange(k + 2)
    v = np.stack([j // 2 + 0.5 * (j % 2), (j % 2) + y0, np.zeros(k + 2)], 1)
    i = np.arange(k)
    f = np.stack([i, i + 1, i + 2], 1)
    f[1::2] = f[1::2][:, [1, 0, 2]]
    return v, f + base


def test_cluster_filter_edge_cases():
    min_tris, parts, verts, base = 7, [], [], 0
    for y, k in enumerate((min_tris - 1, min_tris, min_tris + 1)):
        v, f = _strip(k, base, 3.0 * y)
        verts.append(v); parts.append(f); base += v.shape[0]
    # two fans of 4 triangles that meet at one vertex: two clusters of 4, not one of 8
    fan = np.array([[0, 0, 0], [1, 0, 0], [1, 1, 0], [0, 1, 0], [-1, 1, 0], [-1, 0, 0], [-1, -1, 0], [0, -1, 0], [1, -1, 0]],
                   dtype=np.float64) + [0, 20, 0]
    verts.append(fan)
    parts.append(base + np.array([[0, 1, 2], [0, 2, 3], [0, 3, 4], [0, 4, 5], [0, 5, 6], [0, 6, 7], [0, 7, 8], [0, 8, 1]])[[0, 1, 4, 5]])
    base += fan.shape[0]
    # an edge shared by four triangles (a book of four pages), 4 triangles in one cluster
    book = np.array([[0, 0, 0], [0, 0, 1], [1, 0, 0], [0, 1, 0], [-1, 0, 0], [0, -1, 0]], dtype=np.float64) + [0, 30, 0]
    verts.append(book)
    parts.append(base + np.array([[0, 1, 2], [1, 0, 3], [0, 1, 4], [1, 0, 5]]))
    v, f = np.concatenate(verts), np.concatenate(parts)
    rng = np.random.default_rng(480)
    order = rng.permutation(f.shape[0])
    for ff in (f, f[::-1], f[order]):
        label, sizes = mo.triangle_clusters(ff, v.shape[0])
        assert sorted(sizes.tolist()) == sorted([6, 7, 8, 2, 2, 4])
        for t in (min_tris - 1, min_tris, min_tris + 1, 3, 4, 5):
            _, keep = _clusters(v, ff, t)
            assert np.array_equal(keep, sizes[label] >= t), t
    _, keep = _clusters(v, f, 2)
    assert keep.all()
    # one triangle
    nrm, keep = _clusters(v[:3], [[0, 1, 2]], 1)
    assert keep.tolist() == [True] and np.allclose(np.abs(nrm[:, 2]), 1.0)
    assert _clusters(v[:3], [[0, 1, 2]], 2)[1].tolist() == [False]
    # no triangles, five vertices: zero normals, an empty mask
    nrm, keep = _clusters(v[:5], np.zeros((0, 3)), 1)
    assert keep.shape == (0,) and nrm.shape == (5, 3) and (nrm == 0).all()
    print("strips of min_tris - 1 .. + 1, a shared vertex, a four-triangle edge, nt = 1, nt = 0: keep masks equal")


def test_cluster_filter_on_a_long_strip():
    k = 2_000_000
    v, f = _strip(k, 0)
    label, sizes = mo.triangle_clusters(f, v.shape[0])
    assert sizes.tolist() == [k]
    rng = np.random.default_rng(481)
    for name, ff in (("natural", f), ("reversed", f[::-1]), ("shuffled", f[rng.permutation(k)])):
        _, keep = _clusters(v, ff, k)
        assert keep.all(), name
        _, keep = _clusters(v, ff, k + 1)
        assert not keep.any(), name
    print(f"strip of {k} triangles in natural, reversed and shuffled order: one cluster")


def test_cluster_filter_refuses_a_small_edge_table():
    from shine_mapping_b200 import _abi
    v, f = _strip(10, 0)
    verts = torch.from_numpy(v.astype(np.float32)).to(DEV).contiguous()
    faces = torch.from_numpy(f.astype(np.int32)).to(DEV).contiguous()
    nt, nv = faces.shape[0], verts.shape[0]
    scratch = torch.empty(2 * nt, dtype=torch.int32, device=DEV)
    keep = torch.empty(nt, dtype=torch.uint8, device=DEV)
    normals = torch.empty(nv, 3, dtype=torch.float32, device=DEV)

    def call(cap):
        slots = torch.full((cap * 16,), 0xFF, dtype=torch.uint8, device=DEV)
        return _abi.lib().shine_mesh_clusters(_abi.ptr(verts), nv, _abi.ptr(faces), nt, 1, _abi.ptr(slots), cap,
                                              _abi.ptr(scratch), _abi.ptr(keep), _abi.ptr(normals), _abi.stream_ptr(DEV))
    assert call(32) == -1          # 6 nt = 60 slots needed
    assert call(96) == -1          # not a power of two
    assert call(64) == 0
    torch.cuda.synchronize()
    assert bool(keep.bool().all())
    print("edge capacity below 6 nt and not a power of two refused")


# ---- E. vertex normals -------------------------------------------------------------------------------------------------

def test_normals_match_fp64_at_the_abi(street):
    from shine_mapping_b200 import Mesher
    cfg, octree, dec, _ = street
    meshes = []
    field, dmask, bricks, sdf, mask, hi = _random_field(472)
    meshes.append(("random field", *_mc_chunks(bricks, sdf, mask, 8, hi, 9)))
    m = Mesher(cfg, octree, dec)
    meshes.append(("street", *m.marching_cubes(m.octree_grid(octree.free_level_num, 0.15))))
    for name, verts, faces in meshes:
        v, f = verts.cpu().numpy(), faces.cpu().numpy()
        nrm, _ = _clusters(v, f, 1)
        want = mo.vertex_normals(v.astype(np.float64), f)
        ok = np.linalg.norm(want, axis=1) > 0
        worst = float(_angle(nrm[ok], want[ok]).max())
        print(f"{name}: {v.shape[0]} vertices, max angle to the fp64 normals {worst:.2e} rad")
        assert ok.mean() > 0.99 and worst <= 2e-3
        assert np.allclose(np.linalg.norm(nrm[ok], axis=1), 1.0, atol=1e-6)


@pytest.mark.parametrize("octree_mode", [True, False])
def test_mesher_normals_do_not_depend_on_the_map_offset(street, tmp_path, monkeypatch, octree_mode):
    """The map's offset moves the vertices, not the surface: the written normals stay those of the fp64 vertices."""
    from shine_mapping_b200 import Mesher, mesher as mm
    cfg, octree, dec, bbx = street
    m = Mesher(cfg, octree, dec)
    m.global_transform = TRANSFORM
    base = m.octree_grid(octree.free_level_num, 0.1) if octree_mode else m.bbx_grid(*bbx, 0.1)
    seen = {}
    real_mc, real_compact = mm.Mesher.marching_cubes, mm.compact

    def spy_mc(self, grid, sdf_map=None):
        seen["verts"], seen["faces"] = real_mc(self, grid, sdf_map)
        return seen["verts"], seen["faces"]

    def spy_compact(verts_m, faces, normals, keep):
        seen["verts_m"], seen["keep"] = verts_m, keep
        return real_compact(verts_m, faces, normals, keep)
    monkeypatch.setattr(mm.Mesher, "marching_cubes", spy_mc)
    monkeypatch.setattr(mm, "compact", spy_compact)
    R, t = TRANSFORM[:3, :3], TRANSFORM[:3, 3]
    runs, report, failures = [], [], []
    for off in (0.0, 50.0, 400.0, 1500.0):
        grid = dict(base, origin_m=np.asarray(base["origin_m"], dtype=np.float64) + off)
        path = str(tmp_path / f"mesh_{int(off)}.ply")
        _, _, normals = m._mesh(grid, 1, path)
        f = seen["faces"].cpu().numpy().astype(np.int64)
        keep = seen["keep"].cpu().numpy()
        used = np.zeros(seen["verts"].shape[0], dtype=bool)
        used[f[keep].reshape(-1)] = True
        want = mo.vertex_normals(seen["verts_m"].cpu().numpy() @ R.T + t, f)[used]
        got = normals.cpu().numpy()
        ok = np.linalg.norm(want, axis=1) > 0
        ang = _angle(got[ok], want[ok])
        ang = np.where(np.isnan(ang), np.pi, ang)
        written = mm.read_ply(path)[2]
        ln = np.linalg.norm(written.astype(np.float64), axis=1)
        bad = int((~np.isfinite(ln) | (np.abs(ln - 1.0) > 1e-6)).sum())
        report.append(f"offset {off:g} m: max angle {ang.max():.2e} rad, {int((ang > 1e-2).sum())} vertices > 0.01 rad, "
                      f"{bad} non-unit normals of {written.shape[0]}")
        if ang.max() > 2e-3 or bad:
            failures.append(off)
        runs.append(_sorted_normals(seen["verts"].cpu().numpy()[used], got))
    across = max(float(np.abs(r[1] - runs[0][1]).max()) for r in runs)
    print(f"octree={octree_mode}: " + "; ".join(report) + f"; max|dnormal| across offsets {across:.1e}")
    assert not failures, f"normals off at offsets {failures}"
    assert all(np.array_equal(r[0], runs[0][0]) for r in runs)
    assert across <= 1e-6
