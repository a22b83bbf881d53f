"""Mesh evaluation on the GPU (csrc/shine_eval.cu, shine_mapping_b200/evaluate.py) against tests/eval_oracle.py: exact
nearest neighbours, Philox-driven surface samples bit for bit, an analytic plane, and a trained street end to end."""
import math

import numpy as np
import pytest
import torch

from tests import eval_oracle as eo

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


@pytest.fixture(scope="module", autouse=True)
def _lib(built_lib):
    assert torch.cuda.is_available()
    return built_lib


def _t(a):
    return torch.from_numpy(np.ascontiguousarray(a, dtype=np.float64)).to(DEV)


# ---- nearest neighbours ------------------------------------------------------------------------------------------------

def _sphere_lattice(r, s):
    g = np.arange(-r - s, r + s, s)
    p = np.stack(np.meshgrid(g, g, g, indexing="ij"), -1).reshape(-1, 3)
    n = np.linalg.norm(p, axis=1)
    return p[np.abs(n - r) < s / 2]


def _nn_case(name, rng):
    if name == "uniform":
        return rng.uniform(-5, 5, (20000, 3)), rng.uniform(-6, 6, (20000, 3)), 0.5
    if name == "plane_lattice":
        g = np.arange(0, 4, 0.02)
        p = np.stack(np.meshgrid(g, g, indexing="ij"), -1).reshape(-1, 2)
        ref = np.column_stack((p, np.zeros(len(p))))
        return ref, rng.uniform(-0.5, 4.5, (30000, 3)) * [1, 1, 0.1], 0.2
    if name == "sphere_lattice":
        return _sphere_lattice(1.0, 0.02), rng.normal(size=(20000, 3)) * 0.7, 2.0
    if name == "clustered":
        centres = rng.uniform(-20, 20, (30, 3))
        ref = (centres[rng.integers(0, 30, 40000)] + rng.normal(scale=0.05, size=(40000, 3)))
        return ref, rng.uniform(-22, 22, (20000, 3)), 2.0
    if name == "duplicates":
        base = rng.uniform(-1, 1, (500, 3))
        return np.repeat(base, 9, axis=0)[rng.permutation(4500)], rng.uniform(-1.2, 1.2, (5000, 3)), 0.3
    if name == "coincident":
        ref = rng.uniform(-1, 1, (10000, 3))
        return ref, ref[rng.permutation(10000)[:4000]], 0.1
    if name == "all_beyond":
        return rng.uniform(-1, 1, (5000, 3)), rng.uniform(5, 6, (3000, 3)), 2.0
    if name == "empty_ref":
        return np.zeros((0, 3)), rng.uniform(-1, 1, (100, 3)), 1.0
    if name == "one_point":
        return np.array([[0.25, -0.5, 1.0]]), rng.uniform(-1, 1, (1000, 3)), 1.0
    if name == "million":
        return rng.uniform(-30, 30, (1_000_000, 3)), rng.uniform(-31, 31, (1_000_000, 3)), 2.0
    raise KeyError(name)


@pytest.mark.parametrize("name", ["uniform", "plane_lattice", "sphere_lattice", "clustered", "duplicates", "coincident",
                                  "all_beyond", "empty_ref", "one_point", "million"])
def test_nearest_neighbours_are_exact(name):
    from shine_mapping_b200.evaluate import NearestNeighbours
    rng = np.random.default_rng(sum(name.encode()))
    ref, q, r = _nn_case(name, rng)
    dist, index = NearestNeighbours(_t(ref)).query(_t(q), r)
    dist, index = dist.cpu().numpy(), index.cpu().numpy().astype(np.int64)
    want_d2, _ = eo.nearest(ref, q)
    inside = want_d2 < r * r
    assert np.array_equal(index >= 0, inside)                       # the within-radius flags
    assert np.isinf(dist[~inside]).all() and (index[~inside] == -1).all()
    got_d2 = eo.dist2(q[inside], ref[index[inside]])
    assert np.array_equal(got_d2, want_d2[inside])                  # exact minimum; the index is one of its ties
    assert np.array_equal(dist[inside], np.sqrt(got_d2))
    if name == "coincident":
        assert (dist == 0).all()
    if name == "all_beyond":
        assert not inside.any()


# ---- sampling ------------------------------------------------------------------------------------------------------------

def _random_mesh(rng, nv=3000, nt=6000):
    verts = rng.uniform(-2, 2, (nv, 3))
    faces = rng.integers(0, nv, (nt, 3))
    faces[:50, 1] = faces[:50, 0]                                   # zero area: a repeated vertex
    verts[faces[50:60, 2]] = verts[faces[50:60, 0]]                 # zero area: coincident vertices
    return verts, faces


def test_samples_match_the_oracle_bit_for_bit():
    from shine_mapping_b200.evaluate import sample_mesh
    rng = np.random.default_rng(5)
    verts, faces = _random_mesh(rng)
    box = np.array([-1.5, -1.8, -1.6, 1.7, 1.5, 1.9])
    n = 400_000
    pts, ids = sample_mesh(_t(verts), torch.from_numpy(faces).to(DEV, torch.int32), n, seed=7, crop_box=_t(box),
                           return_tri_ids=True)
    pts, ids = pts.cpu().numpy(), ids.cpu().numpy().astype(np.int64)
    assert pts.shape == (n, 3)                                      # exactly N
    assert np.array_equal(pts, eo.sample_points(verts, faces, ids, 7))
    area = eo.triangle_areas(verts, faces, box)
    want, cn = eo.sample_counts(area, n)
    got = np.bincount(ids, minlength=len(faces))
    near_half = np.abs(cn - np.floor(cn) - 0.5) < 1e-6
    exempt = near_half | np.r_[False, near_half[:-1]]               # a tie moves one sample between neighbours
    assert np.array_equal(got[~exempt], want[~exempt])
    assert (got[area == 0] == 0).all() and (area == 0).sum() > 60   # cropped and zero-area triangles get none
    assert eo.crop_keep(verts, faces[ids], box).all()
    again = sample_mesh(_t(verts), torch.from_numpy(faces).to(DEV, torch.int32), n, seed=7, crop_box=_t(box))
    assert again.cpu().numpy().tobytes() == pts.tobytes()
    other = sample_mesh(_t(verts), torch.from_numpy(faces).to(DEV, torch.int32), n, seed=8, crop_box=_t(box))
    assert (other.cpu().numpy() != pts).any(axis=1).mean() > 0.99


def test_zero_area_mesh_gives_no_samples():
    from shine_mapping_b200.evaluate import sample_mesh
    verts = np.array([[0, 0, 0], [1, 0, 0], [2, 0, 0]], dtype=np.float64)
    pts = sample_mesh(_t(verts), torch.tensor([[0, 1, 2]], dtype=torch.int32, device=DEV), 1000)
    assert pts.shape == (0, 3)


# ---- analytic plane ------------------------------------------------------------------------------------------------------

def _square(k=40):
    g = np.linspace(0.0, 1.0, k + 1)
    v = np.stack(np.meshgrid(g, g, indexing="ij"), -1).reshape(-1, 2)
    verts = np.column_stack((v, np.zeros(len(v))))
    i = np.arange(k)[:, None] * (k + 1) + np.arange(k)[None, :]
    i = i.reshape(-1)
    faces = np.concatenate((np.stack((i, i + k + 1, i + 1), 1), np.stack((i + 1, i + k + 1, i + k + 2), 1)))
    return verts, faces


def _lattice(lo, hi, s, z):
    gx, gy = np.arange(lo[0], hi[0] + s / 2, s), np.arange(lo[1], hi[1] + s / 2, s)
    p = np.stack(np.meshgrid(gx, gy, indexing="ij"), -1).reshape(-1, 2)
    return np.column_stack((p, np.full(len(p), z)))


def test_plane_distances_truncation_and_crop():
    from shine_mapping_b200.evaluate import NearestNeighbours, eval_mesh, sample_mesh
    verts, faces = _square()
    fv, ff = _t(verts), torch.from_numpy(faces).to(DEV, torch.int32)
    s, d = 0.05, 0.1
    gt = _lattice((-2.0, -2.0), (3.0, 3.0), s, d)
    samples = sample_mesh(fv, ff, 200_000, seed=1)
    dist, _ = NearestNeighbours(_t(gt)).query(samples, 0.5)
    dist = dist.cpu().numpy()
    assert np.isfinite(dist).all()
    assert (dist >= d * (1 - 1e-15)).all() and (dist <= math.sqrt(d * d + s * s / 2) * (1 + 1e-15)).all()
    # d >= truncation_acc: no prediction point is kept
    m = eval_mesh((fv, ff), _t(gt), down_sample_res=0.0, truncation_acc=0.1, truncation_com=0.5, gt_bbx_mask_on=False,
                  mesh_sample_point=100_000, device=DEV)
    assert np.isnan(m["MAE_accuracy (m)"]) and np.isnan(m["Precision [Accuracy] (%)"])
    # ground-truth points farther than truncation_com from the square are beyond (+inf, clamped by the metrics)
    tc = 0.5
    dr, idx = NearestNeighbours(samples).query(_t(gt), tc)
    dr, idx = dr.cpu().numpy(), idx.cpu().numpy()
    dx = np.maximum(np.maximum(-gt[:, 0], gt[:, 0] - 1.0), 0.0)
    dy = np.maximum(np.maximum(-gt[:, 1], gt[:, 1] - 1.0), 0.0)
    to_square = np.sqrt(dx * dx + dy * dy + d * d)
    far, near = to_square > tc + 0.02, to_square < tc - 0.02
    assert far.any() and np.isinf(dr[far]).all() and (idx[far] == -1).all() and np.isfinite(dr[near]).all()
    m = eval_mesh((fv, ff), _t(gt), down_sample_res=0.0, truncation_acc=0.5, truncation_com=tc, gt_bbx_mask_on=False,
                  mesh_sample_point=100_000, device=DEV)
    assert m["MAE_completeness (m)"] <= tc and m["MAE_completeness (m)"] > 0.8 * tc
    # crop on, d <= down_sample_res: the box is the lattice's (x, y) by [d - r, d + r] in z
    dsr, gt_part = 0.1, _lattice((0.0, 0.0), (0.5, 1.2), s, 0.05)
    box = np.r_[gt_part.min(0) - [0, 0, dsr], gt_part.max(0) + [0, 0, dsr]]
    pts, ids = sample_mesh(fv, ff, 100_000, seed=3, crop_box=_t(box), return_tri_ids=True)
    pts, ids = pts.cpu().numpy(), ids.cpu().numpy()
    assert np.all((pts >= box[:3]) & (pts <= box[3:]))
    outside = ~eo.crop_keep(verts, faces, box)
    assert outside.any() and not outside[ids].any()


# ---- end to end ------------------------------------------------------------------------------------------------------------

def _street_mesh():
    from shine_mapping_b200 import Decoder, FeatureOctree, Mesher, synth
    from shine_mapping_b200.batch_loop import run_shine_mapping_batch
    from shine_mapping_b200.config import SHINEConfig
    torch.manual_seed(0)
    cfg = SHINEConfig(tree_level_world=12, tree_level_feat=3, leaf_vox_size=0.3, device=DEV, bs=8192, iters=300,
                      mc_res_m=0.15, surface_sample_range_m=0.3, free_sample_end_dist_m=1.0, min_range=2.0, pc_radius=25.0)
    octree, dec = FeatureOctree(cfg), Decoder(cfg)
    pool = synth.build_scene_map(cfg, octree, 512, 10, frame_step_m=1.0, seed=3)
    run_shine_mapping_batch(cfg, octree, dec, pool, iters=300)
    mesher = Mesher(cfg, octree, dec)
    verts, faces, _ = mesher.recon_bbx_mesh(pool.map_bbx[0], pool.map_bbx[1], cfg.mc_res_m)
    return verts, faces


@pytest.fixture(scope="module")
def street():
    from shine_mapping_b200 import synth
    verts, faces = _street_mesh()
    gt = synth.scene_surface_points(-10.0, 20.0, 0.1).to(DEV)
    return verts, faces, gt


def test_street_metrics_match_the_oracle(street):
    from shine_mapping_b200.evaluate import eval_mesh, load_mesh, sample_mesh
    verts, faces, gt = street
    kw = dict(down_sample_res=0.05, threshold=0.1, truncation_acc=0.2, truncation_com=2.0, gt_bbx_mask_on=True,
              mesh_sample_point=300_000, seed=11, device=DEV)
    got = eval_mesh((verts, faces), gt, **kw)
    again = eval_mesh((verts, faces), gt, **kw)
    assert np.array(list(got.values())).tobytes() == np.array(list(again.values())).tobytes()
    print(got)
    # the oracle from the GPU's own samples
    v64, f32 = load_mesh((verts, faces), torch.device(DEV))
    widen = torch.tensor([0.0, 0.0, 0.05], dtype=torch.float64, device=DEV)
    box = torch.cat((gt.amin(0) - widen, gt.amax(0) + widen))
    samples = sample_mesh(v64, f32, 300_000, 11, box).cpu().numpy()
    pred = eo.voxel_down(samples, 0.05)
    gtd = eo.voxel_down(gt.cpu().numpy(), 0.05)
    want = eo.metrics_from_points(pred, gtd, 0.05, 0.1, 0.2, 2.0)
    assert list(got) == list(want)
    for k in ("Precision [Accuracy] (%)", "Recall [Completeness] (%)", "Spacing (m)", "Inlier_threshold (m)",
              "Outlier_truncation_acc (m)", "Outlier_truncation_com (m)"):
        assert got[k] == want[k], k
    for k in want:
        assert got[k] == pytest.approx(want[k], rel=1e-12, abs=0), k
    assert got["F-score (%)"] > 0.0 and got["MAE_accuracy (m)"] < 0.2


def test_crop_intersection_matches_the_oracle(street, tmp_path):
    from shine_mapping_b200.evaluate import crop_intersection, load_mesh, sample_mesh
    from shine_mapping_b200.scans import read_ply
    verts, faces, gt = street
    shifted = verts + torch.tensor([0.3, 0.0, 0.0], device=DEV)
    out = str(tmp_path / "crop.ply")
    kept = crop_intersection(gt, [(verts, faces), (shifted, faces)], out, dist_thre=0.1, mesh_sample_point=200_000,
                             seed=5, device=DEV)
    want = gt.cpu().numpy()
    for v in (verts, shifted):
        v64, f32 = load_mesh((v, faces), torch.device(DEV))
        s = sample_mesh(v64, f32, 200_000, 5).cpu().numpy()
        d2, _ = eo.nearest(s, want)
        want = want[d2 < 0.1 ** 2]
    assert 0 < want.shape[0] < gt.shape[0]
    assert np.array_equal(kept.cpu().numpy(), want)
    back = read_ply(out, pinned=False)
    assert back.fp64 and np.array_equal(back.points(), want)
