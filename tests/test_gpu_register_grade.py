"""shine_register_normal_eq graded against fp64 (tests/grad_field_bound.py): all 29 outputs and every block partial of
the scratch, on whole scans with their ReLU-kink points (each kink point enters with the interval over its mask
alternatives), with the count exact and two launches bit for bit equal.

The matrix: 1, 3, 4, 5 and 8 levels at world levels 6, 12 and 15, poly and linear, with and without biases, fresh tables
and tables x300.  Besides a scan at a random pose, each map is launched at the identity (q = p exactly) on voxel
corners and face centres of every level, points on the clamp faces and outside the cube whose boundary voxel exists
(each map carries one extra frame at the cube's faces), and points whose leaf voxel is missing while a coarser level
hits (they must add nothing, not even to the count).  Also: dense tables (one slot per node), the adversarial tables of
test_gpu_infer_grade, a descriptor whose levels are not consecutive, n = 1 .. 10^6 around the 256-thread block and the
1024-block cap, a kappa so large that w = 1 exactly and one so small that most w fall below 2^-60, and rows of the
K-pose entry past its 512-pose launch chunk.  Each case prints its worst error / bound and its kink points."""
import ctypes as C

import numpy as np
import pytest
import torch

from oracle import shine_oracle as orc
from tests.grad_field_bound import GradRef, RegBound, gm_weight, grade_reg, reg_blocks
from tests.parity_utils import build_cuda_models, make_case, make_config
from tests.test_gpu_infer_grade import (KeptLevels, _adversarial_map, _voxel_points, check_octree_slots, clone,
                                        load_tables, scaled, special_points)
from tests.test_gpu_odometry import _q32, _random_pose

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
F32 = np.float32
EYE = np.eye(4)


@pytest.fixture(scope="module", autouse=True)
def _lib(built_lib):
    assert torch.cuda.is_available()
    return built_lib


# ---- calling the kernel ----------------------------------------------------------------------------------------------------

def register(od, dd, pts, poses, sigma, kappa):
    """shine_register_normal_eq (one pose) or shine_register_normal_eq_poses -> (out [K, 29], block partials [K, G, 29])"""
    from shine_mapping_b200 import _abi
    lib = _abi.lib()
    pts = np.ascontiguousarray(pts, dtype=F32).reshape(-1, 3)
    poses = np.asarray(poses, dtype=np.float64).reshape(-1, 16)
    n, K = pts.shape[0], poses.shape[0]
    p = torch.from_numpy(pts).to(DEV)
    need = max(lib.shine_register_scratch_bytes(n, K), _abi.REGISTER_SCRATCH_BYTES)
    scratch = torch.full((need // 8,), float("nan"), dtype=torch.float64, device=DEV)
    out = torch.full((K, 29), float("nan"), dtype=torch.float64, device=DEV)
    buf = (C.c_double * (16 * K))(*poses.reshape(-1).tolist())
    od_, dd_ = C.byref(od), C.byref(dd)
    if K == 1:
        rc = lib.shine_register_normal_eq(od_, dd_, _abi.ptr(p), n, buf, float(sigma), float(kappa), _abi.ptr(out),
                                          _abi.ptr(scratch), need, _abi.stream_ptr(DEV))
    else:
        rc = lib.shine_register_normal_eq_poses(od_, dd_, _abi.ptr(p), n, buf, K, float(sigma), float(kappa),
                                                _abi.ptr(out), _abi.ptr(scratch), need, _abi.stream_ptr(DEV))
    _abi.check(rc, "shine_register_normal_eq")
    torch.cuda.synchronize()
    G = reg_blocks(n)
    return out.cpu().numpy(), scratch[: K * G * 29].cpu().numpy().reshape(K, G, 29)


def check(od, dd, rb, pts, idx, pose, what, blocks=True):
    """launch pts at pose (idx: the ref point of each launched point), grade out and the block partials, launch again
    for the same bits -> worst ratio"""
    out, part = register(od, dd, pts, pose, rb.sigma, rb.kappa)
    want, bound = rb.expect(idx)
    worst = grade_reg(out[0], want, bound, what)
    if blocks:
        bw, bb = rb.expect_blocks(idx)
        worst = max(worst, grade_reg(part[0], bw, bb, f"{what}: {bw.shape[0]} block partials"))
    again, _ = register(od, dd, pts, pose, rb.sigma, rb.kappa)
    assert np.array_equal(out.view(np.int64), again.view(np.int64)), f"{what}: two launches differ"
    return worst


def graded(case, q, sigma, kappa, what):
    """GradRef and RegBound at q; the points left out (> 4 uncertain units) are counted and must be rare"""
    ref = GradRef(case, q)
    assert ref.n_dropped <= max(2, ref.n // 1000), f"{what}: {ref.n_dropped} points with more than 4 uncertain units"
    print(f"[register bounds] {what}: {ref.n} points, {int(ref.valid.sum())} at lv[0], {ref.kinks} kink points graded "
          f"({ref.alternatives} rows), {ref.n_dropped} left out")
    return ref, RegBound(ref, sigma, kappa)


# ---- maps and point sets ---------------------------------------------------------------------------------------------------

def _scale(world):
    return 1.0 / (0.2 * 2 ** (world - 1))


def with_boundary(case, seed):
    """the case with one more frame of surface points just inside each face of the cube, tables regrown, and its oracle
    -> (case, boundary points: on the clamp faces +-1, nextafter(+-1, 0), and outside at +-1.25, +-1.5)"""
    c = case["cfg"]
    rng = np.random.default_rng(seed)
    yz = rng.uniform(-0.03, 0.03, (6, 2))
    e = 1.0 - 2.0 ** -(c["tree_level_world"] + 2)
    frame, edges = [], []
    for a in range(3):
        others = [b for b in range(3) if b != a]
        for s in (1.0, -1.0):
            p = np.zeros((yz.shape[0], 3))
            p[:, others] = yz
            p[:, a] = s * e
            frame.append(p)
            for v in (1.0, float(np.nextafter(F32(1), F32(0))), 1.25, 1.5):
                q = p.copy()
                q[:, a] = s * v
                edges.append(q)
    frames = list(case["frames"]) + [np.concatenate(frame).astype(F32)]
    torch.manual_seed(seed)
    o = orc.OracleOctree(c["tree_level_world"], c["tree_level_feat"], c["feature_dim"], 0.05, c["poly_int_on"])
    for fr in frames:
        o.update(torch.from_numpy(np.asarray(fr)))
    tables = [t.detach().numpy().copy() for t in o.hier_features]
    return dict(case, frames=frames, tables=tables, oracle=o), np.concatenate(edges).astype(F32)


def leaf_missing(o, rng, surf, world, m=400):
    """points near the surface whose leaf voxel is missing while a coarser level hits"""
    idx = rng.integers(0, surf.shape[0], 8 * m)
    off = rng.normal(0, 1, (8 * m, 3))
    off *= (rng.uniform(1.5, 4.0, 8 * m) * 2.0 ** (1 - world) / np.linalg.norm(off, axis=1))[:, None]
    p = (surf[idx] + off).astype(F32)
    ix = o.get_indices(torch.from_numpy(p))
    keep = (ix[0][:, 0] < 0).numpy() & np.any([(t[:, 0] >= 0).numpy() for t in ix[1:]], axis=0) if len(ix) > 1 else \
        np.zeros(p.shape[0], bool)
    return p[keep][:m]


def scan(case, rng, n, world):
    """n surface points of the map's frames with noise, in the frame of a random pose T -> (local points, T)"""
    sc = _scale(world)
    surf = np.concatenate([np.asarray(f, np.float64) for f in case["frames"][:1]])
    wpts = surf[rng.integers(0, surf.shape[0], n)] + rng.normal(0, 0.05 * sc, (n, 3))
    T = _random_pose(rng, sc)
    return ((wpts - T[:3, 3]) @ T[:3, :3]).astype(F32), T


def identity_set(case, rng, edges):
    o = case["oracle"]
    world = case["cfg"]["tree_level_world"]
    pts = [special_points(o, rng), edges, leaf_missing(o, rng, np.concatenate(case["frames"][:1]), world)]
    p = np.concatenate(pts).astype(F32)
    assert np.array_equal(_q32(p, EYE), p)
    return p


def grade_map(od, dd, case, scan_pts, T, ident, kappa, what, sigma=None):
    """the scan at T and the identity set, each graded -> worst ratio"""
    sigma = F32(case["cfg"]["sigma"] if sigma is None else sigma)
    worst = 0.0
    for pts, pose, name in ((scan_pts, T, "scan"), (ident, EYE, "corners, faces, clamp, leaf-missing")):
        if pts is None:
            continue
        q = _q32(pts, pose)
        ref, rb = graded(case, q, sigma, kappa, f"{what} {name}")
        keep = np.flatnonzero(~ref.dropped)
        worst = max(worst, check(od, dd, rb, pts[keep], keep, pose, f"{what} {name}"))
        if name != "scan":
            lm = ~ref.valid & ref.hits.any(1)
            assert lm.sum() >= (20 if ref.hits.shape[1] > 1 else 0), f"{what}: {int(lm.sum())} leaf-missing points"
    return worst


# ---- the matrix ------------------------------------------------------------------------------------------------------------

LEVELS = [(1, 6), (3, 12), (4, 15), (5, 6), (8, 15)]
VARIANTS = [(True, True), (False, False), (True, False), (False, True)]


@pytest.mark.parametrize("poly,bias", VARIANTS, ids=lambda v: str(v))
@pytest.mark.parametrize("levels,world", LEVELS)
def test_register_graded_on_natural_maps(levels, world, poly, bias):
    seed = 700 + 10 * levels + 2 * poly + bias
    case = make_case(n_points=1500, n_batch=16, feat_levels=levels, world_level=world, seed=seed, poly=poly, bias=bias)
    case, edges = with_boundary(case, seed)
    rng = np.random.default_rng(seed)
    local, T = scan(case, rng, 3000, world)
    ident = identity_set(case, rng, edges)
    cfg, octree, dec = build_cuda_models(case, DEV)
    dd = dec.c_descriptor(None)
    for ts in (1, 300):
        cs = scaled(case, ts)
        load_tables(octree, cs)
        od = octree._descriptor(None, None)
        grade_map(od, dd, cs, local, T, ident, 0.1 * _scale(world), f"L{levels} W{world} poly {poly} bias {bias} x{ts}")


@pytest.mark.parametrize("n", [1, 255, 256, 257, 1024 * 256, 1024 * 256 + 1, 10 ** 6])
def test_register_sizes(n):
    """Partial and full blocks, the 1024-block cap and one past it (a thread then takes two points), 10^6 points: copies
    of one graded set of 4096 scan points, launched at the identity."""
    case = make_case(n_points=1500, n_batch=16, feat_levels=3, world_level=12, seed=77)
    case, _ = with_boundary(case, 77)
    rng = np.random.default_rng(n % 1009)
    local, T = scan(case, rng, 4096, 12)
    q = _q32(local, T)
    cfg, octree, dec = build_cuda_models(case, DEV)
    od, dd = octree._descriptor(None, None), dec.c_descriptor(None)
    ref, rb = graded(case, q, F32(case["cfg"]["sigma"]), 0.1 * _scale(12), f"n = {n}")
    base = np.flatnonzero(~ref.dropped)
    base = base[rng.permutation(base.size)]
    idx = base[np.arange(n) % base.size]
    check(od, dd, rb, q[idx], idx, EYE, f"n = {n}")


@pytest.mark.parametrize("which", ["w = 1", "w < 2^-60"])
def test_register_kappa_extremes(which):
    case = make_case(n_points=1500, n_batch=16, feat_levels=4, world_level=12, seed=78, poly=False)
    case, edges = with_boundary(case, 78)
    rng = np.random.default_rng(3)
    local, T = scan(case, rng, 3000, 12)
    cfg, octree, dec = build_cuda_models(case, DEV)
    od, dd = octree._descriptor(None, None), dec.c_descriptor(None)
    kappa = 1e15 if which == "w = 1" else 1e-12 * _scale(12)
    sigma = F32(case["cfg"]["sigma"])
    q = _q32(local, T)
    ref, rb = graded(case, q, sigma, kappa, which)
    use = ref.valid & ~ref.dropped
    r = sigma * ref.pred[np.isin(ref.pt, np.flatnonzero(use))]
    w = gm_weight(r * r, kappa * kappa)
    if which == "w = 1":
        assert np.all(w == 1.0)
    else:
        assert np.mean(w < 2.0 ** -60) > 0.5, np.mean(w < 2.0 ** -60)
    keep = np.flatnonzero(~ref.dropped)
    check(od, dd, rb, local[keep], keep, T, which)


# ---- dense, adversarial and non-consecutive tables ------------------------------------------------------------------------

@pytest.mark.parametrize("levels", [2, 7])
def test_register_dense_tables(levels, monkeypatch):
    from shine_mapping_b200 import FeatureOctree
    monkeypatch.setattr(FeatureOctree, "_HASH_SLOTS_PER_NODE", 1)
    case = make_case(n_points=4000, n_batch=16, feat_levels=levels, seed=31 + levels, n_frames=2)
    case, edges = with_boundary(case, 31 + levels)
    rng = np.random.default_rng(levels)
    cfg, octree, dec = build_cuda_models(case, DEV)
    probe = check_octree_slots(octree, "dense")
    loads = [octree._levels[l].node_keys.numel() / octree._levels[l].hash_capacity
             for l in range(octree.free_level_num, octree.max_level + 1)]
    assert max(loads) > 0.5 and probe >= 2, (loads, probe)
    local, T = scan(case, rng, 3000, 12)
    ident = identity_set(case, rng, edges)
    dd = dec.c_descriptor(None)
    for ts in (1, 300):
        cs = scaled(case, ts)
        load_tables(octree, cs)
        grade_map(octree._descriptor(None, None), dd, cs, local, T, ident, 0.1 * _scale(12), f"dense L{levels} x{ts}")


@pytest.mark.parametrize("levels,poly", [(3, True), (5, False)])
def test_register_adversarial_tables(levels, poly):
    from shine_mapping_b200 import Decoder
    world = 12
    case, od, slots, sets = _adversarial_map(levels, world, poly, 40 + levels, [1024, 512, 256, 128, 64][:levels])
    rng = np.random.default_rng(levels)
    pts = []
    for i, ks in enumerate(sets):
        for name in ("stored", "absent_chain", "absent"):
            pts.append(_voxel_points(ks[name] if name != "stored" else ks[name][:200], world - i, rng))
    coord = rng.permutation(np.concatenate(pts)).astype(F32)
    dec = Decoder(make_config(levels, world, device=DEV, poly_int_on=poly))
    sd = dec.state_dict()
    for k, v in case["dec"].items():
        sd[k] = torch.from_numpy(v).to(DEV)
    dec.load_state_dict(sd)
    dd = dec.c_descriptor(None)
    keep = []
    for ts in (1, 300):
        cs = scaled(case, ts)
        feats = [torch.from_numpy(t).to(DEV) for t in cs["tables"]]
        keep += feats
        for i in range(levels):
            od.lv[i].features = feats[levels - 1 - i].data_ptr()
        grade_map(od, dd, cs, None, None, coord, 0.1 * _scale(world), f"adversarial L{levels} x{ts}", sigma=1.0)


@pytest.mark.parametrize("levels,drop", [(4, 1), (6, 3)])
def test_register_non_consecutive_levels(levels, drop):
    case = make_case(n_points=2000, n_batch=16, feat_levels=levels, seed=50 + levels + drop)
    case, edges = with_boundary(case, 50 + levels + drop)
    rng = np.random.default_rng(drop)
    cfg, octree, dec = build_cuda_models(case, DEV)
    dd = dec.c_descriptor(None)
    keep_lv = [i for i in range(levels) if i != drop]
    W = cfg.tree_level_world
    tables = case["tables"]
    keep_tables = [tables[levels - 1 - i] for i in reversed(keep_lv)]
    o2 = KeptLevels(case["oracle"], [W - i for i in keep_lv], keep_tables)
    case2 = dict(case, oracle=o2, cfg=dict(case["cfg"], tree_level_feat=levels - 1), tables=keep_tables)
    local, T = scan(case, rng, 3000, W)
    ident = np.concatenate((special_points(case["oracle"], rng), edges)).astype(F32)
    for ts in (1, 300):
        load_tables(octree, scaled(case, ts))
        full = octree._descriptor(None, None)
        od = clone(full)
        od.num_levels = levels - 1
        for j, i in enumerate(keep_lv):
            C.memmove(C.byref(od.lv[j]), C.byref(full.lv[i]), C.sizeof(full.lv[i]))
        grade_map(od, dd, scaled(case2, ts), local, T, ident, 0.1 * _scale(W),
                  f"levels {[od.lv[j].level for j in range(levels - 1)]} x{ts}")


# ---- the K-pose entry past its 512-pose chunk ------------------------------------------------------------------------------

def test_register_poses_rows_graded():
    """600 poses in one shine_register_normal_eq_poses call (two launches of 512 and 88): rows 0, 1, 511, 512 and 599
    graded against fp64 directly, with their block partials, and every seventh pose off the map all zero."""
    case = make_case(n_points=1500, n_batch=16, feat_levels=3, world_level=12, seed=79)
    case, _ = with_boundary(case, 79)
    rng = np.random.default_rng(9)
    sc = _scale(12)
    local, _ = scan(case, rng, 2000, 12)
    P = np.stack([_random_pose(rng, sc) for _ in range(600)])
    P[3::7, :3, 3] = (3.0, -3.0, 3.0)
    cfg, octree, dec = build_cuda_models(case, DEV)
    od, dd = octree._descriptor(None, None), dec.c_descriptor(None)
    sigma, kappa = F32(case["cfg"]["sigma"]), 0.1 * sc
    out, part = register(od, dd, local, P, sigma, kappa)
    assert np.array_equal(out[3::7], np.zeros_like(out[3::7]))
    for k in (0, 1, 511, 512, 599):
        ref, rb = graded(case, _q32(local, P[k]), sigma, kappa, f"pose {k} of 600")
        idx = np.arange(local.shape[0])
        if ref.n_dropped:
            continue                       # a point left out is in the launch: this row cannot be graded
        want, bound = rb.expect(idx)
        grade_reg(out[k], want, bound, f"pose {k} of 600")
        bw, bb = rb.expect_blocks(idx)
        grade_reg(part[k], bw, bb, f"pose {k} of 600: block partials")
