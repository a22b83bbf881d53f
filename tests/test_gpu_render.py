"""shine_render (csrc/shine_raycast.cu, DESIGN §14) against the fp64 oracle march of tests/raycast_oracle.py on the
kernel's camera rays (tests/render_rays.py), its normals against the fp64 gradient of tests/eikonal_bound.py, an analytic
plane, sizes and refusals, and end to end through `python -m shine_mapping_b200.render` and `evaluate depth`.

March grading follows tests/test_gpu_raycast.py: on rays whose visited masked samples all have |s| above their bound,
hit / miss and the bracket index are exact and the range lies within that module's bounds.  The oracle's rays are the
kernel's (bit for bit: the same fp32 formula), with r = t_max and beyond = 0, so its lattice is the view's.
Normals: n = -g / |g| at the GPU's hit point x = o + t d (fp32).  With |g_gpu - g| <= e_g per component (EikRef's
per-point bound), |n_gpu - n| <= 2 |e_g| / |g| plus the normalisation's roundings (8 u); points at a ReLU kink or with
|g| <= 4 |e_g| are dropped."""
import contextlib
import ctypes as C
import math

import numpy as np
import pytest
import torch

from tests import raycast_oracle as ro
from tests import render_rays as rr
from tests.error_bound import U, oracle64
from tests.parity_utils import build_cuda_models, make_case

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
LEAF = 2.0 / 4096
NAN_BITS = 0x7FC00000


@pytest.fixture(scope="module", autouse=True)
def _lib(built_lib):
    assert torch.cuda.is_available()
    return built_lib


def _camera(model, W, H, a=0.0, b=0.0, c=0.0, d=0.0):
    from shine_mapping_b200 import _abi
    if model == "pinhole":
        return _abi.ShineCamera(_abi.CAMERA_PINHOLE, W, H, a, b, c, d, 0.0, 0.0)
    return _abi.ShineCamera(_abi.CAMERA_RANGE_IMAGE, W, H, 0.0, 0.0, 0.0, 0.0, a, b)


def _dirs(model, W, H, a, b, c=0.0, d=0.0):
    return rr.pinhole_dirs(W, H, a, b, c, d) if model == "pinhole" else rr.range_image_dirs(W, H, a, b)


def _render(octree, dec, cam, pose12, h, t_max, iters=6, mask_level=0, t_min=0.0, outs=(True, True, True, True),
            n=None):
    """-> (rc, range, depth, normal, status) as numpy; the buffers (n pixels, default the view's) start as sentinels
    (7.0, 9)."""
    from shine_mapping_b200 import _abi
    n = cam.width * cam.height if n is None else n
    bufs = [torch.full((n,), 7.0, device=DEV), torch.full((n,), 7.0, device=DEV), torch.full((n, 3), 7.0, device=DEV),
            torch.full((n,), 9, dtype=torch.uint8, device=DEV)]
    pose = (C.c_float * 12)(*np.asarray(pose12, dtype=np.float32).reshape(12).tolist())
    rc = _abi.lib().shine_render(C.byref(octree._descriptor(None, None)), C.byref(dec.c_descriptor(None)), C.byref(cam),
                                 pose, float(np.float32(h)), float(np.float32(t_min)), float(np.float32(t_max)), iters,
                                 mask_level, *[_abi.ptr(b) if w else None for b, w in zip(bufs, outs)],
                                 _abi.stream_ptr(DEV))
    torch.cuda.synchronize()
    return (rc, *[b.cpu().numpy() for b in bufs])


@contextlib.contextmanager
def _oracle_rays(d, r):
    """raycast_oracle.march with the view's rays in place of its point-to-origin rays."""
    saved = ro.rays
    ro.rays = lambda origin, points: (d, r)
    try:
        yield
    finally:
        ro.rays = saved


def _look_at(origin, target, roll=0.0):
    """A camera-to-map rotation whose camera z axis points from origin to target."""
    z = np.asarray(target, np.float64) - np.asarray(origin, np.float64)
    z /= np.linalg.norm(z)
    up = np.array([math.sin(roll), 0.0, math.cos(roll)])
    x = np.cross(up, z) if abs(np.dot(up, z)) < 0.99 else np.cross([0.0, 1.0, 0.0], z)
    x /= np.linalg.norm(x)
    return np.stack([x, np.cross(z, x), z], 1)


def _tilted(rng):
    """A sensor-to-map rotation: any heading, pitch and roll within 0.2 rad."""
    yaw, pitch, roll = rng.uniform(-np.pi, np.pi), rng.uniform(-0.2, 0.2), rng.uniform(-0.2, 0.2)
    cz, sz, cy, sy, cx, sx = np.cos(yaw), np.sin(yaw), np.cos(pitch), np.sin(pitch), np.cos(roll), np.sin(roll)
    return np.array([[cz, -sz, 0], [sz, cz, 0], [0, 0, 1]]) @ np.array([[cy, 0, sy], [0, 1, 0], [-sy, 0, cy]]) @ \
        np.array([[1, 0, 0], [0, cx, -sx], [0, sx, cx]])


def _pose12(R, o):
    return np.concatenate([np.asarray(R, np.float64), np.asarray(o, np.float64).reshape(3, 1)], 1).astype(np.float32)


def _lively(case):
    from tests.test_gpu_raycast import _lively as lively
    return lively(case)


def _views(case, rng):
    """(model, W, H, camera parameters, pose12, h, t_max) per view: from the sensor origin (empty space), from inside a
    node and from outside the map's cube, in both camera models."""
    surf = case["frames"][0].astype(np.float64)
    inside = surf[0] + 0.1 * LEAF
    outside = np.array([1.25, 0.01, 0.0])
    reach = 1.2 * float(np.linalg.norm(surf, axis=1).max())
    out = []
    # each pinhole looks at a surface sample, which the scan saw from the sensor origin
    for o, t_max, size in (((0.0, 0.0, 0.0), reach, 2), (inside, 60 * LEAF, 1), (outside, 1.3 + reach, 1)):
        target = surf[rng.integers(surf.shape[0])]
        h = 0.6 * LEAF if t_max < 0.2 else 0.002
        R = _look_at(o, target, rng.uniform(-0.3, 0.3))
        out.append(("pinhole", 20 * size, 15 * size, (8.0 * size, 8.0 * size, 9.5 * size, 7.0 * size), _pose12(R, o), h,
                    t_max))
        out.append(("range", 24 * size, 12 * size, (15.0, -30.0), _pose12(_tilted(rng), o), h, t_max))
    return out


def grade_view(o, dec, octree, cdec, view, mask_level, iters=6, what=""):
    """-> (rays, hits, ambiguous, hit mask of the unambiguous rays, got range) of one view, asserting the rules."""
    model, W, H, p, pose12, h, t_max = view
    rc, got_t, got_depth, got_n, got_s = _render(octree, cdec, _camera(model, W, H, *p), pose12, h, t_max, iters,
                                                 mask_level)
    assert rc == 0
    c, cz = _dirs(model, W, H, *p)
    origin, d = rr.map_rays(c, pose12)
    n = W * H
    with _oracle_rays(d, np.full(n, np.float32(t_max), np.float32)):
        want = ro.march(o, dec, origin, np.zeros((n, 3)), h, 0.0, 0.0, t_max, iters, mask_level)
    assert set(np.unique(got_s).tolist()) <= {0, 1}
    miss, hit_ = got_s == 0, got_s == 1
    assert np.isnan(got_t[miss]).all() and np.isfinite(got_t[hit_]).all()
    assert np.isnan(got_depth[miss]).all() and np.isnan(got_n[miss]).all()
    assert np.array_equal(got_depth.view(np.uint32)[hit_], (got_t[hit_] * cz[hit_]).astype(np.float32).view(np.uint32))
    ok = ~want["ambiguous"]
    bad = ok & (want["hit"] != hit_)
    assert not bad.any(), f"{what}: {int(bad.sum())} unambiguous rays disagree on hit / miss"
    hit = ok & want["hit"]
    k = want["k"][hit]
    lo, hi = ro.lattice_t(k - 1, h, 0.0), ro.lattice_t(k, h, 0.0)
    g = got_t[hit]
    assert ((g >= lo) & (g <= hi)).all(), f"{what}: a hit outside its lattice bracket"
    den = want["sa"] - want["sb"] - want["Pa"] - want["Pb"]
    fine = hit & ~want["refine_ambiguous"] & (den > 0)
    if fine.any():
        w = want["tb"][fine] - want["ta"][fine]
        bound = w * (want["Pa"][fine] + want["Pb"][fine]) / den[fine] + 8 * U * (np.abs(want["t"][fine]) + w)
        err = np.abs(got_t[fine].astype(np.float64) - want["t"][fine])
        assert (err <= bound).all(), f"{what}: refined range off by {err.max():.3g}"
    split = hit & want["refine_ambiguous"]
    if split.any():
        err = np.abs(got_t[split].astype(np.float64) - want["t"][split])
        bound = want["div_w"][split] + 8 * U * (np.abs(want["t"][split]) + want["div_w"][split])
        assert (err <= bound).all(), f"{what}: refined range off by {err.max():.3g} after a split bracket"
    return n, int(hit_.sum()), int((~ok).sum()), hit_, got_t, got_n, origin, d


@pytest.mark.parametrize("levels", [1, 3, 4, 5, 8])
@pytest.mark.parametrize("poly,bias", [(True, True), (False, False), (True, False), (False, True)])
def test_render_matches_oracle(levels, poly, bias):
    case = _lively(make_case(n_points=1500, n_batch=16, feat_levels=levels, seed=900 + 10 * levels + 2 * poly + bias,
                             poly=poly, bias=bias))
    cfg, octree, cdec = build_cuda_models(case, DEV)
    o, dec = oracle64(case)
    rng = np.random.default_rng(levels * 4 + 2 * poly + bias + 50)
    rays = hits = amb = 0
    for ml in sorted({0, levels - 1}):
        for j, view in enumerate(_views(case, rng)):
            r = grade_view(o, dec, octree, cdec, view, ml, what=f"view {j} ({view[0]}) mask level {ml}")
            rays, hits, amb = rays + r[0], hits + r[1], amb + r[2]
    print(f"levels {levels} poly {poly} bias {bias}: {rays} rays, {hits} hits, ambiguous {amb}")
    # one level, linear blend, no biases: the field changes sign on few of these rays (3 in the first run)
    assert hits >= (3 if levels == 1 and not poly and not bias else 20)
    # views see more surface per ray than test_gpu_raycast's sets: at 8 levels up to 17 % are ambiguous (first run)
    assert amb <= 0.2 * rays


def test_render_normals_against_fp64():
    """Normals at the GPU's hit points against -g / |g| of EikRef, on both camera models and both mask levels."""
    from tests.eikonal_bound import EikRef
    graded = 0
    for levels, poly in ((3, True), (4, False), (5, True)):
        case = _lively(make_case(n_points=1500, n_batch=16, feat_levels=levels, seed=950 + levels, poly=poly))
        cfg, octree, cdec = build_cuda_models(case, DEV)
        o, dec = oracle64(case)
        rng = np.random.default_rng(levels)
        for ml in (0, levels - 1):
            for view in _views(case, rng):
                _, _, _, hit, t, nrm, origin, d = grade_view(o, dec, octree, cdec, view, ml)
                if not hit.any():
                    continue
                x = ro.positions(origin, d[hit], t[hit])
                m = x.shape[0]
                ref = EikRef(dict(case, coord=x, label=np.zeros(m, np.float32), weight=-np.ones(m, np.float32)),
                             weight_e=0.0)
                g, eg = ref.g, ref.eg
                len_g, len_e = np.linalg.norm(g, axis=1), np.linalg.norm(eg, axis=1)
                keep = ~ref.kink & (len_g > 4 * len_e)
                want = -g[keep] / len_g[keep, None]
                bound = 2 * len_e[keep, None] / len_g[keep, None] + 8 * U
                err = np.abs(nrm[hit][keep].astype(np.float64) - want)
                assert (err <= bound).all(), f"normal off by {err.max():.3g} (bound {bound.max():.3g})"
                graded += int(keep.sum())
    print(f"normals graded: {graded}")
    assert graded >= 100


def _plane_map():
    """test_gpu_raycast's analytic plane: the field is exactly x0 - x near x = x0."""
    from shine_mapping_b200 import Decoder, FeatureOctree
    from shine_mapping_b200.feature_octree import morton_to_points
    from tests.parity_utils import make_config
    cfg = make_config(feat_levels=1, device=DEV, poly_int_on=False, mc_vis_level=1)
    octree = FeatureOctree(cfg)
    x0 = np.float32(0.0123)
    g = np.arange(-40, 41) * 0.4 * LEAF
    gy = np.arange(-12, 13) * 0.4 * LEAF
    box = np.stack(np.meshgrid(x0 + g, gy, gy, indexing="ij"), -1).reshape(-1, 3).astype(np.float32)
    octree.update(torch.from_numpy(box).to(DEV))
    level = octree.max_level
    st = octree._levels[level]
    nodes = morton_to_points(st.node_keys).cpu().numpy()
    ids = st.node_ids.cpu().numpy()
    table = octree.hier_features[0]
    feat = np.zeros(tuple(table.shape), dtype=np.float32)
    res = 2.0 ** level
    for c in range(8):
        xc = -1.0 + 2.0 * (nodes[:, 0] + ((c >> 2) & 1)) / res
        feat[ids[:, c], 0] = (xc - np.float64(x0)).astype(np.float32)
    with torch.no_grad():
        table.copy_(torch.from_numpy(feat))
    dec = Decoder(cfg)
    sd = {k: torch.zeros_like(v) for k, v in dec.state_dict().items()}
    sd["layers.0.weight"][0, 0] = 1.0
    sd["layers.0.bias"][0] = 1.0
    sd["layers.1.weight"][0, 0] = 1.0
    sd["lout.weight"][0, 0] = 1.0
    sd["lout.bias"][0] = -1.0
    dec.load_state_dict(sd)
    return cfg, octree, dec, x0


def test_render_exact_plane():
    """A pinhole camera looking along +x at the plane x = x0: depth = x0 - o_x at every pixel, normal (-1, 0, 0).
    Depth: the plane test's bound on t (32 u (2 + B) / d_x + 8 u t) times c_z = d_x, plus one rounding.  Normal: the
    features at the hit are at most one leaf cell (2 / res) from 0, so each blend-gradient component sums 8 products of
    at most 2 / res . res / 2 with fp32 roundings: 64 u covers it with the normalisation."""
    from shine_mapping_b200 import render
    from shine_mapping_b200.rgbd import RGBDCamera
    cfg, octree, dec, x0 = _plane_map()
    origin = np.array([x0 - 60 * 0.4 * LEAF, 0.0, 0.0], dtype=np.float32)
    pose = np.eye(4)
    pose[:3, :3] = [[0, 0, 1], [1, 0, 0], [0, 1, 0]]                 # camera z -> map x, x -> y, y -> z
    pose[:3, 3] = origin.astype(np.float64) / cfg.scale
    cam = RGBDCamera(9, 9, 4 / 0.15, 4 / 0.15, 4.0, 4.0)
    view = render.render_view(cfg, octree, dec, pose, cam, max_range_m=100 * 0.4 * LEAF / cfg.scale,
                              step_m=0.7 * LEAF / cfg.scale, refine_iters=8)
    assert bool(view["hit"].all())
    c, cz = rr.pinhole_dirs(9, 9, cam.fx, cam.fy, cam.cx, cam.cy)
    want = np.float64(x0) - np.float64(origin[0])
    t_want = want / cz.astype(np.float64)
    tol = (32 * U * 3 / cz + 8 * U * t_want) * cz + U * want
    got = view["depth"].cpu().numpy().reshape(-1) * cfg.scale
    err = np.abs(got - want)
    print(f"plane: worst |depth - exact| {err.max():.3g} (scaled), {float((err / tol).max()):.3f} of the bound")
    assert (err <= tol).all()
    nrm = view["normal"].cpu().numpy().reshape(-1, 3).astype(np.float64)
    nerr = np.abs(nrm - [-1.0, 0.0, 0.0]).max()
    print(f"plane: worst normal error {nerr:.3g}")
    assert nerr <= 64 * U


def test_render_sizes_determinism_and_refusals():
    from shine_mapping_b200 import _abi
    case = _lively(make_case(n_points=1500, n_batch=16, feat_levels=4, seed=977))
    cfg, octree, cdec = build_cuda_models(case, DEV)
    surf = case["frames"][0].astype(np.float64)
    R = _look_at((0, 0, 0), surf[0])
    pose = _pose12(R, (0, 0, 0))
    h, t_max = 0.6 * LEAF, 1.2 * float(np.linalg.norm(surf, axis=1).max())
    big = _camera("pinhole", 1920, 1080, 800.0, 800.0, 959.5, 539.5)
    rc, t0, d0, n0, s0 = _render(octree, cdec, big, pose, h, t_max)
    assert rc == 0
    rc, t1, d1, n1, s1 = _render(octree, cdec, big, pose, h, t_max)
    for a, b in ((t0, t1), (d0, d1), (n0, n1)):
        assert np.array_equal(a.view(np.uint32), b.view(np.uint32))
    assert np.array_equal(s0, s1)
    print(f"1920 x 1080: {int(s0.sum())} hits")
    assert s0.sum() > 1000
    t0, s0 = t0.reshape(1080, 1920), s0.reshape(1080, 1920)
    # a window of the same camera: the principal point moved by whole pixels gives the same rays
    for (W, H, u0, v0) in ((1, 1, 960, 540), (3 * 128 + 17, 1, 700, 520), (33, 7, 900, 530)):
        cam = _camera("pinhole", W, H, 800.0, 800.0, 959.5 - u0, 539.5 - v0)
        rc, t, _, _, s = _render(octree, cdec, cam, pose, h, t_max)
        assert rc == 0
        assert np.array_equal(t.view(np.uint32), t0[v0:v0 + H, u0:u0 + W].reshape(-1).view(np.uint32))
        assert np.array_equal(s, s0[v0:v0 + H, u0:u0 + W].reshape(-1))
    # only some outputs wanted
    rc, t, d, nn, s = _render(octree, cdec, _camera("pinhole", 1, 1, 800.0, 800.0, -0.5, -0.5), pose, h, t_max,
                              outs=(False, True, False, False))
    assert rc == 0 and t[0] == 7.0 and nn[0, 0] == 7.0 and s[0] == 9 and d[0] != 7.0

    good = dict(cam=_camera("range", 16, 8, 10.0, -20.0), pose=pose, h=h, t_max=t_max, iters=6, mask_level=0)
    bad_pose = pose.copy()
    bad_pose[1, 3] = np.inf
    cases = [
        ("width 0", dict(cam=_camera("range", 0, 8, 10.0, -20.0)), -1),
        ("height -1", dict(cam=_camera("pinhole", 8, -1, 1.0, 1.0, 0.0, 0.0)), -1),
        ("over 2^31 pixels", dict(cam=_camera("pinhole", 65536, 32769, 1.0, 1.0, 0.0, 0.0)), -1),
        ("fx 0", dict(cam=_camera("pinhole", 8, 8, 0.0, 1.0, 0.0, 0.0)), -1),
        ("fy < 0", dict(cam=_camera("pinhole", 8, 8, 1.0, -1.0, 0.0, 0.0)), -1),
        ("cx nan", dict(cam=_camera("pinhole", 8, 8, 1.0, 1.0, float("nan"), 0.0)), -1),
        ("fov up == down", dict(cam=_camera("range", 8, 8, 5.0, 5.0)), -1),
        ("fov inf", dict(cam=_camera("range", 8, 8, float("inf"), 0.0)), -1),
        ("model 7", dict(cam=_abi.ShineCamera(7, 8, 8, 1.0, 1.0, 0.0, 0.0, 1.0, 0.0)), -1),
        ("pose inf", dict(pose=bad_pose), -1),
        ("h 0", dict(h=0.0), -1),
        ("t_max inf", dict(t_max=float("inf")), -1),
        ("t_max <= t_min", dict(t_max=0.0), -1),
        ("refine 33", dict(iters=33), -1),
        ("refine -1", dict(iters=-1), -1),
        ("mask level 4", dict(mask_level=4), -1),
        ("mask level -1", dict(mask_level=-1), -1),
    ]
    for name, over, code in cases:
        a = dict(good, **over)
        rc, t, d, nn, s = _render(octree, cdec, a["cam"], a["pose"], a["h"], a["t_max"], a["iters"], a["mask_level"],
                                  n=128)
        assert rc == code, name
        assert (t == 7.0).all() and (d == 7.0).all() and (nn == 7.0).all() and (s == 9).all(), name
    # a decoder other than 8 -> 32 -> 32 -> 1
    dd = cdec.c_descriptor(None)
    dd.hidden = 16
    buf = torch.full((128,), 7.0, device=DEV)
    rc = _abi.lib().shine_render(C.byref(octree._descriptor(None, None)), C.byref(dd), C.byref(good["cam"]),
                                 (C.c_float * 12)(*pose.reshape(12).tolist()), float(h), 0.0, float(t_max), 6, 0,
                                 _abi.ptr(buf), None, None, None, _abi.stream_ptr(DEV))
    torch.cuda.synchronize()
    assert rc == -2 and (buf == 7.0).all()
    with pytest.raises(_abi.ShineB200Error):
        _abi.check(_abi.lib().shine_render(None, None, None, None, 1.0, 0.0, 2.0, 6, 0, None, None, None, None, None),
                   "shine_render")


# ---- end to end ------------------------------------------------------------------------------------------------------------

# The first measured run (H100): drive hit ratio 0.9891, median 0.0170 m; RGB-D AbsRel 0.0014, r1 0.9997, complete
# 0.7442.  These limits leave a margin, as test_gpu_raycast's do (DESIGN §14).
DRIVE_LIMITS = dict(hit_ratio=0.90, median_m=0.05)
RGBD_LIMITS = dict(abs_rel=0.01, r1=0.98, complete=0.65)


def test_render_drive_end_to_end(tmp_path, capsys):
    """The 20-frame drive mapped from every other frame; range images of the held-out frames against their scans: each
    measured point's pixel (nearest elevation row and azimuth column) keeps its nearest range."""
    import yaml
    from shine_mapping_b200 import batch_loop, render, synth
    from shine_mapping_b200.raycast import map_pose
    from shine_mapping_b200.scans import LiDARDataset
    from shine_mapping_b200.config import SHINEConfig
    paths = synth.write_drive(str(tmp_path / "drive"), n_frames=20)
    doc = {"setting": dict(pc_path=paths["pc_path"], pose_path=paths["pose_path"], calib_path="", begin_frame=0,
                           end_frame=100, every_frame=2, first_frame_ref=True, device=DEV),
           "process": {"min_range_m": 2.75, "pc_radius_m": 30.0, "min_z_m": -10.0, "rand_downsample": False,
                       "vox_down_m": 0.1},
           "sampler": {"surface_sample_range_m": 0.3, "surface_sample_n": 3, "free_sample_begin_ratio": 0.3,
                       "free_sample_end_dist_m": 0.8, "free_sample_n": 3},
           "octree": {"tree_level_world": 12, "tree_level_feat": 3, "leaf_vox_size": 0.2, "feature_dim": 8},
           "continual": {"continual_learning_reg": False, "window_replay_on": False},
           "optimizer": {"batch_size": 8192, "learning_rate": 0.01},
           "eval": {"save_freq_iters": 1000, "vis_freq_iters": 100000, "mc_res_m": 0.1}}
    cfg_path = tmp_path / "cfg.yaml"
    cfg_path.write_text(yaml.safe_dump(doc))
    run = tmp_path / "run"
    batch_loop.main([str(cfg_path), "--scans", "--iters", "1000", "--run-path", str(run)])
    ckpt = run / "model" / "model_iter_1000.pth"
    out = tmp_path / "render"
    capsys.readouterr()
    assert render.main([str(cfg_path), str(ckpt), "--out", str(out), "--frames", "1:20:2", "--npz"]) == 0
    printed = capsys.readouterr().out
    assert printed.count("frame ") == 10
    config = SHINEConfig()
    config.load(str(cfg_path))
    ds = LiDARDataset(config)
    hits = meas = 0
    errs = []
    for f in range(1, 20, 2):
        z = np.load(out / "npz" / f"{f}.npz")
        assert z["depth"].shape == (64, 1024) and z["normal"].shape == (64, 1024, 3)
        assert (out / "depth" / f"{f}.png").exists() and (out / "normal" / f"{f}.png").exists()
        pose = map_pose(ds, f)
        cam = render.lidar_camera(ds, f, pose)
        pts = ds.processor.points(ds.read_frame(f), pose).double().cpu().numpy() / config.scale
        v = (pts - pose[:3, 3]) @ pose[:3, :3]
        rng_m = np.linalg.norm(v, axis=1)
        el = np.degrees(np.arctan2(v[:, 2], np.hypot(v[:, 0], v[:, 1])))
        az = np.arctan2(v[:, 1], v[:, 0])
        row = np.rint((cam.fov_up - el) / (cam.fov_up - cam.fov_down) * (cam.height - 1)).astype(int)
        col = np.rint((np.pi - az) / (2 * np.pi) * cam.width).astype(int) % cam.width
        best = np.full((cam.height, cam.width), np.inf)
        np.minimum.at(best, (row, col), rng_m)
        has = np.isfinite(best)
        got = z["range"]
        hit = has & z["hit"]
        meas += int(has.sum())
        hits += int(hit.sum())
        errs.append(np.abs(got[hit] - best[hit]))
    hit_ratio = hits / meas
    median = float(np.median(np.concatenate(errs)))
    print(f"drive range images: {meas} measured pixels, hit ratio {hit_ratio:.4f}, median |range - measured| "
          f"{median:.4f} m")
    assert hit_ratio >= DRIVE_LIMITS["hit_ratio"] and median <= DRIVE_LIMITS["median_m"]


def test_evaluate_depth_end_to_end(tmp_path, capsys):
    """A synthetic RGB-D sequence (test_gpu_rgbd's scene and cameras) mapped from every other frame, the held-out frames
    rendered and scored with eval_depth's metrics."""
    import csv
    from shine_mapping_b200 import batch_loop, evaluate, rgbd
    from tests.test_gpu_rgbd import _rgbd_args, _yaml, write_rgbd_sequence
    seq = write_rgbd_sequence(str(tmp_path / "seq"))
    cfg = _yaml(tmp_path, setting__every_frame=2, eval__save_freq_iters=1000, eval__vis_freq_iters=100000)
    run = tmp_path / "run"
    batch_loop.main([cfg, *_rgbd_args(seq), "--iters", "1000", "--run-path", str(run)])
    ckpt = run / "model" / "model_iter_1000.pth"
    assert ckpt.exists()
    capsys.readouterr()
    out_csv, out_dir = tmp_path / "eval" / "depth.csv", tmp_path / "eval" / "views"
    assert evaluate.main(["depth", cfg, str(ckpt), *_rgbd_args(seq), "--csv", str(out_csv), "--out", str(out_dir)]) == 0
    printed = capsys.readouterr().out
    assert printed.count("frame ") == 5 and "mean:" in printed
    with open(out_csv) as fh:
        rows = list(csv.DictReader(fh))
    assert [r["frame"] for r in rows] == ["1", "3", "5", "7", "9", "mean"]
    mean = rows[-1]
    png = rgbd.read_depth(str(out_dir / "depth" / "1.png"), pinned=False)
    assert tuple(png.shape) == (120, 160)
    abs_rel, r1, complete = float(mean["AbsRel"]), float(mean["r1"]), float(mean["complete"])
    print(f"rgbd held-out depth: AbsRel {abs_rel:.4f}, AbsDiff {float(mean['AbsDiff']):.4f} m, RMSE "
          f"{float(mean['RMSE']):.4f} m, r1 {r1:.4f}, complete {complete:.4f}")
    assert abs_rel <= RGBD_LIMITS["abs_rel"] and r1 >= RGBD_LIMITS["r1"] and complete >= RGBD_LIMITS["complete"]
