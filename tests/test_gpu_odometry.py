"""Pose-free mapping on the GPU: shine_register_normal_eq against an fp64 restatement built on EikRef (per-element bounds
derived from its bounds for pred and g), registration of a scan to a map of earlier frames, and a remap from the written poses that reproduces the pose-free run bit for bit."""
import itertools
import math
import os

import numpy as np
import pytest
import torch

from shine_mapping_b200 import odometry, synth
from shine_mapping_b200.trainer import SdfTrainer
from tests.eikonal_bound import EikRef
from tests.error_bound import U, grade_values
from tests.parity_utils import build_cuda_models, dec_keys, make_case

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
E64 = 2.0 ** -53


# ---- the kernel against fp64 -------------------------------------------------------------------------------------------------

def _trained(seed, bias=True, steps=80):
    """A case whose tables and decoder were trained on its street samples by the fused step (the map registration sees)."""
    case = make_case(n_points=4000, n_batch=8192, feat_levels=3, seed=seed, bias=bias)
    cfg, octree, dec = build_cuda_models(case, DEV)
    trainer = SdfTrainer(cfg, octree, dec)
    c, l, w = (torch.from_numpy(case[k]).to(DEV) for k in ("coord", "label", "weight"))
    trainer.zero_grad()
    for _ in range(steps):
        trainer.forward_backward(c, l, w)
        trainer.optimizer_step(zero_grad=True)
    torch.cuda.synchronize()
    case["tables"] = [p.detach().cpu().numpy().copy() for p in octree.hier_features]
    params = dict(dec.named_parameters())
    case["dec"] = {k: params[k].detach().cpu().numpy().copy() for k in dec_keys(case)}
    case["cfg"] = dict(case["cfg"], sigma=float(np.float32(cfg.sigma_sigmoid)))       # the fp32 sigma the kernel gets
    return case, odometry.ScanToMapRegistration(cfg, octree, dec)


@pytest.fixture(scope="module")
def trained():
    return _trained(0)


@pytest.fixture(scope="module")
def trained_nobias():
    return _trained(1, bias=False)


def _q32(local, pose):
    """The kernel's q = R p + t: fp32, ((R0 x + R1 y) + R2 z) + t, every operation rounded on its own."""
    R, t = pose[:3, :3].astype(np.float32), pose[:3, 3].astype(np.float32)
    x, y, z = local[:, 0], local[:, 1], local[:, 2]
    return np.stack([((R[a, 0] * x + R[a, 1] * y) + R[a, 2] * z) + t[a] for a in range(3)], 1).astype(np.float32)


def _random_pose(rng, scale):
    yaw, pitch, roll = rng.uniform(-0.3, 0.3), rng.uniform(-0.03, 0.03), rng.uniform(-0.03, 0.03)
    cz, sz, cy, sy, cx, sx = math.cos(yaw), math.sin(yaw), math.cos(pitch), math.sin(pitch), math.cos(roll), math.sin(roll)
    T = np.eye(4)
    T[:3, :3] = np.array([[cz, -sz, 0], [sz, cz, 0], [0, 0, 1]]) @ np.array([[cy, 0, sy], [0, 1, 0], [-sy, 0, cy]]) @ \
        np.array([[1, 0, 0], [0, cx, -sx], [0, sx, cx]])
    T[:3, 3] = rng.uniform(-0.5, 0.5, 3) * scale
    return T


class RegRef:
    """fp64 values of the 29 outputs and their bounds for points whose q (fp32) the kernel computes bit for bit.
    r = sigma pred with e_r = sigma P + u |r|; Jr = [g, q x g] with e_J = [e_g, |q| x e_g (crosswise)]; w = (k^2 / (k^2 +
    r^2))^2 with e_w = |w'(r)| e_r + 2 e_r^2 / k^2 (|w''| <= 4 / k^2); per point e(w a c) <= e_w |a c| + w (e_a |c| + |a| e_c)
    (+ second-order terms); the fp64 products and sums add 8 (n + 8) 2^-53 of the sum of |terms|.  `mult` copies of every
    point (the million-point launch tiles a smaller set)."""

    def __init__(self, case, q, kappa):
        n = q.shape[0]
        c = dict(case, coord=q, label=np.zeros(n, np.float32), weight=-np.ones(n, np.float32))
        self.ref = ref = EikRef(c, weight_e=0.0)
        self.valid = ref.geo[0]["ix"][:, 0] >= 0
        self.kink = ref.kink & self.valid
        self.q, self.kappa, self.sigma = q, kappa, ref.sigma

    def expect(self, keep, mult=1):
        ref, m = self.ref, keep & self.valid
        g, eg = ref.g[m], ref.eg[m]
        r = self.sigma * ref.pred[m]
        er = self.sigma * ref.P[m] + U * np.abs(r)
        q = self.q[m].astype(np.float64)
        aq = np.abs(q)
        J = np.concatenate((g, np.cross(q, g)), 1)
        eJ = np.concatenate((eg, np.stack([aq[:, 1] * eg[:, 2] + aq[:, 2] * eg[:, 1], aq[:, 2] * eg[:, 0] + aq[:, 0] * eg[:, 2],
                                           aq[:, 0] * eg[:, 1] + aq[:, 1] * eg[:, 0]], 1)), 1)
        k2 = self.kappa ** 2
        den = k2 + r * r
        w = (k2 / den) ** 2
        ew = 4 * k2 * k2 * np.abs(r) / den ** 3 * er + 2 * er * er / k2
        iu = np.triu_indices(6)
        Hp = w[:, None] * (J[:, iu[0]] * J[:, iu[1]])
        eH = (ew[:, None] * np.abs(J[:, iu[0]] * J[:, iu[1]]) + w[:, None] * (eJ[:, iu[0]] * np.abs(J[:, iu[1]]) +
              np.abs(J[:, iu[0]]) * eJ[:, iu[1]]) + w[:, None] * eJ[:, iu[0]] * eJ[:, iu[1]])
        bp = w[:, None] * J * r[:, None]
        eb = (ew[:, None] * np.abs(J * r[:, None]) + w[:, None] * (eJ * np.abs(r)[:, None] + np.abs(J) * er[:, None]) +
              w[:, None] * eJ * er[:, None])
        cp = w * r * r
        ec = ew * r * r + w * (2 * np.abs(r) * er + er * er)
        terms = np.concatenate((Hp, bp, cp[:, None]), 1)
        bounds = np.concatenate((eH, eb, ec[:, None]), 1)
        total = int(m.sum()) * mult
        want = mult * terms.sum(0)
        bound = mult * bounds.sum(0) + 8 * (total + 8) * E64 * mult * np.abs(terms).sum(0)
        return np.concatenate((want, [total])), np.concatenate((bound, [0.0]))


def _launch(reg, points, pose_scaled, kappa):
    reg.out.fill_(float("nan"))
    reg.launch(torch.from_numpy(np.ascontiguousarray(points, dtype=np.float32)).to(DEV), pose_scaled, kappa)
    return reg.out.cpu().numpy().copy()


def _grade(got, ref, keep, what, mult=1):
    want, bound = ref.expect(keep, mult)
    assert got[28] == want[28], f"{what}: count {got[28]} != {want[28]}"
    grade_values(got[:21], want[:21], bound[:21], what, "H", "register bounds")
    grade_values(got[21:27], want[21:27], bound[21:27], what, "b", "register bounds")
    grade_values(got[27:28], want[27:28], bound[27:28], what, "cost", "register bounds")
    return want


def _scan(case, rng, n, noise_m, scale):
    world = np.concatenate([np.asarray(f, np.float64) for f in case["frames"]])
    pts = world[rng.integers(0, world.shape[0], n)] + rng.normal(0, noise_m * scale, (n, 3))
    return pts


@pytest.mark.parametrize("seed", [0, 1, 2])
def test_kernel_against_fp64_random_poses(trained, seed):
    case, reg = trained
    rng = np.random.default_rng(seed)
    kappa = 0.1 * reg.scale
    T = _random_pose(rng, reg.scale)
    world = _scan(case, rng, 20000, 0.05, reg.scale)
    local = ((world - T[:3, 3]) @ T[:3, :3]).astype(np.float32)          # T^-1 applied: the scan in its own frame
    q = _q32(local, T)
    ref = RegRef(case, q, kappa)
    keep = ~ref.kink
    assert ref.valid[keep].sum() > 10000, "most points of a scan of the map lie on it"
    got = _launch(reg, local[keep], T, kappa)
    ref2 = RegRef(case, q[keep], kappa)
    _grade(got, ref2, np.ones(int(keep.sum()), bool), f"seed {seed}")
    again = _launch(reg, local[keep], T, kappa)
    assert np.array_equal(got.view(np.int64), again.view(np.int64)), "two launches differ"


def _clean(case, local, pose, kappa):
    """local points without the ReLU-kink points, their q and the reference."""
    q = _q32(local, pose)
    keep = ~RegRef(case, q, kappa).kink
    return local[keep], RegRef(case, q[keep], kappa)


@pytest.mark.parametrize("n", [0, 1, 256 * 3 + 37, 1000])
def test_kernel_sizes(trained, n):
    case, reg = trained
    rng = np.random.default_rng(10 + n)
    kappa = 0.2 * reg.scale
    T = _random_pose(rng, reg.scale)
    world = _scan(case, rng, max(n, 1) + 64, 0.02, reg.scale)
    local, ref = _clean(case, ((world - T[:3, 3]) @ T[:3, :3]).astype(np.float32), T, kappa)
    local = local[:n]
    if n:
        ref = RegRef(case, _q32(local, T), kappa)
    got = _launch(reg, local.reshape(-1, 3), T, kappa)
    if n == 0:
        assert np.array_equal(got, np.zeros(29))
        return
    _grade(got, ref, np.ones(n, bool), f"n = {n}")


def test_kernel_million_points(trained):
    """10^6 points (the grid-stride loop with the block cap): 250 copies of 4000 clean points."""
    case, reg = trained
    rng = np.random.default_rng(5)
    kappa = 0.1 * reg.scale
    T = _random_pose(rng, reg.scale)
    world = _scan(case, rng, 4400, 0.05, reg.scale)
    local, _ = _clean(case, ((world - T[:3, 3]) @ T[:3, :3]).astype(np.float32), T, kappa)
    local = local[:4000]
    ref = RegRef(case, _q32(local, T), kappa)
    got = _launch(reg, np.tile(local, (250, 1)), T, kappa)
    _grade(got, ref, np.ones(4000, bool), "10^6 points", mult=250)
    again = _launch(reg, np.tile(local, (250, 1)), T, kappa)
    assert np.array_equal(got.view(np.int64), again.view(np.int64))


def test_kernel_all_points_masked(trained):
    case, reg = trained
    rng = np.random.default_rng(6)
    local = rng.uniform(-0.02, 0.02, (3000, 3)).astype(np.float32)
    T = np.eye(4)
    T[:3, 3] = (0.9, -0.9, 0.9)                                 # far outside the map: no voxel at lv[0]
    assert not RegRef(case, _q32(local, T), 0.1 * reg.scale).valid.any()
    got = _launch(reg, local, T, 0.1 * reg.scale)
    assert np.array_equal(got, np.zeros(29))


def test_kernel_points_on_level_boundaries(trained):
    """Points snapped to the leaf grid (every coarser level's boundaries too) at the identity: q = p exactly."""
    case, reg = trained
    rng = np.random.default_rng(7)
    res = 2.0 ** case["cfg"]["tree_level_world"]
    world = _scan(case, rng, 6000, 0.0, reg.scale)
    snapped = (np.round((world + 1) * res / 2) * 2 / res - 1).astype(np.float32)
    snapped[::3, 0] = world[::3, 0]                              # and points on one or two boundary planes only
    snapped[1::3, 1] = world[1::3, 1]
    kappa = 0.1 * reg.scale
    local, ref = _clean(case, snapped, np.eye(4), kappa)
    assert np.array_equal(_q32(local, np.eye(4)), local)
    got = _launch(reg, local, np.eye(4), kappa)
    _grade(got, ref, np.ones(local.shape[0], bool), "level boundaries")


def test_kernel_biasless_decoder(trained_nobias):
    case, reg = trained_nobias
    rng = np.random.default_rng(8)
    kappa = 0.1 * reg.scale
    T = _random_pose(rng, reg.scale)
    world = _scan(case, rng, 8000, 0.05, reg.scale)
    local, ref = _clean(case, ((world - T[:3, 3]) @ T[:3, :3]).astype(np.float32), T, kappa)
    got = _launch(reg, local, T, kappa)
    _grade(got, ref, np.ones(local.shape[0], bool), "bias-less decoder")


# ---- a drive along the street -------------------------------------------------------------------------------------------------

def _yaml(tmp_path, name, pc_path, pose_path="", **over):
    import yaml
    doc = {"setting": dict(pc_path=pc_path, pose_path=pose_path, calib_path="", begin_frame=0, end_frame=100, every_frame=1,
                           first_frame_ref=True, device=DEV, seed=7),
           "process": {"min_range_m": 2.75, "pc_radius_m": 25.0, "min_z_m": -10.0, "rand_downsample": False,
                       "vox_down_m": 0.1},
           "sampler": {"surface_sample_range_m": 0.3, "surface_sample_n": 3, "free_sample_begin_ratio": 0.3,
                       "free_sample_end_dist_m": 0.8, "free_sample_n": 3},
           "octree": {"tree_level_world": 12, "tree_level_feat": 3, "leaf_vox_size": 0.2, "feature_dim": 8},
           "continual": {"continual_learning_reg": False, "window_replay_on": False},
           "eval": {"mesh_freq_frame": 20, "mc_res_m": 0.1, "mc_with_octree": True},
           "optimizer": {"batch_size": 4096, "learning_rate": 0.01}}
    for k, v in over.items():
        sec, key = k.split("__")
        doc.setdefault(sec, {})[key] = v
    p = tmp_path / f"{name}.yaml"
    p.write_text(yaml.safe_dump(doc))
    return str(p)


def _config(path):
    from shine_mapping_b200.config import SHINEConfig
    cfg = SHINEConfig()
    cfg.load(path)
    return cfg


def _errors(est, truth):
    """Per frame: translation error (m) and rotation error (deg) of est against truth (map frame = frame 0)."""
    base = np.linalg.inv(truth[0])
    t_err, r_err = [], []
    for E, W in zip(est, truth):
        D = np.linalg.inv(base @ W) @ E
        t_err.append(float(np.linalg.norm(D[:3, 3])))
        r_err.append(math.degrees(float(np.linalg.norm(odometry.se3_log(D)[3:]))))
    return np.array(t_err), np.array(r_err)


ITERS = 150

def test_registration_recovers_perturbed_pose(tmp_path):
    from shine_mapping_b200 import Decoder, FeatureOctree
    from shine_mapping_b200.incre_loop import run_shine_mapping_incremental
    from shine_mapping_b200.scans import LiDARDataset
    drive = synth.write_drive(str(tmp_path / "seq"), n_frames=9)
    cfg = _config(_yaml(tmp_path, "true", drive["pc_path"], drive["pose_path"]))
    torch.manual_seed(cfg.seed)
    octree, decoder = FeatureOctree(cfg), Decoder(cfg)
    ds = LiDARDataset(cfg)
    run_shine_mapping_incremental(cfg, octree, decoder, itertools.islice(ds.frames(), 8), iters=ITERS,
                                  pool=synth.ReplayPool(ds.device))
    truth = ds.poses_ref[8]
    local = ds.processor.points(ds.read_frame(8), np.eye(4))
    reg = odometry.ScanToMapRegistration(cfg, octree, decoder)
    worst = []
    for dx, dy, dyaw in [(0.5, 0.0, 0.0), (0.0, 0.5, 0.0), (0.3, -0.3, 5.0), (-0.35, 0.35, -5.0), (0.0, 0.0, 5.0)]:
        init = truth.copy()
        init[:3, 3] += (dx, dy, 0.0)
        c, s = math.cos(math.radians(dyaw)), math.sin(math.radians(dyaw))
        init[:3, :3] = np.array([[c, -s, 0], [s, c, 0], [0, 0, 1]]) @ init[:3, :3]
        pose, info = reg.register(local, init)
        t_err, r_err = _errors([np.eye(4), pose], [np.eye(4), truth])
        worst.append((t_err[1], r_err[1]))
        print(f"[odometry] start ({dx}, {dy}) m, {dyaw} deg: error {100 * t_err[1]:.2f} cm, {r_err[1]:.3f} deg, {info}")
        assert info["ok"]
    assert max(w[0] for w in worst) <= 0.03 and max(w[1] for w in worst) <= 0.2, worst


def test_remap_from_written_poses_is_bit_identical(tmp_path):
    """The pose-free run and a LiDARDataset remap from its poses.txt (calib_path "") under the same seeds sample the same
    frames: equal pools and equal octree tables, bit for bit."""
    from shine_mapping_b200 import Decoder, FeatureOctree
    from shine_mapping_b200.incre_loop import run_shine_mapping_incremental
    from shine_mapping_b200.scans import LiDARDataset
    drive = synth.write_drive(str(tmp_path / "seq"), n_frames=6)
    runs = []
    for estimate in (True, False):
        pose_path = "" if estimate else str(tmp_path / "poses.txt")
        cfg = _config(_yaml(tmp_path, f"c{int(estimate)}", drive["pc_path"], pose_path))
        torch.manual_seed(cfg.seed)
        octree, decoder = FeatureOctree(cfg), Decoder(cfg)
        ds = odometry.OdometryScans(cfg, octree, decoder) if estimate else LiDARDataset(cfg)
        pool = synth.ReplayPool(ds.device)
        run_shine_mapping_incremental(cfg, octree, decoder, ds.frames(), iters=60, pool=pool)
        if estimate:
            ds.write_kitti_poses(str(tmp_path / "poses.txt"))
            assert all(ds.reg_info[f]["ok"] for f in ds.used_frames)
        runs.append((ds, pool, octree))
    (a, pa, oa), (b, pb, ob) = runs
    for f in a.used_frames:
        assert np.array_equal(a.poses_ref[f].view(np.int64), b.poses_ref[f].view(np.int64))
    for name in ("coord_pool", "sdf_label_pool", "weight_pool"):
        x, y = getattr(pa, name), getattr(pb, name)
        assert x.shape == y.shape and torch.equal(x.view(torch.int32), y.view(torch.int32)), name
    assert [tuple(p.shape) for p in oa.hier_features] == [tuple(p.shape) for p in ob.hier_features]
    assert oa.nodes_lookup_tables == ob.nodes_lookup_tables
    assert oa.corners_lookup_tables == ob.corners_lookup_tables
    assert all(np.array_equal(x, y) for x, y in zip(a.map_bbx, b.map_bbx))
