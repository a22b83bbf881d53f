"""csrc/shine_rgbd.cu against a numpy fp64 restatement of the converter's back-projection (bit for bit, NaN exactly where
a pixel is dropped), its argument checks, the direct RGB-D path against the converted one (points, pools and octree
tables bit-identical), and both mapping loops on a synthetic RGB-D sequence."""
import ctypes as C
import math
import os
import warnings

import numpy as np
import pytest
import torch

from shine_mapping_b200 import _abi, rgbd, scans, synth
from tests.parity_utils import make_config
from tests.test_gpu_scans import _surface_distance
from tests.test_rgbd_host import rigid, write_png

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
FLIP = np.diag([1.0, -1.0, -1.0, 1.0])


# ------------------------------------------------------------------------------------------------------------ oracle

def oracle(raw, fx, fy, cx, cy, depth_scale, trunc, pose):
    """The contract in numpy: fp32 d = raw / scale, dropped when (double)d >= trunc or d <= 0; fp64 x y z with every
    operation rounded on its own; rows of pose · (x, y, z, 1) summed in k order.  -> [H*W,3], NaN where dropped."""
    H, W = raw.shape
    d = raw.astype(np.float32) / np.float32(depth_scale)
    valid = (d > 0) & ~(d.astype(np.float64) >= trunc)
    z = d.astype(np.float64)
    j = np.broadcast_to(np.arange(W, dtype=np.float64)[None, :], (H, W))
    i = np.broadcast_to(np.arange(H, dtype=np.float64)[:, None], (H, W))
    x = ((j - cx) * z) / fx
    y = ((i - cy) * z) / fy
    m = np.asarray(pose, dtype=np.float64)
    q = np.stack([((m[r, 0] * x + m[r, 1] * y) + m[r, 2] * z) + m[r, 3] * 1.0 for r in range(3)], -1)
    q[~valid] = np.nan
    return q.reshape(-1, 3)


def run_kernel(raw, cam_args, pose, row_pitch=None, rgb=None):
    """raw [H, W] uint16 (optionally inside rows of row_pitch), rgb [H, row_pitch, 3] uint8 or None."""
    H, W = raw.shape
    pitch = W if row_pitch is None else row_pitch
    buf = np.full((H, pitch), 12345, dtype=np.uint16)
    buf[:, :W] = raw
    d = torch.from_numpy(buf.view(np.int16)).to(DEV)
    xyz = torch.full((H * W, 3), 7.0, dtype=torch.float64, device=DEV)
    rgb_in = torch.from_numpy(rgb).to(DEV) if rgb is not None else None
    rgb_out = torch.zeros(H * W, 3, dtype=torch.uint8, device=DEV) if rgb is not None else None
    p = (C.c_double * 16)(*np.asarray(pose, dtype=np.float64).reshape(16).tolist())
    _abi.check(_abi.lib().shine_rgbd_backproject(_abi.ptr(d), H, W, pitch, *cam_args, p, _abi.ptr(xyz),
                                                 _abi.ptr(rgb_out), _abi.ptr(rgb_in), _abi.stream_ptr(DEV)),
               "shine_rgbd_backproject")
    torch.cuda.synchronize()
    return xyz.cpu().numpy(), (rgb_out.cpu().numpy() if rgb is not None else None)


def assert_bit_exact(got, want):
    nan_w, nan_g = np.isnan(want), np.isnan(got)
    np.testing.assert_array_equal(nan_g, nan_w)
    assert (nan_w.all(1) | ~nan_w.any(1)).all()
    np.testing.assert_array_equal(got[~nan_g].view(np.int64), want[~nan_w].view(np.int64))


CAMERAS = {
    "primesense": ((525.0, 525.0, 319.5, 239.5), 1000.0, FLIP),
    "neural_rgbd": ((554.2562584220408, 554.2562584220408, 319.5, 239.5), 1000.0, FLIP),
    "replica": ((600.0, 600.0, 599.5, 339.5), 6553.5, np.eye(4)),
    "rigid": ((512.25, 498.75, 321.125, 243.5), 1000.0, rigid(7)),
}


def _image(kind, H, W, rng):
    if kind == "zeros":
        return np.zeros((H, W), np.uint16)
    if kind == "valid":
        return rng.integers(1, 4999, (H, W), dtype=np.uint16)
    img = rng.integers(0, 65536, (H, W), dtype=np.uint16)
    img[rng.random((H, W)) < 0.2] = 0
    img[rng.random((H, W)) < 0.1] = 5000                       # exactly the truncation at scale 1000
    img.reshape(-1)[:4] = (0, 65535, 4999, 5001)[:img.size]
    return img


@pytest.mark.parametrize("camera", list(CAMERAS))
@pytest.mark.parametrize("shape,kind", [((480, 640), "mixed"), ((1080, 1920), "mixed"), ((1, 1), "mixed"),
                                        ((1, 37), "mixed"), ((41, 1), "mixed"), ((33, 65), "mixed"),
                                        ((17, 19), "zeros"), ((48, 64), "valid")])
def test_backproject_bit_exact(camera, shape, kind):
    (fx, fy, cx, cy), scale, extrinsic = CAMERAS[camera]
    pose = np.linalg.inv(extrinsic)
    raw = _image(kind, *shape, np.random.default_rng(shape[0] * 7 + shape[1]))
    got, _ = run_kernel(raw, (fx, fy, cx, cy, scale, 5.0), pose)
    want = oracle(raw, fx, fy, cx, cy, scale, 5.0, pose)
    assert_bit_exact(got, want)
    if kind == "zeros":
        assert np.isnan(got).all()
    if kind == "valid":
        assert not np.isnan(got).any()


def test_truncation_edges_compare_in_fp64():
    """d exactly at the truncation is dropped; one fp64 ulp above keeps it, one below drops it.  At d = fp32(4.321),
    trunc = nextafter(d, +inf) rounds to d in fp32: only an fp64 comparison keeps the pixel."""
    pose = np.linalg.inv(FLIP)
    for raw_v, d in ((5000, 5.0), (4321, float(np.float32(4321) / np.float32(1000)))):
        raw = np.full((3, 5), raw_v, np.uint16)
        for trunc, kept in ((d, False), (np.nextafter(d, np.inf), True), (np.nextafter(d, 0.0), False)):
            got, _ = run_kernel(raw, (10.0, 10.0, 2.0, 1.0, 1000.0, trunc), pose)
            assert_bit_exact(got, oracle(raw, 10.0, 10.0, 2.0, 1.0, 1000.0, trunc, pose))
            assert (~np.isnan(got).any(1)).all() == kept and np.isnan(got).all() != kept


def test_row_pitch_and_colour_passthrough():
    rng = np.random.default_rng(5)
    H, W, pitch = 37, 53, 64
    raw = _image("mixed", H, W, rng)
    rgb = rng.integers(0, 256, (H, pitch, 3), dtype=np.uint8)
    (fx, fy, cx, cy), scale, extrinsic = CAMERAS["rigid"]
    pose = np.linalg.inv(extrinsic)
    got, col = run_kernel(raw, (fx, fy, cx, cy, scale, 5.0), pose, row_pitch=pitch, rgb=rgb)
    assert_bit_exact(got, oracle(raw, fx, fy, cx, cy, scale, 5.0, pose))
    np.testing.assert_array_equal(col, rgb[:, :W].reshape(-1, 3))


def test_abi_rejections_launch_nothing():
    lib, st = _abi.lib(), _abi.stream_ptr(DEV)
    d = torch.ones(64, dtype=torch.int16, device=DEV)
    xyz = torch.full((64, 3), 7.0, dtype=torch.float64, device=DEV)
    rgb = torch.zeros(64 * 3, dtype=torch.uint8, device=DEV)
    pose = (C.c_double * 16)(*np.eye(4).reshape(16).tolist())
    P, X = _abi.ptr(d), _abi.ptr(xyz)
    cases = {
        "null depth": (None, 8, 8, 8, 1000.0, pose, X, None, None),
        "null pose": (P, 8, 8, 8, 1000.0, None, X, None, None),
        "null xyz": (P, 8, 8, 8, 1000.0, pose, None, None, None),
        "rgb_out without rgb_in": (P, 8, 8, 8, 1000.0, pose, X, _abi.ptr(rgb), None),
        "rgb_in without rgb_out": (P, 8, 8, 8, 1000.0, pose, X, None, _abi.ptr(rgb)),
        "height 0": (P, 0, 8, 8, 1000.0, pose, X, None, None),
        "width 0": (P, 8, 0, 8, 1000.0, pose, X, None, None),
        "negative height": (P, -1, 8, 8, 1000.0, pose, X, None, None),
        "row_pitch < width": (P, 8, 8, 7, 1000.0, pose, X, None, None),
        "depth_scale 0": (P, 8, 8, 8, 0.0, pose, X, None, None),
        "depth_scale < 0": (P, 8, 8, 8, -1000.0, pose, X, None, None),
        "depth_scale NaN": (P, 8, 8, 8, float("nan"), pose, X, None, None),
        "depth_scale beyond fp32": (P, 8, 8, 8, 1e300, pose, X, None, None),
        "misaligned depth": (C.c_void_p(d.data_ptr() + 1), 8, 8, 8, 1000.0, pose, X, None, None),
        "misaligned xyz": (P, 8, 8, 8, 1000.0, pose, C.c_void_p(xyz.data_ptr() + 4), None, None),
    }
    for name, (dp, h, w, pitch, scale, ps, xp, ro, ri) in cases.items():
        rc = lib.shine_rgbd_backproject(dp, h, w, pitch, 1.0, 1.0, 0.0, 0.0, scale, 5.0, ps, xp, ro, ri, st)
        assert rc == -1, name                                          # SHINE_ERR_INVALID_ARG
    for h, w, pitch in ((65536, 32768, 32768), (2, 2, 0x7fffffff), (46341, 46341, 46341)):
        assert lib.shine_rgbd_backproject(P, h, w, pitch, 1.0, 1.0, 0.0, 0.0, 1000.0, 5.0, pose, X, None, None,
                                          st) == -2, (h, w, pitch)
    torch.cuda.synchronize()
    assert (xyz == 7.0).all()


# ---------------------------------------------------------------------------------------------- a synthetic sequence

H_IMG, W_IMG, FOCAL = 120, 160, 100.0


def camera_to_world(k: int) -> np.ndarray:
    """Camera k's pose in the Neural RGB-D convention (camera x right, y up, looking along -z) along a short arc."""
    yaw, pitch = -0.5 + 0.04 * k, 0.5
    fwd = np.array([math.cos(pitch) * math.cos(yaw), math.cos(pitch) * math.sin(yaw), -math.sin(pitch)])
    right = np.cross(fwd, [0.0, 0.0, 1.0])
    right /= np.linalg.norm(right)
    up = np.cross(right, fwd)
    T = np.eye(4)
    T[:3, :3] = np.stack((right, up, -fwd), 1)
    T[:3, 3] = (2.5 + 0.25 * k, -1.0 - 0.1 * k, 0.0)
    return T


def render_depth(T: np.ndarray, H: int = H_IMG, W: int = W_IMG, focal: float = FOCAL) -> np.ndarray:
    """z-depth in millimetres (uint16, 0 where no surface or beyond 65.535 m) through the pinhole of the sequence."""
    j, i = np.meshgrid(np.arange(W, dtype=np.float64), np.arange(H, dtype=np.float64))
    cv = np.stack(((j - (W - 1) / 2) / focal, (i - (H - 1) / 2) / focal, np.ones_like(j)), -1).reshape(-1, 3)
    dirs = (cv * [1.0, -1.0, -1.0]) @ T[:3, :3].T
    hits = synth.raycast_scene(torch.tensor(T[:3, 3]), torch.tensor(dirs), synth.default_boxes().double(),
                               min_range=0.0, max_range=float("inf")).numpy()
    ok = np.isfinite(hits).all(1)
    t = np.zeros(len(cv))
    t[ok] = ((hits[ok] - T[:3, 3]) * dirs[ok]).sum(1) / (dirs[ok] ** 2).sum(1)
    mm = np.round(t * 1000.0)
    return np.where(ok & (mm < 65535), mm, 0).astype(np.uint16).reshape(H, W)


def write_rgbd_sequence(root, n_frames=10, n_colour=None):
    """Neural RGB-D layout: depth/*.png (uint16 mm), images/*.png (RGB pattern), focal.txt, poses.txt (4x4 per frame)."""
    for d in ("depth", "images"):
        os.makedirs(os.path.join(root, d), exist_ok=True)
    ii, jj = np.meshgrid(np.arange(H_IMG), np.arange(W_IMG), indexing="ij")
    colour = np.stack(((ii * 7) % 256, (jj * 3) % 256, (ii + jj) % 256), -1).astype(np.uint8)
    poses = [camera_to_world(k) for k in range(n_frames)]
    for k, T in enumerate(poses):
        write_png(os.path.join(root, "depth", f"depth{k}.png"), render_depth(T))
        if k < (n_frames if n_colour is None else n_colour):
            write_png(os.path.join(root, "images", f"img{k}.png"), np.roll(colour, k, 1))
    with open(os.path.join(root, "poses.txt"), "w") as fh:
        for T in poses:
            fh.write("\n".join(" ".join(repr(float(v)) for v in row) for row in T) + "\n")
    with open(os.path.join(root, "focal.txt"), "w") as fh:
        fh.write(f"{FOCAL}\n")
    return dict(depth=os.path.join(root, "depth"), rgb=os.path.join(root, "images"),
                poses=os.path.join(root, "poses.txt"), focal=os.path.join(root, "focal.txt"), frames=poses)


def _convert(seq, out):
    return rgbd.main(["convert", "--depth_img_folder", seq["depth"], "--rgb_img_folder", seq["rgb"], "--intrinsic_file",
                      seq["focal"], "--pose_file", seq["poses"], "--output_root", out, "--is_focal_file", "True",
                      "--already_kitti_format_pose", "False", "--vis_on", "False"])


def _rgbd_cfg(**kw):
    """config/rgbd/rgbd_batch.yaml's process, sampler and octree settings."""
    base = dict(device=DEV, rand_downsample=False, vox_down_m=0.01, min_range=0.2, pc_radius=5.0, min_z=-10.0,
                first_frame_ref=False, begin_frame=0, end_frame=1500, every_frame=1, surface_sample_range_m=0.05,
                free_sample_begin_ratio=0.5, free_sample_end_dist_m=0.3, sigma_sigmoid_m=0.02)
    base.update(kw)
    return make_config(4, leaf_vox=0.02, **base)


def test_converter_output(tmp_path):
    seq = write_rgbd_sequence(str(tmp_path / "seq"), n_frames=4, n_colour=3)
    out = str(tmp_path / "out")
    assert _convert(seq, out) == 0
    assert sorted(os.listdir(os.path.join(out, "rgbd_ply"))) == ["000000.ply", "000001.ply", "000002.ply"]  # zip
    poses = scans.read_poses_file(os.path.join(out, "poses.txt"), {"Tr": np.eye(4)})
    for got, want in zip(poses, seq["frames"]):
        assert got[:3].tobytes() == want[:3].tobytes()
    from shine_mapping_b200.mesher import read_point_ply
    cam = rgbd.RGBDCamera.from_converter_args(seq["focal"], True, (H_IMG, W_IMG))
    for k in range(3):
        ply = read_point_ply(os.path.join(out, "rgbd_ply", f"{k:06d}.ply"))
        assert ply.dtype.names == ("x", "y", "z", "red", "green", "blue")
        raw = rgbd.read_depth(os.path.join(seq["depth"], f"depth{k}.png"), pinned=False).numpy()
        want = oracle(raw, cam.fx, cam.fy, cam.cx, cam.cy, 1000.0, 5.0, cam.camera_pose)
        keep = ~np.isnan(want[:, 0])
        assert 0 < keep.sum() < keep.size                  # the sequence has dropped pixels (no hit, beyond 5 m)
        got = np.stack([ply[a] for a in "xyz"], 1)
        np.testing.assert_array_equal(got.view(np.int64), want[keep].view(np.int64))
        colour = rgbd.read_color(os.path.join(seq["rgb"], f"img{k}.png"), pinned=False).numpy().reshape(-1, 3)
        np.testing.assert_array_equal(np.stack([ply[c] for c in ("red", "green", "blue")], 1), colour[keep])


def _tables(octree):
    return ([p.detach().cpu().numpy().tobytes() for p in octree.hier_features],
            [list(octree.nodes_lookup_tables[l].items()) for l in range(octree.free_level_num, octree.max_level + 1)],
            [list(octree.corners_lookup_tables[l].items()) for l in range(octree.free_level_num, octree.max_level + 1)])


def test_direct_path_equals_converted_path(tmp_path):
    from shine_mapping_b200 import FeatureOctree
    seq = write_rgbd_sequence(str(tmp_path / "seq"))
    out = str(tmp_path / "out")
    _convert(seq, out)
    cfg = _rgbd_cfg(pc_path=os.path.join(out, "rgbd_ply"), pose_path=os.path.join(out, "poses.txt"), calib_path="")
    torch.manual_seed(0)
    oct_a = FeatureOctree(cfg)
    torch.manual_seed(0)
    oct_b = FeatureOctree(cfg)
    conv = scans.LiDARDataset(cfg, oct_a)
    cam = rgbd.RGBDCamera.from_converter_args(seq["focal"], True, (H_IMG, W_IMG))
    direct = rgbd.RGBDDataset(cfg, seq["depth"], seq["poses"], cam, octree=oct_b)
    assert conv.used_frames == direct.used_frames == list(range(10))
    for a, b in zip(conv.poses_ref, direct.poses_ref):
        assert a.tobytes() == b.tobytes()
    for f in direct.used_frames:
        pa = conv.processor.points(conv.read_frame(f), conv.poses_ref[f])
        pb = direct.processor.points(direct.read_frame(f), direct.poses_ref[f])
        assert pa.shape[0] > 1000
        assert torch.equal(pa.view(torch.int32), pb.view(torch.int32)), f
        W = np.linalg.inv(direct.begin_pose_inv)
        pw = (pb.double().cpu().numpy() / cfg.scale) @ W[:3, :3].T + W[:3, 3]
        assert _surface_distance(pw).max() < cfg.vox_down_m * 1.8
        for ds in (conv, direct):
            torch.manual_seed(100 + f)
            ds.process_frame(f)
        assert _tables(oct_a) == _tables(oct_b), f
    for name in ("coord_pool", "sdf_label_pool", "weight_pool"):
        assert torch.equal(getattr(conv.pool, name).view(torch.int32), getattr(direct.pool, name).view(torch.int32))
    assert np.array_equal(conv.map_bbx[0], direct.map_bbx[0]) and np.array_equal(conv.map_bbx[1], direct.map_bbx[1])


def test_one_host_read_per_frame(tmp_path):
    seq = write_rgbd_sequence(str(tmp_path / "seq"), n_frames=2)
    cam = rgbd.RGBDCamera.from_converter_args(seq["focal"], True, (H_IMG, W_IMG))
    ds = rgbd.RGBDDataset(_rgbd_cfg(), seq["depth"], seq["poses"], cam)
    ds.frame_samples(0)
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("warn")
    try:
        with warnings.catch_warnings(record=True) as caught:
            warnings.simplefilter("always")
            ds.frame_samples(1)
    finally:
        torch.cuda.set_sync_debug_mode("default")
    syncs = [w for w in caught if "synchroniz" in str(w.message)]
    assert len(syncs) == 1, [str(w.message) for w in syncs]


# ---------------------------------------------------------------------------------------------------- command lines

def _yaml(tmp_path, **over):
    """config/rgbd/rgbd_batch.yaml with the given `section__key` values."""
    import yaml
    doc = {"setting": {"name": "rgbd_batch", "pc_path": "unused/rgbd_ply", "pose_path": "unused/poses.txt",
                       "calib_path": "", "load_model": False, "first_frame_ref": False, "begin_frame": 0,
                       "end_frame": 1500, "every_frame": 5, "device": DEV},
           "process": {"min_range_m": 0.2, "pc_radius_m": 5.0, "min_z_m": -10.0, "rand_downsample": False,
                       "vox_down_m": 0.01},
           "sampler": {"surface_sample_range_m": 0.05, "surface_sample_n": 3, "free_sample_begin_ratio": 0.5,
                       "free_sample_end_dist_m": 0.3, "free_sample_n": 3},
           "octree": {"leaf_vox_size": 0.02, "tree_level_world": 12, "tree_level_feat": 4, "feature_dim": 8,
                      "poly_int_on": True, "octree_from_surface_samples": True},
           "decoder": {"mlp_level": 2, "mlp_hidden_dim": 32, "freeze_after_frame": 0},
           "loss": {"ray_loss": False, "main_loss_type": "sdf_bce", "sigma_sigmoid_m": 0.02, "loss_weight_on": False,
                    "behind_dropoff_on": False, "ekional_loss_on": False, "weight_e": 0.1},
           "continual": {"continual_learning_reg": False, "lambda_forget": 0, "window_replay_on": False,
                         "window_radius_m": 0},
           "optimizer": {"iters": 20000, "batch_size": 4096, "learning_rate": 0.01, "weight_decay": 1e-7},
           "eval": {"wandb_vis_on": False, "o3d_vis_on": False, "vis_freq_iters": 5000, "save_freq_iters": 10000,
                    "mesh_freq_frame": 1, "mc_res_m": 0.01, "mc_with_octree": True, "mc_local": False,
                    "mc_vis_level": 2, "save_map": False}}
    for k, v in over.items():
        sec, key = k.split("__")
        doc[sec][key] = v
    p = tmp_path / "cfg.yaml"
    p.write_text(yaml.safe_dump(doc))
    return str(p)


def _ground_truth_in_view(seq, trunc=5.0):
    """synth.scene_surface_points seen by some camera of the sequence: in front, inside the image, not occluded (its
    depth within 2 cm of the rendered depth there) and nearer than the truncation."""
    gt = synth.scene_surface_points(0.0, 12.0, 0.02).numpy()
    seen = np.zeros(len(gt), bool)
    for T in seq["frames"]:
        depth = render_depth(T).astype(np.float64) / 1000.0
        cam = ((gt - T[:3, 3]) @ T[:3, :3]) * [1.0, -1.0, -1.0]
        z = cam[:, 2]
        with np.errstate(divide="ignore", invalid="ignore"):
            u = np.round(FOCAL * cam[:, 0] / z + (W_IMG - 1) / 2)
            v = np.round(FOCAL * cam[:, 1] / z + (H_IMG - 1) / 2)
        inside = (z > 0.2) & (u >= 0) & (u < W_IMG) & (v >= 0) & (v < H_IMG)
        idx = np.where(inside)[0]
        dz = depth[v[idx].astype(int), u[idx].astype(int)]
        ok = (dz > 0) & (dz < trunc) & (np.abs(dz - z[idx]) < 0.02)
        seen[idx[ok]] = True
    return torch.from_numpy(gt[seen])


# (accuracy, completeness) in metres: about 1.5 x the worst of each measured on one H100 80GB HBM3 at 700 W over three
# or four runs, 0.0150 m and 0.0262 m (both incre_reg); the other modes measured 0.0113-0.0131 m and 0.0219-0.0250 m
# (DESIGN §11)
MESH_BOUNDS = (0.022, 0.039)


def _grade(seq, mesh_path, mode):
    from shine_mapping_b200.evaluate import eval_mesh
    m = eval_mesh(mesh_path, _ground_truth_in_view(seq), down_sample_res=0.02, threshold=0.05, truncation_acc=0.5,
                  truncation_com=0.5, mesh_sample_point=1_000_000, device=DEV)
    acc, com = m["MAE_accuracy (m)"], m["MAE_completeness (m)"]
    print(f"[rgbd mesh] {mode}: accuracy {acc:.4f} m, completeness {com:.4f} m, F-score {m['F-score (%)']:.1f} %")
    assert acc < MESH_BOUNDS[0] and com < MESH_BOUNDS[1], (mode, acc, com)


def _rgbd_args(seq):
    return ["--rgbd", seq["depth"], "--intrinsic-file", seq["focal"], "--focal-file", "--pose-file", seq["poses"],
            "--max-depth-m", "5.0"]


def test_batch_loop_rgbd_eikonal_mesh(tmp_path, capsys):
    from shine_mapping_b200 import batch_loop
    seq = write_rgbd_sequence(str(tmp_path / "seq"))
    cfg = _yaml(tmp_path, setting__every_frame=1, loss__ekional_loss_on=True, eval__vis_freq_iters=2000,
                eval__mc_res_m=0.02)
    batch_loop.main([cfg, *_rgbd_args(seq), "--iters", "2000", "--run-path", str(tmp_path / "run")])
    out = capsys.readouterr().out
    mesh = str(tmp_path / "run" / "mesh" / "mesh_iter_2000.ply")
    assert os.path.exists(mesh), out
    with capsys.disabled():
        _grade(seq, mesh, "batch")


@pytest.mark.parametrize("mode", ["incre_reg", "incre_replay"])
def test_incre_loop_rgbd_mesh(tmp_path, capsys, mode):
    from shine_mapping_b200 import incre_loop
    seq = write_rgbd_sequence(str(tmp_path / "seq"))
    over = dict(setting__every_frame=1, decoder__freeze_after_frame=20, optimizer__iters=50, eval__mesh_freq_frame=5,
                eval__mc_res_m=0.02, eval__vis_freq_iters=0)
    if mode == "incre_reg":
        over.update(continual__continual_learning_reg=True, continual__lambda_forget=1e3)
    else:
        over.update(process__vox_down_m=0.02, continual__window_replay_on=True, continual__window_radius_m=7.0)
    history = incre_loop.main([_yaml(tmp_path, **over), *_rgbd_args(seq), "--run-path", str(tmp_path / "run")])
    assert len(history) == 10 and all(math.isfinite(h["loss_last"]) for h in history)
    assert ("pool" in history[-1]) == (mode == "incre_replay")
    meshes = [h["mesh"] for h in history if "mesh" in h]
    assert [os.path.basename(m) for m in meshes] == ["mesh_frame_1.ply", "mesh_frame_5.ply", "mesh_frame_10.ply"]
    with capsys.disabled():
        _grade(seq, meshes[-1], mode)


def test_converted_sequence_through_scans_with_rgbd_batch_settings(tmp_path, capsys):
    import ast
    from shine_mapping_b200 import batch_loop
    seq = write_rgbd_sequence(str(tmp_path / "seq"))
    out = str(tmp_path / "out")
    _convert(seq, out)
    cfg = _yaml(tmp_path, setting__pc_path=os.path.join(out, "rgbd_ply"), setting__pose_path=os.path.join(out, "poses.txt"))
    batch_loop.main([cfg, "--scans", "--iters", "500"])
    text = capsys.readouterr().out
    res = ast.literal_eval([l for l in text.splitlines() if l.startswith("{'loss_first'")][-1])
    assert res["loss_last"] < res["loss_first"]
    # every_frame 5: frames 0 and 5 of the ten
    assert "SamplePool" in text
