"""Cost of rendering views of a map (`shine_render`, render.py) on the synthetic drive.

    python tools/render_bench.py [--frames 20] [--iters 1000] [--reps 50] [--out DIR]

1. Builds the map of tools/raycast_bench.py: `synth.write_drive` (--frames scans 1.5 m apart) in a temporary directory,
   every other frame mapped by the batch loop (`--scans`, --iters iterations), the saved checkpoint loaded.
2. At the first held-out frame's pose, with the command's defaults (step mc_res_m = 0.1 m, max range pc_radius_m = 30 m,
   8 bisection steps, the mesher's mask level), three views:
   * a 640 x 480 pinhole (the PrimeSense intrinsics) looking along the sensor's x axis;
   * the frame's 64 x 1024 range image (its FOV from the scan's elevation extremes, as `render` picks it);
   * a 1920 x 1080 pinhole (f = 1000 px) along the same axis, the large case.
   Each: CUDA events around --reps launches after 5 warm-up launches -> ms per view, rays (pixels) per second and the
   hit ratio.
3. --out DIR: each view's depth and normal PNGs (render.write_view), DIR/{view}.png.

Prints one JSON object with the card's name and power limit read in the same run.  Writes nothing else outside a
temporary directory.  Needs a GPU.
"""
from __future__ import annotations

import argparse
import ctypes as C
import json
import os
import sys
import tempfile

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

# camera x -> sensor -y, camera y -> sensor -z, camera z -> sensor x: a forward-looking pinhole on a LiDAR's frame
CAMERA_IN_SENSOR = np.array([[0.0, 0.0, 1.0, 0.0], [-1.0, 0.0, 0.0, 0.0], [0.0, -1.0, 0.0, 0.0], [0.0, 0.0, 0.0, 1.0]])


def main(argv=None):
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--frames", type=int, default=20)
    ap.add_argument("--iters", type=int, default=1000)
    ap.add_argument("--reps", type=int, default=50)
    ap.add_argument("--out", default=None, metavar="DIR", help="write each view's depth and normal PNGs here")
    args = ap.parse_args(argv)
    if not torch.cuda.is_available():
        raise SystemExit("render_bench times sm_90a kernels: no CUDA device")
    import yaml
    from raycast_bench import card
    from shine_mapping_b200 import _abi, batch_loop, render, synth
    from shine_mapping_b200.checkpoint import load_checkpoint
    from shine_mapping_b200.config import SHINEConfig
    from shine_mapping_b200.decoder import Decoder
    from shine_mapping_b200.raycast import REFINE_ITERS, held_out_frames, map_pose, mask_level
    from shine_mapping_b200.rgbd import RGBDCamera
    from shine_mapping_b200.scans import LiDARDataset
    dev = "cuda:0"
    report = {"card": card()}
    with tempfile.TemporaryDirectory() as tmp:
        paths = synth.write_drive(os.path.join(tmp, "drive"), n_frames=args.frames)
        doc = {"setting": dict(pc_path=paths["pc_path"], pose_path=paths["pose_path"], calib_path="", begin_frame=0,
                               end_frame=100000, every_frame=2, first_frame_ref=True, device=dev),
               "process": {"min_range_m": 2.75, "pc_radius_m": 30.0, "min_z_m": -10.0, "rand_downsample": False,
                           "vox_down_m": 0.1},
               "sampler": {"surface_sample_range_m": 0.3, "surface_sample_n": 3, "free_sample_begin_ratio": 0.3,
                           "free_sample_end_dist_m": 0.8, "free_sample_n": 3},
               "octree": {"tree_level_world": 12, "tree_level_feat": 3, "leaf_vox_size": 0.2, "feature_dim": 8},
               "continual": {"continual_learning_reg": False, "window_replay_on": False},
               "optimizer": {"batch_size": 8192, "learning_rate": 0.01},
               "eval": {"save_freq_iters": args.iters, "vis_freq_iters": 10 ** 9, "mc_res_m": 0.1}}
        cfg_path = os.path.join(tmp, "cfg.yaml")
        with open(cfg_path, "w") as fh:
            yaml.safe_dump(doc, fh)
        run = os.path.join(tmp, "run")
        batch_loop.main([cfg_path, "--scans", "--iters", str(args.iters), "--run-path", run])
        config = SHINEConfig()
        config.load(cfg_path)
        state, octree = load_checkpoint(os.path.join(run, "model", f"model_iter_{args.iters}.pth"), config, dev)
        decoder = Decoder(config)
        decoder.load_state_dict(state)
        dataset = LiDARDataset(config)
        frame = held_out_frames(config, dataset.total_pc_count)[0]
        pose = map_pose(dataset, frame)
        range_cam = render.lidar_camera(dataset, frame, pose)

    extrinsic = np.linalg.inv(CAMERA_IN_SENSOR)
    views = {"pinhole_640x480": RGBDCamera(640, 480, 525.0, 525.0, 319.5, 239.5, extrinsic=extrinsic),
             "range_1024x64": range_cam,
             "pinhole_1920x1080": RGBDCamera(1920, 1080, 1000.0, 1000.0, 959.5, 539.5, extrinsic=extrinsic)}
    report["frame"] = frame
    report["range_image_fov_deg"] = [round(range_cam.fov_up, 3), round(range_cam.fov_down, 3)]
    lib, st = _abi.lib(), _abi.stream_ptr(dev)
    od, dd = octree._descriptor(None, None), decoder.c_descriptor(None)
    scale = float(config.scale)
    h, t_max = float(np.float32(config.mc_res_m * scale)), float(np.float32(config.pc_radius * scale))
    level = mask_level(config, octree)
    for name, cam in views.items():
        T = render.sensor_to_map(pose, cam)
        P = np.array(T[:3, :4])
        P[:, 3] *= scale
        p12 = (C.c_float * 12)(*P.astype(np.float32).reshape(12).tolist())
        cs = render._camera_struct(cam)
        n = cam.width * cam.height
        rng, depth = torch.empty(n, device=dev), torch.empty(n, device=dev)
        normal, status = torch.empty(n, 3, device=dev), torch.empty(n, dtype=torch.uint8, device=dev)

        def launch():
            _abi.check(lib.shine_render(C.byref(od), C.byref(dd), C.byref(cs), p12, h, 0.0, t_max, REFINE_ITERS, level,
                                        _abi.ptr(rng), _abi.ptr(depth), _abi.ptr(normal), _abi.ptr(status), st),
                       "shine_render")
        for _ in range(5):
            launch()
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize()
        a.record()
        for _ in range(args.reps):
            launch()
        b.record()
        torch.cuda.synchronize()
        ms = a.elapsed_time(b) / args.reps
        report[name] = {"pixels": n, "ms": round(ms, 4), "rays_per_s": round(n / ms * 1e3),
                        "hit_ratio": round(float(status.double().mean()), 4)}
        if args.out:
            view = render.render_view(config, octree, decoder, pose, cam, config.pc_radius)
            render.write_view(args.out, name, view, cam.depth_scale)
    print(json.dumps(report))


if __name__ == "__main__":
    main()
