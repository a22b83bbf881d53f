"""Mesh evaluation against a ground-truth point cloud, after reference eval/eval_utils.py (`eval_mesh`, `nn_correspondance`,
`crop_intersection`) and eval/evaluator.py, on the GPU.

* `eval_mesh`          — accuracy, completeness, Chamfer-L1/L2, precision, recall and F-score with the reference's
                         parameters: crop to the ground truth's box, uniform surface sampling, voxel down-sampling of both
                         clouds, nearest neighbours in both directions with the reference's truncation rules.
* `crop_intersection`  — the ground-truth points near every one of several meshes, written as an fp64 PLY point cloud.
* `python -m shine_mapping_b200.evaluate PRED GT [...]` / `... crop GT PRED [PRED ...] --out FILE` — the CLI.
* `... scans CONFIG CHECKPOINT [...]` — a saved map against held-out scans (raycast.py, DESIGN.md §13).

Sampling and nearest neighbours are csrc/shine_eval.cu; the down-sampling is csrc/shine_scan.cu's voxel_down_sample.
DESIGN.md §9 states the rules and where this differs from the reference.
"""
from __future__ import annotations

import argparse
import csv
import ctypes as C
import math
import os
import sys

import numpy as np
import torch

from . import _abi

CSV_COLUMNS = ["MAE_accuracy (m)", "MAE_completeness (m)", "Chamfer_L1 (m)", "Chamfer_L2 (m)",
               "Precision [Accuracy] (%)", "Recall [Completeness] (%)", "F-score (%)", "Spacing (m)",
               "Inlier_threshold (m)", "Outlier_truncation_acc (m)", "Outlier_truncation_com (m)"]
VOXEL_AXIS_LIMIT = (1 << 21) - 2        # voxels per axis of shine_scan's keys (21 bits), with its one-voxel margin


def _device(device):
    if device is None:
        if not torch.cuda.is_available():
            raise _abi.ShineB200Error("mesh evaluation runs as sm_90a CUDA kernels: no CUDA device is available")
        device = "cuda"
    device = torch.device(device)
    if device.type != "cuda":
        raise _abi.ShineB200Error(f"mesh evaluation runs as sm_90a CUDA kernels, not on {device}")
    return device


def _scratch(nbytes: int, what: str, device) -> torch.Tensor:
    if nbytes < 0:
        raise _abi.ShineB200Error(f"{what}: input too large")
    return torch.empty(max(int(nbytes), 1), dtype=torch.uint8, device=device)


# ---- inputs ----------------------------------------------------------------------------------------------------------

def load_mesh(pred, device) -> tuple[torch.Tensor, torch.Tensor]:
    """A PLY path or a (verts, faces[, ...]) pair -> (fp64 [V,3], int32 [T,3]) on the device."""
    if isinstance(pred, (str, os.PathLike)):
        from .mesher import read_ply
        v, f, _ = read_ply(os.fspath(pred))
        verts, faces = torch.from_numpy(np.ascontiguousarray(v, dtype=np.float64)), torch.from_numpy(f)
    else:
        verts, faces = pred[0], pred[1]
    verts = torch.as_tensor(verts).to(device=device, dtype=torch.float64).reshape(-1, 3).contiguous()
    faces = torch.as_tensor(faces).to(device=device).reshape(-1, 3)
    if faces.shape[0] and (int(faces.min()) < 0 or int(faces.max()) >= verts.shape[0]):
        raise ValueError(f"face indices outside [0, {verts.shape[0]})")
    return verts, faces.to(torch.int32).contiguous()


def load_points(gt, device) -> torch.Tensor:
    """A point-cloud path (.ply, .pcd, .bin, read by scans.read_scan) or an [M,3] tensor -> fp64 [M,3] on the device."""
    if isinstance(gt, (str, os.PathLike)):
        from .scans import read_scan
        rec = read_scan(os.fspath(gt), pinned=False)
        return torch.from_numpy(rec.points()).to(device)
    return torch.as_tensor(gt).to(device=device, dtype=torch.float64).reshape(-1, 3).contiguous()


# ---- kernels -----------------------------------------------------------------------------------------------------------

def sample_mesh(verts: torch.Tensor, faces: torch.Tensor, n: int, seed: int = 42, crop_box: torch.Tensor | None = None,
                return_tri_ids: bool = False):
    """Open3D's sample_points_uniformly on the GPU (shine_mesh_sample_*): n fp64 points, none when the (cropped) area is
    0.  crop_box: fp64 [6] device tensor (min x y z, max x y z); a triangle with a vertex outside it gets no samples.
    -> points [n,3] (and the int32 triangle id of every sample)."""
    dev = verts.device
    lib, st = _abi.lib(), _abi.stream_ptr(dev)
    nt = faces.shape[0]
    scratch = _scratch(lib.shine_mesh_sample_scratch_bytes(nt), "shine_mesh_sample_scratch_bytes", dev)
    total = torch.zeros(1, dtype=torch.float64, device=dev)
    box = None if crop_box is None else crop_box.to(device=dev, dtype=torch.float64).contiguous()
    _abi.check(lib.shine_mesh_sample_areas(_abi.ptr(verts), verts.shape[0], _abi.ptr(faces), nt, _abi.ptr(box),
                                           _abi.ptr(total), _abi.ptr(scratch), scratch.numel(), st),
               "shine_mesh_sample_areas")
    area = float(total.item())                     # the one host read: a zero area means no samples
    n = int(n) if area > 0.0 else 0
    points = torch.empty(n, 3, dtype=torch.float64, device=dev)
    ids = torch.empty(n, dtype=torch.int32, device=dev) if return_tri_ids else None
    _abi.check(lib.shine_mesh_sample_points(_abi.ptr(verts), _abi.ptr(faces), nt, _abi.ptr(total), n, int(seed) & (2**64 - 1),
                                            _abi.ptr(scratch), scratch.numel(), _abi.ptr(points), _abi.ptr(ids), st),
               "shine_mesh_sample_points")
    return (points, ids) if return_tri_ids else points


def voxel_down(points: torch.Tensor, voxel: float) -> torch.Tensor:
    """open3d's voxel_down_sample of fp64 device points (shine_scan's filter/sort/average with a box that holds every
    point, identity pose, scale 1): per voxel the fp64 mean in input order, voxels in ascending key order."""
    dev = points.device
    n = points.shape[0]
    if n == 0:
        return points.new_zeros(0, 3)
    lo, hi = (t.cpu().numpy() for t in (points.amin(0), points.amax(0)))
    if not (np.isfinite(lo).all() and np.isfinite(hi).all()):
        raise ValueError("voxel down-sampling: the cloud holds non-finite points")
    radius = float(max(abs(lo[0]), abs(hi[0]), abs(lo[1]), abs(hi[1])))
    min_z = float(np.nextafter(lo[2], -np.inf))                    # the filter keeps z > min_z
    if 2.0 * radius / voxel >= VOXEL_AXIS_LIMIT or (float(hi[2]) - min_z) / voxel >= VOXEL_AXIS_LIMIT:
        raise ValueError(f"voxel down-sampling at {voxel} m covers at most 2^21 - 2 = {VOXEL_AXIS_LIMIT} voxels per axis "
                         f"of a box centred on the origin: this cloud spans x {lo[0]}..{hi[0]}, y {lo[1]}..{hi[1]}, "
                         f"z {lo[2]}..{hi[2]}")
    lib, st = _abi.lib(), _abi.stream_ptr(dev)
    pts = points.contiguous()
    inp = _abi.ShineScanInput(pts.data_ptr(), n, 24, 1)
    scratch = _scratch(lib.shine_scan_scratch_bytes(n), "shine_scan_scratch_bytes", dev)
    count = torch.zeros(1, dtype=torch.int64, device=dev)
    _abi.check(lib.shine_scan_filter_keys(C.byref(inp), min_z, float(hi[2]), 0.0, radius, float(voxel), _abi.ptr(scratch),
                                          scratch.numel(), st), "shine_scan_filter_keys")
    _abi.check(lib.shine_scan_sort_voxels(n, _abi.ptr(count), _abi.ptr(scratch), scratch.numel(), st),
               "shine_scan_sort_voxels")
    m = int(count.item())
    vox = torch.empty(m, 3, dtype=torch.float64, device=dev)
    unused = torch.empty(m, 3, dtype=torch.float32, device=dev)
    eye = (C.c_double * 16)(*np.eye(4).reshape(16).tolist())
    _abi.check(lib.shine_scan_average_transform(C.byref(inp), eye, 1.0, m, _abi.ptr(vox), _abi.ptr(unused),
                                                _abi.ptr(scratch), scratch.numel(), st), "shine_scan_average_transform")
    return vox


class NearestNeighbours:
    """Exact nearest neighbours within a radius over fp64 reference points (shine_nn_build / shine_nn_query)."""

    def __init__(self, points: torch.Tensor):
        self.points = points.to(torch.float64).reshape(-1, 3).contiguous()
        dev = self.points.device
        lib = _abi.lib()
        self.n = self.points.shape[0]
        self.tree = _scratch(lib.shine_nn_tree_bytes(self.n), "shine_nn_tree_bytes", dev)
        scratch = _scratch(lib.shine_nn_scratch_bytes(self.n), "shine_nn_scratch_bytes", dev)
        _abi.check(lib.shine_nn_build(_abi.ptr(self.points), self.n, _abi.ptr(self.tree), self.tree.numel(),
                                      _abi.ptr(scratch), scratch.numel(), _abi.stream_ptr(dev)), "shine_nn_build")

    def query(self, queries: torch.Tensor, radius: float):
        """-> (dist fp64 [m], index int32 [m]): the distance to and input index of a nearest reference point when its
        squared distance is < radius^2 (fp64), else +inf and -1."""
        q = queries.to(device=self.points.device, dtype=torch.float64).reshape(-1, 3).contiguous()
        m = q.shape[0]
        dev = q.device
        lib = _abi.lib()
        dist = torch.empty(m, dtype=torch.float64, device=dev)
        index = torch.empty(m, dtype=torch.int32, device=dev)
        scratch = _scratch(lib.shine_nn_scratch_bytes(m), "shine_nn_scratch_bytes", dev)
        _abi.check(lib.shine_nn_query(_abi.ptr(self.tree), self.n, _abi.ptr(q), m, float(radius) ** 2, _abi.ptr(dist),
                                      _abi.ptr(index), _abi.ptr(scratch), scratch.numel(), _abi.stream_ptr(dev)),
                   "shine_nn_query")
        return dist, index


# ---- metrics -----------------------------------------------------------------------------------------------------------

def assemble_metrics(dist_p, dist_r, down_sample_res: float, threshold: float, truncation_acc: float,
                     truncation_com: float) -> dict:
    """eval_utils.py:73-106 from the raw nearest-neighbour distances (+inf beyond the truncation radius):
    dist_p per prediction point (accuracy: beyond is dropped), dist_r per ground-truth point (completeness: beyond
    becomes truncation_com).  Either set empty: both lists are empty (:121-122) and every metric is NaN."""
    dp = torch.as_tensor(dist_p, dtype=torch.float64).reshape(-1)
    dr = torch.as_tensor(dist_r, dtype=torch.float64).reshape(-1)
    if dp.numel() == 0 or dr.numel() == 0:
        dp, dr = dp[:0], dr[:0]
    else:
        dp = dp[torch.isfinite(dp)]
        dr = torch.where(torch.isfinite(dr), dr, torch.full_like(dr, truncation_com))
    mean = lambda t: float(t.sum()) / t.numel() if t.numel() else float("nan")     # numpy's sum / n, not sum * (1/n)
    dist_p_mean, dist_r_mean = mean(dp), mean(dr)
    dist_p_s_mean, dist_r_s_mean = mean(torch.square(dp)), mean(torch.square(dr))
    precision = mean((dp < threshold).double()) * 100.0
    recall = mean((dr < threshold).double()) * 100.0
    with np.errstate(invalid="ignore", divide="ignore"):
        chamfer_l1 = float(np.float64(0.5) * (np.float64(dist_p_mean) + dist_r_mean))
        chamfer_l2 = float(np.sqrt(np.float64(0.5) * (np.float64(dist_p_s_mean) + dist_r_s_mean)))
        fscore = float(np.float64(2.0) * precision * recall / (np.float64(precision) + recall))
    values = [dist_p_mean, dist_r_mean, chamfer_l1, chamfer_l2, precision, recall, fscore, down_sample_res, threshold,
              truncation_acc, truncation_com]
    return dict(zip(CSV_COLUMNS, values))


def eval_mesh(pred, gt, down_sample_res: float = 0.02, threshold: float = 0.05, truncation_acc: float = 0.50,
              truncation_com: float = 0.50, gt_bbx_mask_on: bool = True, mesh_sample_point: int = 10_000_000,
              seed: int = 42, device=None) -> dict:
    """eval_utils.py:24-107.  pred: a mesh PLY path or (verts, faces) tensors (e.g. what Mesher.recon_*_mesh returns);
    gt: a point-cloud path or [M,3] tensor.  -> the reference's 11 metrics and setup values, keyed as its CSV columns."""
    dev = _device(device)
    verts, faces = load_mesh(pred, dev)
    gt_pts = load_points(gt, dev)
    box = None
    if gt_bbx_mask_on:                                              # :49-56
        widen = torch.tensor([0.0, 0.0, down_sample_res], dtype=torch.float64, device=dev)
        if gt_pts.shape[0]:
            box = torch.cat((gt_pts.amin(0) - widen, gt_pts.amax(0) + widen))
        else:                                                       # an empty box crops every triangle
            box = torch.tensor([np.inf] * 3 + [-np.inf] * 3, dtype=torch.float64, device=dev)
    samples = sample_mesh(verts, faces, mesh_sample_point, seed, box)
    if down_sample_res > 0:                                         # :63-68
        pred_pts, gt_pts = voxel_down(samples, down_sample_res), voxel_down(gt_pts, down_sample_res)
    else:
        pred_pts = samples
    dist_p, _ = NearestNeighbours(gt_pts).query(pred_pts, truncation_acc)
    dist_r, _ = NearestNeighbours(pred_pts).query(gt_pts, truncation_com)
    return assemble_metrics(dist_p, dist_r, down_sample_res, threshold, truncation_acc, truncation_com)


def write_point_ply(path: str, points) -> None:
    """Binary little-endian PLY point cloud with `double x y z` (scans.read_ply reads it back)."""
    p = np.ascontiguousarray(torch.as_tensor(points).detach().cpu().numpy(), dtype="<f8").reshape(-1, 3)
    header = (f"ply\nformat binary_little_endian 1.0\nelement vertex {p.shape[0]}\n"
              "property double x\nproperty double y\nproperty double z\nend_header\n")
    os.makedirs(os.path.dirname(os.path.abspath(path)), exist_ok=True)
    with open(path, "wb") as fh:
        fh.write(header.encode("ascii"))
        fh.write(p.tobytes())


def crop_intersection(file_gt, files_pred, out_file: str, dist_thre: float = 0.1, mesh_sample_point: int = 1_000_000,
                      seed: int = 42, device=None) -> torch.Tensor:
    """eval_utils.py:180-216: keep the ground-truth points whose nearest sample of every predicted mesh lies at
    d^2 < dist_thre^2 (no crop, no down-sampling); write them to out_file.  -> the kept points [K,3] fp64."""
    dev = _device(device)
    pts = load_points(file_gt, dev)
    for pred in files_pred:
        verts, faces = load_mesh(pred, dev)
        samples = sample_mesh(verts, faces, mesh_sample_point, seed)
        _, index = NearestNeighbours(samples).query(pts, dist_thre)
        pts = pts[index >= 0]
    write_point_ply(out_file, pts)
    return pts


# ---- CLI ---------------------------------------------------------------------------------------------------------------

def _eval_parser():
    ap = argparse.ArgumentParser(prog="python -m shine_mapping_b200.evaluate",
                                 description="Evaluate a mesh against a ground-truth point cloud (eval_mesh).  "
                                             "`crop GT PRED [PRED ...] --out FILE` runs crop_intersection instead.")
    ap.add_argument("pred", help="predicted mesh (.ply)")
    ap.add_argument("gt", help="ground-truth point cloud (.ply, .pcd or .bin)")
    ap.add_argument("--down-sample", type=float, default=0.02, help="voxel size of the down-sampling, m (0: none)")
    ap.add_argument("--threshold", type=float, default=0.05, help="inlier threshold of precision / recall, m")
    ap.add_argument("--trunc-acc", type=float, default=0.50, help="outlier truncation of accuracy, m")
    ap.add_argument("--trunc-com", type=float, default=0.50, help="outlier truncation of completeness, m")
    ap.add_argument("--no-bbx-mask", action="store_true", help="do not crop the mesh to the ground truth's box")
    ap.add_argument("--samples", type=int, default=10_000_000, help="points sampled on the mesh")
    ap.add_argument("--seed", type=int, default=42, help="seed of the surface sampling")
    ap.add_argument("--csv", default=None, help="write the metrics as a CSV row with the reference's columns")
    return ap


def _crop_parser():
    ap = argparse.ArgumentParser(prog="python -m shine_mapping_b200.evaluate crop",
                                 description="Keep the ground-truth points near every predicted mesh (crop_intersection).")
    ap.add_argument("gt", help="ground-truth point cloud (.ply, .pcd or .bin)")
    ap.add_argument("pred", nargs="+", help="predicted meshes (.ply)")
    ap.add_argument("--out", required=True, help="output point cloud (.ply, fp64)")
    ap.add_argument("--dist-thre", type=float, default=0.1, help="nearest-neighbour distance threshold, m")
    ap.add_argument("--samples", type=int, default=1_000_000, help="points sampled on each mesh")
    ap.add_argument("--seed", type=int, default=42, help="seed of the surface sampling")
    return ap


def _scans_parser():
    from .rgbd import add_loop_arguments
    ap = argparse.ArgumentParser(prog="python -m shine_mapping_b200.evaluate scans",
                                 description="Cast the rays of held-out scans through a saved map and report range errors. "
                                             "The checkpoint is unpickled: load only files you trust.")
    ap.add_argument("config")
    ap.add_argument("checkpoint")
    add_loop_arguments(ap)
    ap.set_defaults(scans=False)
    ap.add_argument("--frames", default=None, metavar="START:STOP[:STEP]",
                    help="frames to evaluate (default: the ids in [begin_frame, end_frame] that mapping skips)")
    ap.add_argument("--step-m", type=float, default=None, help="ray sample spacing, m (default: the config's mc_res_m)")
    ap.add_argument("--beyond-m", type=float, default=1.0, help="search this far past each measured point, m")
    ap.add_argument("--threshold", type=float, default=0.1, help="a hit within this of the measured range is an inlier, m")
    ap.add_argument("--refine-iters", type=int, default=None, help="bisection steps of each hit (default 8)")
    ap.add_argument("--csv", default=None, help="write one row per frame and a total row")
    ap.add_argument("--points-dir", default=None, metavar="DIR", help="write each frame's hit points, DIR/{frame}.ply")
    return ap


def parse_args(argv):
    """-> ("crop" | "scans" | "eval", namespace); invalid values exit through argparse's error."""
    argv = list(argv)
    if argv and argv[0] == "scans":
        from .raycast import REFINE_ITERS, parse_frames
        from .rgbd import check_loop_arguments
        ap = _scans_parser()
        args = ap.parse_args(argv[1:])
        check_loop_arguments(ap, args)
        if args.frames is not None:
            try:
                args.frames = parse_frames(args.frames)
            except ValueError as e:
                ap.error(str(e))
        for name in ("step_m", "threshold"):
            v = getattr(args, name)
            if v is not None and not (v > 0 and math.isfinite(v)):
                ap.error(f"--{name.replace('_', '-')} must be > 0")
        if not (args.beyond_m >= 0 and math.isfinite(args.beyond_m)):
            ap.error("--beyond-m must be >= 0")
        if args.refine_iters is None:
            args.refine_iters = REFINE_ITERS
        if not 0 <= args.refine_iters <= _abi.RAYCAST_MAX_REFINE:
            ap.error(f"--refine-iters must be in [0, {_abi.RAYCAST_MAX_REFINE}]")
        return "scans", args
    if argv and argv[0] == "crop":
        ap = _crop_parser()
        args = ap.parse_args(argv[1:])
        if not args.dist_thre > 0:
            ap.error("--dist-thre must be > 0")
        if args.samples < 1:
            ap.error("--samples must be >= 1")
        return "crop", args
    ap = _eval_parser()
    args = ap.parse_args(argv)
    if not args.down_sample >= 0:
        ap.error("--down-sample must be >= 0")
    for name in ("threshold", "trunc_acc", "trunc_com"):
        if not getattr(args, name) > 0:
            ap.error(f"--{name.replace('_', '-')} must be > 0")
    if args.samples < 1:
        ap.error("--samples must be >= 1")
    return "eval", args


def write_csv(path: str, metrics: dict) -> None:
    """evaluator.py:66-76: a header of the reference's columns and one row."""
    os.makedirs(os.path.dirname(os.path.abspath(path)), exist_ok=True)
    with open(path, "w", newline="") as fh:
        writer = csv.DictWriter(fh, fieldnames=CSV_COLUMNS)
        writer.writeheader()
        writer.writerow(metrics)


def write_scans_csv(path: str, result: dict) -> None:
    """eval_scans' result: a `frame` column and the metric columns, one row per frame and a `total` row."""
    from .raycast import METRIC_COLUMNS
    os.makedirs(os.path.dirname(os.path.abspath(path)), exist_ok=True)
    with open(path, "w", newline="") as fh:
        writer = csv.DictWriter(fh, fieldnames=["frame"] + METRIC_COLUMNS)
        writer.writeheader()
        for row in result["frames"]:
            writer.writerow(row)
        writer.writerow({"frame": "total", **result["total"]})


def _format_metrics(m: dict) -> str:
    return (f"rays {m['rays']}, hit ratio {m['hit_ratio']:.4f}, |err| mean {m['mean_abs_err_m']:.4f} m, median "
            f"{m['median_abs_err_m']:.4f} m, rmse {m['rmse_m']:.4f} m, bias {m['bias_m']:+.4f} m, within threshold "
            f"{m['within_threshold']:.4f}")


def main_scans(args) -> int:
    from .checkpoint import load_checkpoint
    from .config import SHINEConfig
    from .decoder import Decoder
    from .raycast import eval_scans, held_out_frames, scan_frames
    config = SHINEConfig()
    config.load(args.config)
    state, octree = load_checkpoint(args.checkpoint, config, config.device)
    if octree is None or octree.is_empty():
        raise SystemExit(f"{args.checkpoint}: the checkpoint holds a decoder but no map (feature_octree): nothing to cast "
                         "rays through")
    decoder = Decoder(config)
    decoder.load_state_dict(state)
    if args.rgbd:
        from .rgbd import dataset_from_args
        dataset = dataset_from_args(config, args)
    else:
        from .scans import LiDARDataset
        dataset = LiDARDataset(config)
    frames = list(args.frames) if args.frames is not None else held_out_frames(config, dataset.total_pc_count)
    if not frames:
        raise SystemExit(f"no held-out frames: every frame in [begin_frame {config.begin_frame}, end_frame "
                         f"{config.end_frame}] was used for mapping (every_frame {config.every_frame}); choose frames "
                         "with --frames START:STOP[:STEP]")
    result = eval_scans(config, octree, decoder, scan_frames(dataset, frames), args.threshold, args.step_m,
                        args.beyond_m, args.refine_iters, args.points_dir, np.linalg.inv(dataset.begin_pose_inv))
    for row in result["frames"]:
        print(f"frame {row['frame']}: {_format_metrics(row)}")
    print(f"total: {_format_metrics(result['total'])}")
    if args.csv:
        write_scans_csv(args.csv, result)
    return 0


def main(argv=None) -> int:
    mode, args = parse_args(sys.argv[1:] if argv is None else argv)
    if mode == "scans":
        return main_scans(args)
    if mode == "crop":
        kept = crop_intersection(args.gt, args.pred, args.out, args.dist_thre, args.samples, args.seed)
        print(f"kept {kept.shape[0]} ground-truth points -> {args.out}")
        return 0
    metrics = eval_mesh(args.pred, args.gt, down_sample_res=args.down_sample, threshold=args.threshold,
                        truncation_acc=args.trunc_acc, truncation_com=args.trunc_com,
                        gt_bbx_mask_on=not args.no_bbx_mask, mesh_sample_point=args.samples, seed=args.seed)
    print(metrics)
    if args.csv:
        write_csv(args.csv, metrics)
    return 0


if __name__ == "__main__":
    sys.exit(main())
