"""Localize LiDAR scans in a saved map: register every scan of a sequence to the map's SDF in lock-step on the GPU.

    python -m shine_mapping_b200.localize CONFIG CHECKPOINT --init-poses FILE
        [--scan-dir DIR] [--frames START:STOP[:STEP]] [--truth-poses FILE] [--out POSES.txt] [--csv FILE]

* `read_init_poses`   — KITTI rows in the world frame under the config's calib convention (`scans.read_poses_file`), one
                        per scan; a short file or a non-finite row is refused.
* `write_poses`       — one KITTI row per scan: the estimate of each localized frame (`repr` floats), every other row
                        copied from the input as it was.
* `localize`          — `ScanToMapRegistration.register_scans` over the selected frames, in the map's frame.
* `pose_errors`       — translation (m) and rotation (deg) error of a pose against the truth.

The map and its frame come from CONFIG and CHECKPOINT as in `evaluate scans`: a pose P in the world becomes
begin_pose_inv @ P in the map.  Each scan is preprocessed at the identity (`ScanProcessor.points`), as `OdometryScans`
does, and registered by `register`'s policy, which searches a grid around the start: x within 2 m and y within 0.5 m
of the map frame, yaw within 6 degrees.  DESIGN.md §15 states the layout, the schedule and the limits.
"""
from __future__ import annotations

import argparse
import csv
import math
import os
import sys

import numpy as np

# one row per frame; the summary row counts ok and converged frames and holds the median of each error column, and its
# max in the max_* columns
CSV_COLUMNS = ["frame", "ok", "converged", "iters", "valid", "rmse_m", "start_t_err_m", "start_r_err_deg", "t_err_m",
               "r_err_deg", "max_start_t_err_m", "max_start_r_err_deg", "max_t_err_m", "max_r_err_deg"]
ERROR_COLUMNS = ["start_t_err_m", "start_r_err_deg", "t_err_m", "r_err_deg"]


def _calib(config) -> dict:
    from .scans import read_calib_file
    return read_calib_file(config.calib_path) if config.calib_path != "" else {"Tr": np.eye(4)}


def read_init_poses(path: str, calib: dict, count: int) -> list:
    """The first `count` poses of a KITTI pose file (world frame, `read_poses_file`'s calib convention).  Raises
    ValueError for a file of fewer rows, and for any row that is not 12 numbers or holds a non-finite value."""
    with open(path) as fh:
        lines = fh.read().splitlines()
    if len(lines) < count:
        raise ValueError(f"{path} holds {len(lines)} poses for {count} scans")
    for i, line in enumerate(lines):
        try:
            values = [float(v) for v in line.split()]
        except ValueError:
            raise ValueError(f"{path} row {i}: not a list of numbers") from None
        if len(values) != 12:
            raise ValueError(f"{path} row {i}: {len(values)} values, a KITTI pose has 12")
        if not all(math.isfinite(v) for v in values):
            raise ValueError(f"{path} row {i}: a non-finite value")
    from .scans import read_poses_file
    return read_poses_file(path, calib)[:count]


def kitti_row(pose_w: np.ndarray, calib: dict) -> str:
    """The KITTI row of a LiDAR pose in the world: Tr P Tr^-1 (the inverse of `read_poses_file`'s Tr^-1 P Tr), 12 `repr`
    floats.  With Tr the identity the row holds P itself and reads back bit for bit."""
    Tr = calib["Tr"]
    P = np.asarray(pose_w, dtype=np.float64)
    if not np.array_equal(Tr, np.eye(4)):
        P = Tr @ P @ np.linalg.inv(Tr)
    return " ".join(repr(float(v)) for v in P[:3].reshape(-1))


def write_poses(path: str, init_path: str, count: int, estimates: dict, calib: dict) -> None:
    """`count` rows: estimates[f] (a world pose) for the frames it holds, the input file's row f for the others."""
    with open(init_path) as fh:
        lines = fh.read().splitlines()
    rows = [kitti_row(estimates[f], calib) if f in estimates else lines[f].strip() for f in range(count)]
    os.makedirs(os.path.dirname(os.path.abspath(path)), exist_ok=True)
    with open(path, "w") as fh:
        fh.write("\n".join(rows) + "\n")


def pose_errors(est: np.ndarray, truth: np.ndarray) -> tuple:
    """(translation error m, rotation error deg) of est against truth: the twist of truth^-1 est."""
    from .odometry import se3_log
    D = np.linalg.inv(truth) @ est
    return float(np.linalg.norm(D[:3, 3])), math.degrees(float(np.linalg.norm(se3_log(D)[3:])))


def localize(registration, processor, scan_files: list, frames: list, starts_map: list) -> list:
    """Read and preprocess each frame's scan at the identity, and register all of them in lock-step from their starts
    (map frame) -> [(pose in the map frame, info)] per frame."""
    from .scans import read_scan
    local = [processor.points(read_scan(scan_files[f]), np.eye(4)) for f in frames]
    return registration.register_scans(local, starts_map)


def _parser():
    ap = argparse.ArgumentParser(
        prog="python -m shine_mapping_b200.localize",
        description="Localize LiDAR scans in a saved map: register each scan to the map's SDF on the GPU, all scans in "
                    "lock-step, starting from --init-poses.  The registration searches a grid around each start (x "
                    "within 2 m and y within 0.5 m of the map frame, yaw within 6 degrees): starts farther off are "
                    "outside its basin.  LiDAR scans only.  The checkpoint is unpickled: load only files you trust.")
    ap.add_argument("config")
    ap.add_argument("checkpoint")
    ap.add_argument("--init-poses", required=True, metavar="FILE",
                    help="KITTI poses in the world frame, one row per scan, read with the config's calib_path")
    ap.add_argument("--scan-dir", default=None, metavar="DIR",
                    help="the scans to localize (default: the config's pc_path)")
    ap.add_argument("--frames", default=None, metavar="START:STOP[:STEP]",
                    help="frames to localize (default: the held-out frames of the config's own scans, every scan of "
                         "--scan-dir)")
    ap.add_argument("--truth-poses", default=None, metavar="FILE",
                    help="true KITTI poses to report errors against (default: the config's pose file when no "
                         "--scan-dir is given)")
    ap.add_argument("--out", default=None, metavar="POSES.txt",
                    help="write one KITTI row per scan: the estimate of each localized frame, the input row otherwise")
    ap.add_argument("--csv", default=None, metavar="FILE", help="write one row per frame and a summary row")
    return ap


def parse_args(argv):
    from .raycast import parse_frames
    ap = _parser()
    args = ap.parse_args(argv)
    if args.frames is not None:
        try:
            args.frames = parse_frames(args.frames)
        except ValueError as e:
            ap.error(str(e))
    if args.scan_dir is not None and not os.path.isdir(args.scan_dir):
        ap.error(f"--scan-dir {args.scan_dir}: not a directory")
    for name in ("init_poses", "truth_poses"):
        v = getattr(args, name)
        if v is not None and not os.path.isfile(v):
            ap.error(f"--{name.replace('_', '-')} {v}: no such file")
    return args


def _fmt(v, spec):
    return "-" if v is None or (isinstance(v, float) and math.isnan(v)) else format(v, spec)


def main(argv=None) -> int:
    args = parse_args(sys.argv[1:] if argv is None else argv)
    from .evaluate import load_map_and_dataset
    from .odometry import ScanToMapRegistration
    from .raycast import held_out_frames
    from .scans import natural_sorted
    args.rgbd = None
    config, octree, decoder, dataset = load_map_and_dataset(args)
    scan_dir = args.scan_dir if args.scan_dir is not None else config.pc_path
    files = [os.path.join(scan_dir, f) for f in natural_sorted(os.listdir(scan_dir))]
    if args.frames is not None:
        frames = list(args.frames)
    elif args.scan_dir is None:
        frames = held_out_frames(config, len(files))
    else:
        frames = list(range(len(files)))
    if not frames:
        raise SystemExit("no frames to localize: every frame of the config's scans was used for mapping; choose frames "
                         "with --frames START:STOP[:STEP]")
    bad = [f for f in frames if f >= len(files)]
    if bad:
        raise SystemExit(f"frame {bad[0]}: {scan_dir} has frames 0 .. {len(files) - 1}")
    calib = _calib(config)
    try:
        init_w = read_init_poses(args.init_poses, calib, len(files))
        truth_path = args.truth_poses if args.truth_poses is not None else (config.pose_path if args.scan_dir is None
                                                                             else None)
        truth_w = read_init_poses(truth_path, calib, len(files)) if truth_path is not None else None
    except ValueError as e:
        raise SystemExit(str(e))
    to_map = np.asarray(dataset.begin_pose_inv, dtype=np.float64)
    to_world = np.linalg.inv(to_map)
    starts = [to_map @ init_w[f] for f in frames]
    reg = ScanToMapRegistration(config, octree, decoder)
    results = localize(reg, dataset.processor, files, frames, starts)

    rows, estimates = [], {}
    for f, start, (pose, info) in zip(frames, starts, results):
        row = {"frame": f, "ok": bool(info["ok"]), "converged": bool(info["converged"]), "iters": int(info["iters"]),
               "valid": int(info["valid"]), "rmse_m": float(info["rmse_m"])}
        if info["ok"]:
            estimates[f] = to_world @ pose
        if truth_w is not None:
            truth = to_map @ truth_w[f]
            row["start_t_err_m"], row["start_r_err_deg"] = pose_errors(start, truth)
            row["t_err_m"], row["r_err_deg"] = pose_errors(pose, truth)
        rows.append(row)
        print(f"frame {f}: ok {row['ok']}, converged {row['converged']}, iters {row['iters']}, valid {row['valid']}, "
              f"rmse {_fmt(row['rmse_m'], '.4f')} m"
              + (f", start {row['start_t_err_m']:.4f} m {row['start_r_err_deg']:.3f} deg -> "
                 f"{row['t_err_m']:.4f} m {row['r_err_deg']:.3f} deg" if truth_w is not None else "")
              + ("" if info["ok"] else f" ({info['reason']})"))
    summary = {"frame": "summary", "ok": sum(r["ok"] for r in rows), "converged": sum(r["converged"] for r in rows)}
    text = f"{summary['ok']} of {len(rows)} frames ok, {summary['converged']} converged"
    if truth_w is not None:
        for key in ERROR_COLUMNS:
            v = np.array([r[key] for r in rows])
            summary[key], summary[f"max_{key}"] = float(np.median(v)), float(v.max())
        text += (f"; error median {summary['t_err_m']:.4f} m {summary['r_err_deg']:.3f} deg, max "
                 f"{summary['max_t_err_m']:.4f} m {summary['max_r_err_deg']:.3f} deg (starts: median "
                 f"{summary['start_t_err_m']:.4f} m {summary['start_r_err_deg']:.3f} deg, max "
                 f"{summary['max_start_t_err_m']:.4f} m {summary['max_start_r_err_deg']:.3f} deg)")
    print(text)
    if args.out:
        write_poses(args.out, args.init_poses, len(files), estimates, calib)
    if args.csv:
        os.makedirs(os.path.dirname(os.path.abspath(args.csv)), exist_ok=True)
        with open(args.csv, "w", newline="") as fh:
            writer = csv.DictWriter(fh, fieldnames=CSV_COLUMNS)
            writer.writeheader()
            for row in rows + [summary]:
                writer.writerow(row)
    return 0


if __name__ == "__main__":
    sys.exit(main())
