"""Mapping without a pose file: each new LiDAR scan is registered to the current SDF map on the GPU before it is mapped.

The map is a signed distance field with an analytic gradient, so a scan can be aligned to it by Gauss-Newton on the SDF
residuals of its points (scan-to-implicit-map odometry).  For a pose T and the scan's points p_i, r_i = SDF(T p_i) and
its Jacobian for a left-multiplied twist xi = (rho, phi) is [g_i, (T p_i) x g_i], g_i the SDF gradient.
`shine_register_normal_eq` (csrc/shine_register.cu) forms the robust (Geman-McClure) normal equations of one iterate in
one pass over the scan; the 6x6 system is solved here in fp64, one 29-double read per iteration.
`shine_register_normal_eq_poses` forms them at many poses in one call (the coarse grid, the weak-direction search).

* `se3_exp` / `se3_log` — the SE(3) exponential and logarithm in fp64, twist (rho, phi).
* `ScanToMapRegistration` — the normal equations and the Gauss-Newton loop.
* `OdometryScans` — a frame source for `incre_loop.run_shine_mapping_incremental` that estimates each frame's pose.

The map frame is the first scan's frame.  The loop trains the map frame by frame, so each scan is registered to the map
of all earlier frames.  Registration draws no random numbers: a remap from the written poses (`write_kitti_poses`, then
`LiDARDataset` with `pose_path` set to that file, `calib_path: ""` and `first_frame_ref: True`) samples the same frames
with the same random streams.
"""
from __future__ import annotations

import ctypes as C
import math
import os

import numpy as np
import torch

from . import _abi
from .config import SHINEConfig
from .scans import LiDARDataset, check_process_config, natural_sorted, read_scan

# ------------------------------------------------------------------------------------------------------------- SE(3)


def hat(v) -> np.ndarray:
    """The skew-symmetric matrix of a 3-vector: hat(a) @ b == a x b."""
    return np.array([[0.0, -v[2], v[1]], [v[2], 0.0, -v[0]], [-v[1], v[0], 0.0]])


def _so3_parts(phi):
    """theta, A = sin(theta) / theta, B = (1 - cos(theta)) / theta^2, C = (1 - A) / theta^2 (Taylor series near 0)."""
    th2 = float(np.dot(phi, phi))
    th = math.sqrt(th2)
    if th < 1e-5:
        return th, 1.0 - th2 / 6.0, 0.5 - th2 / 24.0, 1.0 / 6.0 - th2 / 120.0
    return th, math.sin(th) / th, (1.0 - math.cos(th)) / th2, (1.0 - math.sin(th) / th) / th2


def se3_exp(xi) -> np.ndarray:
    """exp of the twist xi = (rho, phi) -> 4x4 fp64 pose [R, V rho; 0, 1]."""
    xi = np.asarray(xi, dtype=np.float64).reshape(6)
    rho, phi = xi[:3], xi[3:]
    _, A, B, Cc = _so3_parts(phi)
    K = hat(phi)
    K2 = K @ K
    T = np.eye(4)
    T[:3, :3] = np.eye(3) + A * K + B * K2
    T[:3, 3] = (np.eye(3) + B * K + Cc * K2) @ rho
    return T


def se3_log(T) -> np.ndarray:
    """log of a 4x4 pose -> twist (rho, phi), |phi| < pi."""
    T = np.asarray(T, dtype=np.float64)
    R = T[:3, :3]
    cos_th = min(1.0, max(-1.0, (np.trace(R) - 1.0) / 2.0))
    th = math.acos(cos_th)
    W = (R - R.T) / 2.0
    w = np.array([W[2, 1], W[0, 2], W[1, 0]])
    if th < 1e-5:
        phi = w * (1.0 + th * th / 6.0)
    elif math.pi - th < 1e-5:                              # near pi: the axis from the symmetric part
        S = (R + np.eye(3)) / 2.0
        k = int(np.argmax(np.diag(S)))
        axis = S[:, k] / math.sqrt(max(S[k, k], 1e-300))
        axis *= 1.0 if np.dot(axis, w) >= 0 else -1.0
        phi = axis * th
    else:
        phi = w * (th / math.sin(th))
    th, A, B, _ = _so3_parts(phi)
    K = hat(phi)
    if th < 1e-5:
        Vinv = np.eye(3) - 0.5 * K + K @ K / 12.0
    else:
        Vinv = np.eye(3) - 0.5 * K + (1.0 - A / (2.0 * B)) / (th * th) * (K @ K)
    return np.concatenate((Vinv @ T[:3, 3], phi))


# ------------------------------------------------------------------------------------------------------ registration


def unpack_normal_equations(out) -> tuple:
    """The 29 values of shine_register_normal_eq -> (H 6x6, b 6, cost, count)."""
    out = np.asarray(out, dtype=np.float64)
    H = np.zeros((6, 6))
    H[np.triu_indices(6)] = out[:21]
    H = H + np.triu(H, 1).T
    return H, out[21:27].copy(), float(out[27]), int(round(out[28]))


class ScanToMapRegistration:
    """Gauss-Newton registration of a scan to the SDF map of `octree` and `decoder`.

    Points are fp32 [n,3] in the sensor frame, in the map's scaled coordinates (what `ScanProcessor.points` returns for
    the identity pose).  Poses are 4x4 fp64 with the translation in metres.  kappa_m: the Geman-McClure scale of the SDF
    residuals, metres; the first iterations run with a wider kernel (8, 4, 2 kappa).  tol: Gauss-Newton stops once an
    update moves the pose by less than tol metres and tol radians.  min_valid: fewer points on the map than this, or a
    singular system, returns the initial pose with ok=False.

    The SDF only pulls points that lie within a few tens of centimetres of a surface, and a scan can constrain one
    translation direction through few points (a street: only the faces across it fix the position along it).  So
    Gauss-Newton starts from the best candidate of a coarse grid around the start (x, y within 2 m and 0.5 m, yaw within
    6 degrees, scored as below at twice kappa).  After that first Gauss-Newton run, the pose is therefore searched along the weakest translation direction of its normal
    equations, search_m either way in steps of search_step_m, for the largest inlier score sum w |g|^2 (the trace of
    the translation block of H: points on a surface count about 1, points off it or off the map about 0); if a candidate
    beats the current pose by more than a relative 1e-3, Gauss-Newton runs again from the best one."""

    WIDE = (8.0, 4.0, 2.0)
    # the coarse grid around the start: x and y of the map frame (metres) and yaw about its z axis (radians)
    GRID_X = np.arange(-8, 9) * 0.25
    GRID_Y = np.arange(-2, 3) * 0.25
    GRID_YAW = np.radians(np.arange(-6, 7) * 1.0)
    # launch_poses splits a batch of poses so that its block partials stay within this many bytes of scratch
    SCRATCH_BOUND_BYTES = 64 << 20

    def __init__(self, config: SHINEConfig, octree, decoder, kappa_m: float = 0.1, max_iters: int = 30,
                 tol: float = 1e-4, min_valid: int = 100, search_m: float = 2.0, search_step_m: float = 0.1):
        self.config, self.octree, self.decoder = config, octree, decoder
        self.kappa_m, self.max_iters, self.tol, self.min_valid = float(kappa_m), int(max_iters), float(tol), int(min_valid)
        self.search_m, self.search_step_m = float(search_m), float(search_step_m)
        self.scale = float(config.scale)
        self.sigma = float(config.sigma_sigmoid)
        self.device = torch.device(config.device)
        self.out = torch.zeros(_abi.REGISTER_OUT, dtype=torch.float64, device=self.device)
        self.scratch = torch.empty(_abi.REGISTER_SCRATCH_BYTES, dtype=torch.uint8, device=self.device)

    def launch(self, points: torch.Tensor, pose_scaled: np.ndarray, kappa_scaled: float, out=None) -> None:
        """One shine_register_normal_eq into out (default self.out; no host read).  pose_scaled: translation in scaled
        units."""
        _abi.require_cuda(points, "ScanToMapRegistration")
        points = points.float().contiguous()
        od = self.octree._descriptor(None, None)
        dd = self.decoder.c_descriptor(None)
        pose = (C.c_double * 16)(*np.ascontiguousarray(pose_scaled, dtype=np.float64).reshape(16).tolist())
        _abi.check(_abi.lib().shine_register_normal_eq(
            C.byref(od), C.byref(dd), _abi.ptr(points), points.shape[0], pose, self.sigma, float(kappa_scaled),
            _abi.ptr(self.out if out is None else out), _abi.ptr(self.scratch), self.scratch.numel(),
            _abi.stream_ptr(self.device)),
            "shine_register_normal_eq")

    def launch_poses(self, points: torch.Tensor, poses_scaled: np.ndarray, kappa_scaled: float, out: torch.Tensor) -> None:
        """The normal equations at K poses (fp64 [K,4,4], translation in scaled units) into out (fp64 [K,29]; no host
        read): shine_register_normal_eq_poses, whose row k equals `launch` at pose k bit for bit.  The poses go in
        batches whose block partials fit SCRATCH_BOUND_BYTES (a 10^6-point scan needs 237 KB per pose, so the 1105
        candidates of the coarse grid take 4 calls; a 3*10^4-point scan takes one).

        A subclass that replaces the field by overriding `launch` (a host-side restatement) keeps working: when `launch`
        is overridden, this calls it once per pose into the rows of out."""
        poses = np.ascontiguousarray(poses_scaled, dtype=np.float64).reshape(-1, 16)
        K = poses.shape[0]
        if out.dtype != torch.float64 or tuple(out.shape) != (K, _abi.REGISTER_OUT) or not out.is_contiguous():
            raise ValueError(f"launch_poses writes fp64 [{K}, {_abi.REGISTER_OUT}] rows: out is {out.dtype} "
                             f"{tuple(out.shape)}{'' if out.is_contiguous() else ', not contiguous'}")
        if type(self).launch is not ScanToMapRegistration.launch:
            for k in range(K):
                self.launch(points, poses[k].reshape(4, 4), kappa_scaled, out[k])
            return
        _abi.require_cuda(points, "ScanToMapRegistration")
        if out.device != points.device:
            raise ValueError(f"launch_poses: out is on {out.device}, the points on {points.device}")
        points = points.float().contiguous()
        n = points.shape[0]
        lib = _abi.lib()
        per_pose = max(1, lib.shine_register_scratch_bytes(n, 1))
        chunk = max(1, min(K, self.SCRATCH_BOUND_BYTES // per_pose))
        need = lib.shine_register_scratch_bytes(n, chunk)
        if self.scratch.numel() < need:
            self.scratch = torch.empty(need, dtype=torch.uint8, device=self.device)
        od = self.octree._descriptor(None, None)
        dd = self.decoder.c_descriptor(None)
        for k0 in range(0, K, chunk):
            kc = min(chunk, K - k0)
            buf = (C.c_double * (16 * kc))(*poses[k0:k0 + kc].reshape(-1).tolist())
            _abi.check(lib.shine_register_normal_eq_poses(
                C.byref(od), C.byref(dd), _abi.ptr(points), n, buf, kc, self.sigma, float(kappa_scaled),
                _abi.ptr(out[k0:k0 + kc]), _abi.ptr(self.scratch), self.scratch.numel(), _abi.stream_ptr(self.device)),
                "shine_register_normal_eq_poses")

    def _scaled(self, poses) -> np.ndarray:
        P = np.array(poses, dtype=np.float64).reshape(-1, 4, 4)
        P[:, :3, 3] *= self.scale
        return P

    def normal_equations_at(self, points: torch.Tensor, poses, kappa_m: float | None = None) -> list:
        """[(H, b, cost, count)] at each of the poses (metres), one launch_poses and one read."""
        P = self._scaled(poses)
        out = torch.empty(P.shape[0], _abi.REGISTER_OUT, dtype=torch.float64, device=self.device)
        self.launch_poses(points, P, (self.kappa_m if kappa_m is None else kappa_m) * self.scale, out)
        return [unpack_normal_equations(row) for row in out.cpu().numpy()]

    def normal_equations(self, points: torch.Tensor, pose: np.ndarray, kappa_m: float | None = None) -> tuple:
        """(H, b, cost, count) of the scan at `pose` (metres): H = sum w J^T J, b = sum w J^T r over the points on the
        map, in scaled units, J for a left-multiplied twist with rho in scaled units; cost = sum w r^2."""
        T = np.array(pose, dtype=np.float64)
        T[:3, 3] *= self.scale
        self.launch(points, T, (self.kappa_m if kappa_m is None else kappa_m) * self.scale)
        return unpack_normal_equations(self.out.cpu().numpy())

    def gauss_newton(self, points: torch.Tensor, pose: np.ndarray) -> tuple:
        """-> (pose, iterations, converged, failure reason or None)."""
        pose = np.array(pose, dtype=np.float64)
        for it in range(self.max_iters):
            wide = it < len(self.WIDE)
            H, b, cost, count = self.normal_equations(points, pose, self.kappa_m * (self.WIDE[it] if wide else 1.0))
            if count < self.min_valid:
                return pose, it + 1, False, f"{count} points on the map (< {self.min_valid})"
            if not np.all(np.isfinite(H)) or np.linalg.cond(H) > 1e12:
                return pose, it + 1, False, "singular normal equations"
            xi = -np.linalg.solve(H, b)
            step = se3_exp(xi)
            step[:3, 3] /= self.scale                       # rho was in scaled units
            pose = step @ pose
            if not wide and np.linalg.norm(xi[:3]) / self.scale < self.tol and np.linalg.norm(xi[3:]) < self.tol:
                return pose, it + 1, True, None
        return pose, self.max_iters, False, None

    def search_weak_direction(self, points: torch.Tensor, pose: np.ndarray) -> tuple:
        """The best pose along the weakest translation direction (class docstring), all candidates in one launch_poses
        -> (pose, moved)."""
        H, _, _, _ = self.normal_equations(points, pose)
        score0 = float(np.trace(H[:3, :3]))
        v = np.linalg.eigh(H[:3, :3])[1][:, 0]              # eigenvalues ascending
        n = int(round(self.search_m / self.search_step_m))
        steps = [k * self.search_step_m for k in range(-n, n + 1) if k != 0]
        cands = []
        for d in steps:
            cand = pose.copy()
            cand[:3, 3] += d * v
            cands.append(cand)
        best, best_score = 0.0, score0
        for d, (H, _, _, _) in zip(steps, self.normal_equations_at(points, cands)):
            score = float(np.trace(H[:3, :3]))
            if score > best_score:
                best, best_score = d, score
        if best_score <= score0 * (1.0 + 1e-3):
            return pose, False
        out = pose.copy()
        out[:3, 3] += best * v
        return out, True

    def coarse_search(self, points: torch.Tensor, pose: np.ndarray) -> np.ndarray:
        """The candidate of the grid around pose (GRID_X x GRID_Y x GRID_YAW) with the largest inlier score sum w |g|^2
        at twice kappa: one launch_poses into one row per candidate, one read for all of them."""
        cands = []
        for yaw in self.GRID_YAW:
            c, s_ = math.cos(yaw), math.sin(yaw)
            Rz = np.array([[c, -s_, 0.0], [s_, c, 0.0], [0.0, 0.0, 1.0]])
            for dx in self.GRID_X:
                for dy in self.GRID_Y:
                    T = pose.copy()
                    T[:3, :3] = Rz @ pose[:3, :3]
                    T[:3, 3] = pose[:3, 3] + (dx, dy, 0.0)
                    cands.append(T)
        outs = torch.empty(len(cands), _abi.REGISTER_OUT, dtype=torch.float64, device=self.device)
        self.launch_poses(points, self._scaled(cands), 2.0 * self.kappa_m * self.scale, outs)
        score = (outs[:, 0] + outs[:, 6] + outs[:, 11]).cpu().numpy()        # H(0,0) + H(1,1) + H(2,2)
        return cands[int(np.argmax(score))]

    def register(self, points: torch.Tensor, init_pose: np.ndarray) -> tuple:
        """The coarse grid search, Gauss-Newton from its best candidate, the search along the weakest direction,
        Gauss-Newton again when that moved the pose ->
        (pose, {iters, valid, rmse_m, ok, converged}).  ok=False (with `reason`): too few points on the map or a singular
        system, the initial pose is returned.  converged=False: the last Gauss-Newton run stopped at max_iters without
        meeting tol (the pose is returned, ok stays True).  valid and rmse_m = sqrt(sum w r^2 / valid) (metres) are
        those of the returned pose."""
        init = np.array(init_pose, dtype=np.float64)
        pose, iters, converged, reason = self.gauss_newton(points, self.coarse_search(points, init))
        if reason is None:
            pose, moved = self.search_weak_direction(points, pose)
            if moved:
                pose, more, converged, reason = self.gauss_newton(points, pose)
                iters += more
        if reason is not None:
            return init, {"iters": iters, "valid": 0, "rmse_m": float("nan"), "ok": False, "converged": False,
                          "reason": reason}
        _, _, cost, count = self.normal_equations(points, pose)
        return pose, {"iters": iters, "valid": count, "rmse_m": math.sqrt(cost / count) / self.scale if count else float("nan"),
                      "ok": True, "converged": converged}


# ------------------------------------------------------------------------------------------------------ frame source


class OdometryScans(LiDARDataset):
    """The scans of config.pc_path (frame selection begin_frame / end_frame / every_frame, readers of scans.py) with
    poses estimated on the way: frame 0 is the identity (the map frame is the first scan's frame); each later frame is
    preprocessed at the identity, registered to the map starting from a constant-velocity prediction, and then sampled
    at the estimated pose exactly as `LiDARDataset.frame_samples` samples it with that pose in `poses_ref`.
    config.pose_path and config.calib_path are not read.  `poses_ref[f]` (metres, map frame) and `reg_info[f]` hold the
    results of the frames read so far.

    Refused (ValueError): `first_frame_ref: False` (its global_shift_default would move the map frame of a remap from the
    written poses away from this one) and a map that is not empty (a loaded map has its own frame, which the first scan,
    taken as the identity, would not be registered to)."""

    def __init__(self, config: SHINEConfig, octree, decoder, pool=None, **registration):
        check_process_config(config)
        if not config.first_frame_ref:
            raise ValueError("pose estimation takes the first scan's frame as the map frame: it needs first_frame_ref: True")
        if octree is not None and not octree.is_empty():
            raise ValueError("pose estimation starts a new map: it cannot continue a loaded one (load_model)")
        self.pc_filenames = natural_sorted(os.listdir(config.pc_path))
        total = len(self.pc_filenames)
        self._init_frames(config, [np.eye(4)] * total, total, None, pool)
        self.begin_pose_inv = np.eye(4)
        self.poses_ref = [np.eye(4) for _ in range(total)]
        self.registration = ScanToMapRegistration(config, octree, decoder, **registration)
        self.reg_info = {}
        self._estimated = []          # frame ids with a pose, in order
        self._record = None

    def read_frame(self, frame_id: int):
        if self._record is not None and self._record[0] == frame_id:
            return self._record[1]
        return read_scan(os.path.join(self.config.pc_path, self.pc_filenames[frame_id]))

    def estimate_pose(self, frame_id: int) -> np.ndarray:
        """Register frame_id to the current map (identity for the first frame) -> its pose, kept in poses_ref."""
        rec = self.read_frame(frame_id)
        self._record = (frame_id, rec)
        if not self._estimated:
            pose, info = np.eye(4), {"iters": 0, "valid": 0, "rmse_m": 0.0, "ok": True, "converged": True}
        else:
            last = self.poses_ref[self._estimated[-1]]
            prev = self.poses_ref[self._estimated[-2]] if len(self._estimated) > 1 else last
            predicted = last @ (np.linalg.inv(prev) @ last)
            local = self.processor.points(rec, np.eye(4))
            pose, info = self.registration.register(local, predicted)
            if not info["ok"]:
                print(f"[odometry] frame {frame_id}: registration failed ({info['reason']}); "
                      "keeping the constant-velocity prediction")
            elif not info["converged"]:
                print(f"[odometry] frame {frame_id}: Gauss-Newton stopped after {info['iters']} iterations without "
                      f"meeting tol; keeping its last pose")
        self.poses_ref[frame_id] = pose
        self.reg_info[frame_id] = info
        self._estimated.append(frame_id)
        return pose

    def frame_samples(self, frame_id: int):
        if frame_id not in self.reg_info:
            self.estimate_pose(frame_id)
        try:
            return super().frame_samples(frame_id)
        finally:
            self._record = None

    def frame_info(self, frame_id: int) -> dict:
        """The history fields of a frame: its pose (3x4 rows, metres) and reg_iters / reg_valid / reg_rmse_m / reg_ok /
        reg_converged."""
        info = self.reg_info[frame_id]
        return {"pose": self.poses_ref[frame_id][:3].tolist(),
                **{f"reg_{k}": v for k, v in info.items() if k in ("iters", "valid", "rmse_m", "ok", "converged")}}

    def write_kitti_poses(self, path: str) -> None:
        """One KITTI row (3x4, row-major, repr floats: they read back bit for bit) per scan of the sequence: the estimated
        pose of a used frame, the last estimate before it for a frame that is not used (identity before the first)."""
        rows, pose = [], np.eye(4)
        for f in range(self.total_pc_count):
            if f in self.reg_info:
                pose = self.poses_ref[f]
            rows.append(" ".join(repr(float(v)) for v in pose[:3].reshape(-1)))
        os.makedirs(os.path.dirname(os.path.abspath(path)), exist_ok=True)
        with open(path, "w") as fh:
            fh.write("\n".join(rows) + "\n")
