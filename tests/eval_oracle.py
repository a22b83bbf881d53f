"""numpy / scipy restatement of mesh evaluation (reference eval/eval_utils.py eval_mesh, nn_correspondance,
crop_intersection, with open3d's TriangleMesh.crop, sample_points_uniformly and voxel_down_sample restated from their
published semantics): the yardstick of csrc/shine_eval.cu and shine_mapping_b200/evaluate.py."""
from __future__ import annotations

import numpy as np
from scipy.spatial import cKDTree

from tests.scan_oracle import voxel_down  # noqa: F401  (open3d voxel_down_sample)

M32 = 0xFFFFFFFF


def crop_keep(verts: np.ndarray, faces: np.ndarray, box) -> np.ndarray:
    """TriangleMesh.crop: a triangle stays iff its three vertices lie in the box, bounds inclusive."""
    lo, hi = np.asarray(box[:3]), np.asarray(box[3:])
    inside = np.all((verts >= lo) & (verts <= hi), axis=1)
    return inside[faces].all(1)


def triangle_areas(verts: np.ndarray, faces: np.ndarray, box=None) -> np.ndarray:
    """0.5 |(p0 - p1) x (p0 - p2)|, the norm as sqrt((x*x + y*y) + z*z); 0 for a cropped triangle."""
    p0, p1, p2 = (verts[faces[:, k]] for k in range(3))
    a, b = p0 - p1, p0 - p2
    cx = a[:, 1] * b[:, 2] - a[:, 2] * b[:, 1]
    cy = a[:, 2] * b[:, 0] - a[:, 0] * b[:, 2]
    cz = a[:, 0] * b[:, 1] - a[:, 1] * b[:, 0]
    area = 0.5 * np.sqrt((cx * cx + cy * cy) + cz * cz)
    if box is not None:
        area = np.where(crop_keep(verts, faces, box), area, 0.0)
    return area


def cdf(area: np.ndarray) -> np.ndarray:
    """SamplePointsUniformlyImpl: S summed in sequence, C_t = area_t / S + C_{t-1}."""
    s = 0.0
    for a in area.tolist():
        s += a
    return np.cumsum(area / s)


def sample_counts(area: np.ndarray, n: int):
    """-> (samples per triangle, C_t N): triangle t gets [round(C_{t-1} N), round(C_t N)), the last end N."""
    c = cdf(area)
    ends = np.round(c * n).astype(np.int64)
    ends[-1] = n
    return np.diff(np.r_[0, ends]), c * n


def _mulhilo(a: int, b: np.ndarray):
    p = np.uint64(a) * b.astype(np.uint64)
    return (p >> np.uint64(32)).astype(np.uint32), (p & np.uint64(M32)).astype(np.uint32)


def philox4x32_10(counter: np.ndarray, seed: int):
    """Philox4x32-10 with counter (lo, hi, 0, 0) = counter (uint64 array) and key (lo, hi) = seed -> 4 uint32 arrays."""
    counter = counter.astype(np.uint64)
    c0 = (counter & np.uint64(M32)).astype(np.uint32)
    c1 = (counter >> np.uint64(32)).astype(np.uint32)
    c2 = np.zeros_like(c0)
    c3 = np.zeros_like(c0)
    k0, k1 = seed & M32, (seed >> 32) & M32
    for r in range(10):
        if r:
            k0, k1 = (k0 + 0x9E3779B9) & M32, (k1 + 0xBB67AE85) & M32
        hi0, lo0 = _mulhilo(0xD2511F53, c0)
        hi1, lo1 = _mulhilo(0xCD9E8D57, c2)
        c0, c1, c2, c3 = hi1 ^ c1 ^ np.uint32(k0), lo1, hi0 ^ c3 ^ np.uint32(k1), lo0
    return c0, c1, c2, c3


def unit53(a: np.ndarray, b: np.ndarray) -> np.ndarray:
    return (((a >> np.uint32(5)).astype(np.uint64) << np.uint64(26)) | (b >> np.uint32(6)).astype(np.uint64)) * 2.0 ** -53


def sample_points(verts: np.ndarray, faces: np.ndarray, tri_ids: np.ndarray, seed: int) -> np.ndarray:
    """Sample k on triangle tri_ids[k]: (a v0 + b v1) + c v2 with Philox(seed, k)'s r1, r2."""
    x0, x1, x2, x3 = philox4x32_10(np.arange(tri_ids.shape[0], dtype=np.uint64), seed)
    r1, r2 = unit53(x0, x1), unit53(x2, x3)
    s = np.sqrt(r1)
    a, b, c = 1.0 - s, s * (1.0 - r2), s * r2
    f = faces[tri_ids]
    v0, v1, v2 = verts[f[:, 0]], verts[f[:, 1]], verts[f[:, 2]]
    return (a[:, None] * v0 + b[:, None] * v1) + c[:, None] * v2


def dist2(q: np.ndarray, p: np.ndarray) -> np.ndarray:
    d = q - p
    return (d[..., 0] * d[..., 0] + d[..., 1] * d[..., 1]) + d[..., 2] * d[..., 2]


def nearest(ref: np.ndarray, queries: np.ndarray, k: int = 8):
    """-> (minimum d2 with the kernel's formula over cKDTree's k candidates, its index).  Empty ref: (+inf, -1)."""
    m = queries.shape[0]
    if ref.shape[0] == 0:
        return np.full(m, np.inf), np.full(m, -1, dtype=np.int64)
    k = min(k, ref.shape[0])
    _, idx = cKDTree(ref).query(queries, k=k)
    idx = idx.reshape(m, k)
    d2 = dist2(queries[:, None, :], ref[idx])
    j = np.argmin(d2, axis=1)
    return d2[np.arange(m), j], idx[np.arange(m), j]


def nn_correspondance(ref: np.ndarray, queries: np.ndarray, truncation: float, ignore_outlier: bool) -> np.ndarray:
    """eval_utils.py:110-141: the distances kept (d2 < truncation^2) or clamped to truncation."""
    if ref.shape[0] == 0 or queries.shape[0] == 0:
        return np.zeros(0)
    d2, _ = nearest(ref, queries)
    inside = d2 < truncation ** 2
    if ignore_outlier:
        return np.sqrt(d2[inside])
    return np.where(inside, np.sqrt(d2), truncation)


def metrics(dist_p: np.ndarray, dist_r: np.ndarray, down_sample_res, threshold, truncation_acc, truncation_com) -> dict:
    """eval_utils.py:79-106 from the kept / clamped distance lists."""
    with np.errstate(invalid="ignore", divide="ignore"):
        mp = np.mean(dist_p) if dist_p.size else np.nan
        mr = np.mean(dist_r) if dist_r.size else np.nan
        mps = np.mean(np.square(dist_p)) if dist_p.size else np.nan
        mrs = np.mean(np.square(dist_r)) if dist_r.size else np.nan
        precision = (np.mean((dist_p < threshold).astype("float")) if dist_p.size else np.nan) * 100.0
        recall = (np.mean((dist_r < threshold).astype("float")) if dist_r.size else np.nan) * 100.0
        fscore = 2 * precision * recall / (precision + recall)
        return {"MAE_accuracy (m)": mp, "MAE_completeness (m)": mr, "Chamfer_L1 (m)": 0.5 * (mp + mr),
                "Chamfer_L2 (m)": np.sqrt(0.5 * (mps + mrs)), "Precision [Accuracy] (%)": precision,
                "Recall [Completeness] (%)": recall, "F-score (%)": fscore, "Spacing (m)": down_sample_res,
                "Inlier_threshold (m)": threshold, "Outlier_truncation_acc (m)": truncation_acc,
                "Outlier_truncation_com (m)": truncation_com}


def metrics_from_points(pred: np.ndarray, gt: np.ndarray, down_sample_res, threshold, truncation_acc, truncation_com):
    """Down-sampled clouds -> the metrics (both directions, the reference's truncation rules)."""
    dp = nn_correspondance(gt, pred, truncation_acc, True)
    dr = nn_correspondance(pred, gt, truncation_com, False)
    return metrics(dp, dr, down_sample_res, threshold, truncation_acc, truncation_com)
