"""The camera rays of `shine_render` (include/shine_b200.h) restated with numpy's fp32 arithmetic, operation by operation,
for tests/test_render_host.py and tests/test_gpu_render.py.  Sines and cosines are evaluated in fp64 and rounded to fp32,
as the kernel does.  Test infrastructure, no GPU needed."""
from __future__ import annotations

import math

import numpy as np

F32 = np.float32


def pixel_grid(W: int, H: int):
    """(u, v) of every pixel in row-major order, int64."""
    v, u = np.meshgrid(np.arange(H), np.arange(W), indexing="ij")
    return u.reshape(-1), v.reshape(-1)


def pinhole_dirs(W, H, fx, fy, cx, cy):
    """-> (c fp32 [H W, 3] camera-frame unit directions, c_z fp32 [H W]: depth = t c_z)."""
    u, v = pixel_grid(W, H)
    a = ((u.astype(F32) - F32(cx)).astype(F32) / F32(fx)).astype(F32)
    b = ((v.astype(F32) - F32(cy)).astype(F32) / F32(fy)).astype(F32)
    n = np.sqrt(((a * a).astype(F32) + (b * b).astype(F32)).astype(F32) + F32(1)).astype(F32)
    c = np.stack([(a / n).astype(F32), (b / n).astype(F32), (F32(1) / n).astype(F32)], 1)
    return c, c[:, 2].copy()


def range_image_steps(W, H, fov_up, fov_down):
    """(el0, del, az0, daz) as the entry rounds them from fp64."""
    deg = math.pi / 180.0
    up, down = float(F32(fov_up)), float(F32(fov_down))
    el0 = F32(up * deg)
    de = F32((up - down) * deg / (H - 1)) if H > 1 else F32(0)
    return el0, de, F32(math.pi), F32(2.0 * math.pi / W)


def range_image_dirs(W, H, fov_up, fov_down):
    """-> (c fp32 [H W, 3], ones: depth = t)."""
    el0, de, az0, daz = range_image_steps(W, H, fov_up, fov_down)
    u, v = pixel_grid(W, H)
    el = (el0 - (v.astype(F32) * de).astype(F32)).astype(F32).astype(np.float64)
    az = (az0 - (u.astype(F32) * daz).astype(F32)).astype(F32).astype(np.float64)
    ce, se, ca, sa = (np.cos(el).astype(F32), np.sin(el).astype(F32), np.cos(az).astype(F32),
                      np.sin(az).astype(F32))
    c = np.stack([(ce * ca).astype(F32), (ce * sa).astype(F32), se], 1)
    return c, np.ones(c.shape[0], F32)


def map_rays(c, pose12):
    """pose12: the fp32 3x4 camera-to-map transform the kernel gets -> (origin fp32 [3], d fp32 [n,3] = R c per row
    ((R0 c0 + R1 c1) + R2 c2))."""
    P = np.asarray(pose12, dtype=F32).reshape(3, 4)
    d = np.stack([(((P[a, 0] * c[:, 0]).astype(F32) + (P[a, 1] * c[:, 1]).astype(F32)).astype(F32) +
                   (P[a, 2] * c[:, 2]).astype(F32)).astype(F32) for a in range(3)], 1)
    return P[:, 3].copy(), d
