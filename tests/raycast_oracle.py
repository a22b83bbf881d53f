"""fp64 restatement of `shine_raycast` (include/shine_b200.h, csrc/shine_raycast.cu) for tests/test_gpu_raycast.py and
tools/raycast_bench.py: the fp32 lattice and sample positions exactly as the kernel forms them, the mask exactly, the
field in fp64 with the oracle's query (tests/mesh_oracle.py `query`) and the per-sample error bound of the fused
decoder (`error_bound.decoder_passes`, its P).  The march visits every sample (no empty-space skipping).
Test infrastructure, no GPU needed."""
from __future__ import annotations

import numpy as np
import torch

from oracle import shine_oracle as orc
from tests.error_bound import abs_feature, decoder_passes

F32 = np.float32
MAX_K = 2 ** 24 - 1


def rays(origin, points):
    """-> (d [n,3] fp32, r [n] fp32) as the kernel forms them."""
    o = np.asarray(origin, dtype=F32).reshape(1, 3)
    v = (np.asarray(points, dtype=F32).reshape(-1, 3) - o).astype(F32)
    r = np.sqrt(((v[:, 0] * v[:, 0] + v[:, 1] * v[:, 1]).astype(F32) + v[:, 2] * v[:, 2]).astype(F32)).astype(F32)
    with np.errstate(divide="ignore", invalid="ignore"):
        d = (v / r[:, None]).astype(F32)
    return d, r


def lattice_count(r, h, t_min, beyond, t_max):
    """K per ray (-1: no sample)."""
    with np.errstate(invalid="ignore"):
        e = np.minimum((r + F32(beyond)).astype(F32), F32(t_max)).astype(F32)
        kf = np.floor(((e - F32(t_min)).astype(F32) / F32(h)).astype(F32))
    ok = (r > 0) & np.isfinite(r) & (kf >= 0)
    return np.where(ok, np.minimum(np.nan_to_num(kf, nan=-1.0, posinf=MAX_K), MAX_K), -1).astype(np.int64)


def lattice_t(k, h, t_min):
    return (F32(t_min) + (np.asarray(k).astype(F32) * F32(h)).astype(F32)).astype(F32)


def positions(origin, d, t):
    o = np.asarray(origin, dtype=F32).reshape(1, 3)
    return (o + (np.asarray(t, dtype=F32)[:, None] * d).astype(F32)).astype(F32)


def present(o, x, level_index):
    """x's voxel exists at featured level `level_index` (bottom-up)."""
    level = o.max_level - level_index
    keys = orc.points_to_morton(orc.quantize_points(x, level)).tolist()
    table = o.nodes_lookup_tables[level]
    return np.fromiter((k in table for k in keys), dtype=bool, count=len(keys))


def field(o, dec, x, n_levels):
    """-> (s fp64 = -Decoder.sdf, bound of |s_kernel - s|) at fp32 points x."""
    if x.shape[0] == 0:
        return np.zeros(0), np.zeros(0)
    with torch.no_grad():
        c = torch.from_numpy(np.ascontiguousarray(x))
        feat = o.query_feature(c)
        s = -orc.decoder_sdf(feat, dec)
        P = decoder_passes(feat, abs_feature(o, c), dec, False, n_levels)["P"]
    return s.numpy().astype(np.float64), P.numpy().astype(np.float64)


def march(o, dec, origin, points, h, t_min, beyond, t_max, refine_iters, mask_level, chunk=400_000):
    """The kernel's definition without skipping.  -> dict of per-ray arrays:
    hit, k (the bracket's upper sample, -1 on a miss), t (refined in fp64 field values, NaN on a miss), ta / tb / sa / sb
    / Pa / Pb (the final bracket and its bounds), ambiguous (a visited masked sample has |s| <= its bound),
    refine_ambiguous (a bisection midpoint does), div_w (the width of the bracket that the first such midpoint splits: a
    march that takes the other branch there still ends inside it), samples (lattice samples visited: K + 1)."""
    n_levels = o.featured_level_num
    d, r = rays(origin, points)
    n = d.shape[0]
    K = lattice_count(r, h, t_min, beyond, t_max)
    ray_of = np.repeat(np.arange(n), np.maximum(K + 1, 0))
    kk = np.concatenate([np.arange(k + 1) for k in K]) if n else np.zeros(0, dtype=np.int64)
    tt = lattice_t(kk, h, t_min)
    m = np.zeros(kk.shape[0], dtype=bool)
    s = np.zeros(kk.shape[0])
    P = np.zeros(kk.shape[0])
    for a in range(0, kk.shape[0], chunk):
        x = positions(origin, d[ray_of[a:a + chunk]], tt[a:a + chunk])
        mm = present(o, x, mask_level)
        m[a:a + chunk] = mm
        idx = np.nonzero(mm)[0]
        s[a + idx], P[a + idx] = field(o, dec, x[idx], n_levels)
    start = np.concatenate(([0], np.cumsum(np.maximum(K + 1, 0))))
    out = {k: np.full(n, np.nan) for k in ("t", "ta", "tb", "sa", "sb", "Pa", "Pb", "div_w")}
    out.update(hit=np.zeros(n, bool), k=np.full(n, -1), ambiguous=np.zeros(n, bool),
               refine_ambiguous=np.zeros(n, bool), samples=np.maximum(K + 1, 0))
    for i in range(n):
        a, b = start[i], start[i + 1]
        mi, si, Pi = m[a:b], s[a:b], P[a:b]
        cross = np.nonzero(mi[:-1] & mi[1:] & (si[:-1] > 0) & (si[1:] <= 0))[0]
        last = b - a if cross.size == 0 else cross[0] + 2
        out["ambiguous"][i] = bool((mi[:last] & (np.abs(si[:last]) <= Pi[:last])).any())
        if cross.size:
            k = cross[0] + 1
            out["hit"][i], out["k"][i] = True, k
            out["ta"][i], out["tb"][i] = tt[a + k - 1], tt[a + k]
            out["sa"][i], out["sb"][i], out["Pa"][i], out["Pb"][i] = si[k - 1], si[k], Pi[k - 1], Pi[k]
    # bisection, all hit rays at once
    live = out["hit"].copy()
    ta, tb = out["ta"].astype(F32), out["tb"].astype(F32)
    for _ in range(refine_iters):
        ix = np.nonzero(live)[0]
        if ix.size == 0:
            break
        tm = (F32(0.5) * (ta[ix] + tb[ix]).astype(F32)).astype(F32)
        inside = (tm > ta[ix]) & (tm < tb[ix])
        live[ix[~inside]] = False
        ix, tm = ix[inside], tm[inside]
        x = positions(origin, d[ix], tm)
        mm = present(o, x, mask_level)
        live[ix[~mm]] = False
        ix, tm, x = ix[mm], tm[mm], x[mm]
        sm, Pm = field(o, dec, x, n_levels)
        amb = (np.abs(sm) <= Pm) & ~out["refine_ambiguous"][ix]
        out["div_w"][ix[amb]] = tb[ix[amb]].astype(np.float64) - ta[ix[amb]]
        out["refine_ambiguous"][ix[amb]] = True
        pos = sm > 0
        for sel, which in ((pos, "a"), (~pos, "b")):
            j = ix[sel]
            (ta if which == "a" else tb)[j] = tm[sel]
            out["s" + which][j], out["P" + which][j] = sm[sel], Pm[sel]
    hit = out["hit"]
    out["ta"][hit], out["tb"][hit] = ta[hit], tb[hit]
    q = out["sa"][hit] / (out["sa"][hit] - out["sb"][hit])
    out["t"][hit] = out["ta"][hit] + (out["tb"][hit] - out["ta"][hit]) * q
    return out


def skip_samples(o, origin, points, h, t_min, beyond, t_max):
    """Lattice samples the kernel's march probes with empty-space skipping, per ray, up to the end of the lattice (hits
    ignored: an upper bound of the probes of a ray that hits): the coarsest-level cell walk of csrc/shine_raycast.cu."""
    d, r = rays(origin, points)
    K = lattice_count(r, h, t_min, beyond, t_max)
    L = o.featured_level_num
    level = o.max_level - (L - 1)
    table = o.nodes_lookup_tables[level]
    res = F32(2 ** level)
    out = np.zeros(d.shape[0], dtype=np.int64)
    o32 = np.asarray(origin, dtype=F32)

    def cell(i, k):
        x = positions(origin, d[i:i + 1], lattice_t(np.array([k]), h, t_min))
        return tuple(orc.quantize_points(x, level)[0].tolist()), x

    for i in range(d.shape[0]):
        k, visits = 0, 0
        while k <= K[i]:
            visits += 1
            c0, x = cell(i, k)
            if int(orc.points_to_morton(np.array([c0]))[0]) in table:
                k += 1
                continue
            t_exit = np.inf
            for a in range(3):
                if d[i, a] > 0 and c0[a] + 1 < res:
                    t_exit = min(t_exit, (-1.0 + 2.0 * (c0[a] + 1) / float(res) - float(o32[a])) / float(d[i, a]))
                elif d[i, a] < 0 and c0[a] > 0:
                    t_exit = min(t_exit, (-1.0 + 2.0 * c0[a] / float(res) - float(o32[a])) / float(d[i, a]))
            je = np.floor((t_exit - t_min) / h)
            j = int(K[i]) if je >= K[i] else (k if je <= k else int(je))
            while j > k and cell(i, j)[0] != c0:
                j = k + (j - k) // 2
            k = j + 1
        out[i] = visits
    return out, np.maximum(K + 1, 0)
