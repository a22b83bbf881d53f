"""Mint tests/golden/ref_eval_depth.npz from the UNMODIFIED reference's eval/eval_utils.py `eval_depth`.
*** TEST INFRASTRUCTURE ***

eval_utils imports open3d at module level for its mesh metrics; `eval_depth` uses only numpy.  So the module is loaded
with an empty stand-in `open3d` in sys.modules (as oracle/kaolin_shim stands in for kaolin), from the reference checkout
at $SHINE_REFERENCE (default /root/reference).  Each case is a seeded (pred, target) pair of fp64 depth images with the
cases the metric's mask distinguishes: no prediction (0), targets at 0, at and beyond 10 m, and predictions far off.

    python oracle/make_depth_golden.py

npz keys: pred_{i}, target_{i} (fp64 [H,W]) and metrics_{i} (fp64, in `KEYS` order) for i < count; keys, count.
"""
from __future__ import annotations

import importlib.util
import os
import sys
import types

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF = os.environ.get("SHINE_REFERENCE", "/root/reference")
OUT = os.path.join(ROOT, "tests", "golden", "ref_eval_depth.npz")
KEYS = ["AbsRel", "AbsDiff", "SqRel", "RMSE", "LogRMSE", "r1", "r2", "r3", "complete"]


def load_eval_depth():
    sys.modules.setdefault("open3d", types.ModuleType("open3d"))
    spec = importlib.util.spec_from_file_location("ref_eval_utils", os.path.join(REF, "eval", "eval_utils.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod.eval_depth


def cases():
    rng = np.random.default_rng(2024)
    out = []
    for H, W, hole, far in ((24, 32, 0.1, 0.05), (30, 40, 0.3, 0.2), (7, 5, 0.0, 0.0), (31, 17, 0.6, 0.4)):
        target = rng.uniform(0.2, 12.0, (H, W))
        target[rng.random((H, W)) < hole] = 0.0
        target.flat[: min(3, target.size)] = 10.0                       # exactly at the mask's upper limit
        pred = target * np.exp(rng.normal(0.0, 0.1, (H, W)))
        pred[rng.random((H, W)) < hole] = 0.0                           # no hit
        off = rng.random((H, W)) < far
        pred[off] = rng.uniform(0.01, 20.0, int(off.sum()))             # far off: beyond the 1.25^3 ratio
        out.append((pred, target))
    return out


def main() -> None:
    eval_depth = load_eval_depth()
    arrays = {"keys": np.array(KEYS)}
    cs = cases()
    for i, (pred, target) in enumerate(cs):
        m = eval_depth(pred.copy(), target.copy())
        arrays[f"pred_{i}"], arrays[f"target_{i}"] = pred, target
        arrays[f"metrics_{i}"] = np.array([m[k] for k in KEYS], dtype=np.float64)
    arrays["count"] = np.array(len(cs))
    np.savez_compressed(OUT, **arrays)
    print(f"wrote {OUT}: {len(cs)} cases")


if __name__ == "__main__":
    main()
