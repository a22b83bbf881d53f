"""shine_render's normals graded against the fp64 reference of sdf_grad_at (tests/grad_field_bound.py), on the level matrix
of test_gpu_register_grade and both camera models, kink points included.

At the GPU's hit point x (fp32), n = -g / |g|.  If the kernel's g lies within e_g of the reference's g (per component) for
one mask alternative of the point, then |n_gpu - n| <= 2 |e_g| / |g| plus the normalisation's roundings (8 u), where
|g| > 4 |e_g|.  A point passes if one of its alternatives holds that bound.  Points where no alternative has |g| > 4 |e_g|
are cut: there the direction of g is ill-conditioned, a loss of conditioning and not a gap in the error model.  The cut
must stay a small share of the hits."""
import numpy as np
import pytest
import torch

from tests import raycast_oracle as ro
from tests import render_rays as rr
from tests.error_bound import U
from tests.grad_field_bound import GradRef
from tests.parity_utils import build_cuda_models, make_case
from tests.test_gpu_infer_grade import load_tables, scaled
from tests.test_gpu_register_grade import LEVELS, VARIANTS
from tests.test_gpu_render import _camera, _dirs, _lively, _render, _views

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


@pytest.fixture(scope="module", autouse=True)
def _lib(built_lib):
    assert torch.cuda.is_available()
    return built_lib


def grade_normals(ref, nrm, what):
    """-> (graded, cut, worst ratio): every point with a well-conditioned alternative must match one of them"""
    lg, le = np.linalg.norm(ref.g, axis=1), np.linalg.norm(ref.eg, axis=1)
    cond = lg > 4 * le
    safe = np.where(cond, lg, 1.0)
    want = -ref.g / safe[:, None]
    bound = (2 * le / safe + 8 * U)[:, None]
    ratio = (np.abs(np.asarray(nrm, np.float64)[ref.pt] - want) / bound).max(1)
    ratio = np.where(cond, ratio, np.inf)
    best = np.full(ref.n, np.inf)
    np.minimum.at(best, ref.pt, ratio)
    has = np.zeros(ref.n, bool)
    has[ref.pt[cond]] = True
    has &= ~ref.dropped
    bad = np.flatnonzero(has & ~(best <= 1.0))
    if bad.size:
        i = bad[0]
        raise AssertionError(f"{what}: {bad.size} normals outside their bound; first {i} (kink {ref.kink[i]}): got "
                             f"{nrm[i]} want {want[ref.pt == i][0]} bound {bound[ref.pt == i][0, 0]:.3g}")
    worst = float(best[has].max()) if has.any() else 0.0
    return int(has.sum()), int((~has).sum()), worst, int((ref.kink & has).sum())


@pytest.mark.parametrize("poly,bias", VARIANTS, ids=lambda v: str(v))
@pytest.mark.parametrize("levels,world", LEVELS)
def test_render_normals_graded(levels, world, poly, bias):
    seed = 960 + 10 * levels + 2 * poly + bias
    case = _lively(make_case(n_points=1500, n_batch=16, feat_levels=levels, world_level=world, seed=seed, poly=poly,
                             bias=bias))
    cfg, octree, cdec = build_cuda_models(case, DEV)
    graded = cut = kinks = 0
    worst = 0.0
    for ts in (1, 300):
        cs = scaled(case, ts)
        load_tables(octree, cs)
        rng = np.random.default_rng(seed + ts)
        for model, W, H, p, pose12, h, t_max in _views(cs, rng):
            h *= 2.0 ** min(0, 12 - world)          # the views' steps are set for world level 12's leaf
            rc, t, _, nrm, status = _render(octree, cdec, _camera(model, W, H, *p), pose12, h, t_max)
            assert rc == 0
            hit = status == 1
            if not hit.any():
                continue
            origin, d = rr.map_rays(_dirs(model, W, H, *p)[0], pose12)
            x = ro.positions(origin, d[hit], t[hit])
            ref = GradRef(cs, x)
            g_, c_, w_, k_ = grade_normals(ref, nrm[hit], f"L{levels} W{world} {model} x{ts}")
            graded, cut, kinks, worst = graded + g_, cut + c_, kinks + k_, max(worst, w_)
    print(f"[render normals] L{levels} W{world} poly {poly} bias {bias}: {graded} normals graded ({kinks} kink), "
          f"{cut} cut, worst {worst:.3f} of the bound")
    assert graded >= 10
    assert cut <= 0.05 * (graded + cut), f"the conditioning cut removes {cut} of {graded + cut} hits"
