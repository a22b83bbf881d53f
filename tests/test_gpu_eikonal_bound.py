"""The eikonal paths graded element by element against the fp64 reference of tests/eikonal_bound.py (error model in its
docstring): the fused eikonal step in all six instantiations, the query kernels at the C ABI for F = 4, 8, 16 and 32,
and the class-surface recipe `batch_loop.eikonal_iteration`.  Every case prints its worst error / bound.

The fused step is linear in weight_e: each case runs at the reference's weight_e = 0.1 and again at a weight_e at which
the eikonal term dominates the rows the surface samples touch (`dominant_weight`), so that the eikonal scatter is graded
per element without a difference of two runs."""
import ctypes as C

import numpy as np
import pytest
import torch

from tests import sdf_diff_oracle as sdo
from tests.eikonal_bound import EikRef, QueryRef, autograd_decoder_grads, clean_case, dominant_weight, level_geometry
from tests.error_bound import RowSums, grade_values, oracle64, subset
from tests.parity_utils import DEC_KEYS, build_cuda_models, make_case, sort_case_morton

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
UNSUPPORTED = -2                        # SHINE_ERR_UNSUPPORTED


@pytest.fixture(scope="module", autouse=True)
def _lib(built_lib):
    assert torch.cuda.is_available()
    return built_lib


def _case(levels, poly, seed, scale=300.0, weighted=False, reduction="mean", bias=True, n=None, ordered=False,
          feature_dim=8):
    """n: the last n points of the batch (make_case's 6 stragglers and 10 surface points come last)."""
    case = make_case(n_points=2000, n_batch=60000 if (n or 0) > 10000 else 1500, feat_levels=levels, seed=seed, poly=poly,
                     weighted=weighted, reduction=reduction, bias=bias, feature_dim=feature_dim)
    case["tables"] = [(t * np.float32(scale)).astype(np.float32) for t in case["tables"]]
    if n is not None:
        case = subset(case, np.arange(case["coord"].shape[0] - n, case["coord"].shape[0]))
    return sort_case_morton(case) if ordered else case


def _dev(case):
    return tuple(torch.from_numpy(case[k]).to(DEV) for k in ("coord", "label", "weight"))


# ---- the fused eikonal step ------------------------------------------------------------------------------------------------------

class _Fused:
    def __init__(self, case, loss_type, frozen):
        from shine_mapping_b200 import SdfTrainer
        self.cfg, octree, self.dec = build_cuda_models(case, DEV, freeze_decoder=frozen)
        self.tr = SdfTrainer(self.cfg, octree, self.dec, main_loss_type=loss_type)
        self.frozen = frozen
        self.inputs = _dev(case)

    def run(self, weight_e):
        coord, label, weight = self.inputs
        n = coord.shape[0]
        self.cfg.weight_e = weight_e
        self.tr.zero_grad()
        g = torch.full((n, 3), float("nan"), device=DEV)
        pred = torch.full((n,), float("nan"), device=DEV)
        loss, eik = self.tr.forward_backward_eikonal(coord, label, weight, pred_out=pred, grad_out=g)
        torch.cuda.synchronize()
        dec = {k: v.cpu().numpy().copy() for k, v in zip(DEC_KEYS, self.tr.dec_grads) if v is not None}
        return {"table_grads": [t.cpu().numpy().copy() for t in self.tr.table_grads], "dec_grads": dec,
                "pred": pred.cpu().numpy(), "g": g.cpu().numpy(), "loss": float(loss), "eikonal": float(eik)}


def _check_decoder(got, case, weight_e, loss_type, ref, what):
    """compare_step's check of the decoder gradients (1e-3 of each tensor's maximum) against the oracle's fp64 double
    backward, with the L1 signs of the kernel's pred near the label."""
    sign = None
    if loss_type == "sdf_l1":
        sign = sdo.l1_sign(ref.pred, case["label"], got["pred"], ref.P, 0.0)
    want = autograd_decoder_grads(case, weight_e, loss_type, sign)
    worst = 0.0
    for k, w in want.items():
        scale = max(float(np.abs(w).max()), 1e-30)
        d = float(np.abs(got["dec_grads"][k] - w).max()) / scale
        assert d <= 1e-3 + 1e-9 / scale, f"{what}: decoder gradient {k} off by {d:.2e} of its maximum"
        worst = max(worst, d)
    print(f"[eikonal bounds] {what}: decoder grads worst {worst:.1e} of their maxima")


FUSED_CASES = [   # loss, frozen, levels, poly, scale, bias, weighted, reduction, n, ordered, seed
    pytest.param("sdf_bce", False, 1, True, 1.0, True, False, "mean", None, False, 301, id="bce-L1-x1"),
    pytest.param("sdf_bce", False, 4, False, 300.0, True, True, "sum", None, False, 302, id="bce-L4-linear-weighted-sum"),
    pytest.param("sdf_bce", False, 8, True, 300.0, True, True, "mean", None, False, 303, id="bce-L8-weighted-mean"),
    pytest.param("sdf_bce", False, 4, True, 300.0, True, False, "mean", None, True, 304, id="bce-L4-morton"),
    pytest.param("sdf_bce", False, 4, True, 300.0, True, False, "mean", 33, False, 305, id="bce-n33"),
    pytest.param("sdf_bce", False, 4, True, 300.0, True, True, "mean", 60016, False, 306, id="bce-n60016"),
    pytest.param("sdf_bce", True, 4, True, 300.0, False, False, "mean", None, False, 307, id="bce-L4-nobias-frozen"),
    pytest.param("sdf_bce", True, 1, False, 1.0, True, True, "sum", 1, False, 308, id="bce-L1-linear-frozen-n1"),
    pytest.param("sdf_l1", False, 8, True, 300.0, True, True, "mean", None, False, 311, id="l1-L8"),
    pytest.param("sdf_l1", False, 4, False, 1.0, False, True, "mean", 129, False, 312, id="l1-L4-linear-nobias-n129"),
    pytest.param("sdf_l1", True, 4, True, 300.0, True, True, "mean", None, True, 313, id="l1-L4-morton-frozen"),
    pytest.param("sdf_l1", True, 1, False, 300.0, True, True, "mean", 31, False, 314, id="l1-L1-linear-frozen-n31"),
    pytest.param("sdf_l2", False, 1, True, 300.0, True, True, "mean", None, False, 321, id="l2-L1"),
    pytest.param("sdf_l2", False, 4, False, 300.0, True, True, "mean", None, True, 322, id="l2-L4-linear-morton"),
    pytest.param("sdf_l2", False, 4, True, 300.0, True, True, "mean", 60016, False, 323, id="l2-n60016"),
    pytest.param("sdf_l2", True, 8, True, 300.0, False, True, "mean", None, False, 324, id="l2-L8-nobias-frozen"),
]


@pytest.mark.parametrize("loss_type,frozen,levels,poly,scale,bias,weighted,reduction,n,ordered,seed", FUSED_CASES)
def test_fused_eikonal_step_per_element(loss_type, frozen, levels, poly, scale, bias, weighted, reduction, n, ordered,
                                        seed):
    """shine_sdf_eikonal_step (DEC_GRAD x {BCE, sdf_l1, sdf_l2}): pred, g, the loss and
    eikonal scalars and every table-gradient element within their bounds, at weight_e = 0.1 and at a dominant weight_e."""
    case = _case(levels, poly, seed, scale, weighted or loss_type != "sdf_bce", reduction, bias, n, ordered)
    case, dropped = clean_case(case, loss_type)
    big = dominant_weight(case, loss_type)
    step = _Fused(case, loss_type, frozen)
    for weight_e in (0.1, big):
        got = step.run(weight_e)
        ref = EikRef(case, weight_e, loss_type, pred=got["pred"])
        med, top = ref.eikonal_share()
        what = (f"fused {loss_type} {'frozen' if frozen else 'trainable'} N={ref.n} surface={ref.n_surface} "
                f"weight_e={weight_e:.3g} (dropped {dropped}, eikonal share of touched rows: median {med:.2f})")
        ref.grade(got, what)
        if frozen:
            assert all(float(g.abs().max()) == 0.0 for g in step.tr.dec_grads if g is not None)
        elif weight_e == 0.1:
            _check_decoder(got, case, weight_e, loss_type, ref, what)


# ---- the query kernels at the C ABI ----------------------------------------------------------------------------------------------

def _face_points(case, rng, per_level=6):
    """Points placed exactly on a cell face of each level (d = 0 on x) and just below one (d -> 1), from surface points."""
    c = case["cfg"]
    base = case["coord"][case["weight"] > 0][:per_level]
    out = []
    for i in range(c["tree_level_feat"]):
        res = np.float32(2.0 ** (c["tree_level_world"] - i))
        for p in base:
            half, one = np.float32(0.5), np.float32(1)
            k = np.floor(res * (np.float32(p[0]) * half + half))
            v = np.float32(k / res)                     # 0.5 x + 0.5 on the face; below: the fp32 values under it
            face, below = np.float32(2) * v - one, None
            vb = v
            for _ in range(64):
                vb = np.nextafter(vb, np.float32(0))
                xb = np.float32(2) * vb - one
                if res * (xb * half + half) < k:
                    below = xb
                    break
            for xx in (face, below):
                if xx is not None:
                    q = p.copy()
                    q[0] = xx
                    out.append(q)
    pts = np.asarray(out, dtype=np.float32)
    fr = []
    for i in range(c["tree_level_feat"]):
        res = np.float32(2.0 ** (c["tree_level_world"] - i))
        cc = res * (pts[:, 0] * np.float32(0.5) + np.float32(0.5))
        fr.append(cc - np.trunc(cc))
    fr = np.stack(fr, 1)
    assert (fr == 0).any() and (fr > 0.99).any(), "no point on a face / just below one"
    return pts


def _spread(rng, shape):
    """Values over four decades with both signs, a tenth of them exact zeros (fp32)."""
    v = rng.standard_normal(shape) * 10.0 ** rng.uniform(-2, 2, shape)
    v[rng.random(shape) < 0.1] = 0.0
    return v.astype(np.float32)


def _query_case(F, levels, poly, seed):
    case = make_case(n_points=2000, n_batch=3000, feat_levels=levels, seed=seed, poly=poly, feature_dim=F)
    case["tables"] = [(t * np.float32(300.0)).astype(np.float32) for t in case["tables"]]
    rng = np.random.default_rng(seed)
    faces = _face_points(case, rng)
    case["coord"] = np.concatenate((case["coord"], faces)).astype(np.float32)
    case["label"] = np.concatenate((case["label"], np.zeros(faces.shape[0], np.float32)))
    case["weight"] = np.concatenate((case["weight"], np.ones(faces.shape[0], np.float32)))
    return case


def _call(lib, name, *args):
    rc = getattr(lib, name)(*args)
    assert rc == 0, f"{name} returned {rc}"


@pytest.mark.parametrize("F", [4, 8, 16, 32])
@pytest.mark.parametrize("levels,poly", [(1, True), (3, False), (8, True)])
def test_query_kernels_per_element(F, levels, poly, built_lib):
    """shine_query_fwd, shine_query_coord_grad, shine_query_tangent_fwd and shine_query_tangent_bwd on their own, with
    chosen dfeat / tangents, for n = 1, 7, 33 and the whole batch (the LP = F / 4 lanes of a point: groups that end
    mid-warp).  The last points are make_case's stragglers (misses, cube faces, exact corners) and points on / just below
    a cell face of each level."""
    from shine_mapping_b200 import _abi
    full = _query_case(F, levels, poly, 400 + 10 * F + levels)
    cfg, octree, dec = build_cuda_models(full, DEV)
    N = full["coord"].shape[0]
    rng = np.random.default_rng(F * 100 + levels)
    st = _abi.stream_ptr(DEV)
    for n in (1, 7, 33, N):
        case = subset(full, np.arange(N - n, N))
        dfeat, tangent = _spread(rng, (n, F)), _spread(rng, (n, 3))
        ref = QueryRef(case, dfeat, tangent)
        coord, d, t = (torch.from_numpy(a).to(DEV) for a in (case["coord"], dfeat, tangent))
        feat = torch.full((n, F), float("nan"), device=DEV)
        G = torch.full((n, 3), float("nan"), device=DEV)
        tf = torch.full((n, F), float("nan"), device=DEV)
        grads = [torch.zeros_like(p) for p in octree.hier_features]
        desc = octree._descriptor(None, None)
        _call(built_lib, "shine_query_fwd", C.byref(desc), _abi.ptr(coord), n, _abi.ptr(feat), st)
        _call(built_lib, "shine_query_coord_grad", C.byref(desc), _abi.ptr(coord), n, _abi.ptr(d), _abi.ptr(G), st)
        _call(built_lib, "shine_query_tangent_fwd", C.byref(desc), _abi.ptr(coord), n, _abi.ptr(t), _abi.ptr(tf), st)
        gdesc = octree._descriptor(None, grads)
        _call(built_lib, "shine_query_tangent_bwd", C.byref(gdesc), _abi.ptr(coord), n, _abi.ptr(t), _abi.ptr(d), st)
        torch.cuda.synchronize()
        what = f"F={F} L={levels} poly={poly} n={n}"
        grade_values(feat.cpu().numpy(), ref.feat, ref.efeat, what, "query_fwd")
        grade_values(G.cpu().numpy(), ref.G, ref.eG, what, "query_coord_grad")
        grade_values(tf.cpu().numpy(), ref.tfwd, ref.etfwd, what, "query_tangent_fwd")
        ref.rows.grade([g.cpu().numpy() for g in grads], f"{what} query_tangent_bwd")


@pytest.fixture
def force(monkeypatch):
    """force(target, rmax): gradient replicas at small batches for octrees that build their descriptors afterwards."""
    from shine_mapping_b200 import FeatureOctree

    def set_(target, rmax=64):
        monkeypatch.setattr(FeatureOctree, "_REPLICA_TARGET", target)
        monkeypatch.setattr(FeatureOctree, "_REPLICA_MAX", rmax)
    return set_


def _spy_replicas(octree):
    """Records the largest R of every descriptor handed to the octree's replica fold."""
    seen = []
    fold = octree._reduce_replicas
    L = octree.featured_level_num

    def spy(desc, device):
        seen.append(max(max(1, desc.lv[k].num_replicas) for k in range(L)))
        fold(desc, device)
    octree._reduce_replicas = spy
    return seen


def test_query_bwd_f32_with_replicas(force):
    """shine_query_bwd at F = 32 (LP = 8 lanes a point) with forced gradient replicas, every element against its bound."""
    force(1, 64)
    case = _query_case(32, 4, True, 432)
    cfg, octree, dec = build_cuda_models(case, DEV)
    seen = _spy_replicas(octree)
    n = case["coord"].shape[0]
    dfeat = _spread(np.random.default_rng(32), (n, 32))
    coord = torch.from_numpy(case["coord"]).to(DEV)
    feature = octree.query_feature(coord)
    got = torch.autograd.grad(feature, list(octree.hier_features), torch.from_numpy(dfeat).to(DEV))
    torch.cuda.synchronize()
    assert seen and seen[-1] > 1, f"query_bwd ran without replicas ({seen})"
    o, _ = oracle64(case)
    rows = RowSums([t.shape[0] for t in o.hier_features], 32)
    pts = np.repeat(np.arange(n), 8)
    for i, g in enumerate(level_geometry(o, case["coord"])):
        rows.add(case["cfg"]["tree_level_feat"] - 1 - i, g["ix"].reshape(-1), pts, g["w"].reshape(-1), dfeat)
    rows.grade([t.cpu().numpy() for t in got], f"query_bwd F=32 R={seen[-1]}")


# ---- the class surface -------------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("F,levels,poly,replicas", [(4, 3, True, False), (8, 4, False, False), (16, 3, True, False),
                                                    (32, 2, False, False), (8, 3, True, True)])
def test_class_surface_eikonal_per_element(F, levels, poly, replicas, force):
    """batch_loop.eikonal_iteration (query kernels + torch MLP in fp32, TF32 off): g, the eikonal mean and every
    table-gradient element, at weight_e = 0.1 and at a dominant weight_e; one case with replicas in query_bwd."""
    from shine_mapping_b200 import SdfTrainer
    from shine_mapping_b200.batch_loop import eikonal_iteration
    assert not torch.backends.cuda.matmul.allow_tf32, "the class-surface bound assumes fp32 cuBLAS GEMMs (TF32 off)"
    if replicas:
        force(1, 64)
    case, dropped = clean_case(_case(levels, poly, 500 + F + levels, feature_dim=F))
    cfg, octree, dec = build_cuda_models(case, DEV)
    seen = _spy_replicas(octree)
    cfg.ekional_loss_on = True
    tr = SdfTrainer(cfg, octree, dec)
    coord, label, weight = _dev(case)
    for weight_e in (0.1, dominant_weight(case)):
        cfg.weight_e = weight_e
        tr.zero_grad()
        total, eik, g = eikonal_iteration(cfg, octree, dec, tr, coord, label, weight)
        torch.cuda.synchronize()
        ref = EikRef(case, weight_e, class_surface=True)
        what = f"class surface F={F} L={levels} poly={poly} weight_e={weight_e:.3g} (dropped {dropped})"
        ref.grade({"table_grads": [t.cpu().numpy() for t in tr.table_grads], "g": g.cpu().numpy(),
                   "eikonal": float(eik)}, what)
    if replicas:
        assert seen and max(seen) > 1, f"query_bwd ran without replicas ({seen})"


# ---- small related checks ----------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("n", [0, 1, 1025, 3_000_017])
def test_count_positive_is_exact(n, built_lib):
    """shine_count_positive (the eikonal mean's N_surf) against numpy: +0.0, -0.0, denormals of both signs, NaN-free."""
    from shine_mapping_b200 import _abi
    rng = np.random.default_rng(n)
    v = rng.standard_normal(n).astype(np.float32)
    special = np.array([0.0, -0.0, 1e-45, -1e-45, 1e-40, -1e-40, np.float32(1.17e-38), -np.float32(1.17e-38)],
                       dtype=np.float32)
    if n:
        k = min(n, 4 * special.shape[0])
        v[rng.choice(n, k, replace=False)] = np.resize(special, k)
    dv = torch.from_numpy(v).to(DEV)
    out = torch.zeros(1, dtype=torch.int32, device=DEV)
    _call(built_lib, "shine_count_positive", _abi.ptr(dv) if n else None, n, _abi.ptr(out), _abi.stream_ptr(DEV))
    torch.cuda.synchronize()
    want = int((v > 0).sum())
    assert int(out.item()) == want, f"n={n}: counted {int(out.item())}, numpy {want}"


@pytest.mark.parametrize("F", [12, 64])
def test_query_entries_refuse_other_feature_dims(F, built_lib):
    """check_octree accepts any multiple of 4, the query dispatchers only 4, 8, 16 and 32: the five entries return
    SHINE_ERR_UNSUPPORTED and leave their outputs as they were."""
    from shine_mapping_b200 import _abi
    case = make_case(n_points=1500, n_batch=64, feat_levels=2, seed=7)
    cfg, octree, dec = build_cuda_models(case, DEV)
    n = case["coord"].shape[0]
    grads = [torch.full((p.shape[0], F), 7.0, device=DEV) for p in octree.hier_features]
    tables = [torch.zeros((p.shape[0], F), device=DEV) for p in octree.hier_features]
    desc = octree._descriptor(tables, grads)
    desc.feature_dim = F
    coord = torch.from_numpy(case["coord"]).to(DEV)
    vin = torch.ones((n, F), device=DEV)
    tangent = torch.ones((n, 3), device=DEV)
    outs = {"feat": torch.full((n, F), 5.0, device=DEV), "dcoord": torch.full((n, 3), 5.0, device=DEV),
            "tfwd": torch.full((n, F), 5.0, device=DEV)}
    st, o, p = _abi.stream_ptr(DEV), C.byref(desc), _abi.ptr
    lib = built_lib
    calls = {"shine_query_fwd": lambda: lib.shine_query_fwd(o, p(coord), n, p(outs["feat"]), st),
             "shine_query_bwd": lambda: lib.shine_query_bwd(o, p(coord), n, p(vin), st),
             "shine_query_coord_grad": lambda: lib.shine_query_coord_grad(o, p(coord), n, p(vin), p(outs["dcoord"]), st),
             "shine_query_tangent_fwd": lambda: lib.shine_query_tangent_fwd(o, p(coord), n, p(tangent), p(outs["tfwd"]), st),
             "shine_query_tangent_bwd": lambda: lib.shine_query_tangent_bwd(o, p(coord), n, p(tangent), p(vin), st)}
    for name, call in calls.items():
        assert call() == UNSUPPORTED, f"{name} accepted feature_dim {F}"
    torch.cuda.synchronize()
    assert all(bool((t == 5.0).all()) for t in outs.values()), "an output was written"
    assert all(bool((g == 7.0).all()) for g in grads), "a gradient table was written"
