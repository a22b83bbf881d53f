"""The forward-only kernels graded element by element against fp64 (tests/infer_bound.py):
`shine_sdf_infer` (pred and validity mask), `shine_mesh_grid` (the same kernel body over generated grid points) and
`shine_sdf_fwd` / `shine_sdf_bce_fwd` (pred and loss).

These kernels walk the node tables their own way, the sector walk: each lane of a point reads one 32-byte half of the home
slot and resolves a collision with that half's own copy of maxdisp (`resolve_sector`), while the training kernels use the
level-split walk (`probe_slot_from` on sector 0).  So besides fresh tables and tables x300 (trained magnitudes), the
tables here are
  * dense: one slot per node (`FeatureOctree._HASH_SLOTS_PER_NODE = 1`, load above 0.5): long chains, wrapping chains;
  * adversarial: key sets of tests/hash_layout.py written through `shine_hash_insert` (8 keys of one home, chains that wrap
    past the last slot, interleaved buddy chains, misses that walk a foreign chain), with an oracle that is a dict of
    those keys;
and every table's slots are checked against the invariants of tests/hash_layout.py after each way a table gets built.
The points include voxel corners and face centres of every featured level (exact dyadic coordinates), the clamp edges
+-1 and nextafter(+-1, 0), points outside [-1, 1], tiles of 16 misses (the zero-tile branch), mixed tiles and a single
miss, batch sizes around the 16-point tile and past the persistent grid, world levels 6, 12 and 15, and a descriptor whose
levels are not consecutive (the kernels then quantise every level instead of shifting the leaf key).
Pred is graded at every point against P (kink points with the kink bound), masks must match at every mask level, and
the training step's pred must equal inference's bit for bit on every dense and adversarial table.  Each test prints its
worst error / bound and the number of points it graded."""
import ctypes as C
import pickle

import numpy as np
import pytest
import torch

from oracle import shine_oracle as orc
from tests import hash_layout as hl
from tests.infer_bound import LossRef, PredRef
from tests.parity_utils import build_cuda_models, make_case, make_config
from tests.test_gpu_replicas import with_weights
from tests.test_gpu_sdf_diff import _scale

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
F32 = np.float32


@pytest.fixture(scope="module", autouse=True)
def _lib(built_lib):
    assert torch.cuda.is_available()
    return built_lib


# ---- calling the kernels ---------------------------------------------------------------------------------------------------

def _t(a, dtype=torch.float32):
    return torch.from_numpy(np.ascontiguousarray(a)).to(DEV, dtype)


def infer(od, dd, coord, mask_level=None, tf32x1=False):
    """shine_sdf_infer -> (pred, mask or None) as numpy"""
    from shine_mapping_b200 import _abi
    n = coord.shape[0]
    c = _t(coord)
    pred = torch.full((n,), float("nan"), device=DEV)
    mask = torch.full((n,), 7, dtype=torch.uint8, device=DEV) if mask_level is not None else None
    _abi.check(_abi.lib().shine_sdf_infer(C.byref(od), C.byref(dd), _abi.ptr(c), n, _abi.ptr(pred), _abi.ptr(mask),
                                          int(mask_level or 0), _abi.FLAG_TF32X1 if tf32x1 else 0, _abi.stream_ptr(DEV)),
               "shine_sdf_infer")
    torch.cuda.synchronize()
    if mask is not None:
        m = mask.cpu().numpy()
        assert set(np.unique(m).tolist()) <= {0, 1}, "the mask holds a value other than 0 / 1"
        return pred.cpu().numpy(), m
    return pred.cpu().numpy(), None


def step_pred(od_grads, dd, coord, tf32x1=False):
    """pred of shine_sdf_step (the level-split walk) on a descriptor that carries gradient tables"""
    from shine_mapping_b200 import _abi
    n = coord.shape[0]
    c, label = _t(coord), torch.zeros(n, device=DEV)
    pred, loss = torch.full((n,), float("nan"), device=DEV), torch.zeros((), device=DEV)
    _abi.check(_abi.lib().shine_sdf_step(C.byref(od_grads), C.byref(dd), _abi.ptr(c), _abi.ptr(label), None, n, 1.0, 1.0,
                                         1.0, None, _abi.ptr(pred), _abi.ptr(loss), _abi.FLAG_TF32X1 if tf32x1 else 0,
                                         _abi.stream_ptr(DEV)), "shine_sdf_step")
    torch.cuda.synchronize()
    return pred.cpu().numpy()


def fwd(od, dd, case, loss_type, bce_entry=False):
    """shine_sdf_fwd (or shine_sdf_bce_fwd) with the case's loss config -> (pred, loss)"""
    from shine_mapping_b200 import _abi
    c = case["cfg"]
    n = case["coord"].shape[0]
    coord, label, weight = _t(case["coord"]), _t(case["label"]), _t(case["weight"])
    pred, loss = torch.full((n,), float("nan"), device=DEV), torch.zeros((), device=DEV)
    lib, st = _abi.lib(), _abi.stream_ptr(DEV)
    if loss_type == "sdf_bce":
        flags = (_abi.FLAG_REDUCTION_SUM if c["reduction"] == "sum" else 0) | (_abi.FLAG_WEIGHTED if c["weighted"] else 0)
        ls = 1.0 if c["reduction"] == "sum" else 1.0 / n
        if bce_entry:
            rc = lib.shine_sdf_bce_fwd(C.byref(od), C.byref(dd), _abi.ptr(coord), _abi.ptr(label), _abi.ptr(weight), n,
                                       c["sigma"], ls, _abi.ptr(pred), _abi.ptr(loss), flags, st)
        else:
            rc = lib.shine_sdf_fwd(C.byref(od), C.byref(dd), _abi.ptr(coord), _abi.ptr(label), _abi.ptr(weight), n,
                                   c["sigma"], 1.0, ls, _abi.ptr(pred), _abi.ptr(loss), flags, st)
    else:
        flags = _abi.FLAG_LOSS_L1 if loss_type == "sdf_l1" else _abi.FLAG_LOSS_L2
        rc = lib.shine_sdf_fwd(C.byref(od), C.byref(dd), _abi.ptr(coord), _abi.ptr(label), _abi.ptr(weight), n, 1.0,
                               _scale(case), 1.0 / n, _abi.ptr(pred), _abi.ptr(loss), flags, st)
    _abi.check(rc, "shine_sdf_fwd")
    torch.cuda.synchronize()
    return pred.cpu().numpy(), float(loss)


def clone(od):
    from shine_mapping_b200 import _abi
    out = _abi.ShineOctree()
    C.memmove(C.byref(out), C.byref(od), C.sizeof(od))
    return out


def with_grads(od, keep):
    """a copy of descriptor od whose levels carry zeroed gradient tables (kept alive in `keep`)"""
    out = clone(od)
    for i in range(od.num_levels):
        g = torch.zeros(od.lv[i].rows, 8, device=DEV)
        keep.append(g)
        out.lv[i].feature_grads = g.data_ptr()
    return out


# ---- maps and their oracles -------------------------------------------------------------------------------------------------

def scaled(case, table_scale):
    out = dict(case)
    out["tables"] = [(t * F32(table_scale)).astype(F32) for t in case["tables"]]
    return out


def with_oracle(case):
    """the case with its OracleOctree grown once (PredRef reuses its lookup tables instead of replaying the frames)"""
    c = case["cfg"]
    o = orc.OracleOctree(c["tree_level_world"], c["tree_level_feat"], c["feature_dim"], 0.05, c["poly_int_on"])
    for fr in case["frames"]:
        o.update(torch.from_numpy(np.asarray(fr)))
    return dict(case, oracle=o)


def load_tables(octree, case):
    with torch.no_grad():
        for p, t in zip(octree.hier_features, case["tables"]):
            p.copy_(torch.from_numpy(np.asarray(t)))


def check_octree_slots(octree, what):
    """check_slots on every featured level of a FeatureOctree's device node tables -> the largest probe index"""
    octree._ensure_hash()
    worst = 0
    for lvl in range(octree.free_level_num, octree.max_level + 1):
        st = octree._levels[lvl]
        info = hl.check_slots(hl.Slots.decode(st.hash.cpu().numpy()), st.node_keys.cpu().numpy(),
                              st.node_ids.cpu().numpy(), f"{what} level {lvl}")
        worst = max(worst, info["max_probe"])
    return worst


def node_voxels(o, level, rng, m):
    """integer coordinates of up to m nodes of the oracle's table at world `level`"""
    keys = np.array(list(o.nodes_lookup_tables[level]), dtype=np.int64)
    if keys.size == 0:
        return np.zeros((0, 3), dtype=np.int64)
    pick = rng.choice(keys.size, min(m, keys.size), replace=False)
    return orc.morton_to_points(keys[pick]).astype(np.int64)


_CORNERS = np.array([[(i >> 2) & 1, (i >> 1) & 1, i & 1] for i in range(8)], dtype=np.float64)
_FACES = np.array([[0, .5, .5], [1, .5, .5], [.5, 0, .5], [.5, 1, .5], [.5, .5, 0], [.5, .5, 1]])
EDGES = np.array([1.0, -1.0, np.nextafter(F32(1), F32(0)), np.nextafter(F32(-1), F32(0)), 1.25, -1.5, 1.3, -1.3,
                  1.0 + 2.0 ** -20], dtype=F32)


def special_points(o, rng, per_level=12):
    """voxel corners and face centres of nodes of every featured level (exact in fp32: -1 + k 2^(1 - level)), node centres
    with one or all coordinates on a clamp edge (+-1, nextafter(+-1, 0)) or outside [-1, 1]"""
    pts = []
    for level in range(o.free_level_num, o.max_level + 1):
        v = node_voxels(o, level, rng, per_level)
        for off in (_CORNERS, _FACES):
            pts.append((-1.0 + 2.0 * (v[:, None, :] + off[None]) / 2.0 ** level).reshape(-1, 3))
    centres = np.concatenate([-1.0 + 2.0 * (node_voxels(o, l, rng, 4) + 0.5) / 2.0 ** l
                              for l in range(o.free_level_num, o.max_level + 1)])
    for e in EDGES:
        for a in range(3):
            p = centres.copy()
            p[:, a] = e
            pts.append(p)
        pts.append(np.full((1, 3), e))
    out = np.concatenate(pts).astype(F32)
    assert np.array_equal(out[: len(pts[0])].astype(np.float64), pts[0])        # the dyadic points are exact in fp32
    return out


def hits_any(o, coord):
    idx = o.get_indices(torch.from_numpy(np.ascontiguousarray(coord, dtype=F32)))
    return np.any([(ix >= 0).any(1).numpy() for ix in idx], axis=0)


def tile_order(o, coord, rng):
    """coord rearranged into tiles of 16: all hits, all misses (the zero-tile branch), 8 / 8 interleaved, 15 hits and one
    miss, then the rest, with one more tile of misses; misses added from the cube where the map has none when the batch
    has too few.  -> (points, order): order[j] is the index in coord of point j, -1 for an added miss."""
    coord = np.asarray(coord, dtype=F32)
    cand = rng.uniform(-1, 1, size=(4096, 3)).astype(F32)
    cand = cand[~hits_any(o, cand)][:64]
    pts = np.concatenate((coord, cand))
    src = np.concatenate((np.arange(coord.shape[0]), np.full(cand.shape[0], -1)))
    hit = hits_any(o, pts)
    H, M = np.flatnonzero(hit), np.flatnonzero(~hit)
    assert H.size >= 40 and M.size >= 41, (H.size, M.size)
    mixed = np.empty(16, dtype=np.int64)
    mixed[0::2], mixed[1::2] = H[16:24], M[16:24]
    one = np.concatenate((H[24:31], M[24:25], H[31:39]))
    idx = np.concatenate((H[:16], M[:16], mixed, one, H[39:], M[25:41], M[41:]))
    return pts[idx], src[idx]


def tiled(o, coord, rng):
    return tile_order(o, coord, rng)[0]


def tiled_case(case, rng):
    """the case's batch rearranged by tile_order; an added miss gets label 0 and weight 1"""
    pts, src = tile_order(case["oracle"], case["coord"], rng)
    out = dict(case, coord=pts)
    for k, fill in (("label", 0.0), ("weight", 1.0)):
        out[k] = np.where(src >= 0, case[k][np.maximum(src, 0)], F32(fill)).astype(F32)
    return out


def infer_and_grade(od, dd, case, coord, what, tf32x1=False, levels=None, ref=None):
    """infer at every mask level: pred graded (the same bits at every mask level), masks exact -> (PredRef, pred)"""
    L = od.num_levels
    ref = ref or PredRef(case, coord, tf32x1=tf32x1)
    first, masks = None, []
    for k in range(L):
        pred, mask = infer(od, dd, coord, k, tf32x1)
        masks.append(mask)
        if first is None:
            first = pred
        assert np.array_equal(pred.view(np.uint32), first.view(np.uint32)), f"{what}: pred depends on mask level {k}"
    p_nomask, _ = infer(od, dd, coord, None, tf32x1)
    assert np.array_equal(p_nomask.view(np.uint32), first.view(np.uint32)), f"{what}: pred depends on the mask output"
    ref.grade(first, what)
    ref.grade_masks(masks, what)
    return ref, first


def same_bits(a, b, what):
    bad = np.flatnonzero(a.view(np.uint32) != b.view(np.uint32))
    assert bad.size == 0, f"{what}: {bad.size} points differ, first {bad[0]}: {a[bad[0]]!r} vs {b[bad[0]]!r}"
    print(f"[infer bounds] {what}: {a.shape[0]} points bit for bit")


# ---- shine_sdf_infer on natural maps ---------------------------------------------------------------------------------------

# (feature levels, world level): both LMAX builds (<= 4 and 5 .. 8 levels), world levels 6, 12 and 15
LEVELS = [(1, 6), (3, 12), (4, 15), (5, 6), (8, 15)]
VARIANTS = [(True, True, False), (False, False, True), (True, False, True), (False, True, False)]


@pytest.mark.parametrize("poly,bias,tf32x1", VARIANTS, ids=lambda v: str(v))
@pytest.mark.parametrize("levels,world", LEVELS)
def test_infer_graded_on_natural_maps(levels, world, poly, bias, tf32x1):
    seed = 600 + 10 * levels + 2 * poly + bias
    case = with_oracle(make_case(n_points=1500, n_batch=1200, feat_levels=levels, world_level=world, seed=seed, poly=poly,
                                 bias=bias))
    rng = np.random.default_rng(seed)
    o = case["oracle"]
    coord = tiled(o, np.concatenate((case["coord"], special_points(o, rng))), rng)
    cfg, octree, dec = build_cuda_models(case, DEV)
    dd = dec.c_descriptor(None)
    for ts in (1, 300):
        cs = scaled(case, ts)
        load_tables(octree, cs)
        od = octree._descriptor(None, None)
        infer_and_grade(od, dd, cs, coord, f"L{levels} W{world} poly {poly} bias {bias} tf32x1 {tf32x1} x{ts}",
                        tf32x1=tf32x1)


@pytest.mark.parametrize("n", [1, 15, 16, 17, 4097, 16 * 8 * 8 * 132 + 17])
def test_infer_batch_sizes(n):
    """Partial tiles, and n past the largest persistent grid (8 blocks / SM of 8 warps on 132 SMs, one tile per warp): the
    grid-stride loop turns."""
    case = with_oracle(make_case(n_points=1500, n_batch=max(n, 64), feat_levels=3, seed=70 + n % 97))
    rng = np.random.default_rng(n)
    sub = tiled_case(case, rng) if n >= 64 else case
    sub = dict(sub, **{k: np.ascontiguousarray(sub[k][:n]) for k in ("coord", "label", "weight")})
    coord = sub["coord"]
    cfg, octree, dec = build_cuda_models(case, DEV)
    od, dd = octree._descriptor(None, None), dec.c_descriptor(None)
    ref, pred = infer_and_grade(od, dd, case, coord, f"n = {n}")
    if n > 16:
        p2, loss = fwd(od, dd, sub, "sdf_bce")
        same_bits(p2, pred, f"n = {n}: shine_sdf_fwd pred vs shine_sdf_infer")
        c = case["cfg"]
        LossRef(ref.pred, ref.P, sub["label"], sub["weight"], "sdf_bce", sigma=c["sigma"]).grade(loss, f"n = {n}")


# ---- shine_sdf_fwd / shine_sdf_bce_fwd -------------------------------------------------------------------------------------

LOSSES = [("sdf_bce", False, "mean"), ("sdf_bce", False, "sum"), ("sdf_bce", True, "mean"), ("sdf_bce", True, "sum"),
          ("sdf_l1", True, "mean"), ("sdf_l2", True, "mean")]


@pytest.mark.parametrize("levels", [3, 5])
@pytest.mark.parametrize("loss_type,weighted,reduction", LOSSES)
def test_fwd_pred_and_loss_graded(loss_type, weighted, reduction, levels):
    seed = 800 + levels
    case = make_case(n_points=1500, n_batch=2000, feat_levels=levels, seed=seed, weighted=weighted, reduction=reduction)
    case = tiled_case(with_oracle(with_weights(case, loss_type, seed)), np.random.default_rng(seed))
    cfg, octree, dec = build_cuda_models(case, DEV)
    dd = dec.c_descriptor(None)
    c = case["cfg"]
    for ts in (1, 300):
        cs = scaled(case, ts)
        load_tables(octree, cs)
        od = octree._descriptor(None, None)
        what = f"L{levels} {loss_type} {'weighted ' if weighted else ''}{reduction} x{ts}"
        pred, loss = fwd(od, dd, cs, loss_type)
        ref = PredRef(cs)
        ref.grade(pred, what)
        lr = LossRef(ref.pred, ref.P, cs["label"], cs["weight"], loss_type, sigma=c["sigma"], scale=_scale(cs),
                     weighted=c["weighted"], reduction=c["reduction"])
        lr.grade(loss, what)
        p_inf, _ = infer(od, dd, cs["coord"])
        same_bits(pred, p_inf, f"{what}: shine_sdf_fwd pred vs shine_sdf_infer")
        if loss_type == "sdf_bce":
            p2, loss2 = fwd(od, dd, cs, loss_type, bce_entry=True)
            same_bits(p2, pred, f"{what}: shine_sdf_bce_fwd pred vs shine_sdf_fwd")
            assert abs(loss2 - loss) <= 2 * lr.summation, (loss2, loss, lr.summation)
            lr.grade(loss2, what + " (shine_sdf_bce_fwd)")


# ---- shine_mesh_grid -------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("levels", [1, 3, 4, 5, 8])
def test_mesh_grid_graded(levels):
    """-Decoder.sdf on the brick sets of test_gpu_mesh_oracle's grid query, every grid point that belongs to a brick of the
    map, against P."""
    from shine_mapping_b200 import _abi
    from shine_mapping_b200.feature_octree import morton_to_points
    from shine_mapping_b200.mesher import _brick_keys
    from tests import mesh_oracle as mo
    from tests.test_gpu_mesh_oracle import GRID_SIZES, _brick_grid, _local
    poly, bias = levels % 2 == 1, levels != 4
    case = with_oracle(make_case(n_points=1500, n_batch=16, feat_levels=levels, seed=900 + levels, poly=poly, bias=bias))
    cfg, octree, dec = build_cuda_models(case, DEV)
    q = cfg.tree_level_world - cfg.tree_level_feat + 1
    nodes = morton_to_points(octree._levels[q].node_keys.to(DEV)).to(torch.int32)
    all_keys = torch.sort(_brick_keys(nodes)).values
    keyset = set(map(tuple, nodes.cpu().numpy().tolist()))
    node_res = 2.0 ** (1 - q)
    dd = dec.c_descriptor(None)
    lib, st = _abi.lib(), _abi.stream_ptr(DEV)
    rng = np.random.default_rng(levels)
    P = nodes.cpu().numpy().astype(np.int64)
    for ts in (1, 300):
        cs = scaled(case, ts)
        load_tables(octree, cs)
        od = octree._descriptor(None, None)
        for n, nb in GRID_SIZES:
            centre = P[rng.integers(P.shape[0])]
            pick = np.argsort(np.abs(P - centre).max(1), kind="stable")[:min(nb, P.shape[0])]
            bricks = torch.from_numpy(P[pick].astype(np.int32)).to(DEV).contiguous()
            h = node_res / n
            per = (n + 1) ** 3
            sdf = torch.full((bricks.shape[0] * per,), np.nan, dtype=torch.float32, device=DEV)
            mask = torch.full((bricks.shape[0] * per,), 7, dtype=torch.uint8, device=DEV)
            g = _brick_grid(bricks, sdf, mask, n, -1.0 + 0.5 * h, h, all_keys, missing=1234.5)
            G = (P[pick][:, None, :] * n + _local(n)[None]).reshape(-1, 3)
            inmap = np.array([tuple(x) in keyset for x in (G // n).tolist()])
            _abi.check(lib.shine_mesh_grid(C.byref(od), C.byref(dd), C.byref(g), 0, 0, st), "shine_mesh_grid")
            got = sdf.cpu().numpy()
            coord = mo.grid_coords(G, F32(-1.0 + 0.5 * h), h)[inmap]
            PredRef(cs, coord).grade(got[inmap], f"mesh grid L{levels} n {n} x{ts}", sign=-1.0)


# ---- dense and adversarial tables ------------------------------------------------------------------------------------------

@pytest.mark.parametrize("levels", [2, 4, 7])
def test_dense_tables(levels, monkeypatch):
    """One slot per node: every level's table at load > 0.5 with chains of several probes; pred / masks graded on fresh
    and x300 tables, the training step's pred equal to inference's bit for bit."""
    from shine_mapping_b200 import FeatureOctree
    monkeypatch.setattr(FeatureOctree, "_HASH_SLOTS_PER_NODE", 1)
    case = with_oracle(make_case(n_points=4000, n_batch=3000, feat_levels=levels, seed=31 + levels, n_frames=2))
    rng = np.random.default_rng(levels)
    o = case["oracle"]
    coord = tiled(o, np.concatenate((case["coord"], special_points(o, rng))), rng)
    cfg, octree, dec = build_cuda_models(case, DEV)
    probe = check_octree_slots(octree, "dense")
    loads = [octree._levels[l].node_keys.numel() / octree._levels[l].hash_capacity
             for l in range(octree.free_level_num, octree.max_level + 1)]
    assert max(loads) > 0.5 and probe >= 2, (loads, probe)
    print(f"[infer bounds] dense L{levels}: loads {[round(x, 2) for x in loads]}, longest probe {probe}")
    dd = dec.c_descriptor(None)
    keep = []
    for ts in (1, 300):
        cs = scaled(case, ts)
        load_tables(octree, cs)
        od = octree._descriptor(None, None)
        _, pred = infer_and_grade(od, dd, cs, coord, f"dense L{levels} x{ts}")
        same_bits(step_pred(with_grads(od, keep), dd, coord), pred, f"dense L{levels} x{ts}: step pred vs infer pred")


def _adversarial_map(levels, world, poly, seed, caps):
    """Per level (bottom-up, world level world - i) an adversarial key set of tests/hash_layout.py in a table of caps[i]
    slots written by shine_hash_insert, random corner rows; the finest level's named keys (clusters, wrapping and buddy
    chains) have their ancestors stored at every coarser level.  -> (case, descriptor, slot tensors, key sets)"""
    from shine_mapping_b200 import _abi
    rng = np.random.default_rng(seed)
    o = orc.OracleOctree(world, levels, 8, 0.05, poly)
    tables, slots, sets = [None] * levels, [], []
    od = _abi.ShineOctree()
    od.num_levels, od.feature_dim, od.poly_interp = levels, 8, int(poly)
    leaf_named = None
    for i in range(levels):
        lvl, cap = world - i, caps[i]
        include = np.unique(leaf_named >> (3 * i)) if leaf_named is not None else np.zeros(0, dtype=np.int64)
        ks = hl.adversarial_keys(rng, cap, lvl, 0.85, include=include)
        if i == 0:
            leaf_named = np.concatenate((ks["cluster"], ks["wrap"], ks["buddy"]))
        keys = ks["stored"]
        rows = 2 * keys.size + 1
        ids = rng.integers(0, rows - 1, size=(keys.size, 8)).astype(np.int32)    # never the trash row
        raw = torch.full((cap * hl.SLOT_BYTES,), 0xFF, dtype=torch.uint8, device=DEV)
        overflow = torch.zeros(1, dtype=torch.int32, device=DEV)
        kt, it = _t(keys, torch.int64), _t(ids, torch.int32)
        _abi.check(_abi.lib().shine_hash_insert(_abi.ptr(raw), cap, _abi.ptr(kt), _abi.ptr(it), keys.size, 0,
                                                _abi.ptr(overflow), _abi.stream_ptr(DEV)), "shine_hash_insert")
        assert int(overflow.item()) == 0
        info = hl.check_slots(hl.Slots.decode(raw.cpu().numpy()), keys, ids, f"adversarial level {lvl}")
        assert info["max_probe"] >= 7, info
        o.nodes_lookup_tables[lvl] = {int(k): ids[j].tolist() for j, k in enumerate(keys)}
        t = (0.05 * rng.standard_normal((rows, 8))).astype(F32)
        t[-1] = 0
        tables[levels - 1 - i] = t
        slots.append((raw, kt, it))
        sets.append(ks)
        lv = od.lv[i]
        lv.hash_slots, lv.hash_capacity, lv.rows, lv.level = raw.data_ptr(), cap, rows, lvl
    dec = orc.make_decoder_params(8, 32, 2, True)
    cfg = dict(tree_level_world=world, tree_level_feat=levels, feature_dim=8, poly_int_on=poly, leaf_vox_size=0.2,
               sigma=1.0, weighted=False, reduction="mean", bias=True)
    o.hier_features = [torch.from_numpy(t) for t in tables]
    case = {"cfg": cfg, "oracle": o, "tables": tables, "dec": {k: v.detach().numpy() for k, v in dec.items()}}
    return case, od, slots, sets


def _voxel_points(keys, level, rng, per=3):
    """random interior points and the lower corner of each voxel"""
    v = orc.morton_to_points(np.asarray(keys, dtype=np.int64)).astype(np.float64)
    inner = (v[:, None, :] + rng.uniform(0.02, 0.98, size=(v.shape[0], per, 3))).reshape(-1, 3)
    return (-1.0 + 2.0 * np.concatenate((inner, v)) / 2.0 ** level).astype(F32)


@pytest.mark.parametrize("levels,poly", [(3, True), (5, False)])
def test_adversarial_tables(levels, poly):
    from shine_mapping_b200 import Decoder
    world = 12
    caps = [1024, 512, 256, 128, 64][:levels]
    case, od, slots, sets = _adversarial_map(levels, world, poly, 40 + levels, caps)
    rng = np.random.default_rng(levels)
    pts = []
    for i, ks in enumerate(sets):
        for name in ("stored", "absent_chain", "absent"):
            keys = ks[name] if name != "stored" else ks[name][:200]
            pts.append(_voxel_points(keys, world - i, rng))
    coord = tiled(case["oracle"], rng.permutation(np.concatenate(pts)), rng)
    cfgo = make_config(levels, world, device=DEV, poly_int_on=poly)
    dec = Decoder(cfgo)
    sd = dec.state_dict()
    for k, v in case["dec"].items():
        sd[k] = torch.from_numpy(v).to(DEV)
    dec.load_state_dict(sd)
    assert all(k in case["dec"] for k in sd if k.startswith(("layers.", "lout.")))
    dd = dec.c_descriptor(None)
    keep = []
    for ts in (1, 300):
        cs = scaled(case, ts)
        feats = [_t(t) for t in cs["tables"]]
        keep += feats
        for i in range(levels):
            od.lv[i].features = feats[levels - 1 - i].data_ptr()
        _, pred = infer_and_grade(od, dd, cs, coord, f"adversarial L{levels} x{ts}")
        same_bits(step_pred(with_grads(od, keep), dd, coord), pred, f"adversarial L{levels} x{ts}: step pred vs infer pred")


# ---- levels that are not consecutive ---------------------------------------------------------------------------------------

class KeptLevels(orc.OracleOctree):
    """The oracle of a subset of another oracle's featured levels (world levels `kept`, finest first): position i of
    the bottom-up lists is world level kept[i], looked up and blended at that level."""

    def __init__(self, o, kept, tables):
        super().__init__(o.max_level, len(kept), o.feature_dim, o.feature_std, o.polynomial_interpolation)
        self.kept = list(kept)
        for lvl in kept:
            self.nodes_lookup_tables[lvl] = o.nodes_lookup_tables[lvl]
        self.hier_features = [torch.from_numpy(np.asarray(t)) for t in tables]

    def get_indices(self, coord):
        c = coord.detach().cpu().numpy()
        self.hierarchical_indices = []
        for lvl in self.kept:
            morton = orc.points_to_morton(orc.quantize_points(c, lvl)).tolist()
            table = self.nodes_lookup_tables[lvl]
            rows = [table.get(m, [-1] * 8) for m in morton]
            self.hierarchical_indices.append(torch.tensor(rows, dtype=torch.int64).reshape(-1, 8))
        return self.hierarchical_indices

    def interpolat(self, x, level, polynomial_on=True):
        return super().interpolat(x, self.kept[self.max_level - level], polynomial_on)


@pytest.mark.parametrize("levels,drop", [(4, 1), (4, 2), (6, 3)])
def test_non_consecutive_levels(levels, drop):
    """The octree's descriptor with level index `drop` removed and the rest shifted down: levels W, .., W - drop + 1,
    W - drop - 1, ..  The kernels quantise each level (`morton_of`) instead of shifting the leaf key; pred and masks are
    graded against the oracle summed over the kept levels, and the step's pred equals inference's bit for bit."""
    case = with_oracle(make_case(n_points=2000, n_batch=1500, feat_levels=levels, seed=50 + levels + drop))
    rng = np.random.default_rng(drop)
    o = case["oracle"]
    coord = tiled(o, np.concatenate((case["coord"], special_points(o, rng))), rng)
    cfg, octree, dec = build_cuda_models(case, DEV)
    dd = dec.c_descriptor(None)
    keep_lv = [i for i in range(levels) if i != drop]                        # bottom-up indices
    W = cfg.tree_level_world
    tables = case["tables"]                                                  # coarse -> fine
    keep_tables = [tables[levels - 1 - i] for i in reversed(keep_lv)]
    o2 = KeptLevels(o, [W - i for i in keep_lv], keep_tables)
    case2 = dict(case, oracle=o2, cfg=dict(case["cfg"], tree_level_feat=levels - 1), tables=keep_tables)
    keep = []
    for ts in (1, 300):
        load_tables(octree, scaled(case, ts))
        full = octree._descriptor(None, None)
        od = clone(full)
        od.num_levels = levels - 1
        for j, i in enumerate(keep_lv):
            C.memmove(C.byref(od.lv[j]), C.byref(full.lv[i]), C.sizeof(full.lv[i]))
        cs = scaled(case2, ts)
        _, pred = infer_and_grade(od, dd, cs, coord, f"levels {[od.lv[j].level for j in range(levels - 1)]} x{ts}")
        same_bits(step_pred(with_grads(od, keep), dd, coord), pred, f"non-consecutive L{levels} drop {drop} x{ts}: step")


# ---- the table invariants after every build path ---------------------------------------------------------------------------

@pytest.mark.parametrize("how", ["frames", "from_lookup_tables", "pickle", "to_device"])
def test_table_invariants_after_each_build(how, monkeypatch):
    """check_slots on every level after: frame-by-frame update() with a table growth in between (at one slot per node, so
    the growth rehash runs on dense tables), FeatureOctree.from_lookup_tables (the reference checkpoint), a pickle round
    trip and a move through host memory; then pred / masks graded on the rebuilt tables."""
    import json
    import os
    from shine_mapping_b200 import Decoder, FeatureOctree, checkpoint
    from shine_mapping_b200.config import SHINEConfig
    from tests.test_gpu_octree_build import _table_growth_frames
    rng = np.random.default_rng(1)
    if how == "from_lookup_tables":
        gold = os.path.join(os.path.dirname(__file__), "golden")
        g = np.load(os.path.join(gold, "ref_checkpoint_l3.npz"))
        cfg = SHINEConfig(device=DEV, **json.loads(str(g["cfg_json"])))
        state, octree = checkpoint.load_checkpoint(os.path.join(gold, "ref_checkpoint_l3.pt"), cfg, DEV)
        dec = Decoder(cfg)
        dec.load_state_dict(state)
        coord = np.asarray(g["coord"], dtype=F32)
        probe = check_octree_slots(octree, how)
    else:
        monkeypatch.setattr(FeatureOctree, "_HASH_SLOTS_PER_NODE", 1)
        cfg = make_config(3, world_level=12, device=DEV)
        torch.manual_seed(3)
        octree, dec = FeatureOctree(cfg), Decoder(cfg)
        frames = _table_growth_frames(12)
        caps, probe = [], 0
        for f, pts in enumerate(frames):
            if f == 2 and how == "pickle":
                octree = pickle.loads(pickle.dumps(octree))
            if f == 2 and how == "to_device":
                octree = octree.to("cpu").to(DEV)
            octree.update(torch.from_numpy(pts).to(DEV))
            probe = max(probe, check_octree_slots(octree, f"{how} frame {f}"))
            caps.append([octree._levels[l].hash_capacity for l in range(octree.free_level_num, 13)])
        assert all(b > a for a, b in zip(caps[0], caps[-1])), caps                  # the tables grew
        coord = np.concatenate([fr[:1500] for fr in frames]).astype(F32)
    # the map as an oracle case: the octree's dict views and tables
    o = orc.OracleOctree(octree.max_level, octree.featured_level_num, octree.feature_dim, 0.05,
                         octree.polynomial_interpolation)
    o.nodes_lookup_tables = octree.nodes_lookup_tables
    o.hier_features = [p.detach().cpu() for p in octree.hier_features]
    case = {"cfg": dict(tree_level_world=octree.max_level, tree_level_feat=octree.featured_level_num, feature_dim=8,
                        poly_int_on=octree.polynomial_interpolation),
            "oracle": o, "tables": [p.detach().cpu().numpy() for p in octree.hier_features],
            "dec": {k: v.detach().cpu().numpy() for k, v in dec.state_dict().items() if k.startswith(("layers.", "lout."))}}
    coord = tiled(o, np.concatenate((coord, special_points(o, rng))), rng)
    print(f"[infer bounds] {how}: longest probe {probe}")
    infer_and_grade(octree._descriptor(None, None), dec.c_descriptor(None), case, coord, f"after {how}")
