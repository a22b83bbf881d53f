"""Incremental mapping with the continual-learning regulariser (`continual_learning_reg: True`) against fp64, element by element,
with the bounds of tests/incre_bound.py.

  * The three kernels of csrc/shine_incre.cu through the C ABI at F = 4, 8, 16, 32, L = 1, 3, 8 and batches of 0, 1, 7, 33
    and ~3000 points (out-of-map points, cube faces and exact voxel corners among them), a batch that misses every level,
    one point repeated 10^5 times, and a batch large enough that the touched-row kernels take a second grid-stride pass.
    The touched set (count, row list, bitmap) is exact; values and gradients are graded against their bounds; the modes
    (clear_marks, zero_grads, out_reg NULL, Omega = 0, f = f_last) are exact.
  * The ABI's argument checks leave every buffer untouched.
  * `run_shine_mapping_incremental`, one step at a time: every table-gradient element against BCE(sum, weighted) (or BCE +
    eikonal) + 2 lambda Omega (f - f_last) on the touched rows, the regulariser value, the decoder gradients while the
    decoder trains, each frame's importance sweep, and the Omega carried into the next frame.
"""
import ctypes as C

import numpy as np
import pytest
import torch

from oracle import shine_oracle as orc
from tests.eikonal_bound import EikRef, autograd_decoder_grads
from tests.error_bound import U, oracle64
from tests.incre_bound import (RegRef, decoder_kink_slack, grade_rows, importance_want, launch_geometry, rows_of_points,
                               touched_sets)
from tests.parity_utils import DEC_KEYS, build_cuda_models, make_case, make_config, oracle_from_case
from tests.test_gpu_replicas import FoldSpy, Ref, assert_scratch_zero, expected_replicas, force  # noqa: F401 (fixture)

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
OK, INVALID, UNSUPPORTED = 0, -1, -2
# Rows left out of a grade because a point near a ReLU kink touches them: about 0.3 % of the points fall within twice the
# forward error of a kink (more once the decoder has trained), and each one takes its 8 L corner rows out: 2-3.5 % of the
# touched rows of a sweep over a few thousand points.
KINK_SHARE = 0.05


def _sm():
    return torch.cuda.get_device_properties(DEV).multi_processor_count


def _np(ts):
    return [t.detach().cpu().numpy().copy() for t in ts]


# ---- driving the kernels through the C ABI ---------------------------------------------------------------------------------

class Kernels:
    """The three entries on one octree with test-owned gradient, f_last and Omega tables (coarse -> fine)."""

    def __init__(self, octree, grads, last, imp):
        from shine_mapping_b200 import _abi
        from shine_mapping_b200.incre_loop import TouchedRows
        self.abi, self.lib, self.st = _abi, _abi.lib(), _abi.stream_ptr(torch.device(DEV))
        self.octree, self.L = octree, octree.featured_level_num
        self.grads = [torch.from_numpy(g).to(DEV).contiguous() for g in grads]
        self.last = [torch.from_numpy(t).to(DEV).contiguous() for t in last]
        self.imp = [torch.from_numpy(t).to(DEV).contiguous() for t in imp]
        self.t = TouchedRows(octree)
        self.od = octree._descriptor(None, self.grads)
        self.aux = _abi.ShineRowTables()
        for i in range(self.L):
            k = self.L - 1 - i
            self.aux.last[i], self.aux.importance[i] = self.last[k].data_ptr(), self.imp[k].data_ptr()
            self.aux.importance_rw[i] = self.imp[k].data_ptr()
        self.out = torch.zeros(1, device=DEV)

    def mark(self, coord, od=None, touched=None, n=None):
        n = coord.shape[0] if n is None and coord is not None else n
        return self.lib.shine_mark_touched(C.byref(od or self.od), self.abi.ptr(coord), n,
                                           C.byref(touched or self.t.desc) if touched is not False else None, self.st)

    def reg(self, lam, clear, out=True, od=None, touched=None, aux=None):
        return self.lib.shine_regularization_apply(
            C.byref(od or self.od), C.byref(touched or self.t.desc) if touched is not False else None,
            C.byref(aux or self.aux) if aux is not False else None, 2.0 * lam, self.abi.ptr(self.out) if out else None,
            clear, self.st)

    def importance(self, zero_grads, clear, od=None, touched=None, aux=None):
        return self.lib.shine_importance_accumulate(
            C.byref(od or self.od), C.byref(touched or self.t.desc) if touched is not False else None,
            C.byref(aux or self.aux) if aux is not False else None, zero_grads, clear, self.st)

    def set(self, grads=None, imp=None, out=None):
        for dst, src in ((self.grads, grads), (self.imp, imp)):
            if src is not None:
                for d, s in zip(dst, src):
                    d.copy_(torch.from_numpy(np.asarray(s)))
        if out is not None:
            self.out.fill_(out)

    def state(self):
        torch.cuda.synchronize()
        return {"counts": self.t.counts.cpu().numpy().copy(), "bitmaps": _np(self.t.bitmaps), "rows": _np(self.t.rows),
                "grads": _np(self.grads), "imp": _np(self.imp), "out": self.out.cpu().numpy().copy()}

    def touched(self):
        """-> per table k: (count, sorted row list, bitmap as uint32)."""
        s = self.state()
        out = [None] * self.L
        for i in range(self.L):
            c = int(s["counts"][i])
            out[self.L - 1 - i] = (c, np.sort(s["rows"][i][:c]), s["bitmaps"][i].view(np.uint32))
        return out


def _bitmap(rows, n_rows):
    words = np.zeros((n_rows + 31) // 32, dtype=np.uint32)
    np.bitwise_or.at(words, rows >> 5, (np.uint32(1) << (rows & 31).astype(np.uint32)))
    return words


def _check_marks(kern, want_rows, what, cleared):
    for kk, (c, rows, bm) in enumerate(kern.touched()):
        assert c == want_rows[kk].shape[0], f"{what}: level {kk} count {c}, reference set {want_rows[kk].shape[0]}"
        assert np.array_equal(rows, want_rows[kk]), f"{what}: level {kk} row list is not a permutation of the set"
        n_rows = kern.octree.hier_features[kk].shape[0]
        want_bm = np.zeros_like(bm) if cleared else _bitmap(want_rows[kk], n_rows)
        assert np.array_equal(bm, want_bm), f"{what}: level {kk} bitmap differs from {'zero' if cleared else 'the set'}"


def run_kernel_case(octree, o, coord_np, grads, last, imp, lam, what):
    """Every exact check and graded quantity of part (a) on one batch -> worst error / bound."""
    L, F = octree.featured_level_num, octree.feature_dim
    caps = [int(p.shape[0]) for p in octree.hier_features]
    want_rows = touched_sets(o, coord_np)
    coord = torch.from_numpy(np.ascontiguousarray(coord_np, dtype=np.float32)).to(DEV)
    kern = Kernels(octree, grads, last, imp)
    tables = _np(octree.hier_features)
    init = 0.25
    # mark: exact set, a second mark of the same batch adds nothing
    kern.set(out=init)
    assert kern.mark(coord) == OK
    _check_marks(kern, want_rows, what, cleared=False)
    assert kern.mark(coord) == OK
    _check_marks(kern, want_rows, what + " (marked twice)", cleared=False)
    # regularisation, clear_marks = 0: graded; the bitmap still holds the set
    assert kern.reg(lam, 0) == OK
    s0 = kern.state()
    ref = RegRef(tables, last, imp, want_rows, lam, grads=grads)
    worst = grade_rows(s0["grads"], ref.want, ref.bound, f"{what} regularisation gradients", tag="incre kernels")
    vb = ref.value_bound(caps, F, _sm(), init)
    err = abs(float(s0["out"][0]) - init - ref.value)
    assert err <= vb, f"{what}: reg {float(s0['out'][0]) - init} want {ref.value} bound {vb}"
    worst = max(worst, err / vb if vb > 0 else 0.0)
    _check_marks(kern, want_rows, what + " (after reg, clear 0)", cleared=False)
    for kk in range(L):                      # untouched rows keep their input bits
        keep = np.ones(caps[kk], dtype=bool)
        keep[want_rows[kk]] = False
        assert np.array_equal(s0["grads"][kk][keep], grads[kk][keep]), f"{what}: untouched rows changed"
    # out_reg NULL: same gradients, bit for bit
    kern.set(grads=grads, out=init)
    assert kern.reg(lam, 0, out=False) == OK
    s1 = kern.state()
    assert all(np.array_equal(a, b) for a, b in zip(s1["grads"], s0["grads"])), f"{what}: out_reg NULL changed the gradients"
    assert float(s1["out"][0]) == init
    # clear_marks = 1: same gradients, value graded again, every bitmap word 0
    kern.set(grads=grads, out=init)
    assert kern.reg(lam, 1) == OK
    s2 = kern.state()
    assert all(np.array_equal(a, b) for a, b in zip(s2["grads"], s0["grads"])), f"{what}: clear_marks changed the gradients"
    assert abs(float(s2["out"][0]) - init - ref.value) <= vb
    _check_marks(kern, want_rows, what + " (after reg, clear 1)", cleared=True)
    # importance, zero_grads = 1 (clear 0): Omega graded, touched gradients exactly 0, the rest bit-identical
    g1 = s0["grads"]
    kern.t.counts.zero_()
    assert kern.mark(coord) == OK
    kern.set(grads=g1, imp=imp)
    assert kern.importance(1, 0) == OK
    s3 = kern.state()
    iw, ib = importance_want(imp, [([np.abs(g.astype(np.float64)) for g in g1], None)], [want_rows])
    worst = max(worst, grade_rows(s3["imp"], iw, ib, f"{what} importance", tag="incre kernels"))
    for kk in range(L):
        r = want_rows[kk]
        assert not s3["grads"][kk][r].any(), f"{what}: zero_grads left a touched gradient non-zero"
        keep = np.ones(caps[kk], dtype=bool)
        keep[r] = False
        assert np.array_equal(s3["grads"][kk][keep], g1[kk][keep]), f"{what}: importance changed an untouched gradient"
        assert np.array_equal(s3["imp"][kk][keep], imp[kk][keep]), f"{what}: importance changed an untouched row"
    _check_marks(kern, want_rows, what + " (after importance, clear 0)", cleared=False)
    # importance, zero_grads = 0 (clear 1): gradients bit-identical, same Omega, bitmap cleared
    kern.set(grads=g1, imp=imp)
    assert kern.importance(0, 1) == OK
    s4 = kern.state()
    assert all(np.array_equal(a, b) for a, b in zip(s4["grads"], g1)), f"{what}: zero_grads 0 changed the gradients"
    assert all(np.array_equal(a, b) for a, b in zip(s4["imp"], s3["imp"])), f"{what}: importance is not deterministic"
    _check_marks(kern, want_rows, what + " (after importance, clear 1)", cleared=True)
    # Omega = 0, then f = f_last: no atomic, out_reg stays at its initial value, gradients == input
    for name, kern2 in (("Omega = 0", Kernels(octree, grads, last, [np.zeros_like(t) for t in imp])),
                        ("f = f_last", Kernels(octree, grads, tables, imp))):
        kern2.set(out=init)
        assert kern2.mark(coord) == OK and kern2.reg(lam, 1) == OK
        s5 = kern2.state()
        assert float(s5["out"][0]) == init, f"{what} {name}: out_reg changed"
        assert all(np.array_equal(a, b) for a, b in zip(s5["grads"], grads)), f"{what} {name}: gradients changed"
    print(f"[incre kernels] {what}: touched {[int(r.shape[0]) for r in want_rows]}, value error {err / vb if vb > 0 else 0.0:.3f} of its bound")
    return worst, want_rows


# ---- (a) the kernels at every shape --------------------------------------------------------------------------------------

_CASES = {}


def _models(F, L):
    """make_case with f_last = f + 0.01 N and Omega spread over six decades per row (trash row 0), cached per shape."""
    if (F, L) not in _CASES:
        case = make_case(n_points=1500, n_batch=3000, feat_levels=L, feature_dim=F, seed=100 + 10 * L + F, reduction="sum")
        cfg, octree, dec = build_cuda_models(case, DEV)
        o, _ = oracle_from_case(case)
        g = np.random.default_rng(F * 7 + L)
        last = [(t + 0.01 * g.standard_normal(t.shape)).astype(np.float32) for t in case["tables"]]
        imp = [(10.0 ** g.uniform(-6, 0, (t.shape[0], 1)) * g.uniform(0.5, 1, t.shape)).astype(np.float32)
               for t in case["tables"]]
        for w in imp:
            w[-1] = 0.0
        _CASES[(F, L)] = (case, cfg, octree, dec, o, last, imp)
    return _CASES[(F, L)]


def _batch(case, name):
    c = case["coord"]
    if name == "n0":
        return c[:0]
    if name == "n1":
        return c[-1:]
    if name == "n7":
        return c[-16:-9]                               # the six stragglers of make_case and one surface point
    if name == "n33":
        return c[-33:]
    if name == "n3000":
        return c
    if name == "miss":
        return np.array([[0.9, 0.9, 0.9], [-0.9, 0.9, -0.9], [0.9, -0.9, 0.9], [1.0, 1.0, 1.0], [-1.0, -1.0, -1.0]] * 7,
                        dtype=np.float32)
    if name == "repeat":
        return np.repeat(c[-1:], 100_000, axis=0)
    raise ValueError(name)


BATCHES = ("n0", "n1", "n7", "n33", "n3000", "miss", "repeat")


@pytest.mark.parametrize("batch", BATCHES)
@pytest.mark.parametrize("L", (1, 3, 8))
@pytest.mark.parametrize("F", (4, 8, 16, 32))
def test_touched_row_kernels(F, L, batch, built_lib):
    """Seeded gradient tables; at F = 8 also the gradients of a real fused step on the batch."""
    case, cfg, octree, dec, o, last, imp = _models(F, L)
    coord = _batch(case, batch)
    g = np.random.default_rng(F + L + len(coord))
    grads = [(g.standard_normal(t.shape) * 10.0 ** g.uniform(-3, 1, t.shape)).astype(np.float32) for t in case["tables"]]
    worst, rows = run_kernel_case(octree, o, coord, grads, last, imp, 1e3, f"F={F} L={L} {batch}")
    if batch == "miss":
        assert all(r.shape[0] == 0 for r in rows)
    elif batch != "n0":
        assert any(r.shape[0] > 0 for r in rows)
    if F == 8 and coord.shape[0] > 0:
        from shine_mapping_b200 import SdfTrainer
        tr = SdfTrainer(cfg, octree, dec)
        tr.zero_grad()
        c = torch.from_numpy(np.ascontiguousarray(coord)).to(DEV)
        tr.forward_backward(c, torch.zeros(c.shape[0], device=DEV))
        worst = max(worst, run_kernel_case(octree, o, coord, _np(tr.table_grads), last, imp, 1e3,
                                           f"F={F} L={L} {batch} fused-step gradients")[0])
    assert worst <= 1.0


def test_touched_row_kernels_grid_stride(built_lib):
    """F = 32 and a batch touching more than 8 * 256 * SM count (row, float4) items on the finest level: the touched-row
    kernels' grid-stride loop takes a second pass."""
    case = make_case(n_points=3000, n_batch=60000, feat_levels=3, feature_dim=32, seed=9, n_azimuth=512, reduction="sum")
    _, octree, _ = build_cuda_models(case, DEV)
    o, _ = oracle_from_case(case)
    coord = np.concatenate([case["coord"], case["frames"][0]]).astype(np.float32)
    g = np.random.default_rng(9)
    last = [(t + 0.01 * g.standard_normal(t.shape)).astype(np.float32) for t in case["tables"]]
    imp = [(10.0 ** g.uniform(-6, 0, (t.shape[0], 1)) * g.uniform(0.5, 1, t.shape)).astype(np.float32) for t in case["tables"]]
    for w in imp:
        w[-1] = 0.0
    grads = [(g.standard_normal(t.shape)).astype(np.float32) for t in case["tables"]]
    rows = touched_sets(o, coord)
    grid = 8 * 256 * _sm()
    items = [r.shape[0] * 32 // 4 for r in rows]
    print(f"[incre kernels] grid stride: items per level {items} against a grid of {grid} threads")
    assert max(items) > grid, "the batch fits in one pass of the grid"
    blocks, m, _ = launch_geometry([r.shape[0] for r in rows], [t.shape[0] for t in case["tables"]], 32, _sm())
    assert blocks == 8 * _sm() and m >= 2
    worst, _ = run_kernel_case(octree, o, coord, grads, last, imp, 1e3, "grid stride F=32 L=3")
    assert worst <= 1.0


# ---- (b) argument checks ---------------------------------------------------------------------------------------------------

def test_abi_rejections_leave_every_buffer_untouched(built_lib):
    from torch.profiler import ProfilerActivity, profile
    case, _, octree, _, o, last, imp = _models(8, 3)
    g = np.random.default_rng(1)
    grads = [g.standard_normal(t.shape).astype(np.float32) for t in case["tables"]]
    kern = Kernels(octree, grads, last, imp)
    coord = torch.from_numpy(case["coord"]).to(DEV)
    kern.set(out=0.5)
    assert kern.mark(coord) == OK
    before = kern.state()

    def same(what):
        after = kern.state()
        for key in before:
            a, b = before[key], after[key]
            pairs = zip(a, b) if isinstance(a, list) else [(a, b)]
            assert all(x.tobytes() == y.tobytes() for x, y in pairs), f"{what}: {key} changed"

    def copy(struct):
        return type(struct).from_buffer_copy(struct)

    calls = [("touched NULL: mark", lambda: kern.mark(coord, touched=False), INVALID),
             ("touched NULL: reg", lambda: kern.reg(1e3, 1, touched=False), INVALID),
             ("touched NULL: importance", lambda: kern.importance(1, 1, touched=False), INVALID)]
    for field in ("bitmap", "rows", "count", "capacity"):
        t = copy(kern.t.desc)
        setattr(t.lv[1], field, 0 if field == "capacity" else None)
        calls += [(f"{field} NULL/0 on level 1: mark", lambda t=t: kern.mark(coord, touched=t), INVALID),
                  (f"{field} NULL/0 on level 1: reg", lambda t=t: kern.reg(1e3, 1, touched=t), INVALID),
                  (f"{field} NULL/0 on level 1: importance", lambda t=t: kern.importance(1, 1, touched=t), INVALID)]
    calls += [("aux NULL: reg", lambda: kern.reg(1e3, 1, aux=False), INVALID),
              ("aux NULL: importance", lambda: kern.importance(1, 1, aux=False), INVALID)]
    for field, entry in (("last", "reg"), ("importance", "reg"), ("importance_rw", "importance")):
        a = copy(kern.aux)
        getattr(a, field)[1] = None
        fn = (lambda a=a: kern.reg(1e3, 1, aux=a)) if entry == "reg" else (lambda a=a: kern.importance(1, 1, aux=a))
        calls.append((f"aux.{field}[1] NULL", fn, INVALID))
    calls += [("n < 0", lambda: kern.mark(coord, n=-1), INVALID),
              ("coord NULL with n > 0", lambda: kern.mark(None, n=5), INVALID)]
    for field, value, rc in (("feature_dim", 6, UNSUPPORTED), ("num_levels", 0, INVALID), ("num_levels", 9, INVALID)):
        od = copy(kern.od)
        setattr(od, field, value)
        calls += [(f"{field} = {value}: mark", lambda od=od: kern.mark(coord, od=od), rc),
                  (f"{field} = {value}: reg", lambda od=od: kern.reg(1e3, 1, od=od), rc),
                  (f"{field} = {value}: importance", lambda od=od: kern.importance(1, 1, od=od), rc)]
    for what, fn, rc in calls:
        got = fn()
        assert got == rc, f"{what}: returned {got}, expected {rc}"
        same(what)
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        assert kern.mark(coord[:0]) == OK
        torch.cuda.synchronize()
    assert not any("mark_touched" in e.key for e in prof.key_averages()), "n = 0 launched a kernel"
    same("n = 0")


# ---- the dense pair of the loop, moved from test_gpu_loop.py ---------------------------------------------------------------

def _stride_refs(case, o, coord, label, bs, down_rate):
    """Per stride of cal_feature_importance: (|g| fp64, bound, touched rows, rows touched by kink points) of the unweighted
    BCE(sum) step, from the replica model's Ref."""
    out = []
    n, interval = coord.shape[0], bs * down_rate
    for head in range(0, n, interval):
        c = np.ascontiguousarray(coord[head:min(head + interval, n):down_rate])
        lab = np.ascontiguousarray(label[head:min(head + interval, n):down_rate])
        cs = dict(case, cfg=dict(case["cfg"], weighted=False, reduction="sum"), coord=c, label=lab,
                  weight=np.ones(c.shape[0], dtype=np.float32), oracle=o)
        ref = Ref(cs)
        B = [(k[:, None] + ref.slack) * U * S + T for S, k, T in zip(ref.S, ref.k, ref.T)]
        out.append(([np.abs(w) for w in ref.want], B, touched_sets(o, c), rows_of_points(o, c, ref.kink)))
    return out


def grade_sweep(case, o, prior, coord, label, bs, down_rate, got, what):
    """Omega after cal_feature_importance against prior + fp64 orc.cal_feature_importance, excluding the rows of kink
    points -> (worst error / bound, number of strides)."""
    strides = _stride_refs(case, o, coord, label, bs, down_rate)
    _, bound = importance_want(prior, [(a, B) for a, B, _, _ in strides], [r for _, _, r, _ in strides])
    o64, d64 = oracle64(dict(case, oracle=o))
    sweep = orc.cal_feature_importance(o64, d64, torch.from_numpy(coord), torch.from_numpy(label).double(),
                                       case["cfg"]["sigma"], bs, down_rate, "sum")
    want = [np.asarray(p, dtype=np.float64) + s.detach().numpy() for p, s in zip(prior, sweep)]
    exclude = [np.zeros(w.shape[0], dtype=bool) for w in want]
    touched = [np.zeros(w.shape[0], dtype=bool) for w in want]
    for _, _, rows, kink in strides:
        for kk in range(len(want)):
            exclude[kk] |= kink[kk]
            touched[kk][rows[kk]] = True
    n_ex, n_t = sum(int(e.sum()) for e in exclude), sum(int(t.sum()) for t in touched)
    assert n_ex <= KINK_SHARE * n_t, f"{what}: {n_ex} of {n_t} touched rows near a ReLU kink"
    for kk in range(len(got)):
        assert float(got[kk][-1].max(initial=0.0)) == 0.0 and float(got[kk][-1].min(initial=0.0)) == 0.0
    return grade_rows(got, want, bound, f"{what} (rows near a kink left out: {n_ex} of {n_t})", exclude, "incre sweep"), \
        len(strides)


def test_regularization_and_importance_match_oracle(built_lib):
    """BASELINE config 4 terms on one batch: `add_regularization` (value + gradient, with no sort / unique kernel) and
    `cal_feature_importance` against fp64, element by element."""
    from torch.profiler import ProfilerActivity, profile

    from shine_mapping_b200 import SdfTrainer
    from shine_mapping_b200.incre_loop import add_regularization, cal_feature_importance
    case = make_case(n_points=2000, n_batch=3000, feat_levels=3, seed=71, reduction="sum")
    cfg, octree, dec = build_cuda_models(case, DEV)
    g = torch.Generator().manual_seed(5)
    last = [(t + 0.01 * torch.randn(t.shape, generator=g).numpy()).astype(np.float32) for t in case["tables"]]
    imp = [torch.rand(t.shape, generator=g).numpy() for t in case["tables"]]
    for w in imp:
        w[-1] = 0.0      # reference invariant: the trash row's importance is reset after every pass (utils/incre_learning.py:40)
    octree.features_last_frame = [torch.from_numpy(t).to(DEV) for t in last]
    octree.importance_weight = [torch.from_numpy(t).to(DEV) for t in imp]
    coord = torch.from_numpy(case["coord"]).to(DEV); label = torch.from_numpy(case["label"]).to(DEV)
    tr = SdfTrainer(cfg, octree, dec)
    # regulariser alone: value + gradient
    tr.zero_grad()
    octree.query_feature(coord)
    lam = 1e3
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        reg = add_regularization(tr, octree, lam)
        torch.cuda.synchronize()
    names = [e.key for e in prof.key_averages() if e.device_type == torch.autograd.DeviceType.CUDA]
    if names:   # CUPTI records nothing when another tool (compute-sanitizer) already owns the injection slot
        assert any("mark_touched" in k for k in names) and any("touched_rows" in k for k in names), names
        assert not any(("sort" in k.lower() or "unique" in k.lower() or "radix" in k.lower()) for k in names), names
    assert abs(float(reg) - float(octree.cal_regularization())) <= 1e-5 * abs(float(reg))
    o, _ = oracle_from_case(case)
    rows = touched_sets(o, case["coord"])
    ref = RegRef(case["tables"], last, imp, rows, lam)
    vb = ref.value_bound([t.shape[0] for t in case["tables"]], 8, _sm())
    assert abs(float(reg) - ref.value) <= vb, (float(reg), ref.value, vb)
    worst = grade_rows(_np(tr.table_grads), ref.want, ref.bound, "add_regularization gradients", tag="incre loop")
    # importance sweep
    octree.importance_weight = [torch.zeros_like(p) for p in octree.hier_features]
    cal_feature_importance(tr, octree, coord, label, bs=512, down_rate=2)
    w2, n_strides = grade_sweep(case, o, [np.zeros_like(t) for t in case["tables"]], case["coord"], case["label"], 512, 2,
                                _np(octree.importance_weight), "cal_feature_importance")
    assert n_strides == -(-case["coord"].shape[0] // 1024)
    assert max(worst, w2) <= 1.0


# ---- (c) the loop, one step at a time ------------------------------------------------------------------------------------

LAMBDA = 1e2
LOOP_CASES = [(1, False), (2, False), (2, True)]


def _drive(cfg, n_az=32, n_frames=3):
    from shine_mapping_b200 import synth
    dirs, boxes = synth.lidar_directions(n_az, device=DEV), synth.default_boxes(DEV)
    gen = torch.Generator(device=DEV).manual_seed(3)
    frames = []
    for f in range(n_frames):
        origin = torch.tensor([2.0 * f, 0.0, 0.0], device=DEV)
        hits = synth.raycast_scene(origin, dirs, boxes, cfg.min_range, cfg.pc_radius)
        frames.append(synth.sample_rays(hits * cfg.scale, origin * cfg.scale, cfg, gen))
    return frames


@pytest.mark.parametrize("down_rate,eikonal", LOOP_CASES, ids=[f"down{d}{'-eikonal' if e else ''}" for d, e in LOOP_CASES])
def test_incremental_loop_steps_match_fp64(down_rate, eikonal, monkeypatch, force, built_lib):
    from shine_mapping_b200 import Decoder, FeatureOctree, SdfTrainer, incre_loop
    force(1, 8)                         # gradient replicas on the coarser levels at 2048 points
    bs, iters, weight_e = (512 if eikonal else 2048), 4, 1.0
    cfg = make_config(3, device=DEV, bs=bs, lr=0.01, iters=iters, continual_learning_reg=True, lambda_forget=LAMBDA,
                      freeze_after_frame=1, loss_weight_on=True, cal_importance_weight_down_rate=down_rate,
                      ekional_loss_on=eikonal, weight_e=weight_e)
    torch.manual_seed(1)
    octree, decoder = FeatureOctree(cfg), Decoder(cfg)
    frames = _drive(cfg)
    for c, _, _ in frames:
        assert c.shape[0] % (bs * down_rate) != 0, "pick a pool size that leaves a short last stride"
    spy = FoldSpy(octree)
    rec = {"steps": [], "sweeps": []}
    state = {"batch": None, "reg": None, "sweep": False}

    def keep_batch(orig):
        def wrapped(self, coord, sdf_label, weight=None, *a, **kw):
            if not state["sweep"]:
                state["batch"] = tuple(None if t is None else t.detach().cpu().numpy().copy() for t in (coord, sdf_label, weight))
            return orig(self, coord, sdf_label, weight, *a, **kw)
        return wrapped

    monkeypatch.setattr(SdfTrainer, "forward_backward", keep_batch(SdfTrainer.forward_backward))
    monkeypatch.setattr(SdfTrainer, "forward_backward_eikonal", keep_batch(SdfTrainer.forward_backward_eikonal))
    add_reg = incre_loop.add_regularization

    def add_regularization(trainer, oc, lam, coord=None):
        reg = add_reg(trainer, oc, lam, coord)
        state["reg"] = reg
        return reg
    monkeypatch.setattr(incre_loop, "add_regularization", add_regularization)

    def snapshot(tr):
        oc = tr.octree
        return {"tables": _np(oc.hier_features), "last": _np(oc.features_last_frame), "imp": _np(oc.importance_weight),
                "dec": {k: v.detach().cpu().numpy().copy() for k, v in decoder.state_dict().items()
                        if k.startswith(("layers.", "lout."))}}

    opt_step = SdfTrainer.optimizer_step

    def optimizer_step(self, *a, **kw):
        torch.cuda.synchronize()
        s = snapshot(self)
        s.update(batch=state["batch"], reg=float(state["reg"]), grads=_np(self.table_grads), trainable=self._dec_trainable,
                 dec_grads={k: g.cpu().numpy().copy() for k, g in zip(DEC_KEYS, self.dec_grads)
                            if g is not None and self._dec_trainable},
                 R=spy.calls[-1] if spy.calls else None)
        spy.calls.clear()
        if s["R"] is not None and max(s["R"]) > 1:
            assert_scratch_zero(self.octree, f"step {len(rec['steps'])}")
        rec["steps"].append(s)
        return opt_step(self, *a, **kw)
    monkeypatch.setattr(SdfTrainer, "optimizer_step", optimizer_step)
    sweep = incre_loop.cal_feature_importance

    def cal_feature_importance(trainer, oc, coord_pool, label_pool, bs_, down_rate_=1):
        torch.cuda.synchronize()
        s = snapshot(trainer)
        s.update(coord=coord_pool.cpu().numpy().copy(), label=label_pool.cpu().numpy().copy(), bs=bs_, down_rate=down_rate_,
                 zero=[])
        rec["sweeps"].append(s)
        state["sweep"] = True
        try:
            sweep(trainer, oc, coord_pool, label_pool, bs_, down_rate_)
        finally:
            state["sweep"] = False
        torch.cuda.synchronize()
        s["after"] = _np(oc.importance_weight)
    monkeypatch.setattr(incre_loop, "cal_feature_importance", cal_feature_importance)
    zero_grad = SdfTrainer.zero_grad

    def zero_grad_spy(self):
        if state["sweep"]:
            torch.cuda.synchronize()
            rec["sweeps"][-1]["zero"].append([int(torch.count_nonzero(g)) for g in self.table_grads])
        return zero_grad(self)
    monkeypatch.setattr(SdfTrainer, "zero_grad", zero_grad_spy)

    hist = incre_loop.run_shine_mapping_incremental(cfg, octree, decoder, frames)
    assert len(rec["steps"]) == 3 * iters and len(rec["sweeps"]) == 3

    # ---- grading, frame by frame on one oracle octree grown like the map
    L, F = 3, cfg.feature_dim
    cased = {"tree_level_world": cfg.tree_level_world, "tree_level_feat": L, "feature_dim": F,
             "poly_int_on": cfg.poly_int_on, "leaf_vox_size": cfg.leaf_vox_size, "sigma": float(cfg.sigma_sigmoid),
             "weighted": True, "reduction": "sum", "bias": True}
    o = orc.OracleOctree(cfg.tree_level_world, L, F, 0.05, cfg.poly_int_on)
    worst = {"steps": 0.0, "value": 0.0, "sweep": 0.0, "decoder": 0.0}
    ratio, dec_graded, replicas = 0.0, 0, []
    for f in range(3):
        coord_f, _, weight_f = (t.cpu().numpy() for t in frames[f])
        o.update(torch.from_numpy(coord_f[weight_f > 0]))
        h = hist[f]
        for it in range(iters):
            s = rec["steps"][f * iters + it]
            what = f"frame {f} step {it}"
            coord, label, weight = s["batch"]
            case = {"cfg": cased, "frames": [], "tables": s["tables"], "dec": s["dec"], "coord": coord, "label": label,
                    "weight": weight, "oracle": o}
            if eikonal:
                ref = EikRef(case, weight_e)
                g64 = ref.rows.want
                B = [ref.rows.bound(kk) for kk in range(L)]
                drop = ref.drop
            else:
                ref = Ref(case)
                g64 = ref.want
                B = [(k[:, None] + ref.slack) * U * S + T for S, k, T in zip(ref.S, ref.k, ref.T)]
                drop = ref.kink
                replicas.append(s["R"])
                assert s["R"] == expected_replicas(s["tables"], coord.shape[0]), f"{what}: R per level {s['R']}"
            rows = touched_sets(o, coord)
            reg = RegRef(s["tables"], s["last"], s["imp"], rows, LAMBDA, grads=g64, B=B)
            exclude = rows_of_points(o, coord, drop)
            n_ex = sum(int(e.sum()) for e in exclude)
            n_t = sum(int(r.shape[0]) for r in rows)
            assert n_ex <= KINK_SHARE * n_t, f"{what}: {n_ex} of {n_t} touched rows near a ReLU kink"
            worst["steps"] = max(worst["steps"], grade_rows(
                s["grads"], reg.want, reg.bound, f"{what} (rows near a kink left out: {n_ex} of {n_t})", exclude, "incre loop"))
            vb = reg.value_bound([t.shape[0] for t in s["tables"]], F, _sm())
            err = abs(s["reg"] - reg.value)
            assert err <= vb, f"{what}: reg {s['reg']} want {reg.value} bound {vb}"
            worst["value"] = max(worst["value"], err / vb if vb > 0 else 0.0)
            if it == 0:
                assert s["reg"] == 0.0, f"{what}: the first step of a frame has a non-zero regulariser"
                if eikonal:     # total = bce + weight_e * eikonal in fp32, then + lambda * 0
                    want_total = h["bce_first"] + weight_e * h["eik_first"]
                    assert abs(h["loss_first"] - want_total) <= 2 * U * abs(want_total), h
                else:
                    assert h["loss_first"] == h["bce_first"], h
            for kk in range(L):
                tmax = float(np.abs(reg.t[kk]).max(initial=0.0))
                gmax = float(np.abs(np.asarray(g64[kk])[:-1]).max(initial=0.0))
                if gmax > 0:
                    ratio = max(ratio, tmax / gmax)
            # decoder gradients: the parity bar of compare_step (1e-3 with the eikonal term, whose steps with a dropped point
            # are skipped), plus, for BCE, the bound of what the kink points can change
            if s["trainable"] and not (eikonal and drop.any()):
                want_dec = autograd_decoder_grads(case, weight_e) if eikonal else ref.step["dec_grads"]
                slack = {} if eikonal or not drop.any() else decoder_kink_slack(case, drop)
                bar = 1e-3 if eikonal else 2e-4
                for k, got in s["dec_grads"].items():
                    w = np.asarray(want_dec[k])
                    scale = max(float(np.abs(w).max()), 1e-30)
                    e = (np.abs(got - w) - slack.get(k, 0.0)) / scale
                    assert float(e.max()) <= bar, f"{what}: decoder gradient {k} off by {float(e.max()):.2e} of its maximum"
                    worst["decoder"] = max(worst["decoder"], float(np.abs(got - w).max()) / scale)
                dec_graded += 1
            assert s["trainable"] == (f < 1)
        # the sweep
        sw = rec["sweeps"][f]
        assert sw["zero"] and all(c == 0 for c in sw["zero"][-1]), \
            f"frame {f}: table gradients left non-zero before the sweep's closing zero_grad: {sw['zero'][-1]}"
        scase = {"cfg": cased, "frames": [], "tables": sw["tables"], "dec": sw["dec"], "coord": sw["coord"],
                 "label": sw["label"], "weight": np.ones(sw["coord"].shape[0], dtype=np.float32)}
        w, n_strides = grade_sweep(scase, o, sw["imp"], sw["coord"], sw["label"], bs, down_rate, sw["after"],
                                   f"frame {f} sweep")
        assert n_strides == -(-sw["coord"].shape[0] // (bs * down_rate))
        worst["sweep"] = max(worst["sweep"], w)
        # the next frame's regulariser starts from that Omega (new rows 0)
        if f + 1 < 3:
            nxt = rec["steps"][(f + 1) * iters]["imp"]
            for kk in range(L):
                old = sw["after"][kk].shape[0] - 1
                assert np.array_equal(nxt[kk][:old], sw["after"][kk][:old]), f"frame {f + 1}: Omega is not the sweep's"
                assert not nxt[kk][old:].any(), f"frame {f + 1}: new rows carry importance"
    if not eikonal:
        assert any(r is not None and max(r) > 1 for r in replicas), "no step ran with gradient replicas"
        print(f"[incre loop] R per level of the steps: {replicas}")
    assert ratio >= 0.1, f"the regulariser's gradient reaches only {ratio:.3f} of the BCE gradient's maximum"
    assert dec_graded >= 1, "no step graded the decoder gradients"
    print(f"[incre loop] down_rate {down_rate}{' eikonal' if eikonal else ''}: worst error / bound {worst}; "
          f"regulariser / first-term gradient maxima up to {ratio:.2f}; decoder graded on {dec_graded} steps")
