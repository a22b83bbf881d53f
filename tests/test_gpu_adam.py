"""Adam on the GPU against the fp64 oracle (`oracle.shine_oracle.adam_reference`): the multi-tensor kernel through the C ABI
(`shine_adam_step`, `shine_adam_step_dev`), and every trainer path that runs it, with one step count across them.

Error bounds.  The ABI takes the betas and eps as fp32, so the kernel's beta1 is fl32(0.9) and its 1 - beta1 is
1 - fl32(0.9), which is exact in fp32 (likewise for beta2 = fl32(0.99)); the reference runs with those same values, and
with lr and weight decay as the fp32 values the kernel reads.  Per element the kernel does about ten fp32 roundings, each
off by at most u = 2^-24 of its result:
    g' = fma(wd, theta, g)                                          1
    m' = m + (g' - m) (1 - beta1)                                   3 (the last may fuse)
    v' = beta2 v + ((1 - beta2) g') g'                              4, and g' enters twice
    theta' = theta - (lr / bc1) m' / (sqrt(v') / bc2_sqrt + eps)    bc1, bc2_sqrt, lr / bc1, sqrt, /, +, /, x: 8; - : 1/2 ulp
m' can cancel (0.9 m against 0.1 g' of the other sign), so its error is measured against the magnitudes that enter it,
S_m = |m'| + (1 - beta1)(|g'| + |m|): |m' - m'64| <= 4u S_m.  v' sums non-negative terms: |v' - v'64| <= 8u |v'64|.  Both
add the smallest subnormal (v underflows below |g| ~ 1e-22).  m' and v' are graded against the oracle run on the same
fp32 inputs widened to fp64.  The update dtheta = theta' - theta, taken in fp64, is graded against the update the oracle's
formula gives for the kernel's own m' and v' (so a cancelling m' does not blur it):
|dtheta - dtheta64| <= 32u |dtheta64| + ulp(theta'), which is about 1.9e-6 relative, four times the eight roundings of the
chain; a bias correction one step off changes the update by 1e-3 or more at every step up to 100.
"""
import math

import numpy as np
import pytest
import torch

from oracle import shine_oracle as orc
from tests.parity_utils import build_cuda_models, make_case

pytestmark = pytest.mark.gpu
DEV = "cuda:0"

U = 2.0 ** -24
TINY = 2.0 ** -149                      # smallest fp32 subnormal
M_BOUND, V_BOUND, D_BOUND = 4 * U, 8 * U, 32 * U


def f32(x):
    return float(np.float32(x))


B1, B2, EPS = f32(0.9), f32(0.99), f32(1e-15)
INVALID = -1                            # SHINE_ERR_INVALID_ARG


@pytest.fixture(scope="module", autouse=True)
def _lib(built_lib):
    assert torch.cuda.is_available()
    return built_lib


def _ulp(x32):
    a = x32.abs()
    return (torch.nextafter(a, torch.full_like(a, math.inf)) - a).double()


def grade(theta, g, m, v, theta_a, m_a, v_a, step, lr, wd, what=""):
    """One Adam step of fp32 state (theta, g, m, v) -> (theta_a, m_a, v_a) against the fp64 oracle, with the bounds of the
    module docstring.  g / m / v may be None (graphed paths, where the gradient is never visible): then only the update
    identity is checked.  -> {quantity: worst error / bound}."""
    theta, theta_a, m_a, v_a = (t.detach().cpu() for t in (theta, theta_a, m_a, v_a))
    worst = {}
    if g is not None:
        g, m, v = (t.detach().cpu() for t in (g, m, v))
        _, m64, v64 = orc.adam_reference(theta, g, m, v, step, lr, wd, betas=(B1, B2), eps=EPS)
        gd = g.double() + wd * theta.double()
        tol_m = M_BOUND * (m64.abs() + (1.0 - B1) * (gd.abs() + m.double().abs())) + TINY
        tol_v = V_BOUND * v64.abs() + TINY
        err_m, err_v = (m_a.double() - m64).abs(), (v_a.double() - v64).abs()
        worst["m"], worst["v"] = float((err_m / tol_m).max()), float((err_v / tol_v).max())
        assert worst["m"] <= 1.0, f"{what} exp_avg: worst {worst['m']:.3g} of the bound"
        assert worst["v"] <= 1.0, f"{what} exp_avg_sq: worst {worst['v']:.3g} of the bound"
    bc1, bc2_sqrt = 1.0 - B1 ** step, math.sqrt(1.0 - B2 ** step)
    d64 = -(lr / bc1) * m_a.double() / (v_a.double().sqrt() / bc2_sqrt + EPS)
    err_d = (theta_a.double() - theta.double() - d64).abs()
    tol_d = D_BOUND * d64.abs() + _ulp(theta_a)
    worst["dtheta"] = float((err_d / tol_d).max())
    assert worst["dtheta"] <= 1.0, f"{what} update at step {step}: worst {worst['dtheta']:.3g} of the bound"
    return worst


def merge(acc, w):
    for k, x in w.items():
        acc[k] = max(acc.get(k, 0.0), x)
    return acc


def report(group, acc):
    print(f"[adam bounds] {group}: " + " ".join(f"{k}={acc[k]:.3f}" for k in ("m", "v", "dtheta") if k in acc)
          + "  (worst error / bound)")


# ---- the kernel through the C ABI ----------------------------------------------------------------------------------

def _entry(t, lr, wd):
    from shine_mapping_b200 import _abi
    e = _abi.ShineAdamTensor()
    e.param, e.grad, e.exp_avg, e.exp_avg_sq = t["p"].data_ptr(), t["g"].data_ptr(), t["m"].data_ptr(), t["v"].data_ptr()
    e.numel, e.lr, e.weight_decay = t["p"].numel(), lr, wd
    return e


def _array(entries):
    from shine_mapping_b200 import _abi
    return (_abi.ShineAdamTensor * len(entries))(*entries)


def _host_step(tensors, step, zero_grad=0):
    from shine_mapping_b200 import _abi
    arr = _array([_entry(t, t["lr"], t["wd"]) for t in tensors])
    return _abi.lib().shine_adam_step(arr, len(tensors), 0.9, 0.99, 1e-15, step, zero_grad, _abi.stream_ptr(DEV))


def _dev_step(tensors, state, zero_grad=0):
    from shine_mapping_b200 import _abi
    arr = _array([_entry(t, t["lr"], t["wd"]) for t in tensors])
    return _abi.lib().shine_adam_step_dev(arr, len(tensors), 0.9, 0.99, 1e-15, _abi.ptr(state), zero_grad,
                                          _abi.stream_ptr(DEV))


# gradient classes, by (element index + shift) mod 8: exact zeros; +-1e-30 (eps dominates the denominator: theta is 0
# there so that the ~1e-18 update is visible); +-1e17; typical values over five decades.  The shift differs per tensor,
# so that the tails of small tensors see every class.
def _gradient(n, gen, shift=0):
    i = torch.arange(n) + shift
    sign = torch.where(torch.rand(n, generator=gen) < 0.5, -1.0, 1.0).double()
    g = torch.randn(n, generator=gen, dtype=torch.float64) * 1e-3 * 10.0 ** (4 * torch.rand(n, generator=gen, dtype=torch.float64) - 2)
    g = torch.where(i % 8 == 0, 0.0, g)
    g = torch.where(i % 8 == 1, 1e-30 * sign, g)
    g = torch.where(i % 8 == 2, 1e17 * sign, g)
    return g.float()


def _tensor(n, lr, wd, gen, shift=0):
    p = torch.randn(n, generator=gen) * 0.1
    p[(torch.arange(n) + shift) % 8 == 1] = 0.0
    return {"p": p.to(DEV), "g": _gradient(n, gen, shift).to(DEV), "m": torch.zeros(n, device=DEV),
            "v": torch.zeros(n, device=DEV), "lr": lr, "wd": wd, "shift": shift}


def _snapshot(tensors):
    return [{k: t[k].clone().cpu() for k in "pgmv"} for t in tensors]


GRID_ROUND = 132 * 8 * 256 * 4          # elements one grid-stride round of the vector body covers on an H100 SXM (132 SMs)
SIZES = [1, 2, 3, 4, 5, 7, 8, 1021, GRID_ROUND - 1, GRID_ROUND, GRID_ROUND + 1, GRID_ROUND + 4, 3_000_003, 6, 9, 4099]
STEPS = [1, 2, 10, 1000, 2 ** 20]


@pytest.mark.parametrize("layout", ["mixed", "alone"])
def test_adam_kernel_matches_fp64(layout):
    """Every size of SIZES (the float4 body, the scalar tail run by block 0, more than one grid-stride round), with
    per-tensor lr and weight decay (0 or 1e-2, so zero gradients with decay still move theta), state carried over steps
    1, 2, 10, 1000 and 2^20, zero_grad on and off.  mixed: all 16 tensors in one launch (count = 16); alone: one launch per
    tensor (a grid of one block for the small ones)."""
    assert len(SIZES) == 16
    gen = torch.Generator().manual_seed(11)
    tensors = [_tensor(n, f32(1e-3 * (1 + 0.25 * i)), f32(1e-2) if i % 2 else 0.0, gen, shift=i) for i, n in enumerate(SIZES)]
    launches = [tensors] if layout == "mixed" else [[t] for t in tensors]
    acc, decay_only = {}, 0
    for call, step in enumerate(STEPS):
        zero_grad = call % 2
        before = _snapshot(tensors)
        for group in launches:
            assert _host_step(group, step, zero_grad) == 0
        torch.cuda.synchronize()
        for i, (t, b) in enumerate(zip(tensors, before)):
            a = {k: t[k].cpu() for k in "pmv"}
            merge(acc, grade(b["p"], b["g"], b["m"], b["v"], a["p"], a["m"], a["v"], step, t["lr"], t["wd"],
                             f"numel {b['p'].numel()} step {step}"))
            g_after = t["g"].cpu()
            if zero_grad:
                assert bool((g_after == 0).all()) and not bool(torch.signbit(g_after).any()), f"numel {g_after.numel()}"
            else:
                assert torch.equal(g_after.view(torch.int32), b["g"].view(torch.int32)), f"numel {g_after.numel()}"
            zero = b["g"] == 0
            if t["wd"] == 0.0:        # a zero gradient without decay: m and v stay exactly 0 and theta does not move
                assert bool((a["m"][zero] == 0).all() and (a["v"][zero] == 0).all())
                assert torch.equal(a["p"][zero], b["p"][zero])
            else:                     # decay alone moves theta
                moved = zero & (b["p"] != 0)
                decay_only += int(moved.sum())
                assert bool((a["p"][moved] != b["p"][moved]).all())
            tiny = (b["g"].abs() == f32(1e-30)) & (b["p"] == 0) & (b["m"] == 0)
            if bool(tiny.any()):      # eps dominates: dtheta = -lr/bc1 * m / eps, visible because theta was 0
                bc1 = 1.0 - B1 ** step
                want = -(t["lr"] / bc1) * a["m"][tiny].double() / EPS
                assert torch.allclose(a["p"][tiny].double(), want, rtol=D_BOUND, atol=0.0)
            t["g"].copy_(_gradient(t["p"].numel(), gen, t["shift"]).to(DEV))
    assert decay_only > 0
    report(f"kernel, {layout}", acc)


def test_adam_kernel_overflowing_gradient_matches_torch_fp32():
    """fp32 limit: once (1 - beta2) g^2 exceeds FLT_MAX (|g| above ~1.8e20 with the product formed as ((1 - beta2) g) g,
    as the kernel and torch both do; g^2 alone overflows above ~1.8e19), v is inf and fp32 Adam moves theta by
    m / inf = 0, whereas fp64 would move it by about lr.  This case is graded against torch's fp32 Adam, not the oracle."""
    gen = torch.Generator().manual_seed(12)
    n = 1021
    sign = torch.where(torch.rand(n, generator=gen) < 0.5, -1.0, 1.0)
    t = {"p": (torch.randn(n, generator=gen) * 0.1).to(DEV), "g": (1e21 * sign).to(DEV), "m": torch.zeros(n, device=DEV),
         "v": torch.zeros(n, device=DEV), "lr": f32(1e-3), "wd": 0.0}
    q = t["p"].clone().requires_grad_(True)
    q.grad = t["g"].clone()
    opt = torch.optim.Adam([q], lr=1e-3, betas=(0.9, 0.99), eps=1e-15)
    p0 = t["p"].clone()
    assert _host_step([t], 1) == 0
    opt.step()
    torch.cuda.synchronize()
    st = opt.state[q]
    assert torch.equal(t["p"], p0) and torch.equal(q.detach(), p0)          # update 0 on both sides
    assert bool(torch.isinf(t["v"]).all()) and bool(torch.isinf(st["exp_avg_sq"]).all())
    # torch rounds 1 - beta1 to fp32 (0.1f); the kernel's 1 - fl32(0.9) is 3.7u larger
    assert bool(((t["m"] - st["exp_avg"]).abs() <= 8 * U * st["exp_avg"].abs()).all())
    p64, _, _ = orc.adam_reference(p0.cpu(), t["g"].cpu(), torch.zeros(n), torch.zeros(n), 1, t["lr"], 0.0, (B1, B2), EPS)
    assert bool(((p64 - p0.cpu().double()).abs() > 0.5e-3).all())        # fp64 would have moved every element by ~lr


@pytest.mark.parametrize("start", [0, 41])
def test_adam_dev_state_advances(start):
    """shine_adam_step_dev: {step, bc1, bc2_sqrt} advance by one step from `start` and equal the fp64 bias corrections to
    fp32 rounding, and the update it runs uses them."""
    gen = torch.Generator().manual_seed(13 + start)
    tensors = [_tensor(n, f32(1e-3), wd, gen) for n, wd in ((1021, 0.0), (5, f32(1e-2)))]
    state = torch.zeros(3, dtype=torch.int32, device=DEV)
    state[0] = start
    acc = {}
    for k in range(1, 4):
        before = _snapshot(tensors)
        assert _dev_step(tensors, state) == 0
        torch.cuda.synchronize()
        step = start + k
        s = state.cpu()
        assert int(s[0]) == step
        bc = s[1:].view(torch.float32).double()
        for got, want in ((bc[0], 1.0 - B1 ** step), (bc[1], math.sqrt(1.0 - B2 ** step))):
            half_ulp = float(_ulp(torch.tensor([want], dtype=torch.float32))[0]) / 2
            assert abs(float(got) - want) <= half_ulp + 1e-15 * want, (step, float(got), want)
        for t, b in zip(tensors, before):
            merge(acc, grade(b["p"], b["g"], b["m"], b["v"], t["p"], t["m"], t["v"], step, t["lr"], t["wd"], f"dev step {step}"))
    report(f"device step from {start}", acc)


def test_adam_dev_graph_replays_equal_host_steps():
    """k replays of a captured shine_adam_step_dev give what k host-step calls with steps s+1 ... s+k give (equal, or 1 ulp
    apart where the device and host pow differ in the last bit)."""
    gen = torch.Generator().manual_seed(14)
    s, k = 5, 4
    graphed = [_tensor(n, f32(2e-3), wd, gen) for n, wd in ((4099, 0.0), (3, f32(1e-2)), (GRID_ROUND + 1, 0.0))]
    host = [{key: (x.clone() if torch.is_tensor(x) else x) for key, x in t.items()} for t in graphed]
    state = torch.zeros(3, dtype=torch.int32, device=DEV)
    scratch = [_tensor(8, f32(1e-3), 0.0, gen)]
    assert _dev_step(scratch, torch.zeros(3, dtype=torch.int32, device=DEV)) == 0      # module loaded outside capture
    torch.cuda.synchronize()
    state[0] = s
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        assert _dev_step(graphed, state) == 0
    for _ in range(k):
        graph.replay()
    for step in range(s + 1, s + k + 1):
        assert _host_step(host, step) == 0
    torch.cuda.synchronize()
    assert int(state[0]) == s + k
    for a, b in zip(graphed, host):
        for key in "pmv":
            x, y = a[key].view(torch.int32).long(), b[key].view(torch.int32).long()
            assert int((x - y).abs().max()) <= 1, key


def test_adam_rejects_bad_arguments():
    """A pointer off by 4 bytes, a null pointer, numel < 0, count 0 or 17, step 0 on the host variant and a null state
    each return SHINE_ERR_INVALID_ARG, and a rejected call changes nothing (the device-step variant checks everything
    before it advances its counter)."""
    from shine_mapping_b200 import _abi
    gen = torch.Generator().manual_seed(15)
    t = _tensor(64, f32(1e-3), 0.0, gen)
    state = torch.zeros(3, dtype=torch.int32, device=DEV)
    state[0] = 7
    before = _snapshot([t])[0]
    lib, stream = _abi.lib(), _abi.stream_ptr(DEV)

    def good():
        return _entry(t, t["lr"], t["wd"])

    bad = []
    for field in ("param", "grad", "exp_avg", "exp_avg_sq"):
        e = good(); setattr(e, field, getattr(e, field) + 4); bad.append(e)      # misaligned
        e = good(); setattr(e, field, None); bad.append(e)                        # null
    e = good(); e.numel = -1; bad.append(e)
    for e in bad:
        for arr, count in ((_array([e]), 1), (_array([good(), e]), 2)):
            assert lib.shine_adam_step(arr, count, 0.9, 0.99, 1e-15, 1, 1, stream) == INVALID
            assert lib.shine_adam_step_dev(arr, count, 0.9, 0.99, 1e-15, _abi.ptr(state), 1, stream) == INVALID
    many = _array([good() for _ in range(17)])
    for count in (0, 17, -1):
        assert lib.shine_adam_step(many, count, 0.9, 0.99, 1e-15, 1, 1, stream) == INVALID
        assert lib.shine_adam_step_dev(many, count, 0.9, 0.99, 1e-15, _abi.ptr(state), 1, stream) == INVALID
    assert lib.shine_adam_step(None, 1, 0.9, 0.99, 1e-15, 1, 1, stream) == INVALID
    assert lib.shine_adam_step_dev(None, 1, 0.9, 0.99, 1e-15, _abi.ptr(state), 1, stream) == INVALID
    for step in (0, -3):
        assert lib.shine_adam_step(_array([good()]), 1, 0.9, 0.99, 1e-15, step, 1, stream) == INVALID
    assert lib.shine_adam_step_dev(_array([good()]), 1, 0.9, 0.99, 1e-15, None, 1, stream) == INVALID
    torch.cuda.synchronize()
    assert state.cpu().tolist() == [7, 0, 0]
    for key in "pgmv":
        assert torch.equal(t[key].cpu(), before[key]), key


# ---- the trainer: grouping, every path that runs Adam, one step count ----------------------------------------------

def _trainer(levels=4, bias=True, frozen=False, seed=21, n_batch=3000, ekional=False):
    from shine_mapping_b200 import SdfTrainer
    case = make_case(n_points=2500, n_batch=n_batch, feat_levels=levels, seed=seed, bias=bias)
    cfg, octree, dec = build_cuda_models(case, DEV, freeze_decoder=frozen)
    cfg.lr, cfg.weight_decay, cfg.lr_level_reduce_ratio = 1e-2, 1e-2, 0.5
    cfg.ekional_loss_on, cfg.weight_e = ekional, 0.1
    tr = SdfTrainer(cfg, octree, dec)
    tr.zero_grad()
    batch = tuple(torch.from_numpy(case[k]).to(DEV) for k in ("coord", "label", "weight"))
    return tr, batch


def _members(tr):
    """[(parameter, index into the flat layout, group)] of every parameter, groups from the oracle's setup_optimizer."""
    tables, dec = tr._params()
    L = len(tables)
    out = []
    for gr in orc.reference_param_groups(L, tr.lr, tr.config.weight_decay, tr.config.lr_level_reduce_ratio):
        if gr["params"] == "decoder":
            out += [(p, L + j, gr) for j, p in enumerate(dec) if p is not None]
        else:
            out.append((tables[gr["params"]], gr["params"], gr))
    return out


def _theta(tr):
    return [p.detach().clone() for p, _, _ in _members(tr)]


def _record_adam_inputs(tr):
    """Every eager optimizer_step first records the gradient and the moments Adam is about to read."""
    rec, inner = [], tr.optimizer_step

    def wrapped(*a, **kw):
        if not torch.cuda.is_current_stream_capturing():
            rec.append((tr.flat_grad.clone(), tr.exp_avg.clone(), tr.exp_avg_sq.clone()))
        return inner(*a, **kw)
    tr.optimizer_step = wrapped
    return rec


def check_trainer_step(tr, before, t, inputs=None, acc=None, what=""):
    """The last Adam step was step t of the state, with the oracle's groups at tr.lr: the update identity for every
    parameter, and with `inputs` (gradient, m, v before the step) the m / v recurrence with decay.  Frozen parameters
    do not move."""
    acc = {} if acc is None else acc
    for (p, idx, gr), p0 in zip(_members(tr), before):
        if not p.requires_grad:
            assert torch.equal(p, p0), f"{what}: a frozen parameter moved"
            continue
        o, s = tr._offs[idx], tr._sizes[idx]
        sl = lambda buf: buf[o:o + s].view(p.shape)        # noqa: E731
        g = m = v = None
        if inputs is not None:
            g, m, v = (sl(b) for b in inputs)
        merge(acc, grade(p0, g, m, v, p, sl(tr.exp_avg), sl(tr.exp_avg_sq), t, f32(gr["lr"]), f32(gr["weight_decay"]),
                         f"{what} (flat segment {idx})"))
    return acc


@pytest.mark.parametrize("levels,bias,frozen", [(1, True, False), (4, True, False), (8, True, False), (4, False, False),
                                                (4, True, True), (8, False, True)])
def test_optimizer_step_groups_match_oracle(levels, bias, frozen):
    """One optimizer_step() on the trainer's own flat gradient equals adam_reference with reference_param_groups:
    decoder at lr with weight decay 1e-2, levels leaf first at lr * 0.5^i without decay; a frozen decoder stays put."""
    tr, (coord, label, weight) = _trainer(levels, bias, frozen, seed=30 + levels)
    acc = {}
    for t in (1, 2):
        tr.forward_backward(coord, label, weight)
        inputs = (tr.flat_grad.clone(), tr.exp_avg.clone(), tr.exp_avg_sq.clone())
        before = _theta(tr)
        tr.optimizer_step()
        torch.cuda.synchronize()
        assert tr.step_count == t
        check_trainer_step(tr, before, t, inputs, acc, f"L={levels} bias={bias} frozen={frozen} step {t}")
        assert bool((tr.flat_grad == 0).all())
    report(f"optimizer_step groups L={levels} bias={bias} frozen={frozen}", acc)


def _pinned(batch):
    return tuple(x.cpu().pin_memory() for x in batch)


PATHS = ["train_step", "device_step", "capture_step", "step_from_host_graph", "step_from_host_eager", "submit_host_step"]


@pytest.mark.parametrize("path", PATHS)
def test_every_adam_path_applies_adam_to_its_own_gradients(path):
    """Three steps through one path from a fresh state: each is Adam step t = 1, 2, 3 with the oracle's groups, the host
    count follows, and the device counter too wherever device-step Adam ran."""
    tr, (coord, label, weight) = _trainer(seed=22)
    rec = _record_adam_inputs(tr)
    coord_h, label_h, _ = _pinned((coord, label, weight))
    graph = []

    def call():
        if path == "train_step":
            tr.train_step(coord, label)
        elif path == "device_step":
            tr.zero_grad(); tr.forward_backward(coord, label); tr.optimizer_step(device_step=True)
        elif path == "capture_step":
            if not graph:                 # capturing runs one real step first
                graph.append(tr.capture_step(coord, label, None, exchange=False, optimizer=True))
            else:
                graph[0].replay()
        elif path == "step_from_host_graph":
            tr.step_from_host(coord_h, label_h, optimizer=True)
        elif path == "step_from_host_eager":
            tr.step_from_host(coord_h, label_h, optimizer=True, use_graph=False)
        else:
            tr.submit_host_step(coord_h, label_h, optimizer=True).result()

    acc = {}
    for t in (1, 2, 3):
        before, n_rec = _theta(tr), len(rec)
        call()
        torch.cuda.synchronize()
        inputs = rec[n_rec] if len(rec) > n_rec else None
        check_trainer_step(tr, before, t, inputs, acc, f"{path} step {t}")
        assert tr.step_count == t
        if path not in ("train_step", "submit_host_step"):
            assert int(tr.adam_state[0]) == t
    report(f"path {path}", acc)


class _DevicePool:
    """A sample pool whose get_batch can be captured in a CUDA graph: batch i % nb of a fixed device tensor, i a device
    counter."""

    def __init__(self, batch, bs):
        nb = batch[0].shape[0] // bs
        self.data = [x[:nb * bs].reshape(nb, bs, *x.shape[1:]) for x in batch]
        self.nb = nb
        self.i = torch.zeros(1, dtype=torch.int64, device=batch[0].device)

    def get_batch(self, bs):
        k = self.i % self.nb
        self.i += 1
        return tuple(torch.index_select(x, 0, k).squeeze(0) for x in self.data)


@pytest.mark.parametrize("ekional", [False, True])
def test_graphed_loop_iterations_are_adam_steps(ekional):
    """_GraphedIteration.run() one iteration at a time, with an lr milestone at iteration 6 (the graph is re-captured at
    the new lr): every iteration is Adam step it + 1 at the current lr, counted on the host and on the device."""
    from shine_mapping_b200.batch_loop import _GraphedIteration, step_lr_decay
    tr, batch = _trainer(seed=23, n_batch=3 * 1024, ekional=ekional)
    rec = _record_adam_inputs(tr)
    loop = _GraphedIteration(tr, _DevicePool(batch, 1024), 1024)
    acc = {}
    for it in range(12):
        step_lr_decay(tr, tr.config.lr, it, [6], 0.5)
        before, n_rec = _theta(tr), len(rec)
        loop.run()
        torch.cuda.synchronize()
        inputs = rec[n_rec] if len(rec) > n_rec else None
        assert (inputs is not None) == (it in (0, 6))       # the iterations that captured ran eagerly
        check_trainer_step(tr, before, it + 1, inputs, acc, f"graphed loop iteration {it}")
        assert tr.step_count == int(tr.adam_state[0]) == it + 1
        assert loop.lr == tr.lr == tr.config.lr * (0.5 if it >= 6 else 1.0)
    report(f"graphed loop ekional={ekional}", acc)


# sequences of optimizer calls; each of the first three walks into one way the host and device counters used to drift
SEQUENCES = {
    "eager_step_from_host_after_host_steps": ["train_step", "train_step", "step_from_host_eager"],
    "cached_graph_after_host_steps": ["train_step", "step_from_host_graph", "train_step", "step_from_host_graph"],
    "capture_replays_then_host_step": ["capture_step", "replay", "replay", "train_step"],
    "all_paths": ["train_step", "train_step", "step_from_host_eager", "step_from_host_graph", "step_from_host_graph",
                  "train_step", "step_from_host_graph", "capture_step", "replay", "replay", "train_step", "device_step",
                  "submit_host_step", "replay"],
}
HOST_STEP_CALLS = ("train_step", "submit_host_step")


@pytest.mark.parametrize("sequence", list(SEQUENCES))
def test_step_count_is_one_across_paths(sequence):
    """Host-step and device-step Adam, eager and replayed, mixed.  After every call the host count is the number of steps
    taken since the state was created and the last update used that step number; after every call that ran
    device-step Adam the device counter agrees (host-step Adam leaves it alone; the next device-step call brings it in
    line first)."""
    tr, (coord, label, weight) = _trainer(seed=24)
    rec = _record_adam_inputs(tr)
    coord_h, label_h, _ = _pinned((coord, label, weight))
    graph = []
    calls = {
        "train_step": lambda: tr.train_step(coord, label),
        "device_step": lambda: (tr.zero_grad(), tr.forward_backward(coord, label), tr.optimizer_step(device_step=True)),
        "step_from_host_eager": lambda: tr.step_from_host(coord_h, label_h, optimizer=True, use_graph=False),
        "step_from_host_graph": lambda: tr.step_from_host(coord_h, label_h, optimizer=True),   # captured once, then cached
        "submit_host_step": lambda: tr.submit_host_step(coord_h, label_h, optimizer=True).result(),
        "capture_step": lambda: graph.append(tr.capture_step(coord, label, None, exchange=False, optimizer=True)),
        "replay": lambda: graph[0].replay(),
    }
    acc = {}
    for t, name in enumerate(SEQUENCES[sequence], start=1):
        before, n_rec = _theta(tr), len(rec)
        calls[name]()
        torch.cuda.synchronize()
        inputs = rec[n_rec] if len(rec) > n_rec else None
        check_trainer_step(tr, before, t, inputs, acc, f"call {t}: {name}")
        assert tr.step_count == t, (name, tr.step_count, t)
        if name not in HOST_STEP_CALLS:
            assert int(tr.adam_state[0]) == t, (name, int(tr.adam_state[0]), t)
    report(f"sequence {sequence}", acc)


def test_graphed_batch_loop_checkpoints_its_step_count(tmp_path):
    """The "step" that save_checkpoint writes after a graphed run_shine_mapping_batch (an lr milestone re-captures the
    iteration graph on the way) is the number of iterations run."""
    from shine_mapping_b200.batch_loop import run_shine_mapping_batch
    tr, batch = _trainer(seed=25)
    cfg = tr.config
    cfg.bs, cfg.iters, cfg.save_freq_iters, cfg.lr_decay_step = 1024, 10, 10, [4]
    run_shine_mapping_batch(cfg, tr.octree, tr.decoder, _DevicePool(batch, 1024), run_path=str(tmp_path),
                            use_cuda_graph=True)
    ck = torch.load(tmp_path / "model" / "model_iter_10.pth", weights_only=False)
    assert ck["optimizer"]["step"] == 10
