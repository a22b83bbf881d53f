"""The oracle's Adam (`adam_reference`, `reference_param_groups`) against torch.optim.Adam in float64 (CPU only).
The GPU Adam tests (tests/test_gpu_adam.py) grade the kernel against this oracle, so it is tied to torch's algorithm
here: the reference loop steps a torch.optim.Adam built by setup_optimizer (utils/tools.py:57-83)."""
import torch

from oracle import shine_oracle as orc


def test_adam_reference_matches_torch_adam_float64():
    L, lr, wd, ratio = 3, 1e-2, 1e-2, 0.5
    g = torch.Generator().manual_seed(3)
    dec = [torch.randn(s, generator=g, dtype=torch.float64) * 0.3 for s in [(32, 8), (32,), (32, 32), (32,), (1, 32), (1,)]]
    tables = [torch.randn(r, 8, generator=g, dtype=torch.float64) * 0.05 for r in (5, 9, 17)]
    groups = orc.reference_param_groups(L, lr, wd, ratio)
    assert [gr["params"] for gr in groups] == ["decoder", 2, 1, 0]                     # leaf level first
    assert [gr["lr"] for gr in groups] == [lr, lr, lr * ratio, lr * ratio * ratio]
    assert [gr["weight_decay"] for gr in groups] == [wd, 0.0, 0.0, 0.0]

    def members(gr, ps):
        return ps[0] if gr["params"] == "decoder" else [ps[1][gr["params"]]]

    mine = ([p.clone() for p in dec], [t.clone() for t in tables])
    theirs = ([p.clone().requires_grad_(True) for p in dec], [t.clone().requires_grad_(True) for t in tables])
    opt = torch.optim.Adam([{"params": members(gr, theirs), "lr": gr["lr"], "weight_decay": gr["weight_decay"]}
                            for gr in groups], betas=(0.9, 0.99), eps=1e-15)
    state = {id(p): (torch.zeros_like(p), torch.zeros_like(p)) for p in mine[0] + mine[1]}
    for step in range(1, 11):
        grads = {}
        for p in mine[0] + mine[1]:
            gr = torch.randn(p.shape, generator=g, dtype=torch.float64) * 1e-3
            grads[id(p)] = gr
        grads[id(mine[1][0])].zero_()                    # a whole level without gradient (no decay: must not move)
        grads[id(mine[1][2])][3:7] = 0.0                 # rows without gradient in a level that has some
        grads[id(mine[0][5])].zero_()                    # decoder bias: decay alone moves it
        for p, q in zip(mine[0] + mine[1], theirs[0] + theirs[1]):
            q.grad = grads[id(p)].clone()
        opt.step()
        for gr in groups:
            ps = members(gr, mine)
            new_p, new_m, new_v = orc.adam_reference(ps, [grads[id(p)] for p in ps], [state[id(p)][0] for p in ps],
                                                     [state[id(p)][1] for p in ps], step, gr["lr"], gr["weight_decay"])
            for p, np_, nm, nv in zip(ps, new_p, new_m, new_v):
                p.copy_(np_)
                state[id(p)] = (nm, nv)
        for p, q in zip(mine[0] + mine[1], theirs[0] + theirs[1]):
            st = opt.state[q]
            assert int(st["step"]) == step
            # relative 1e-12 per element, measured against the tensor's largest magnitude where the element itself is
            # a cancellation residue (a moment of a gradient that changed sign): both sides round those differently
            for a, b in ((p, q.detach()), (state[id(p)][0], st["exp_avg"]), (state[id(p)][1], st["exp_avg_sq"])):
                assert bool(((a - b).abs() <= 1e-12 * torch.maximum(b.abs(), 1e-3 * b.abs().max())).all()), \
                    (step, float((a - b).abs().max()))
    assert torch.equal(mine[1][0], tables[0])                        # the level without gradient did not move
    assert not torch.equal(mine[0][5], dec[5])                       # decay alone moved the bias
