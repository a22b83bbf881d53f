"""CPU tests of the replay pool: the C struct, the oracle of the reference's window filter on hand-computed cases, the
pool without a window (no kernel), and the loop's refusal to mix replay with the regularisation mode."""
import ctypes as C

import pytest
import torch

from tests.parity_utils import make_config
from tests.replay_oracle import replay_pool_update


def test_sample_pool_struct_matches_header():
    from shine_mapping_b200 import _abi
    assert C.sizeof(_abi.ShineSamplePool) == 3 * 8 + 2 * 8
    assert [(n, getattr(_abi.ShineSamplePool, n).offset) for n in ("coord", "label", "weight", "size", "capacity")] == \
        [("coord", 0), ("label", 8), ("weight", 16), ("size", 24), ("capacity", 32)]


def _t(rows):
    return torch.tensor(rows, dtype=torch.float32)


def test_oracle_filters_before_it_appends_with_a_strict_window():
    """origin (1, 0, 0), radius 2: old samples at distances 0, 1.5, 2 (exactly: dropped, the comparison is strict), 3
    and NaN; the new frame's samples are appended whatever their distance."""
    pool_c = _t([[1, 0, 0], [1, 1.5, 0], [1, 0, 2], [4, 0, 0], [float("nan"), 0, 0]])
    pool_l, pool_w = _t([10, 11, 12, 13, 14]), _t([1, -1, 1, -1, 1])
    new_c, new_l, new_w = _t([[9, 9, 9], [1, 0, 0]]), _t([20, 21]), _t([-1, 1])
    c, l, w = replay_pool_update(pool_c, pool_l, pool_w, new_c, new_l, new_w, (1.0, 0.0, 0.0), 2.0)
    assert torch.equal(l, _t([10, 11, 20, 21]))
    assert torch.equal(w, _t([1, -1, -1, 1]))
    assert torch.equal(c, _t([[1, 0, 0], [1, 1.5, 0], [9, 9, 9], [1, 0, 0]]))
    # a radius just above 2 keeps the sample at exactly 2
    _, l2, _ = replay_pool_update(pool_c, pool_l, pool_w, new_c, new_l, new_w, (1.0, 0.0, 0.0), 2.0000002)
    assert torch.equal(l2, _t([10, 11, 12, 20, 21]))
    # no window (window_replay_on: False): every earlier sample stays, NaN included
    c3, l3, w3 = replay_pool_update(pool_c, pool_l, pool_w, new_c, new_l, new_w, (1.0, 0.0, 0.0), None)
    assert torch.equal(l3, _t([10, 11, 12, 13, 14, 20, 21])) and c3.shape == (7, 3) and torch.equal(w3[-2:], new_w)
    # the first frame meets an empty pool
    e = torch.empty(0, 3)
    c4, l4, w4 = replay_pool_update(e, torch.empty(0), torch.empty(0), new_c, new_l, new_w, (1.0, 0.0, 0.0), 2.0)
    assert torch.equal(c4, new_c) and torch.equal(l4, new_l) and torch.equal(w4, new_w)


def test_replay_pool_without_window_appends_on_the_host_side_and_grows():
    from shine_mapping_b200 import synth
    g = torch.Generator().manual_seed(0)
    pool = synth.ReplayPool("cpu", capacity=4)
    want_c, want_l, want_w = torch.empty(0, 3), torch.empty(0), torch.empty(0)
    for n in (3, 0, 5, 17):
        c, l, w = torch.rand(n, 3, generator=g), torch.rand(n, generator=g), torch.rand(n, generator=g)
        cap_before = pool.capacity
        pool.add_frame(c, l, w, (0.0, 0.0, 0.0), None)
        want_c, want_l, want_w = replay_pool_update(want_c, want_l, want_w, c, l, w, None, None)
        assert len(pool) == pool.size == want_l.shape[0] <= pool.capacity
        if want_l.shape[0] > cap_before:
            assert pool.capacity >= int(1.5 * cap_before)
        assert torch.equal(pool.coord_pool, want_c) and torch.equal(pool.sdf_label_pool, want_l)
        assert torch.equal(pool.weight_pool, want_w)
        assert pool.coord_pool.data_ptr() == pool._coord.data_ptr()       # views of the capacity buffers
    b = pool.get_batch(64, torch.Generator().manual_seed(1))
    idx = torch.randint(0, len(pool), (64,), generator=torch.Generator().manual_seed(1))
    assert torch.equal(b[1], want_l[idx])                                  # the reference's draw, in the order drawn
    with pytest.raises(NotImplementedError):
        pool.sort_morton()


def test_replay_pool_with_window_needs_the_gpu():
    from shine_mapping_b200 import _abi, synth
    pool = synth.ReplayPool("cpu")
    with pytest.raises(_abi.ShineB200Error, match="no CPU fallback"):
        pool.add_frame(torch.zeros(4, 3), torch.zeros(4), torch.ones(4), (0.0, 0.0, 0.0), 0.1)


def test_replay_pool_refuses_the_regularisation_mode():
    from shine_mapping_b200 import synth
    from shine_mapping_b200.incre_loop import run_shine_mapping_incremental
    cfg = make_config(2, device="cpu", continual_learning_reg=True)
    with pytest.raises(ValueError, match="continual_learning_reg"):
        run_shine_mapping_incremental(cfg, None, None, [], pool=synth.ReplayPool("cpu"))
