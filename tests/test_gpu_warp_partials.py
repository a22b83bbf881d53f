"""The grouped training kernel contracts each warp's own tile into that warp's decoder-gradient partial (dW2 in shared
memory, the rest in registers); the block sums its eight partials at the end.  These batches leave warps without a tile,
give the warps of the grid unequal tile counts, put zero tiles (every point misses every level) alone and interleaved
within a block, and kill a layer-2 unit, graded against the oracle for both kernel flavours."""
import numpy as np
import pytest
import torch

from tests.parity_utils import compare_step, make_case, run_cuda_step, run_oracle_step, sort_case_morton
from tests.test_gpu_rounds import TILE, _check, _far, _tiles_per_round, _with_tiles

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


@pytest.fixture(scope="module", autouse=True)
def _lib(built_lib):
    assert torch.cuda.is_available()
    return built_lib


def _sorted_case(n_batch, seed, **kw):
    return sort_case_morton(make_case(n_points=2500, n_batch=n_batch, feat_levels=3, seed=seed, weighted=True, **kw))


@pytest.mark.parametrize("n_batch", [1, 15, 17, 16 * 8 + 1])
def test_warps_without_a_tile_match_oracle(n_batch):
    """One partial tile, one full and one partial tile, and a ninth tile of one point: most warps stage nothing."""
    _check(_sorted_case(n_batch, seed=320 + n_batch))


@pytest.mark.parametrize("extra_tiles", [-1, 1])
def test_unequal_tile_counts_match_oracle(extra_tiles):
    """Two passes of the grid's warps, one tile short or one tile over (the last tile partial): the warps of the grid do
    not all contract the same number of tiles."""
    n = (2 * _tiles_per_round() + extra_tiles) * TILE - 5
    _check(_sorted_case(n, seed=330 + extra_tiles))


@pytest.mark.parametrize("frozen", [False, True])
def test_zero_tiles_only_match_oracle(frozen):
    """Every tile is a zero tile: only warp 0's virtual backward tile carries decoder gradients."""
    case = make_case(n_points=2500, n_batch=64, feat_levels=3, seed=340)
    rng = np.random.default_rng(21)
    n = 3 * _tiles_per_round() * TILE + 3
    case["coord"] = _far(rng, n)
    case["label"] = rng.uniform(-0.2, 0.2, size=n).astype(np.float32)
    case["weight"] = rng.uniform(0.5, 1.5, size=n).astype(np.float32)
    _check(case, frozen)


@pytest.mark.parametrize("frozen", [False, True])
def test_zero_tiles_interleaved_within_a_block_match_oracle(frozen):
    """Blocks whose eight warps hold real and zero tiles in an irregular pattern, over more than one pass of the grid."""
    per_block = [True, False, True, True, False, False, True, False]
    pattern = per_block * (_tiles_per_round() // 8 + 5)
    case = _sorted_case(sum(pattern) * TILE + 9, seed=341)
    _check(_with_tiles(case, pattern, 9, seed=22), frozen)


def test_dead_layer2_unit_has_zero_gradients():
    """Layer-2 unit u has a zero W2 row and a zero bias, so h2[:, u] = 0 for every point and ReLU blocks its gradient:
    its dW2 row and db2 entry must be exactly 0 (the grouped kernel rebuilds dh2 from dL/dpred and the staged ReLU mask)."""
    u = 13
    case = _sorted_case(2 * _tiles_per_round() * TILE + 7, seed=342)
    case["dec"] = dict(case["dec"])
    w2 = np.array(case["dec"]["layers.1.weight"], dtype=np.float32, copy=True); w2[u, :] = 0.0
    b2 = np.array(case["dec"]["layers.1.bias"], dtype=np.float32, copy=True); b2[u] = 0.0
    case["dec"]["layers.1.weight"], case["dec"]["layers.1.bias"] = w2, b2
    assert float(np.abs(np.asarray(case["dec"]["lout.weight"])).reshape(-1)[u]) > 0.0
    want = run_oracle_step(case)
    for grouped in (False, True):
        got = run_cuda_step(case, DEV, morton_ordered=grouped)
        print(compare_step(got, want))
        assert np.all(got["dec_grads"]["layers.1.weight"][u] == 0.0)
        assert got["dec_grads"]["layers.1.bias"][u] == 0.0
        assert np.any(got["dec_grads"]["layers.1.weight"] != 0.0)
