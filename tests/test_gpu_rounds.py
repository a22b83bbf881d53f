"""The training kernels with decoder gradients advance in block-wide rounds of one 16-point tile per warp (8 tiles per
block); the round's decoder-weight contraction is split across the block's warps.  These batches put partial last rounds,
rounds of zero tiles (every point misses every level), rounds that mix zero and real tiles, and the virtual backward tile
of the zero-tile shortcut through both kernel flavours (per-point and voxel-grouped scatter), graded against the oracle."""
import numpy as np
import pytest
import torch

from tests.parity_utils import compare_step, make_case, run_cuda_step, run_oracle_step, sort_case_morton

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
TILE = 16


@pytest.fixture(scope="module", autouse=True)
def _lib(built_lib):
    assert torch.cuda.is_available()
    return built_lib


def _tiles_per_round():
    """Tiles one round covers at 2 blocks/SM (the grouped kernel); the per-point kernel's rounds are the same or half."""
    return torch.cuda.get_device_properties(0).multi_processor_count * 2 * 8


def _far(rng, n):
    """Points outside every octree node of make_case's scene (they miss every level)."""
    return rng.uniform(0.6, 0.9, size=(n, 3)).astype(np.float32)


def _with_tiles(case, pattern, n_tail, seed):
    """Lay the (Morton-sorted) batch out tile by tile: pattern[i] True = 16 points of the batch, False = 16 far points;
    n_tail points of the batch follow as a partial last tile."""
    rng = np.random.default_rng(seed)
    coord, label, weight = [], [], []
    src = 0
    for real in pattern:
        if real:
            sl = slice(src, src + TILE); src += TILE
            coord.append(case["coord"][sl]); label.append(case["label"][sl]); weight.append(case["weight"][sl])
        else:
            coord.append(_far(rng, TILE)); label.append(rng.uniform(-0.2, 0.2, size=TILE).astype(np.float32))
            weight.append(rng.uniform(0.5, 1.5, size=TILE).astype(np.float32))
    sl = slice(src, src + n_tail)
    coord.append(case["coord"][sl]); label.append(case["label"][sl]); weight.append(case["weight"][sl])
    assert src + n_tail <= case["coord"].shape[0]
    out = dict(case)
    out["coord"] = np.concatenate(coord).astype(np.float32)
    out["label"] = np.concatenate(label).astype(np.float32)
    out["weight"] = np.concatenate(weight).astype(np.float32)
    return out


def _check(case, frozen=False):
    want = run_oracle_step(case)
    if frozen:
        want = dict(want); want["dec_grads"] = {}
    for grouped in (False, True):
        print(compare_step(run_cuda_step(case, DEV, morton_ordered=grouped, freeze_decoder=frozen), want))


@pytest.mark.parametrize("n_batch", [
    5,                 # fewer than 16 points: one partial tile, seven idle warps
    100,               # 7 tiles: fewer than one round of one block
    None,              # one full round of the grid + 5 tiles, the last one partial
])
def test_partial_rounds_match_oracle(n_batch):
    n = n_batch or _tiles_per_round() * TILE + 4 * TILE + 3
    case = sort_case_morton(make_case(n_points=2500, n_batch=n, feat_levels=3, seed=300 + n % 97, weighted=True))
    _check(case)


@pytest.mark.parametrize("frozen", [False, True])
def test_zero_tile_rounds_match_oracle(frozen):
    """Every tile of several rounds is a zero tile: the decoder gradients come from the virtual backward round alone."""
    case = make_case(n_points=2500, n_batch=64, feat_levels=2, seed=301)
    rng = np.random.default_rng(11)
    n = _tiles_per_round() * TILE + 7 * TILE + 9
    case["coord"] = _far(rng, n)
    case["label"] = rng.uniform(-0.2, 0.2, size=n).astype(np.float32)
    case["weight"] = rng.uniform(0.5, 1.5, size=n).astype(np.float32)
    _check(case, frozen)


@pytest.mark.parametrize("frozen,bias", [(False, True), (True, True), (False, False)])
def test_mixed_rounds_match_oracle(frozen, bias):
    """Rounds that mix zero and real tiles (every third tile, and a whole round of zero tiles in the middle), over more
    than one round of the grid, with a frozen decoder and with a decoder without biases."""
    per_round = _tiles_per_round()
    pattern = [i % 3 != 1 for i in range(per_round)] + [False] * per_round + [i % 2 == 0 for i in range(37)]
    n_real = sum(pattern) * TILE + 11
    case = sort_case_morton(make_case(n_points=2500, n_batch=n_real, feat_levels=4, seed=302, weighted=True,
                                      reduction="sum", bias=bias))
    _check(_with_tiles(case, pattern, 11, seed=12), frozen)
