"""The decoder gradient of the zero tiles (every point misses every level: features 0) is the block's dL/dpred sum times
the gradient of Decoder.sdf(0), added in closed form in the training kernels' epilogue, and only in blocks that had zero
tiles.  Graded element by element against fp64 for batches made only of free-space samples (one tile, one block's worth,
several passes of the grid) and for a block whose every tile is a zero tile among blocks that have none, for both kernel
flavours and every point-wise loss.  test_gpu_rounds covers zero tiles mixed with real tiles inside blocks."""
import numpy as np
import pytest
import torch

from tests.parity_utils import make_case, sort_case_morton
from tests.test_gpu_rounds import TILE, _check, _far, _tiles_per_round, _with_tiles

pytestmark = pytest.mark.gpu
LOSSES = ("sdf_bce", "sdf_l1", "sdf_l2")


@pytest.fixture(scope="module", autouse=True)
def _lib(built_lib):
    assert torch.cuda.is_available()
    return built_lib


@pytest.mark.parametrize("loss_type", LOSSES)
@pytest.mark.parametrize("n_tiles", [1, 8, 3])
def test_free_space_batch_matches_fp64(n_tiles, loss_type):
    """Free-space samples only: one tile, one block's worth of tiles, and (3) three rounds of the grid plus a partial
    tile.  Every decoder gradient comes from the closed form."""
    case = make_case(n_points=2500, n_batch=64, feat_levels=3, seed=350 + n_tiles, weighted=True)
    rng = np.random.default_rng(350 + n_tiles)
    n = n_tiles * TILE if n_tiles != 3 else 3 * _tiles_per_round() * TILE + 5
    case["coord"] = _far(rng, n)
    case["label"] = rng.uniform(-0.2, 0.2, size=n).astype(np.float32)
    case["weight"] = rng.uniform(0.5, 1.5, size=n).astype(np.float32)
    _check(case, loss_type=loss_type)


@pytest.mark.parametrize("loss_type", LOSSES)
def test_block_of_zero_tiles_matches_fp64(loss_type):
    """Every tile of block 0 is a zero tile, every other block holds real tiles: block 0 adds a closed-form term and no
    tile gradient of its own.  Block 0 takes tiles 0-7 of every pass of the grid; a pass is `per_round` tiles in the
    grouped kernel (2 blocks/SM) and half of it in the per-point kernel (1 block/SM), so tiles 0-7, h-h+7 and p-p+7
    (h = per_round / 2, p = per_round) are zero tiles and the batch ends before tile 3h."""
    per_round = _tiles_per_round()
    h = per_round // 2
    pattern = [True] * (per_round + h - 16)
    for s in (0, h, per_round):
        pattern[s:s + 8] = [False] * 8
    case = sort_case_morton(make_case(n_points=2500, n_batch=sum(pattern) * TILE + 7, feat_levels=3, seed=360,
                                      weighted=True))
    _check(_with_tiles(case, pattern, 7, seed=36), loss_type=loss_type)
