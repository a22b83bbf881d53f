"""Round shapes of the grouped kernel's decoder-weight contraction.  A round stages one tile per warp; the warps form two
groups (warps 0-3 with tiles 0-3, warps 4-7 with tiles 4-7) that synchronise separately; in each group every warp owns one
of the four blocks of dW2 over the group's tiles, and the two groups' partials are summed at the end.  These batches stage
only one group's tiles, a single tile at each warp position, and an odd number of tiles in the last round, graded against
the oracle for both kernel flavours."""
import pytest
import torch

from tests.parity_utils import make_case, sort_case_morton
from tests.test_gpu_rounds import TILE, _check, _tiles_per_round, _with_tiles

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module", autouse=True)
def _lib(built_lib):
    assert torch.cuda.is_available()
    return built_lib


def _sorted_case(n_batch, seed):
    return sort_case_morton(make_case(n_points=2500, n_batch=n_batch, feat_levels=3, seed=seed, weighted=True))


@pytest.mark.parametrize("first_half", [True, False])
def test_one_half_of_a_round_matches_oracle(first_half):
    """Block 0 stages tiles 0-3 only (a 4-tile batch), or tiles 4-7 only (tiles 0-3 are zero tiles)."""
    if first_half:
        _check(_sorted_case(3 * TILE + 5, seed=310))
    else:
        pattern = [False] * 4 + [True] * 4
        _check(_with_tiles(_sorted_case(4 * TILE, seed=311), pattern, 0, seed=13))


def test_single_tile_at_each_warp_position_matches_oracle():
    """Block w of the first round stages only the tile of warp w, for w = 0..7; every other tile is a zero tile."""
    pattern = [i % 9 == 0 for i in range(64)]
    _check(_with_tiles(_sorted_case(sum(pattern) * TILE + 6, seed=312), pattern, 6, seed=14))


@pytest.mark.parametrize("last_round_tiles", [3, 7])
def test_odd_last_round_matches_oracle(last_round_tiles):
    """One full round of the grid, then a last round of 3 tiles (first half only) or 7 (both halves, one short),
    the last tile partial."""
    n = _tiles_per_round() * TILE + (last_round_tiles - 1) * TILE + 7
    _check(_sorted_case(n, seed=313 + last_round_tiles))
