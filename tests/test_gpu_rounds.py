"""The training kernels with decoder gradients advance in block-wide rounds of one 16-point tile per warp (8 tiles per
block); the round's decoder-weight contraction is split across the block's warps.  These batches put partial last rounds,
rounds of zero tiles (every point misses every level), rounds that mix zero and real tiles, and the virtual backward tile
of the zero-tile shortcut through both kernel flavours (per-point and voxel-grouped scatter), graded against the oracle,
with sdf_bce and with sdf_l1 / sdf_l2, whose every sample carries a full-size dL/dpred into the zero-tile sums."""
import numpy as np
import pytest
import torch

from tests import test_gpu_sdf_diff as sdd
from tests.parity_utils import compare_step, make_case, run_cuda_step, run_oracle_step, sort_case_morton
from tests.test_gpu_replicas import grade_run

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


def _spans_rounds(case, k=2):
    """The batch covers at least k rounds of the grid at 2 blocks/SM (the last one may be partial)."""
    tiles, per_round = -(-case["coord"].shape[0] // TILE), _tiles_per_round()
    assert -(-tiles // per_round) >= k, f"{tiles} tiles are fewer than {k} rounds of {per_round}"
    print(f"N={case['coord'].shape[0]}: {tiles} tiles, {-(-tiles // per_round)} rounds of {per_round}")


def _check(case, frozen=False, loss_type="sdf_bce", zero_labels=None):
    """Both kernel flavours against the oracle, and element by element against the fp64 bounds (test_gpu_replicas.grade_run).  sdf_l1 / sdf_l2 go through test_gpu_sdf_diff's step and fp64 oracle (the
    L1 sign of the kernel's pred where it is within the pred tolerance of the label).  zero_labels (sdf_l1): indices of
    samples that get the pred the kernel returned for them as label, an exact zero difference inside the zero-tile sum."""
    if loss_type == "sdf_bce":
        want = run_oracle_step(case)
        if frozen:
            want = dict(want); want["dec_grads"] = {}
        ref = None
        for grouped in (False, True):
            got = run_cuda_step(case, DEV, morton_ordered=grouped, freeze_decoder=frozen)
            print(compare_step(got, want))
            ref = grade_run(case, got, "rounds", morton_ordered=grouped, ref=ref)
        return
    for grouped in (False, True):
        kw = dict(morton_ordered=grouped, freeze_decoder=frozen)
        c = case
        got = sdd._cuda_step(c, loss_type, **kw)
        if loss_type == "sdf_l1" and zero_labels is not None:
            c = dict(case, label=case["label"].copy())
            c["label"][zero_labels] = got["pred"][zero_labels]
            got = sdd._cuda_step(c, loss_type, **kw)
            assert np.array_equal(got["pred"][zero_labels], c["label"][zero_labels])
        want = sdd._drop_frozen(sdd._oracle(c, loss_type, got["pred"]), frozen)
        print(loss_type, "grouped" if grouped else "per-point", compare_step(got, want))
        grade_run(c, got, "rounds", loss_type, morton_ordered=grouped)


DIFF_LOSSES = ("sdf_l1", "sdf_l2")


@pytest.mark.parametrize("n_batch,loss_type", [
    pytest.param(5, "sdf_bce", id="5"),            # fewer than 16 points: one partial tile, seven idle warps
    pytest.param(100, "sdf_bce", id="100"),        # 7 tiles: fewer than one round of one block
    pytest.param(None, "sdf_bce", id="None"),      # one full round of the grid + 5 tiles, the last one partial
] + [pytest.param(None, lt, id=f"None-{lt}") for lt in DIFF_LOSSES])
def test_partial_rounds_match_oracle(n_batch, loss_type):
    n = n_batch or _tiles_per_round() * TILE + 4 * TILE + 3
    case = sort_case_morton(make_case(n_points=2500, n_batch=n, feat_levels=3, seed=300 + n % 97, weighted=True))
    n = case["coord"].shape[0]
    if n_batch is None:
        _spans_rounds(case)
        assert n % TILE != 0, "the last tile is partial"
    else:
        assert n < 8 * TILE, "fewer tiles than one block has warps"
    _check(case, loss_type=loss_type)


@pytest.mark.parametrize("frozen,loss_type", [pytest.param(f, "sdf_bce", id=str(f)) for f in (False, True)] +
                         [pytest.param(f, lt, id=f"{f}-{lt}") for lt in DIFF_LOSSES for f in (False, True)])
def test_zero_tile_rounds_match_oracle(frozen, loss_type):
    """Every tile of several rounds is a zero tile: the decoder gradients come from the virtual backward round alone."""
    case = make_case(n_points=2500, n_batch=64, feat_levels=2, seed=301)
    rng = np.random.default_rng(11)
    n = _tiles_per_round() * TILE + 7 * TILE + 9
    case["coord"] = _far(rng, n)
    case["label"] = rng.uniform(-0.2, 0.2, size=n).astype(np.float32)
    case["weight"] = rng.uniform(0.5, 1.5, size=n).astype(np.float32)
    _spans_rounds(case)
    _check(case, frozen, loss_type, zero_labels=np.arange(3, n, 97))


@pytest.mark.parametrize("frozen,bias,loss_type",
                         [pytest.param(f, b, "sdf_bce", id=f"{f}-{b}") for f, b in ((False, True), (True, True), (False, False))] +
                         [pytest.param(f, b, lt, id=f"{f}-{b}-{lt}") for lt in DIFF_LOSSES
                          for f, b in ((False, True), (True, True), (False, False))])
def test_mixed_rounds_match_oracle(frozen, bias, loss_type):
    """Rounds that mix zero and real tiles (every third tile, and a whole round of zero tiles in the middle), over more
    than one round of the grid, with a frozen decoder and with a decoder without biases."""
    per_round = _tiles_per_round()
    pattern = [i % 3 != 1 for i in range(per_round)] + [False] * per_round + [i % 2 == 0 for i in range(37)]
    n_real = sum(pattern) * TILE + 11
    case = sort_case_morton(make_case(n_points=2500, n_batch=n_real, feat_levels=4, seed=302, weighted=True,
                                      reduction="sum", bias=bias))
    case = _with_tiles(case, pattern, 11, seed=12)
    _spans_rounds(case, 3)
    far = [TILE * i + 5 for i, real in enumerate(pattern) if not real][::23]       # one sample in every 23rd zero tile
    _check(case, frozen, loss_type, zero_labels=np.asarray(far))
