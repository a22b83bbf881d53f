"""The spatial partition's plan and the bound of a partitioned step, on the host (tests/boundary_oracle.py).

* BoundaryPlan against its invariants for random per-rank key sets from 1 to 16 ranks (16: kMaxRanks of the peer-memory
  exchange, bit 15 of the int32 holder mask), with a rank that holds no key, a level without a shared key, a level whose
  keys are all shared, and keys listed in no particular order.
* The bound of a partitioned step: a correct fp32 emulation of a 3-rank step (each rank's fp32 partial over its own
  points, then the exchange's rank-order sum) lies inside it; the same step with one rank's partial of one boundary row
  dropped, or added twice, does not."""
import numpy as np
import pytest
import torch

from oracle import shine_oracle as orc
from tests.boundary_oracle import PartitionBound, check_plans, exchange_model, pack_host, shared_keys
from tests.error_bound import drop_kinks, subset
from tests.parity_utils import make_case, oracle_from_case

F = 8
DEC = 1380
LEVELS = 4          # level 0: mixed, 1: nothing shared, 2: everything shared, 3: mixed


def random_key_sets(world, seed):
    """Per rank, per level int64 keys.  Rank world // 2 holds nothing when world >= 3; every list is shuffled."""
    rng = np.random.default_rng(seed)
    empty = world // 2 if world >= 3 else None
    live = [r for r in range(world) if r != empty]
    out = [[[] for _ in range(LEVELS)] for _ in range(world)]
    for lvl in range(LEVELS):
        keys = rng.choice(1 << 45, size=int(rng.integers(60, 400)), replace=False)
        for k in keys.tolist():
            if lvl == 1 or len(live) == 1:
                hold = [live[int(rng.integers(len(live)))]]
            elif lvl == 2:
                hold = rng.choice(live, size=int(rng.integers(2, len(live) + 1)), replace=False).tolist()
            else:
                hold = rng.choice(live, size=int(rng.integers(1, min(len(live), 4) + 1)), replace=False).tolist()
            for r in hold:
                out[r][lvl].append(k)
    return [[torch.tensor(rng.permutation(np.array(ks, dtype=np.int64)), dtype=torch.int64) for ks in lv] for lv in out]


@pytest.mark.parametrize("world", [1, 2, 3, 8, 16])
def test_plan_invariants(world):
    from shine_mapping_b200.partition import BoundaryPlan
    keys = random_key_sets(world, 100 + world)
    plans = [BoundaryPlan(r, keys, F, DEC) for r in range(world)]
    check_plans(plans, keys, F, DEC)
    counts = [shared_keys(keys, lvl)[0].size for lvl in range(LEVELS)]
    assert counts[1] == 0, "level 1 was meant to share nothing"
    if world > 1:
        assert counts[2] == len(set().union(*[k[2].tolist() for k in keys])), "level 2 was meant to share every key"
        assert counts[0] > 0 and counts[3] > 0
    if world >= 3:
        assert all(k.numel() == 0 for k in keys[world // 2]) and all(r.numel() == 0 for r in plans[world // 2].rows)
    if world == 16:
        top = [int((h.numpy() >> 15 & 1).sum()) for h in plans[0].holders]
        assert sum(top) > 0, "no shared corner held by rank 15"
    assert not any(torch.equal(k, torch.sort(k).values) for lv in keys for k in lv if k.numel() > 2), "keys came sorted"
    print(f"[plan] world {world}: shared per level {plans[0].counts}, total floats {plans[0].total_floats}")


def test_plan_of_no_shared_corner_is_the_decoder_segment():
    from shine_mapping_b200.partition import BoundaryPlan
    keys = [[torch.tensor([5, 1, 9]), torch.zeros(0, dtype=torch.int64)], [[7, 3], [2]]]
    keys[1] = [torch.tensor(k) for k in keys[1]]
    plans = [BoundaryPlan(r, keys, 4, 12) for r in range(2)]
    check_plans(plans, keys, 4, 12)
    assert plans[0].total_floats == 12 and plans[0].counts == [0, 0]


def test_exchange_model_sums_the_holders_in_rank_order():
    """The model on a hand-made plan: a corner held by ranks 0 and 2 of 3 sums those two only, the decoder segment all
    three; values whose sum depends on the order (1e8, 1, -1e8) come out as rank order gives them."""
    from shine_mapping_b200.partition import BoundaryPlan
    keys = [[torch.tensor([10, 20])], [torch.tensor([20, 30])], [torch.tensor([10, 20, 30])]]
    plans = [BoundaryPlan(r, keys, 4, 4) for r in range(3)]
    check_plans(plans, keys, 4, 4)
    vals = [np.float32(1e8), np.float32(1.0), np.float32(-1e8)]
    bufs = []
    for r, p in enumerate(plans):
        table = np.full((keys[r][0].numel() + 1, 4), vals[r], dtype=np.float32)
        b = pack_host(p, [table])
        b[:4] = vals[r]
        bufs.append(b)
    got = exchange_model(bufs, plans[0])
    assert np.all(got[:4] == np.float32(0.0))                    # (0 + 1e8 + 1) - 1e8: the 1 is lost in rank order
    # slots in key order: 10 (ranks 0, 2), 20 (all), 30 (ranks 1, 2)
    assert np.all(got[4:8] == np.float32(0.0)) and np.all(got[8:12] == np.float32(0.0))
    assert np.all(got[12:16] == np.float32(1.0 - 1e8))
    assert not np.signbit(got[got == 0]).any(), "a sum came out as -0"


@pytest.fixture(scope="module")
def three_rank_emulation():
    """A global case (sum reduction, so every partial carries the global scale), split into 3 ranges by the coarse key
    as partition_pool splits a pool; per rank the fp32 oracle's partial table gradients over its own points."""
    from shine_mapping_b200.partition import balanced_key_bounds, coarse_keys, owner_of
    from tests.test_gpu_replicas import Ref
    case, _ = drop_kinks(make_case(n_points=1500, n_batch=3000, feat_levels=3, seed=9, reduction="sum"))
    c = case["cfg"]
    coord = torch.from_numpy(case["coord"])
    keys = coarse_keys(coord, c["tree_level_world"] - c["tree_level_feat"] + 1)
    owner = owner_of(keys, balanced_key_bounds(keys, 3)).numpy()
    ref = Ref(case)
    points = [np.flatnonzero(owner == r) for r in range(3)]
    partials = []
    for idx in points:
        sub = subset(case, idx)
        o, dec = oracle_from_case(sub)
        res = orc.train_step(o, dec, torch.from_numpy(sub["coord"]), torch.from_numpy(sub["label"]),
                             torch.from_numpy(sub["weight"]), c["sigma"], c["weighted"], "sum")
        partials.append([g.detach().numpy().astype(np.float32) for g in res["table_grads"]])
    # the rows a rank holds: the ones its points touch (the trash row is nobody's)
    rows = [[np.unique(ref._ix[kk][idx][ref._ix[kk][idx] >= 0]) for kk in range(len(ref.want))] for idx in points]
    return case, ref, points, partials, rows


def _exchange(partials, rows, kk, n_rows, skip=None, twice=None):
    """Rank-order fp32 sum of the holders' partials of table kk (skip / twice: (rank, row) dropped / added again)."""
    acc = np.zeros_like(partials[0][kk])
    for r, tables in enumerate(partials):
        part = tables[kk]
        held = np.zeros(n_rows, dtype=bool)
        held[rows[r][kk]] = True
        add = np.where(held[:, None], part, np.float32(0))
        if skip is not None and skip[0] == r:
            add[skip[1]] = 0
        acc = acc + add
        if twice is not None and twice[0] == r:
            acc[twice[1]] = acc[twice[1]] + part[twice[1]]
    return acc


def test_bound_passes_the_fp32_exchange_and_sees_one_lost_partial(three_rank_emulation):
    case, ref, points, partials, rows = three_rank_emulation
    L = len(ref.want)
    pb = PartitionBound(ref, points, rows, grouped=False)
    n_rows = [w.shape[0] for w in ref.want]
    summed = [_exchange(partials, rows, kk, n_rows[kk]) for kk in range(L)]

    def rank_tables(tables, r):
        return [np.concatenate((t[rows[r][kk]], np.zeros_like(t[:1]))) for kk, t in enumerate(tables)]

    for r in range(3):
        pb.grade_rank(r, rank_tables(summed, r), f"fp32 3-rank exchange, rank {r}")
    kk = L - 1                                                      # the leaf level
    boundary = np.flatnonzero(pb.h[kk] >= 2)
    assert boundary.size > 10, "the split leaves too few boundary rows"
    cand = [u for u in boundary if np.abs(partials[1][kk][u]).max() > 0 and u in set(rows[1][kk].tolist())]
    cand.sort(key=lambda u: float(np.abs(partials[1][kk][u]).max() / pb.bound(kk)[u].max()))
    u = cand[len(cand) // 2]                                        # a median-sized partial of rank 1
    print(f"[partition bounds] {boundary.size} boundary rows on the leaf level; row {u} has holders "
          f"{[r for r in range(3) if u in set(rows[r][kk].tolist())]}")
    for name, kw in (("lost", {"skip": (1, u)}), ("doubled", {"twice": (1, u)})):
        bad = list(summed)
        bad[kk] = _exchange(partials, rows, kk, n_rows[kk], **kw)
        with pytest.raises(AssertionError, match="outside the bound"):
            pb.grade_rank(1, rank_tables(bad, 1), f"rank 1's partial of one boundary row {name}")
