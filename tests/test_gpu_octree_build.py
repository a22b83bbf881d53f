"""FeatureOctree.update on the GPU (csrc/shine_octree_build.cu, `FeatureOctree._update_cuda`) against the oracle's dict
loops (reference model/feature_octree.py:114-166), checked after EVERY frame:

* the node / corner dict views, including their iteration order (new nodes in ascending Morton order, new corner rows in
  lexicographic order), `node_ids`, table shapes and `get_octree_nodes`;
* the feature rows, bit for bit, against a replay of the reference's `randn` call shapes on the CUDA generator, and the
  continual-learning state (`importance_weight`, `features_last_frame`) of reference :143-146,157-160;
* the device tables themselves: node hash slots and corner slots decoded on the host (layout of `HashSlot` in
  csrc/shine_device.cuh), and `get_indices` against the oracle;
* tables rebuilt after a pickle round trip or a device move, CPU-path frames mixed with GPU frames, determinism, and
  scans of a 1024-azimuth LiDAR.
"""
import pickle

import numpy as np
import pytest
import torch

from tests import hash_layout as hl
from tests.parity_utils import make_config, orc

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


@pytest.fixture(scope="module", autouse=True)
def _lib(built_lib):
    assert torch.cuda.is_available()
    return built_lib


# ------------------------------------------------------------------------------------------------------------------
# host restatements of the device table layout (csrc/shine_device.cuh, csrc/shine_octree_build.cu)
# ------------------------------------------------------------------------------------------------------------------

def _lex_key(xyz: np.ndarray) -> np.ndarray:
    """lexicographic corner key of shine_octree_build.cu (16 bits per axis, int16 order)"""
    c = xyz.astype(np.int64) & 0xFFFF ^ 0x8000
    return (c[..., 0] << 32) | (c[..., 1] << 16) | c[..., 2]


def check_device_tables(octree):
    """Every level's node hash table and corner table hold exactly the level's nodes / rows, in the layout the query
    kernels probe."""
    octree._ensure_hash()
    spn = max(1, int(octree._HASH_SLOTS_PER_NODE))
    for lvl in range(octree.free_level_num, octree.max_level + 1):
        st = octree._levels[lvl]
        keys = st.node_keys.cpu().numpy()
        node_ids = st.node_ids.cpu().numpy()
        n, cap = keys.size, st.hash_capacity
        assert n < cap and n * spn <= 2 * cap, (lvl, n, cap, spn)           # one empty slot at least, load <= 2/spn
        hl.check_slots(hl.Slots.decode(st.hash.cpu().numpy()), keys, node_ids, f"level {lvl}")
        # corner table: {lexicographic key, row}, every row once.  Only update() on the GPU builds it (rebuilt there after
        # a move), so a level grown on the CPU path has none until the next GPU frame.
        if st.corner_hash is None:
            continue
        rows = st.corner_morton_by_row.numel()
        ccap = st.corner_hash_capacity
        assert 2 * rows <= ccap
        ct = st.corner_hash.cpu().numpy().reshape(ccap, 2)
        used = np.flatnonzero(ct[:, 0] != -1)
        assert used.size == rows
        want = _lex_key(orc.morton_to_points(st.corner_morton_by_row.cpu().numpy()).astype(np.int64))
        got_rows = (ct[used, 1] & 0xFFFFFFFF).astype(np.int64)
        assert np.array_equal(np.sort(got_rows), np.arange(rows))
        assert np.array_equal(ct[used, 0], want[got_rows]), f"level {lvl}: corner slot key != its row's corner"
        # linear probing from the home slot: no empty slot between a key's home and its slot
        home = hl.hash_key(ct[used, 0].astype(np.uint64)) & (ccap - 1)
        empties = np.concatenate(([0], np.cumsum(np.tile(ct[:, 0] == -1, 2))))
        dist = (used - home) & (ccap - 1)
        assert np.all(empties[home + dist] == empties[home]), f"level {lvl}: corner key unreachable from its home slot"


def assert_tables_match(octree, o, check_nodes=True):
    """Dict views (content and order), node_ids, shapes and get_octree_nodes equal the oracle's."""
    assert [tuple(p.shape) for p in octree.hier_features] == [tuple(t.shape) for t in o.hier_features]
    for lvl in range(octree.free_level_num, octree.max_level + 1):
        want_nodes, want_corners = o.nodes_lookup_tables[lvl], o.corners_lookup_tables[lvl]
        got_nodes, got_corners = octree.nodes_lookup_tables[lvl], octree.corners_lookup_tables[lvl]
        assert got_nodes == want_nodes, f"node table differs at level {lvl}"
        assert got_corners == want_corners, f"corner table differs at level {lvl}"
        assert list(got_corners) == list(want_corners), f"corner rows out of order at level {lvl}"
        assert list(got_nodes) == list(want_nodes), f"nodes out of the reference's order at level {lvl}"
        ids = octree._levels[lvl].node_ids.cpu().numpy()
        assert np.array_equal(ids, np.array(list(want_nodes.values()), dtype=np.int32).reshape(-1, 8))
        if check_nodes and want_nodes:
            pts = orc.morton_to_points(np.array(list(want_nodes), dtype=np.int64)).astype(np.int64)
            size = 2 ** (1 - lvl)
            assert np.array_equal(octree.get_octree_nodes(lvl), pts * size - 1.0 + 0.5 * size)


def check_indices(octree, o, rng, n_random=4000):
    """get_indices at every node centre of every featured level and at random points (hits and misses)."""
    probes = [octree.get_octree_nodes(l) for l in range(octree.free_level_num, octree.max_level + 1)]
    probes.append(rng.uniform(-1.1, 1.1, size=(n_random, 3)))
    coord = torch.from_numpy(np.concatenate(probes).astype(np.float32))
    for a, b in zip(octree.get_indices(coord.to(DEV)), o.get_indices(coord)):
        assert torch.equal(a.cpu(), b)


class FeatureReplay:
    """Expected hier_features: the reference's `feature_std * randn(n_fresh + 1, F)` per grown level and frame (shapes
    read off the oracle's tables), drawn on the CUDA generator in the same order; trash row zeroed (reference :139-156)."""

    def __init__(self, o, std, dim):
        """call right after torch.manual_seed, before the octree draws: the replay continues from this CUDA RNG state"""
        self.o, self.std, self.dim = o, std, dim
        self.tables = []
        self.rng_state = torch.cuda.get_rng_state(DEV)

    def sizes(self):
        return [(len(self.o.nodes_lookup_tables[l]), len(self.o.corners_lookup_tables[l]))
                for l in range(self.o.free_level_num, self.o.max_level + 1)]

    def replay(self, before, after):
        """-> the levels that grew this frame (coarse -> fine index) and their number of fresh rows"""
        grown = {}
        octree_state = torch.cuda.get_rng_state(DEV)
        torch.cuda.set_rng_state(self.rng_state, DEV)
        for k, ((n0, r0), (n1, r1)) in enumerate(zip(before, after)):
            if n1 == n0:
                continue
            fts = self.std * torch.randn(r1 - r0 + 1, self.dim, device=DEV)
            fts[-1] = 0.0
            if k == len(self.tables):
                self.tables.append(fts)
            else:
                self.tables[k] = torch.cat((self.tables[k][:-1], fts), 0)
            grown[k] = r1 - r0
        self.rng_state = torch.cuda.get_rng_state(DEV)
        torch.cuda.set_rng_state(octree_state, DEV)
        return grown


# ------------------------------------------------------------------------------------------------------------------
# frames
# ------------------------------------------------------------------------------------------------------------------


def _leaf_centre(v, world):
    return (-1.0 + (2.0 * np.asarray(v, dtype=np.float64) + 1.0) / 2 ** world).astype(np.float32)


def _gap_frames(o, rng):
    """Two frames: leaf voxels v - x and v + x, then v.  v's 8 corners all exist after the first (its neighbours along x
    own them) and v's ancestors are those of a neighbour: the second frame adds one node at the finest level only, and
    no corner (the reference's randn(1, F) call)."""
    W = o.max_level
    table = o.nodes_lookup_tables[W]
    for _ in range(1000):
        v = rng.integers(1, 2 ** W - 1, size=3)
        trio = [v + [dx, 0, 0] for dx in (-1, 0, 1)]
        if all(int(orc.points_to_morton(np.array(t))) not in table for t in trio):
            return [_leaf_centre([trio[0], trio[2]], W), _leaf_centre([trio[1]], W)]
    raise AssertionError("no free leaf voxel found")


def _boundary_points(rng, world, m):
    """m points exactly on voxel faces k / 2^l of random levels, and on the cube's faces +-1"""
    lv = rng.integers(1, world + 1, size=(m, 1))
    k = rng.integers(0, 2 ** lv + 1, size=(m, 3))
    p = (-1.0 + 2.0 * k / 2.0 ** lv).astype(np.float32)
    p[: m // 4, rng.integers(0, 3)] = rng.choice([-1.0, 1.0])
    if m:
        p[0] = [1.0, 1.0, 1.0]
    return p


def random_frames(seed, world, spread, n, frames, o):
    """Generator of the frames of one case; `o` is the oracle after the frames already yielded (the gap frames are
    placed in voxels still free)."""
    rng = np.random.default_rng(seed)
    cloud = (rng.standard_normal((n, 3)) * spread).astype(np.float32)            # spread 1.2 is clamped at the faces
    nb = min(n, max(1, n // 8))
    cloud[:nb] = _boundary_points(rng, world, nb)
    cloud = cloud[rng.permutation(n)]
    chunks = [c for c in np.array_split(cloud, frames) if len(c)]
    yield chunks[0]
    yield chunks[0][rng.integers(0, len(chunks[0]), size=1)]                      # one old point: no node at any level
    for ch in chunks[1:]:
        yield ch
    yield rng.uniform(-1, 1, size=(1, 3)).astype(np.float32)                     # a single point
    yield np.repeat(rng.uniform(-1, 1, size=(1, 3)).astype(np.float32), 1 + int(rng.integers(1, 3000)), 0)
    first, second = _gap_frames(o, rng)
    yield first
    yield second
    revisit = cloud[rng.integers(0, n, size=max(1, n // 3))]                      # old space, slightly moved
    yield revisit + (rng.standard_normal(revisit.shape) * 2.0 ** -world).astype(np.float32)
    yield cloud[: max(1, n // 2)].copy()                                          # old points only


def _random_cases():
    rng = np.random.default_rng(20261015)
    worlds, spreads = (6, 9, 12, 15), (0.003, 0.05, 1.2)
    cases = []
    for i in range(30):
        world = worlds[i % 4]
        levels = min(1 + (i * 3) % 8, world)
        n = int(np.exp(rng.uniform(0.0, np.log(20000))))
        n = {0: 1, 7: 20000, 13: 2}.get(i, n)
        cases.append(pytest.param(1000 + i, world, levels, spreads[i % 3], n, 1 + i % 5, i % 2 == 0,
                                  id=f"w{world}-L{levels}-s{spreads[i % 3]}-n{n}-f{1 + i % 5}{'-incr' if i % 2 == 0 else ''}"))
    return cases


# ------------------------------------------------------------------------------------------------------------------
# tests
# ------------------------------------------------------------------------------------------------------------------


@pytest.mark.timeout(600)
@pytest.mark.parametrize("seed,world,levels,spread,n,frames,incremental", _random_cases())
def test_update_matches_oracle_after_every_frame(seed, world, levels, spread, n, frames, incremental):
    from shine_mapping_b200 import FeatureOctree
    cfg = make_config(levels, world_level=world, device=DEV)
    torch.manual_seed(seed)
    octree = FeatureOctree(cfg)
    o = orc.OracleOctree(world, levels, cfg.feature_dim, cfg.feature_std, cfg.poly_int_on)
    replay = FeatureReplay(o, cfg.feature_std, cfg.feature_dim)
    rng = np.random.default_rng(seed + 1)
    seen = dict(no_growth=0, fine_only=0, no_corner=0)
    for f, pts in enumerate(random_frames(seed, world, spread, n, frames, o)):
        if f and incremental:       # what a frame of training leaves behind: moved features, importance weights
            for p, e in zip(octree.hier_features, replay.tables):
                p.data.add_(0.5)
                e.add_(0.5)
            for k, w in enumerate(octree.importance_weight):
                w.copy_(torch.arange(w.numel(), device=DEV, dtype=torch.float32).view_as(w) + 1.0 + k)
        prev_w = [w.clone() for w in octree.importance_weight]
        prev_last = [t.clone() for t in octree.features_last_frame]
        prev_params = list(octree.hier_features)
        before = replay.sizes()
        octree.update(torch.from_numpy(pts).to(DEV), incremental_on=incremental)
        o.update(torch.from_numpy(pts))
        after = replay.sizes()
        grown = replay.replay(before, after)
        assert_tables_match(octree, o)
        for k, (p, e) in enumerate(zip(octree.hier_features, replay.tables)):
            assert torch.equal(p.detach(), e), f"frame {f}: features of level index {k} differ from the randn replay"
        if not grown:
            seen["no_growth"] += f > 0
            assert all(a is b for a, b in zip(octree.hier_features, prev_params))
        elif f and min(grown) > 0:
            seen["fine_only"] += 1
        seen["no_corner"] += sum(1 for r in grown.values() if r == 0)
        if incremental:
            assert len(octree.importance_weight) == len(octree.features_last_frame) == levels
            for k in range(levels):
                w, last = octree.importance_weight[k], octree.features_last_frame[k]
                if k not in grown:
                    assert torch.equal(w, prev_w[k]) and torch.equal(last, prev_last[k])
                    continue
                assert w.shape == octree.hier_features[k].shape
                n_old = 0
                if k < len(prev_w):
                    n_old = prev_w[k].shape[0] - 1
                    assert torch.equal(w[:n_old], prev_w[k][:n_old]), "old importance weights must keep their values"
                assert not torch.any(w[n_old:]), "new rows and the trash row of importance_weight must be 0"
                assert torch.equal(last, octree.hier_features[k].detach())
        else:
            assert octree.importance_weight == [] and octree.features_last_frame == []
        check_device_tables(octree)
    check_indices(octree, o, rng)
    assert seen["no_growth"] >= 1 and seen["no_corner"] >= 1, seen
    if levels > 1:
        assert seen["fine_only"] >= 1, seen


def _table_growth_frames(world):
    """a small first frame, then large ones: the node and corner tables of every level outgrow their first capacity"""
    rng = np.random.default_rng(world)
    small = (rng.standard_normal((20, 3)) * 0.02).astype(np.float32)
    big = [(rng.standard_normal((15000, 3)) * s).astype(np.float32) for s in (0.05, 0.3)]
    return [small, *big]


@pytest.mark.parametrize("slots_per_node", [4, 1])
def test_device_tables_after_growth(slots_per_node, monkeypatch):
    from shine_mapping_b200 import FeatureOctree
    monkeypatch.setattr(FeatureOctree, "_HASH_SLOTS_PER_NODE", slots_per_node)
    cfg = make_config(4, world_level=12, device=DEV)
    octree = FeatureOctree(cfg)
    o = orc.OracleOctree(12, 4, cfg.feature_dim, cfg.feature_std, cfg.poly_int_on)
    rng = np.random.default_rng(slots_per_node)
    caps = []
    for pts in _table_growth_frames(12):
        octree.update(torch.from_numpy(pts).to(DEV))
        o.update(torch.from_numpy(pts))
        assert_tables_match(octree, o)
        check_device_tables(octree)
        check_indices(octree, o, rng)
        caps.append([(octree._levels[l].hash_capacity, octree._levels[l].corner_hash_capacity)
                     for l in range(octree.free_level_num, octree.max_level + 1)])
    for (n0, c0), (n1, c1) in zip(caps[0], caps[-1]):
        assert n1 > n0 and c1 > c0, caps
    if slots_per_node == 1:
        loads = [octree._levels[l].node_keys.numel() / octree._levels[l].hash_capacity
                 for l in range(octree.free_level_num, octree.max_level + 1)]
        assert max(loads) > 0.5, loads


def _moved(octree, how):
    if how == "pickle":
        return pickle.loads(pickle.dumps(octree))
    return octree.cpu().cuda()


@pytest.mark.parametrize("how", ["pickle", "cpu-cuda"])
def test_tables_rebuilt_after_a_move(how):
    """Frames 1..k on the GPU, a pickle round trip / a trip through host memory (the device tables are dropped), frames
    k+1..n on the GPU: _ensure_level_tables and corner_rehash_kernel rebuild the tables; the result equals an octree
    that never moved, features included, and the oracle."""
    from shine_mapping_b200 import FeatureOctree
    cfg = make_config(3, world_level=12, device=DEV)
    frames = _table_growth_frames(12)
    frames.append(frames[1][:5000] + np.float32(2.0 ** -12))
    torch.manual_seed(5)
    still = FeatureOctree(cfg)
    for pts in frames:
        still.update(torch.from_numpy(pts).to(DEV))
    torch.manual_seed(5)
    octree = FeatureOctree(cfg)
    o = orc.OracleOctree(12, 3, cfg.feature_dim, cfg.feature_std, cfg.poly_int_on)
    for f, pts in enumerate(frames):
        if f == 2:
            octree = _moved(octree, how)
            assert all(octree._levels[l].hash is None and octree._levels[l].corner_hash is None for l in range(13))
        octree.update(torch.from_numpy(pts).to(DEV))
        o.update(torch.from_numpy(pts))
        assert_tables_match(octree, o)
        check_device_tables(octree)
    for l in range(octree.free_level_num, 13):
        for name in ("node_keys", "node_ids", "corner_morton_by_row"):
            assert torch.equal(getattr(octree._levels[l], name), getattr(still._levels[l], name)), (l, name)
    for p, q in zip(octree.hier_features, still.hier_features):
        assert torch.equal(p, q)
    check_indices(octree, o, np.random.default_rng(0))


@pytest.mark.parametrize("first", ["cpu", "cuda"])
def test_cpu_and_gpu_frames_mixed(first):
    """Frames on one path, then on the other: the GPU path picks up tables the CPU path grew (device tables rebuilt from
    the authoritative arrays), the CPU path picks up tables the GPU path grew (_refresh_sorted)."""
    from shine_mapping_b200 import FeatureOctree
    cfg = make_config(3, world_level=12, device=first)
    frames = _table_growth_frames(12)
    frames.append(frames[2][:4000] * np.float32(1.01))
    octree = FeatureOctree(cfg)
    o = orc.OracleOctree(12, 3, cfg.feature_dim, cfg.feature_std, cfg.poly_int_on)
    for f, pts in enumerate(frames):
        if f == 2:
            octree = octree.cuda() if first == "cpu" else octree.cpu()
        dev = octree.device
        octree.update(torch.from_numpy(pts).to(dev))
        o.update(torch.from_numpy(pts))
        assert_tables_match(octree, o)
    if first == "cuda":             # and back: the GPU path picks up what the CPU path added
        octree = octree.cuda()
        pts = frames[1][:3000] * np.float32(0.9)
        octree.update(torch.from_numpy(pts).to(DEV))
        o.update(torch.from_numpy(pts))
        assert_tables_match(octree, o)
    assert all(octree._levels[l].corner_hash is not None for l in range(octree.free_level_num, 13))
    check_device_tables(octree)
    check_indices(octree, o, np.random.default_rng(1))


def test_two_builds_are_identical():
    """Concurrent inserts race for slots, but the tables a build produces do not depend on the race: node order, corner
    rows and node ids are the same in two builds from the same frames (slot placement may differ)."""
    from shine_mapping_b200 import FeatureOctree, synth
    cfg = make_config(8, world_level=12, device=DEV, pc_radius=40.0)
    scans = [c[w > 0] for c, _, w, _ in synth.generate_scans(cfg, 512, 3, 2.5, 3, DEV)]
    cloud = torch.from_numpy((np.random.default_rng(3).standard_normal((20000, 3)) * 0.05).astype(np.float32)).to(DEV)
    builds = []
    for _ in range(2):
        octree = FeatureOctree(cfg)
        for pts in (*scans, cloud):
            octree.update(pts)
        builds.append(octree)
    a, b = builds
    for l in range(a.free_level_num, a.max_level + 1):
        for name in ("node_keys", "node_ids", "corner_morton_by_row"):
            assert torch.equal(getattr(a._levels[l], name), getattr(b._levels[l], name)), (l, name)


@pytest.mark.timeout(1200)
@pytest.mark.parametrize("levels", [4, 8])
def test_scan_sequence_matches_oracle(levels):
    """Six frames of a 1024-azimuth, 64-beam scan along a street (the shape of the real workload), incremental."""
    from shine_mapping_b200 import FeatureOctree, synth
    cfg = make_config(levels, world_level=12, device=DEV, pc_radius=40.0)
    torch.manual_seed(11)
    octree = FeatureOctree(cfg)
    o = orc.OracleOctree(12, levels, cfg.feature_dim, cfg.feature_std, cfg.poly_int_on)
    replay = FeatureReplay(o, cfg.feature_std, cfg.feature_dim)
    for coord, _, weight, _ in synth.generate_scans(cfg, 1024, 6, 3.0, 21, DEV):
        surf = coord[weight > 0].contiguous()
        before = replay.sizes()
        octree.update(surf, incremental_on=True)
        o.update(surf.cpu())
        replay.replay(before, replay.sizes())
        assert_tables_match(octree, o, check_nodes=False)
        for p, e in zip(octree.hier_features, replay.tables):
            assert torch.equal(p.detach(), e)
        for w, p in zip(octree.importance_weight, octree.hier_features):
            assert w.shape == p.shape
    check_device_tables(octree)
    check_indices(octree, o, np.random.default_rng(2), n_random=20000)
