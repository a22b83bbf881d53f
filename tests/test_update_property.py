"""Property test (hypothesis): for random point clouds split into random frames, the vectorised FeatureOctree.update
must build exactly the oracle's (= the reference's) tables: same nodes, same corner rows, same numbering, same
insertion order — including clouds that touch the cube faces and repeated / overlapping frames."""
import numpy as np
import torch
from hypothesis import given, settings, strategies as st

from tests.parity_utils import make_config, orc


@settings(max_examples=25, deadline=None)
@given(seed=st.integers(0, 2 ** 31 - 1), n=st.integers(1, 400), frames=st.integers(1, 3),
       levels=st.integers(1, 4), world=st.sampled_from([6, 9, 12, 15]), spread=st.sampled_from([0.003, 0.05, 1.2]))
def test_update_matches_oracle_on_random_clouds(seed, n, frames, levels, world, spread):
    from shine_mapping_b200 import FeatureOctree
    levels = min(levels, world)
    rng = np.random.default_rng(seed)
    pts = (rng.standard_normal((n, 3)) * spread).astype(np.float32)      # spread 1.2 exercises the clamp at the faces
    pts[0] = [1.0, -1.0, 0.999999]
    cuts = sorted(rng.integers(0, n + 1, size=frames - 1).tolist())
    chunks = np.split(pts, cuts)
    if frames > 1:
        chunks.append(pts[: max(1, n // 3)])                              # a frame that revisits old space
    cfg = make_config(levels, world_level=world, device="cpu")
    a = FeatureOctree(cfg)
    b = orc.OracleOctree(world, levels)
    for ch in chunks:
        if len(ch) == 0:
            continue
        a.update(torch.from_numpy(ch))
        b.update(torch.from_numpy(ch))
    assert [tuple(p.shape) for p in a.hier_features] == [tuple(p.shape) for p in b.hier_features]
    for lvl in range(world + 1):
        assert a.nodes_lookup_tables[lvl] == b.nodes_lookup_tables[lvl]
        assert list(a.nodes_lookup_tables[lvl]) == list(b.nodes_lookup_tables[lvl])
        assert a.corners_lookup_tables[lvl] == b.corners_lookup_tables[lvl]
