"""CPU side of the mesher: PLY round trip, the configurations it refuses, the loops' --run-path flag and the generated
marching-cubes tables (closed surfaces on every cube configuration)."""
import itertools
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def test_ply_round_trip(tmp_path):
    from shine_mapping_b200.mesher import read_ply, write_ply
    rng = np.random.default_rng(0)
    v = rng.normal(size=(50, 3)).astype(np.float32)
    n = rng.normal(size=(50, 3)).astype(np.float32)
    f = rng.integers(0, 50, size=(70, 3)).astype(np.int32)
    p = str(tmp_path / "m" / "a.ply")
    write_ply(p, torch.from_numpy(v), torch.from_numpy(f), torch.from_numpy(n))
    with open(p, "rb") as fh:
        assert fh.read(60).startswith(b"ply\nformat binary_little_endian 1.0\nelement vertex 50\n")
    rv, rf, rn = read_ply(p)
    assert np.array_equal(rv, v) and np.array_equal(rf, f) and np.array_equal(rn, n)


@pytest.mark.parametrize("key", ["mc_local", "semantic_on"])
def test_unsupported_meshing_is_refused(key):
    from shine_mapping_b200.config import SHINEConfig
    from shine_mapping_b200.mesher import Mesher
    with pytest.raises(NotImplementedError):
        Mesher(SHINEConfig(**{key: True}), None, None)


@pytest.mark.parametrize("module", ["batch_loop", "incre_loop"])
def test_loops_take_run_path(module):
    out = subprocess.run([sys.executable, "-m", f"shine_mapping_b200.{module}", "--help"], cwd=ROOT, capture_output=True,
                         text=True, check=True).stdout
    assert "--run-path DIR" in out


def test_generated_tables_close_every_face():
    """For every case the triangles' boundary edges lie on cube faces, and on each face the boundary segments are the
    ones the neighbouring cube (same four face signs) draws, in the opposite direction: the surface has no cracks."""
    sys.path.insert(0, os.path.join(ROOT, "tools"))
    import gen_mc_table as gm
    _, tri = gm.tables()
    corner = np.array(gm.CORNERS)

    def face_segments(case):
        segs = {}
        ts = tri[case]
        cnt = {}
        for t in ts:
            for a, b in ((t[0], t[1]), (t[1], t[2]), (t[2], t[0])):
                cnt[(a, b)] = cnt.get((a, b), 0) + 1
        for (a, b) in cnt:
            if (b, a) not in cnt:                                   # boundary edge of the patch
                mids = (corner[list(gm.EDGES[a])].mean(0), corner[list(gm.EDGES[b])].mean(0))
                axes = [ax for ax in range(3) for side in (0.0, 1.0) if mids[0][ax] == side and mids[1][ax] == side]
                assert len(axes) == 1, (case, a, b)
                ax = axes[0]
                segs.setdefault((ax, float(mids[0][ax])), []).append((tuple(mids[0]), tuple(mids[1])))
        return segs

    all_segs = [face_segments(c) for c in range(256)]
    for case, other in itertools.product(range(0, 256, 7), range(0, 256, 5)):
        for ax in range(3):
            # `other` is the +ax neighbour: its low face must carry case's high-face signs
            hi_corners = [c for c in range(8) if corner[c][ax] == 1]
            lo_corners = [c for c in range(8) if corner[c][ax] == 0]
            if any(((case >> h) & 1) != ((other >> l) & 1) for h, l in zip(hi_corners, lo_corners)):
                continue
            mine = sorted(all_segs[case].get((ax, 1.0), []))
            theirs = sorted((tuple(np.add(b, np.eye(3)[ax])), tuple(np.add(a, np.eye(3)[ax])))
                            for a, b in all_segs[other].get((ax, 0.0), []))
            assert mine == theirs, (case, other, ax)


def test_generated_tables_keep_inner_edges_off_the_faces():
    """An edge inside a cube's patch (in two of its triangles) never joins two crossings of one cube face.  Such an edge
    lies in the face; when the cube on the other side of a saddle face draws it too, four triangles share it and the
    surface is not a manifold.  Every case of the table is checked, and the committed header is the generator's output."""
    sys.path.insert(0, os.path.join(ROOT, "tools"))
    import gen_mc_table as gm
    _, tri = gm.tables()
    for case in range(256):
        count = {}
        for t in tri[case]:
            for a, b in ((t[0], t[1]), (t[1], t[2]), (t[2], t[0])):
                count[(min(a, b), max(a, b))] = count.get((min(a, b), max(a, b)), 0) + 1
        assert set(count.values()) <= {1, 2}, case
        inner = [e for e, c in count.items() if c == 2]
        assert not [e for e in inner if gm._on_one_face(*e)], case
    with open(gm.HEADER) as fh:
        assert fh.read() == gm.render()
