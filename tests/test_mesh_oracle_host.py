"""The mesh oracles of tests/mesh_oracle.py checked on their own, without a GPU: the cluster partition against a plain
breadth-first search, the normals on solids whose normals are known, the volume bounds on a sampled sphere, and the
canonical key's independence of numbering and triangle order."""
import itertools
import math
import os
import sys
from collections import deque

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from tests import mesh_oracle as mo  # noqa: E402


def _bfs_clusters(faces):
    """Edge-connected triangle clusters by breadth-first search over an edge -> triangles map."""
    by_edge = {}
    for t, f in enumerate(faces.tolist()):
        for a, b in ((f[0], f[1]), (f[1], f[2]), (f[2], f[0])):
            by_edge.setdefault((min(a, b), max(a, b)), []).append(t)
    label = [-1] * len(faces)
    sizes = []
    for s in range(len(faces)):
        if label[s] >= 0:
            continue
        label[s], q, n = len(sizes), deque([s]), 0
        while q:
            t = q.popleft()
            n += 1
            f = faces[t].tolist()
            for a, b in ((f[0], f[1]), (f[1], f[2]), (f[2], f[0])):
                for u in by_edge[(min(a, b), max(a, b))]:
                    if label[u] < 0:
                        label[u] = len(sizes)
                        q.append(u)
        sizes.append(n)
    return np.array(label), np.array(sizes)


@pytest.mark.parametrize("seed", range(6))
def test_clusters_match_breadth_first_search(seed):
    rng = np.random.default_rng(seed)
    nv = int(rng.integers(5, 60))
    nt = int(rng.integers(1, 150))
    faces = np.stack([rng.choice(nv, size=3, replace=False) for _ in range(nt)]).astype(np.int32)
    label, sizes = mo.triangle_clusters(faces, nv)
    want_label, want_sizes = _bfs_clusters(faces)
    assert np.array_equal(label, want_label) and np.array_equal(sizes, want_sizes)
    assert sizes.sum() == nt


def test_clusters_are_joined_by_edges_not_vertices():
    # two fans meeting at vertex 0 only, and an edge (10, 11) shared by four triangles
    faces = np.array([[0, 1, 2], [0, 2, 3], [0, 4, 5], [0, 5, 6], [10, 11, 12], [11, 10, 13], [10, 11, 14], [10, 11, 15]])
    label, sizes = mo.triangle_clusters(faces, 16)
    assert label.tolist() == [0, 0, 1, 1, 2, 2, 2, 2] and sizes.tolist() == [2, 2, 4]
    assert mo.triangle_clusters(np.zeros((0, 3), dtype=np.int32), 3)[1].shape == (0,)


def _angle(a, b):
    return np.arctan2(np.linalg.norm(np.cross(a, b), axis=1), (a * b).sum(1))


def test_normals_of_a_cube_and_a_tetrahedron():
    corner = np.array(list(itertools.product((0.0, 1.0), repeat=3)))       # index = 4 x + 2 y + z
    quads = [(0, 1, 3, 2), (4, 6, 7, 5), (0, 4, 5, 1), (2, 3, 7, 6), (0, 2, 6, 4), (1, 5, 7, 3)]   # outward
    faces = np.array([t for a, b, c, d in quads for t in ((a, b, c), (a, c, d))])
    n = mo.vertex_normals(corner + 5.0, faces)
    # every corner has two unit normals from two of its faces and one from the third: not the diagonal, but inside
    # the octant of the outward diagonal, with |n| = 1
    assert np.allclose(np.linalg.norm(n, axis=1), 1.0, atol=1e-15)
    assert (np.sign(n) == np.where(corner > 0, 1.0, -1.0)).all()
    # a regular tetrahedron: each vertex normal is the direction from the centre, exactly
    tet = np.array([[1.0, 1.0, 1.0], [1.0, -1.0, -1.0], [-1.0, 1.0, -1.0], [-1.0, -1.0, 1.0]])
    tf = np.array([[0, 1, 2], [0, 3, 1], [0, 2, 3], [1, 3, 2]])
    got = mo.vertex_normals(tet + 100.0, tf)
    assert _angle(got, tet / math.sqrt(3.0)).max() < 1e-12
    # degenerate triangles add nothing; a vertex with only those, or none, gets the zero vector
    v = np.concatenate([tet, [[0.0, 0.0, 0.0], [3.0, 3.0, 3.0]]])
    f = np.concatenate([tf, [[0, 4, 0], [4, 4, 4]]])
    got = mo.vertex_normals(v, f)
    assert _angle(got[:4], tet / math.sqrt(3.0)).max() < 1e-12 and (got[4:] == 0).all()
    # opposite triangles cancel: the sum is zero
    assert (mo.vertex_normals(tet[:3], np.array([[0, 1, 2], [0, 2, 1]])) == 0).all()


def test_volume_bounds_bracket_a_sampled_sphere():
    hi, c, r = (24, 26, 28), np.array([11.5, 12.25, 13.0]), 8.3
    G = np.stack(np.meshgrid(*[np.arange(h) for h in hi], indexing="ij"), -1).astype(np.float64)
    sdf = np.linalg.norm(G - c, axis=-1) - r
    lo, up = mo.enclosed_volume_bounds(sdf, np.ones(hi, dtype=bool), hi)
    vol = 4.0 / 3.0 * math.pi * r ** 3
    assert 0 < lo < vol < up
    # masking out the cubes of the upper half: the bounds bracket the half sphere that stays
    mask = np.ones(hi, dtype=bool)
    mask[:, :, 13:] = False
    lo2, up2 = mo.enclosed_volume_bounds(sdf, mask, hi)
    assert lo2 < lo and up2 < up and lo2 < vol / 2 < up2


def test_canonical_mesh_ignores_numbering_and_order_but_not_winding():
    rng = np.random.default_rng(3)
    v = rng.normal(size=(40, 3)).astype(np.float32)
    f = np.stack([rng.choice(40, size=3, replace=False) for _ in range(70)]).astype(np.int32)
    perm = rng.permutation(40)
    inv = np.argsort(perm)                                    # new vertex i is old vertex perm[i]
    f2 = inv[f][rng.permutation(70)]
    f2 = np.roll(f2, 1, axis=1)                               # same winding, another start
    assert mo.canonical_mesh(v, f) == mo.canonical_mesh(v[perm], f2)
    flipped = f.copy()
    flipped[0] = flipped[0][::-1]
    assert mo.canonical_mesh(v, f) != mo.canonical_mesh(v, flipped)
    moved = v.copy()
    moved[f[0, 0], 0] = np.nextafter(moved[f[0, 0], 0], np.float32(np.inf))
    assert mo.canonical_mesh(v, f)[0] != mo.canonical_mesh(moved, f)[0]
