"""Generate csrc/shine_mc_table.cuh: the marching-cubes edge and triangle tables of shine_mesh.cu.

    python tools/gen_mc_table.py            # rewrites shine_mapping_b200/csrc/shine_mc_table.cuh

The tables are derived here rather than typed in.  Corner c of a cube sits at (c & 1, (c >> 1) & 1, (c >> 2) & 1); a
corner is inside when its value is below the iso level.  On every face the crossing points are joined into segments so
that each inside corner is cut off on its own (the saddle rule of the ambiguous faces); the rule depends only on the
face's four signs, so the two cubes that share a face draw the same segments and the surface is closed.  The segments
are oriented with the inside on their left seen from outside the cube, chained into loops and each loop is fanned into
triangles, wound so that the normal (v1 - v0) x (v2 - v0) points from the inside to the outside.  The fan starts at a
vertex none of whose diagonals lies in a cube face, so that every edge of the surface is in exactly two triangles.
"""
from __future__ import annotations

import os

import numpy as np

CORNERS = [(c & 1, (c >> 1) & 1, (c >> 2) & 1) for c in range(8)]
# edge e: axis a = e // 4, from the corner with the other two bits (b0, b1) = ((e & 1), (e >> 1) & 1) to its +a neighbour
EDGES = []
for a in range(3):
    o = [ax for ax in range(3) if ax != a]
    for r in range(4):
        base = [0, 0, 0]
        base[o[0]], base[o[1]] = r & 1, (r >> 1) & 1
        c0 = base[0] + 2 * base[1] + 4 * base[2]
        EDGES.append((c0, c0 + (1 << a)))


def _edge_of(c0, c1):
    key = (min(c0, c1), max(c0, c1))
    return next(e for e, ed in enumerate(EDGES) if ed == key)


def _faces():
    """6 faces as corner lists counter-clockwise seen from outside the cube."""
    out = []
    for a in range(3):
        o = [(a + 1) % 3, (a + 2) % 3]            # right-handed (u, v, n = a)
        for side in (0, 1):
            ring = []
            for (u, v) in [(0, 0), (1, 0), (1, 1), (0, 1)]:
                p = [0, 0, 0]
                p[a], p[o[0]], p[o[1]] = side, u, v
                ring.append(p[0] + 2 * p[1] + 4 * p[2])
            out.append(ring if side == 1 else ring[::-1])   # the -a face is seen from -a: reverse
    return out


FACES = _faces()


def _on_one_face(e0: int, e1: int) -> bool:
    """Whether cube edges e0 and e1 lie on a common face of the cube."""
    a, b = EDGES[e0], EDGES[e1]
    return any(CORNERS[a[0]][ax] == CORNERS[a[1]][ax] == CORNERS[b[0]][ax] == CORNERS[b[1]][ax] for ax in range(3))


def _fan_start(loop):
    """The loop rotated to start at a vertex from which no diagonal of the fan lies in a cube face.  Such a diagonal
    joins two crossings of a face that the loop passes twice (a saddle face); when the cube on the other side does the
    same, the edge is shared by four triangles and the surface is not a manifold there.  Every loop of the table has
    such a start."""
    n = len(loop)
    for r in range(n):
        if not any(_on_one_face(loop[r], loop[(r + i) % n]) for i in range(2, n - 1)):
            return loop[r:] + loop[:r]
    raise AssertionError(f"no fan start without a diagonal in a face: {loop}")


def triangulate(case: int):
    inside = [(case >> c) & 1 for c in range(8)]
    nxt = {}
    for ring in FACES:
        # crossings walking the face boundary counter-clockwise: (edge, 'out' = inside -> outside)
        cross = []
        for i in range(4):
            c0, c1 = ring[i], ring[(i + 1) % 4]
            if inside[c0] != inside[c1]:
                cross.append((_edge_of(c0, c1), inside[c0] == 1, i))
        # segment from each in->out crossing to the out->in crossing that opened the same inside arc (the one before
        # it on the boundary): inside on the left, every inside corner cut off on its own
        for k, (e, out, _) in enumerate(cross):
            if out:
                prev = cross[k - 1]
                assert not prev[1]
                nxt[e] = prev[0]
    tris = []
    seen = set()
    for start in list(nxt):
        if start in seen:
            continue
        loop, e = [], start
        while e not in seen:
            seen.add(e)
            loop.append(e)
            e = nxt[e]
        loop = _fan_start(loop)
        for i in range(1, len(loop) - 1):
            tris.append((loop[0], loop[i], loop[i + 1]))
    return tris


def _orient_sign():
    """+1 when the fan winding already points inside -> outside (checked on the one-corner case), else -1."""
    mid = lambda e: np.mean([CORNERS[EDGES[e][0]], CORNERS[EDGES[e][1]]], axis=0)
    t = triangulate(1)[0]
    n = np.cross(mid(t[1]) - mid(t[0]), mid(t[2]) - mid(t[0]))
    return 1 if float(n @ np.array([1.0, 1.0, 1.0])) > 0 else -1


def tables():
    sign = _orient_sign()
    edge_mask, tri = [], []
    for case in range(256):
        inside = [(case >> c) & 1 for c in range(8)]
        edge_mask.append(sum(1 << e for e, (a, b) in enumerate(EDGES) if inside[a] != inside[b]))
        ts = triangulate(case)
        tri.append([(a, b, c) if sign > 0 else (a, c, b) for a, b, c in ts])
    return edge_mask, tri


HEADER = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "shine_mapping_b200", "csrc",
                      "shine_mc_table.cuh")


def render() -> str:
    """The text of shine_mc_table.cuh."""
    edge_mask, tri = tables()
    width = 3 * max(len(t) for t in tri) + 1
    lines = ["// shine_mc_table.cuh — generated by tools/gen_mc_table.py (see there for the rules); do not edit.",
             "#pragma once", "", f"#define SHINE_MC_TRI_WIDTH {width}", "",
             "// corner c at (c & 1, (c >> 1) & 1, (c >> 2) & 1); edge e = axis (e >> 2), from corner kMcEdgeCorner[e]",
             "__constant__ uint8_t kMcEdgeCorner[12] = {" + ", ".join(str(a) for a, _ in EDGES) + "};",
             "__constant__ uint16_t kMcEdgeMask[256] = {"]
    for i in range(0, 256, 16):
        lines.append("    " + ", ".join(f"0x{m:03x}" for m in edge_mask[i:i + 16]) + ",")
    lines.append("};")
    lines.append(f"// per case: edge ids of its triangles, three per triangle, -1 terminated")
    lines.append(f"__constant__ int8_t kMcTri[256][SHINE_MC_TRI_WIDTH] = {{")
    for ts in tri:
        flat = [e for t in ts for e in t]
        flat += [-1] * (width - len(flat))
        lines.append("    {" + ", ".join(str(v) for v in flat) + "},")
    lines.append("};")
    return "\n".join(lines) + "\n"


def main():
    with open(HEADER, "w") as f:
        f.write(render())
    print(HEADER, "max triangles per cube:", max(len(t) for t in tables()[1]))


if __name__ == "__main__":
    main()
