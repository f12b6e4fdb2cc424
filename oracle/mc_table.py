"""Marching-cubes case table, derived from the corner signs of a cube (no copied table).

    python -m oracle.mc_table            # rewrites neuralsim_b200/csrc/mc_table.cuh

Numbering.  Corner b in [0, 8) sits at offset (b & 1, b >> 1 & 1, b >> 2 & 1) along the lattice axes (i, j, k) = (x, y, z); the case index
of a cell has bit b set when corner b is inside (sdf < level).  Edge e in [0, 12) runs along axis a = e // 4 from the corner at
owner offset EDGE_OWNER[e] to the one a unit step further; the other two axes (u < v) carry offsets (e & 1, e >> 1 & 1).  In the lattice,
edge e of the cell at (i, j, k) is the edge of axis a owned by the lattice point (i, j, k) + EDGE_OWNER[e].

Per case: one vertex on every edge whose two corners differ in sign; on each of the 6 faces the crossing edges are paired into segments
(4 crossings = an ambiguous face: every inside corner of the face is cut off by its own segment, i.e. the inside corners are separated --
a rule that sees only the face's four signs, so both cells sharing the face agree and the mesh has no cracks); each segment is directed
with the face's inside corners on its left seen from outside the cube; the segments chain into closed loops; each loop is fan-triangulated
in reverse order, so that a triangle's right-hand normal points out of the inside region, along +grad sdf.
"""
from __future__ import annotations

import os

import numpy as np

CORNER = np.array([[b & 1, b >> 1 & 1, b >> 2 & 1] for b in range(8)], dtype=np.int64)


def _other(a):
    return [u for u in range(3) if u != a]


def _edge_owner(e):
    a = e // 4
    u, v = _other(a)
    off = [0, 0, 0]
    off[u], off[v] = e & 1, e >> 1 & 1
    return tuple(off)


EDGE_AXIS = [e // 4 for e in range(12)]
EDGE_OWNER = [_edge_owner(e) for e in range(12)]


def _corner_of(off):
    return off[0] + 2 * off[1] + 4 * off[2]


EDGE_CORNERS = []
for _e in range(12):
    _o = list(EDGE_OWNER[_e])
    _p = list(_o)
    _p[EDGE_AXIS[_e]] += 1
    EDGE_CORNERS.append((_corner_of(_o), _corner_of(_p)))
EDGE_MID = np.array([(CORNER[c0] + CORNER[c1]) / 2.0 for c0, c1 in EDGE_CORNERS])


def face_corners(a, s):
    """the 4 corners of face (axis a, side s) in cyclic order around the face"""
    u, v = _other(a)
    out = []
    for du, dv in ((0, 0), (1, 0), (1, 1), (0, 1)):
        off = [0, 0, 0]
        off[a], off[u], off[v] = s, du, dv
        out.append(_corner_of(off))
    return out


def _edge_between(c0, c1):
    for e, (p, q) in enumerate(EDGE_CORNERS):
        if {p, q} == {c0, c1}:
            return e
    raise AssertionError((c0, c1))


def face_segments(case, a, s):
    """undirected segments (pairs of edge ids) the face rule puts on face (a, s) for `case`"""
    cs = face_corners(a, s)
    ins = [bool(case >> c & 1) for c in cs]
    ring = [_edge_between(cs[q], cs[(q + 1) % 4]) for q in range(4)]           # ring[q] joins corners q and q + 1
    cross = [q for q in range(4) if ins[q] != ins[(q + 1) % 4]]
    if len(cross) == 0:
        return []
    if len(cross) == 2:
        return [(ring[cross[0]], ring[cross[1]])]
    # ambiguous face (diagonal corners equal): each inside corner q is cut off by the segment joining its two edges
    return [(ring[(q - 1) % 4], ring[q]) for q in range(4) if ins[q]]


def _directed(case, a, s, seg):
    """orient seg so that the inside corners of the face are on its left, seen from outside the cube"""
    n = np.zeros(3)
    n[a] = 2 * s - 1
    p1, p2 = EDGE_MID[seg[0]], EDGE_MID[seg[1]]
    e0, e1 = seg
    # a corner on the inside side of the segment: one shared by both edges if any (a cut-off corner), else any inside corner of the face
    shared = set(EDGE_CORNERS[e0]) & set(EDGE_CORNERS[e1])
    cands = [c for c in shared if case >> c & 1] or [c for c in face_corners(a, s) if case >> c & 1]
    ci = CORNER[cands[0]].astype(float)
    left = float(np.dot(n, np.cross(p2 - p1, ci - p1)))
    assert left != 0.0
    return (e0, e1) if left > 0 else (e1, e0)


def case_loops(case):
    """closed loops of edge ids (each in the direction of the face segments) for one case"""
    nxt = {}
    for a in range(3):
        for s in range(2):
            for seg in face_segments(case, a, s):
                p, q = _directed(case, a, s, seg)
                assert p not in nxt, (case, p)
                nxt[p] = q
    loops, seen = [], set()
    for start in sorted(nxt):
        if start in seen:
            continue
        loop, e = [], start
        while e not in seen:
            seen.add(e)
            loop.append(e)
            e = nxt[e]
        assert e == start, (case, loop)
        loops.append(loop)
    return loops


def _on_one_face(e0, e1):
    pts = CORNER[list(set(EDGE_CORNERS[e0]) | set(EDGE_CORNERS[e1]))]
    return any((pts[:, a] == s).all() for a in range(3) for s in range(2))


def case_triangles(case):
    """[(e0, e1, e2), ...]: each loop reversed and fan-triangulated from its first vertex whose fan diagonals do not lie on a cube face
    (a diagonal on a face would be a mesh edge the neighbouring cell does not have)"""
    tris = []
    for loop in case_loops(case):
        r = loop[::-1]
        n = len(r)
        rot = next(q for q in range(n) if not any(_on_one_face(r[q], r[(q + k) % n]) for k in range(2, n - 1)))
        r = r[rot:] + r[:rot]
        for k in range(1, n - 1):
            tris.append((r[0], r[k], r[k + 1]))
    return tris


def crossing_edges(case):
    return [e for e, (c0, c1) in enumerate(EDGE_CORNERS) if (case >> c0 & 1) != (case >> c1 & 1)]


MAX_TRIS = 5       # asserted below: the largest triangle count of any case (the table is sized from it)


def build_table():
    tris = [case_triangles(c) for c in range(256)]
    most = max(len(t) for t in tris)
    assert most == MAX_TRIS, most
    count = np.array([len(t) for t in tris], dtype=np.int64)
    edges = -np.ones((256, MAX_TRIS * 3), dtype=np.int64)
    for c, t in enumerate(tris):
        for q, tri in enumerate(t):
            edges[c, 3 * q:3 * q + 3] = tri
    return count, edges


def render_cuh():
    count, edges = build_table()
    lines = ["// Marching-cubes case table.  GENERATED by oracle/mc_table.py (`python -m oracle.mc_table`): do not edit by hand.",
             "// Corner b at offset (b & 1, b >> 1 & 1, b >> 2 & 1); case bit b = corner b inside (sdf < level).  Edge e runs along axis",
             "// e / 4 from the lattice point (cell origin + kMcEdgeOwner[e]).  Per case: kMcTriCount triangles, kMcTriEdges = 3 edge ids each,",
             "// wound so that the right-hand normal points along +grad sdf.  Ambiguous faces separate their inside corners.",
             "#pragma once",
             "#include <stdint.h>",
             "",
             "namespace nsb {",
             f"constexpr int kMcMaxTris = {MAX_TRIS};",
             "__device__ const uint8_t kMcEdgeOwner[12][3] = {" + ", ".join("{%d, %d, %d}" % o for o in EDGE_OWNER) + "};",
             "__device__ const uint8_t kMcTriCount[256] = {"]
    for r in range(0, 256, 32):
        lines.append("    " + ", ".join(str(int(v)) for v in count[r:r + 32]) + ",")
    lines.append("};")
    lines.append("__device__ const int8_t kMcTriEdges[256][kMcMaxTris * 3] = {")
    for c in range(256):
        lines.append("    {" + ", ".join(str(int(v)) for v in edges[c]) + "},")
    lines.append("};")
    lines.append("}  // namespace nsb")
    return "\n".join(lines) + "\n"


CUH = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "neuralsim_b200", "csrc", "mc_table.cuh")

if __name__ == "__main__":
    with open(CUH, "w") as f:
        f.write(render_cuh())
    c, _ = build_table()
    print(CUH, "max triangles per case", int(c.max()))
