"""Generate the marching-cubes case table lara_b200/csrc/mc_table.cuh from first principles.

    python tools/gen_mc_table.py            # rewrite the header
    python tools/gen_mc_table.py --check    # exit 1 if the committed header differs from the output

Conventions (shared with lara_b200/csrc/mesh.cu and oracle/mesh64.py):
  corner c of a cube (0..7): bit 0 = +x, bit 1 = +y, bit 2 = +z; a corner is inside if its TSDF is < 0 and sets bit c
  of the case index.
  edge e = 4 a + b (0..11): along axis a, starting at the corner whose two other axis bits are b (the lower of those
  axes in bit 0 of b); the edge's end is its start plus the unit vector of axis a.

For each of the 256 cases:
  1. On each of the 6 faces the crossing edges (ends of opposite sign) are joined into segments.  A face with two
     crossings has one segment.  A face with four (the two inside corners diagonal, ambiguous) joins the crossings so
     that each inside corner is cut off on its own; the rule reads only the face's four corner signs, so the two cubes
     that share the face draw the same segments and the surface is crack-free by construction.
  2. Each segment is directed so that, seen from outside the cube (face normal n pointing out), n x d points from the
     segment to the face's outside corners.  Every crossing edge then ends one segment and starts one other, and the
     segments link into closed loops that all turn the same way.
  3. Each loop v0 v1 ... vk-1 is fan-triangulated into (v0, vi, vi+1), from the first apex whose diagonals (v0, vi)
     all cross the cube's interior: a diagonal on a face (two crossings of an ambiguous face) could be drawn by the
     cube across the face too.  The right-hand normal of every triangle points toward increasing TSDF, i.e. out of
     the surface.
"""
from __future__ import annotations

import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HEADER = os.path.join(ROOT, "lara_b200", "csrc", "mc_table.cuh")


def corner_pos(c):
    return np.array([c & 1, (c >> 1) & 1, (c >> 2) & 1], dtype=np.float64)


def edge_corners(e):
    """(start, end) corner of edge e."""
    a, b = divmod(e, 4)
    others = [x for x in range(3) if x != a]
    start = ((b & 1) << others[0]) | (((b >> 1) & 1) << others[1])
    return start, start | (1 << a)


EDGES = [edge_corners(e) for e in range(12)]


def edge_of(c0, c1):
    for e, (s, t) in enumerate(EDGES):
        if {s, t} == {c0, c1}:
            return e
    raise ValueError((c0, c1))


def faces():
    """The 6 faces: (outward normal, 4 corners in cyclic order)."""
    out = []
    for a in range(3):
        u, v = [x for x in range(3) if x != a]
        for side in (0, 1):
            base = side << a
            cyc = [base, base | (1 << u), base | (1 << u) | (1 << v), base | (1 << v)]
            n = np.zeros(3)
            n[a] = 1.0 if side else -1.0
            out.append((n, cyc))
    return out


FACES = faces()


def case_loops(case):
    """Closed, consistently directed loops of crossing edges of one sign case."""
    inside = [(case >> c) & 1 == 1 for c in range(8)]
    nxt = {}
    for n, cyc in FACES:
        ins = [inside[c] for c in cyc]
        cross = [i for i in range(4) if ins[i] != ins[(i + 1) % 4]]    # face edge i joins cyc[i], cyc[i+1]
        if not cross:
            continue
        if len(cross) == 2:
            pairs = [(cross[0], cross[1])]
        else:                                                            # ambiguous: cut off each inside corner
            pairs = [((i - 1) % 4, i) for i in range(4) if ins[i]]
        for i, j in pairs:
            ei, ej = edge_of(cyc[i], cyc[(i + 1) % 4]), edge_of(cyc[j], cyc[(j + 1) % 4])
            mid = lambda e: 0.5 * (corner_pos(EDGES[e][0]) + corner_pos(EDGES[e][1]))   # noqa: E731
            pi, pj = mid(ei), mid(ej)
            m = 0.5 * (pi + pj)
            if len(cross) == 2:
                outside = [corner_pos(c) for c in cyc if not inside[c]]
            else:   # the segment cuts off the corner both its edges touch; the other three are across it
                cut = (set(EDGES[ei]) & set(EDGES[ej])).pop()
                outside = [corner_pos(c) for c in cyc if c != cut]
            towards = np.mean(outside, axis=0) - m
            if np.dot(np.cross(n, pj - pi), towards) < 0:
                ei, ej = ej, ei
            assert ei not in nxt, (case, ei)
            nxt[ei] = ej
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


FACE_EDGES = [{edge_of(cyc[i], cyc[(i + 1) % 4]) for i in range(4)} for _, cyc in FACES]


def on_one_face(e0, e1):
    return any(e0 in f and e1 in f for f in FACE_EDGES)


def case_triangles(case):
    """Fan of each loop from the first apex (in loop order) none of whose diagonals lies on a cube face: a diagonal on
    a face could also be drawn by the cube across it, and the edge would then have more than two triangles."""
    tris = []
    for loop in case_loops(case):
        k = len(loop)
        for r in range(k):
            ring = loop[r:] + loop[:r]
            if not any(on_one_face(ring[0], ring[i]) for i in range(2, k - 1)):
                break
        else:
            raise AssertionError(f"case {case}: no fan apex without a diagonal on a face")
        for i in range(1, k - 1):
            tris.append((ring[0], ring[i], ring[i + 1]))
    return tris


def table():
    return [case_triangles(c) for c in range(256)]


def render(tab) -> str:
    maxt = max(len(t) for t in tab)
    lines = [
        "// mc_table.cuh -- GENERATED by tools/gen_mc_table.py; do not edit (python tools/gen_mc_table.py rewrites it).",
        "// Marching-cubes triangles per sign case: corner c = x | y << 1 | z << 2 is inside (bit c of the case) if its",
        "// TSDF is < 0; edge e = 4 a + b runs along axis a from the corner whose other two axis bits are b.  Loops of",
        "// crossing edges, fan-triangulated; each triangle's right-hand normal points toward increasing TSDF.",
        "#pragma once",
        "",
        f"#define SRF_MC_MAX_TRIS {maxt}",
        "",
        "// number of triangles of each case",
        "__device__ __constant__ unsigned char kMcTriCount[256] = {",
    ]
    for r in range(0, 256, 32):
        lines.append("    " + ", ".join(str(len(t)) for t in tab[r:r + 32]) + ",")
    lines += ["};", "", "// the triangles' edges, 3 per triangle, unused slots -1",
              f"__device__ __constant__ signed char kMcTris[256][{3 * maxt}] = {{"]
    for c, t in enumerate(tab):
        flat = [e for tri in t for e in tri] + [-1] * (3 * (maxt - len(t)))
        lines.append("    {" + ", ".join(str(x) for x in flat) + f"}},  // {c}")
    lines += ["};", ""]
    return "\n".join(lines)


def main(argv) -> int:
    text = render(table())
    if "--check" in argv:
        with open(HEADER) as f:
            same = f.read() == text
        print("mc_table.cuh is", "up to date" if same else "STALE")
        return 0 if same else 1
    with open(HEADER, "w") as f:
        f.write(text)
    print("wrote", HEADER)
    return 0


if __name__ == "__main__":
    sys.exit(main(sys.argv[1:]))
