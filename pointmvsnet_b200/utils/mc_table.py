"""Marching-cubes triangle table of the surface extraction (DESIGN.md section 3.23), generated from three rules.

Cube corner c sits at offset (c & 1, (c >> 1) & 1, (c >> 2) & 1) along the grid axes (i, j, k); bit c of a case is
set when that corner is inside (tsdf < 0).  Edge e = 4 a + m runs along axis a from the m-th corner (ascending) whose
bit a is 0 to that corner + (1 << a).  Face f = 2 a + s holds the four corners whose bit a equals s.

1. On every face, pair the cut edges into segments.  With four cut edges (diagonally opposite inside corners) each
   segment cuts off a single inside corner, so the two inside corners are never joined.  The segments of a face depend
   only on its four corner signs, so two cubes sharing a face draw the same ones and the mesh has no cracks.
2. Direct each segment so that, seen from outside the cube, the inside corners it cuts off lie on its right, and chain
   the segments into closed loops on the cube's surface.  Triangles that follow the loops face outward, towards
   tsdf > 0.
3. Triangulate each loop as a fan from the lowest-numbered edge whose fan adds no chord between two edges of a common
   cube face (such a chord could be drawn by the neighbouring cube too, and its edge would end up in four triangles).

`python -m pointmvsnet_b200.utils.mc_table [path]` writes the header csrc/mc_table.cuh (stdout without a path).
"""
import sys

import numpy as np

CORNERS = [(c & 1, (c >> 1) & 1, (c >> 2) & 1) for c in range(8)]
EDGES = []  # (lower corner, upper corner, axis)
for _a in range(3):
    for _c0 in [c for c in range(8) if not (c >> _a) & 1]:
        EDGES.append((_c0, _c0 | (1 << _a), _a))
EDGE_ID = {(c0, c1): e for e, (c0, c1, _) in enumerate(EDGES)}
EDGE_ID.update({(c1, c0): e for (c0, c1), e in list(EDGE_ID.items())})


def _face_cycle(f):
    """the corners of face f = 2a + s in cyclic order around it"""
    a, s = divmod(f, 2)
    b, d = [x for x in range(3) if x != a]
    return [(s << a) | (u << b) | (v << d) for u, v in ((0, 0), (1, 0), (1, 1), (0, 1))]


FACES = [_face_cycle(f) for f in range(6)]
EDGE_FACES = [frozenset(f for f in range(6) if c0 in FACES[f] and c1 in FACES[f]) for c0, c1, _ in EDGES]
MAX_TRIS = 5


def _inside(case, c):
    return (case >> c) & 1 == 1


def face_segments(case, f):
    """rules 1 and 2 on face f: directed segments [(from edge, to edge)], sorted"""
    q = FACES[f]
    ins = [_inside(case, c) for c in q]
    cut = [EDGE_ID[q[t], q[(t + 1) % 4]] for t in range(4) if ins[t] != ins[(t + 1) % 4]]
    if not cut:
        return []
    if len(cut) == 4:  # ambiguous face: one segment around each inside corner
        pairs = [(EDGE_ID[q[(t + 3) % 4], q[t]], EDGE_ID[q[t], q[(t + 1) % 4]], [q[t]]) for t in range(4) if ins[t]]
    else:
        pairs = [(cut[0], cut[1], [c for c in q if _inside(case, c)])]
    a, s = divmod(f, 2)
    n = np.zeros(3)
    n[a] = 1.0 if s else -1.0  # outward normal of the face
    out = []
    for e1, e2, corners in pairs:
        p1 = np.add(*[np.array(CORNERS[c], float) for c in EDGES[e1][:2]]) / 2
        p2 = np.add(*[np.array(CORNERS[c], float) for c in EDGES[e2][:2]]) / 2
        cen = np.mean([np.array(CORNERS[c], float) for c in corners], axis=0)
        right = np.cross(p2 - p1, n)  # seen from outside (looking along -n), the right of p1 -> p2
        out.append((e1, e2) if np.dot(cen - p1, right) > 0 else (e2, e1))
    return sorted(out)


def case_loops(case):
    """rule 2: the directed loops of a case, each a list of edges starting at its lowest, ordered by that edge"""
    succ = {}
    for f in range(6):
        for e1, e2 in face_segments(case, f):
            if e1 in succ:
                raise AssertionError("case %d: edge %d leaves two segments" % (case, e1))
            succ[e1] = e2
    loops, seen = [], set()
    for start in sorted(succ):
        if start in seen:
            continue
        loop, e = [], start
        while e not in seen:
            seen.add(e)
            loop.append(e)
            e = succ[e]
        if e != start:
            raise AssertionError("case %d: open chain from edge %d" % (case, start))
        loops.append(loop)
    return loops


def _fan_apex(loop):
    """rule 3: the loop rotated to start at the lowest edge whose fan has no chord inside a cube face"""
    m = len(loop)
    for apex in sorted(loop):
        p = loop.index(apex)
        r = loop[p:] + loop[:p]
        if all(not (EDGE_FACES[r[0]] & EDGE_FACES[r[k]]) for k in range(2, m - 1)):
            return r
    raise AssertionError("loop %s has no valid fan apex" % (loop,))


def case_triangles(case):
    """rule 3: the triangles of a case, [(e0, e1, e2)] in table order"""
    tris = []
    for loop in case_loops(case):
        r = _fan_apex(loop)
        tris += [(r[0], r[k], r[k + 1]) for k in range(1, len(r) - 1)]
    return tris


def table():
    """-> int8 [256, 3 MAX_TRIS + 1] edge triples, -1 padded, and int8 [256] triangle counts"""
    tris = np.full((256, 3 * MAX_TRIS + 1), -1, dtype=np.int8)
    ntri = np.zeros(256, dtype=np.int8)
    for case in range(256):
        t = case_triangles(case)
        if len(t) > MAX_TRIS:
            raise AssertionError("case %d has %d triangles (> %d)" % (case, len(t), MAX_TRIS))
        ntri[case] = len(t)
        if t:
            tris[case, :3 * len(t)] = np.array(t).reshape(-1)
    return tris, ntri


def header_text():
    tris, ntri = table()
    lines = ["// Generated by pointmvsnet_b200/utils/mc_table.py -- do not edit (DESIGN 3.23).",
             "// Corner c at offset (c & 1, (c >> 1) & 1, (c >> 2) & 1) along (i, j, k); case bit c = corner c inside",
             "// (tsdf < 0).  Edge e runs along axis MC_EDGE_AXIS[e] from corner MC_EDGE_CORNER[e].  MC_TRIS[case] lists",
             "// MC_NTRI[case] triangles as edge triples, counter-clockwise seen from outside (tsdf > 0), -1 padded.",
             "#pragma once", "", "namespace pmvs {", "",
             "constexpr int MC_MAX_TRIS = %d;" % MAX_TRIS, "",
             "__constant__ signed char MC_EDGE_CORNER[12] = {%s};" % ", ".join(str(e[0]) for e in EDGES),
             "__constant__ signed char MC_EDGE_AXIS[12] = {%s};" % ", ".join(str(e[2]) for e in EDGES), "",
             "__constant__ signed char MC_NTRI[256] = {"]
    for r in range(0, 256, 32):
        lines.append("    " + ", ".join(str(int(x)) for x in ntri[r:r + 32]) + ",")
    lines += ["};", "", "__constant__ signed char MC_TRIS[256][%d] = {" % tris.shape[1]]
    for case in range(256):
        lines.append("    {%s},  // %d" % (", ".join(str(int(x)) for x in tris[case]), case))
    lines += ["};", "", "}  // namespace pmvs", ""]
    return "\n".join(lines)


if __name__ == "__main__":
    text = header_text()
    if len(sys.argv) > 1:
        with open(sys.argv[1], "w") as fh:
            fh.write(text)
    else:
        sys.stdout.write(text)
