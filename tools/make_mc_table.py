"""Generate rpg_open_remode_b200/csrc/mc_table.h: the marching-cubes case table of the TSDF mesh (DESIGN.md 4.8).

The table is derived from rules instead of being typed in, so that every property the mesh relies on follows from
the rules and is checked here and in tests/test_mc_table.py:

* Cube corner c = dx + 2 dy + 4 dz; case bit c is set when corner c is inside (tsdf <= 0).
* Edge e = 4 axis + q runs from its lower corner along `axis`; q = dy + 2 dz (x edges), dx + 2 dz (y edges),
  dx + 2 dy (z edges).  Its vertex is the surface point of the edge's lower voxel and axis.
* On each cube face the crossing edges pair into segments: two crossings give one segment; four crossings (an
  ambiguous face) give one segment per INSIDE corner, joining that corner's two face edges.  The rule depends only
  on the face's four signs, so the two cubes sharing a face build the same segments there: the mesh is watertight.
* Segments chain into closed loops (3 to 7 vertices), oriented so that (b - a) x (c - a) points to the tsdf > 0
  side, and each loop is triangulated as a fan whose apex is the first vertex (from the loop's smallest edge on)
  for which no fan chord joins two edges of the same cube face.  Loops are emitted in ascending order of their
  smallest edge, triangles in fan order.

Usage: python tools/make_mc_table.py [--check]   (--check: exit 1 if the committed header differs)
"""
from __future__ import annotations

import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HEADER = os.path.join(ROOT, "rpg_open_remode_b200", "csrc", "mc_table.h")
MAX_TRIS = 5


def corner_xyz(c):
    return (c & 1, (c >> 1) & 1, (c >> 2) & 1)


def edge_ends(e):
    """(lower corner, upper corner, axis) of edge e."""
    axis, q = divmod(e, 4)
    a, b = q & 1, q >> 1
    d = [0, 0, 0]
    others = [x for x in range(3) if x != axis]
    d[others[0]], d[others[1]] = a, b
    c0 = d[0] + 2 * d[1] + 4 * d[2]
    return c0, c0 + (1 << axis), axis


EDGES = [edge_ends(e) for e in range(12)]


def faces():
    """(axis, side, corners, edges) of the 6 cube faces."""
    out = []
    for axis in range(3):
        for side in range(2):
            corners = [c for c in range(8) if corner_xyz(c)[axis] == side]
            edges = [e for e in range(12) if EDGES[e][0] in corners and EDGES[e][1] in corners]
            out.append((axis, side, corners, edges))
    return out


FACES = faces()


def share_face(e1, e2):
    return any(e1 in f[3] and e2 in f[3] for f in FACES)


def midpoint(e):
    c0, _, axis = EDGES[e]
    p = [float(x) for x in corner_xyz(c0)]
    p[axis] += 0.5
    return p


def _sub(a, b):
    return [a[0] - b[0], a[1] - b[1], a[2] - b[2]]


def _cross(a, b):
    return [a[1] * b[2] - a[2] * b[1], a[2] * b[0] - a[0] * b[2], a[0] * b[1] - a[1] * b[0]]


def _dot(a, b):
    return a[0] * b[0] + a[1] * b[1] + a[2] * b[2]


def crossing_edges(case):
    return [e for e in range(12) if ((case >> EDGES[e][0]) ^ (case >> EDGES[e][1])) & 1]


def face_segments(case):
    """Directed segments (from edge, to edge) of every face, oriented for a normal towards tsdf > 0."""
    segs = []
    for axis, side, corners, edges in FACES:
        cross = [e for e in edges if e in crossing_edges(case)]
        inside = [c for c in corners if (case >> c) & 1]
        if len(cross) == 2:
            pairs = [(cross[0], cross[1], inside[0])]
        elif len(cross) == 4:
            pairs = []
            for q in inside:
                at_q = [e for e in cross if q in EDGES[e][:2]]
                assert len(at_q) == 2
                pairs.append((at_q[0], at_q[1], q))
        else:
            assert not cross
            continue
        normal = [0.0, 0.0, 0.0]
        normal[axis] = 1.0 if side else -1.0          # outward face normal
        for e1, e2, q in pairs:
            m1, m2 = midpoint(e1), midpoint(e2)
            # the inside corner q lies to the right of m1 -> m2 seen from outside the cube
            s = _dot(_cross(_sub(m2, m1), _sub([float(x) for x in corner_xyz(q)], m1)), normal)
            assert s != 0.0
            segs.append((e1, e2) if s < 0.0 else (e2, e1))
    return segs


def loops(case):
    nxt = {}
    for a, b in face_segments(case):
        assert a not in nxt, (case, a)
        nxt[a] = b
    assert sorted(nxt) == sorted(nxt.values()) == crossing_edges(case), case
    out, seen = [], set()
    for start in sorted(nxt):
        if start in seen:
            continue
        loop, e = [], start
        while e not in seen:
            seen.add(e)
            loop.append(e)
            e = nxt[e]
        assert e == start and 3 <= len(loop) <= 7, (case, loop)
        out.append(loop)
    return out


def fan(loop):
    for a in range(len(loop)):
        rot = loop[a:] + loop[:a]
        if all(not share_face(rot[0], rot[i]) for i in range(2, len(rot) - 1)):
            return [(rot[0], rot[i], rot[i + 1]) for i in range(1, len(rot) - 1)]
    raise AssertionError("no fan apex for loop %s" % loop)


def table():
    """[256] lists of triangles (3 edge numbers each)."""
    out = []
    for case in range(256):
        tris = [t for loop in loops(case) for t in fan(loop)]
        assert len(tris) <= MAX_TRIS, (case, tris)
        out.append(tris)
    return out


def render() -> str:
    tris = table()
    lines = [
        "/* mc_table.h -- marching-cubes case table of the TSDF mesh (DESIGN.md 4.8).",
        " * GENERATED by tools/make_mc_table.py from the rules stated there; do not edit.  C and CUDA.",
        " *",
        " * Corner c = dx + 2 dy + 4 dz; case bit c set = corner inside (tsdf <= 0).  Edge e = 4 axis + q from its",
        " * lower corner RMD_MC_EDGE[e][0] along axis RMD_MC_EDGE[e][1].  RMD_MC_TRIS[case] holds",
        " * RMD_MC_NTRI[case] triangles as 3 edge numbers each, (b - a) x (c - a) towards tsdf > 0.",
        " * RMD_MC_STORAGE is the storage class of the arrays (default: static const). */",
        "#ifndef RMD_MC_TABLE_H",
        "#define RMD_MC_TABLE_H",
        "",
        "#ifndef RMD_MC_STORAGE",
        "#define RMD_MC_STORAGE static const",
        "#endif",
        "",
        "#define RMD_MC_MAX_TRIS %d" % MAX_TRIS,
        "",
        "RMD_MC_STORAGE unsigned char RMD_MC_EDGE[12][2] = {",
        "  " + ", ".join("{%d, %d}" % (c0, axis) for c0, _, axis in EDGES),
        "};",
        "",
        "RMD_MC_STORAGE unsigned char RMD_MC_NTRI[256] = {",
    ]
    for r in range(0, 256, 32):
        lines.append("  " + ", ".join(str(len(t)) for t in tris[r:r + 32]) + ",")
    lines += ["};", "", "RMD_MC_STORAGE unsigned char RMD_MC_TRIS[256][%d] = {" % (3 * MAX_TRIS)]
    for case, t in enumerate(tris):
        flat = [e for tri in t for e in tri] + [0] * (3 * MAX_TRIS - 3 * len(t))
        lines.append("  {" + ", ".join(str(e) for e in flat) + "},   /* 0x%02x */" % case)
    lines += ["};", "", "#endif /* RMD_MC_TABLE_H */", ""]
    return "\n".join(lines)


def main(argv):
    text = render()
    if "--check" in argv:
        with open(HEADER) as f:
            same = f.read() == text
        print("mc_table.h is up to date" if same else "mc_table.h differs from the generator's output")
        return 0 if same else 1
    with open(HEADER, "w") as f:
        f.write(text)
    print("wrote", HEADER)
    return 0


if __name__ == "__main__":
    sys.exit(main(sys.argv[1:]))
