"""The marching-cubes case table of the TSDF mesh (rpg_open_remode_b200/csrc/mc_table.h; DESIGN.md 4.8): it is what
tools/make_mc_table.py generates, byte for byte, and each of its 256 cases has the properties the mesh relies on.
The cube geometry used here (corners, edges, faces) is restated independently of the generator."""
import importlib.util
import itertools
import os
import re

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HEADER = os.path.join(ROOT, "rpg_open_remode_b200", "csrc", "mc_table.h")


def _array(text, name):
    body = re.search(r"RMD_MC_STORAGE unsigned char " + name + r"\[[^=]*=\s*\{(.*?)\};", text, re.S).group(1)
    body = re.sub(r"/\*.*?\*/", "", body, flags=re.S)
    return [int(x) for x in re.findall(r"\d+", body)]


@pytest.fixture(scope="module")
def table():
    text = open(HEADER).read()
    edge = np.array(_array(text, "RMD_MC_EDGE"), int).reshape(12, 2)
    ntri = np.array(_array(text, "RMD_MC_NTRI"), int)
    m = int(re.search(r"#define RMD_MC_MAX_TRIS (\d+)", text).group(1))
    tris = np.array(_array(text, "RMD_MC_TRIS"), int).reshape(256, 3 * m)
    assert len(ntri) == 256
    return edge, ntri, [tris[c, :3 * ntri[c]].reshape(-1, 3) for c in range(256)]


def _corner(c):
    return np.array([c & 1, (c >> 1) & 1, (c >> 2) & 1])


def _edge_corners(edge):
    """(lower, upper) corner of each edge."""
    return [(int(c0), int(c0) + (1 << int(axis))) for c0, axis in edge]


def _face_of(edge):
    """For each edge, the set of cube faces (axis, side) it lies in."""
    out = []
    for c0, c1 in _edge_corners(edge):
        a, b = _corner(c0), _corner(c1)
        out.append({(d, int(a[d])) for d in range(3) if a[d] == b[d]})
    return out


def test_header_is_the_generators_output():
    spec = importlib.util.spec_from_file_location("make_mc_table", os.path.join(ROOT, "tools", "make_mc_table.py"))
    gen = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(gen)
    assert open(HEADER).read() == gen.render()


def test_edge_numbering(table):
    edge, _, _ = table
    ends = _edge_corners(edge)
    # 12 distinct cube edges, each between corners one unit apart; edge e = 4 axis + q runs along axis e // 4
    assert len({tuple(sorted(e)) for e in ends}) == 12
    for e, (c0, c1) in enumerate(ends):
        assert edge[e][1] == e // 4 and np.abs(_corner(c1) - _corner(c0)).sum() == 1 and c1 > c0


def test_every_case(table):
    edge, ntri, tris = table
    ends = _edge_corners(edge)
    faces = _face_of(edge)
    assert ntri[0] == 0 and ntri[255] == 0
    for case in range(256):
        inside = [(case >> c) & 1 for c in range(8)]
        crossing = {e for e, (c0, c1) in enumerate(ends) if inside[c0] != inside[c1]}
        t = tris[case]
        assert len(t) <= 5, case
        assert set(t.reshape(-1).tolist()) == crossing, case                  # exactly the crossing edges
        assert all(len(set(x)) == 3 for x in t.tolist()), case
        assert len({frozenset(x) for x in t.tolist()}) == len(t), case        # no triangle repeated
        # undirected triangle edges used twice are fan chords; once, loop segments on a cube face
        pairs = {}
        for a, b, c in t.tolist():
            for u, v in ((a, b), (b, c), (c, a)):
                pairs.setdefault(frozenset((u, v)), []).append((u, v))
        for key, uses in pairs.items():
            u, v = tuple(key)
            assert len(uses) <= 2, case
            if len(uses) == 2:
                assert uses[0] == uses[1][::-1], case                       # consistently oriented
                assert not (faces[u] & faces[v]), f"case {case:#x}: fan chord {u}-{v} lies on a cube face"
            else:
                assert faces[u] & faces[v], f"case {case:#x}: boundary {u}-{v} is not on a face"


def test_face_rule_is_shared_by_neighbours(table):
    """The segments a case draws on a face depend only on that face's four signs: for every pair of cases that
    agree on a face, the boundary segments on it are the same (mirrored onto the neighbour's edge numbers)."""
    edge, _, tris = table
    faces = _face_of(edge)
    ends = _edge_corners(edge)

    def segments(case, face):
        out = set()
        t = tris[case].tolist()
        und = {}
        for a, b, c in t:
            for u, v in ((a, b), (b, c), (c, a)):
                und.setdefault(frozenset((u, v)), []).append((u, v))
        for key, uses in und.items():
            u, v = tuple(key)
            if len(uses) == 1 and face in faces[u] and face in faces[v]:
                out.add(uses[0])
        return out

    def corners_of(face):
        d, side = face
        return [c for c in range(8) if _corner(c)[d] == side]

    def mirror_edge(e, d):
        c0, c1 = ends[e]
        m0, m1 = (c ^ (1 << d) for c in (c0, c1))
        return next(k for k, x in enumerate(ends) if set(x) == {m0, m1})

    for d in range(3):
        hi, lo = (d, 1), (d, 0)
        for signs in itertools.product((0, 1), repeat=4):
            a = sum(s << c for s, c in zip(signs, corners_of(hi)))                         # lower cube, face hi
            b = sum(s << (c ^ (1 << d)) for s, c in zip(signs, corners_of(hi)))            # upper cube, face lo
            for rest_a, rest_b in ((0, 0), (sum(1 << c for c in corners_of(lo)), sum(1 << c for c in corners_of(hi)))):
                sa = segments(a | rest_a, hi)
                sb = segments(b | rest_b, lo)
                # the shared face is seen from both sides: same segments between mirrored edges, opposite directions
                assert {(mirror_edge(v, d), mirror_edge(u, d)) for u, v in sa} == sb, (d, signs)
