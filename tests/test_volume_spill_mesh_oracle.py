"""The spill-mesh oracle (oracle/rmd_oracle_volume_spill_mesh.c, DESIGN.md 4.8) pinned against numpy, and the scene
welder api.SceneMesh run on it, on the CPU.

  * the spill mesh's vertices V_s are the numpy surface points filtered by the vertex rule (the point spills, or one
    of the <= 4 cubes of its edge is meshed and has a corner outside the kept box K), bit for bit with their
    intensities and normals; its triangles are the mesh's triangles of those cubes, remapped -- on random ragged grids
    (down to nx = 1, which has no cubes) that mix unknown, +-1, truncated, exact-zero and -0.0 voxels, for every sign
    pattern of d; d = 0 gives nothing and |d| >= n gives mesh();
  * mesh before a shift == spill mesh + mesh after it, with triangles as id triples, and on an exact grid positions,
    weights and intensities bit for bit by id;
  * SceneMesh over several shifts without integration between them (back into unknown space included) gives the
    original grid's mesh();
  * planted bugs in the rule (corners outside K ignored on one axis, seam vertices left out, K off by one) break the
    identity.
"""
import itertools
import os
import sys

import numpy as np
import pytest

import spill_mesh_oracle as smo
import test_mc_table
from test_volume_shift_oracle import _np_surface, _random_volume

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from rpg_open_remode_b200.api import SceneMesh  # noqa: E402  (host code only: no native library is loaded)

F = np.float32
u32 = np.uint32
NTRI = np.array(test_mc_table._array(open(test_mc_table.HEADER).read(), "RMD_MC_NTRI"), int)


def _mixed_volume(rng, dims, s=0.05, origin=(0.3, -0.7, 1.1)):
    """_random_volume's noisy band with exact +-1, 0.0 and -0.0 records planted in it."""
    o = _random_volume(rng, dims, s, origin)
    o.__class__ = smo.OracleVolume
    t = o.tsdf.reshape(-1).copy()
    r = rng.random(t.size)
    t[r < 0.04] = F(1.0)
    t[(r >= 0.04) & (r < 0.08)] = F(-1.0)
    t[(r >= 0.08) & (r < 0.12)] = F(0.0)
    t[(r >= 0.12) & (r < 0.16)] = F(-0.0)
    o.tsdf = np.ascontiguousarray(t.reshape(o.tsdf.shape))
    return o


def _exact_volume(rng, dims, s=F(2.0 ** -4)):
    """Voxel 2^-4 m and an origin of small multiples of it: o + i s is exact, so positions survive a shift."""
    return _mixed_volume(rng, dims, s=s, origin=(F(-3) * s, F(5) * s, F(16) * s))


def _np_cubes(tsdf, weight):
    """Case of every cube [nz - 1, ny - 1, nx - 1] when it is meshed, else 0: 8 known corners, not all on one side,
    no crossing edge with |tsdf| >= 1 at an end."""
    nz, ny, nx = tsdf.shape
    shape = (max(nz - 1, 0), max(ny - 1, 0), max(nx - 1, 0))
    sl = [(slice(c >> 2 & 1, (c >> 2 & 1) + shape[0]), slice(c >> 1 & 1, (c >> 1 & 1) + shape[1]),
           slice(c & 1, (c & 1) + shape[2])) for c in range(8)]
    known = np.ones(shape, bool)
    case = np.zeros(shape, np.int64)
    bad = np.zeros(shape, bool)
    for c in range(8):
        known &= weight[sl[c]] > 0
        case |= (tsdf[sl[c]] <= 0).astype(np.int64) << c
        for axis in range(3):
            if c >> axis & 1:
                continue
            t0, t1 = tsdf[sl[c]], tsdf[sl[c + (1 << axis)]]
            bad |= ((t0 <= 0) != (t1 <= 0)) & ~((np.abs(t0) < 1) & (np.abs(t1) < 1))
    return np.where(known & (case != 0) & (case != 255) & ~bad, case, 0)


def _np_spill_mesh(o, d, bug=None):
    """numpy spill mesh: (vertex mask over the surface points, triangle mask over mesh()'s triangles, all surface
    points, their ids, mesh()'s triangles).  bug plants one of "cube_ignores_x", "no_seam", "k_off_by_one"."""
    pts, vox, axes = _np_surface(o.tsdf, o.weight, o.s, o.origin)
    n, d = np.array(o.dims), np.asarray(d)
    lo, hi = np.maximum(0, d), np.minimum(n, n + d)
    if bug == "k_off_by_one":
        hi = hi - 1
    cases = _np_cubes(o.tsdf, o.weight)

    def leaves(c):
        out = (c < lo) | (c + 1 >= hi)
        if bug == "cube_ignores_x":
            out[:, 0] = False
        return out.any(1)

    b = vox + np.eye(3, dtype=np.int64)[axes]
    vertex = ~(np.all((vox >= lo) & (vox < hi), 1) & np.all((b >= lo) & (b < hi), 1))
    if bug != "no_seam":
        r = np.arange(len(vox))
        u, w = np.where(axes == 0, 1, 0), np.where(axes == 2, 1, 2)
        for q in range(4):
            c = vox.copy()
            c[r, u] -= q & 1
            c[r, w] -= q >> 1
            valid = np.all(c >= 0, 1) & np.all(c + 1 < n, 1)
            cc = np.where(valid[:, None], c, 0)
            meshed = valid & (cases[cc[:, 2], cc[:, 1], cc[:, 0]] != 0) if cases.size else np.zeros(len(c), bool)
            vertex |= meshed & leaves(cc)
    _, tris = smo.mesh_oracle.mesh(o)
    cubes = np.argwhere(cases != 0)[:, ::-1]          # (i, j, k) of the meshed cubes, in cube order
    tri_cube = np.repeat(cubes, NTRI[cases[cases != 0]], axis=0)
    assert len(tri_cube) == len(tris)
    ids = np.concatenate([vox + o.D, axes[:, None]], 1).astype(np.int64)
    return vertex, leaves(tri_cube) if len(tri_cube) else np.zeros(0, bool), pts, ids, tris


def _ids_of_triangles(tris, ids):
    return [tuple(r) for r in ids[tris].reshape(-1, 12)]


def _identity_failures(before, spill, after):
    """Each of (vertex ids [n, 4], triangles as id triples): the ways in which before != spill + after."""
    fails = []
    bv, sv, av = ({tuple(r) for r in x[0]} for x in (before, spill, after))
    if sorted(before[1]) != sorted(spill[1] + after[1]):
        fails.append("triangles")
    if any(v not in sv for t in spill[1] for v in zip(*[iter(t)] * 4)):
        fails.append("spill triangle without its vertex")
    if sv | av != bv or len(sv) + len(av) - len(sv & av) != len(bv) or len(sv) != len(spill[0]):
        fails.append("vertices")
    return fails


RAGGED = [(1, 7, 5), (9, 1, 6), (5, 6, 1), (13, 11, 9), (17, 3, 12), (2, 2, 2)]
SIGNS = list(itertools.product((-1, 0, 1), repeat=3))


@pytest.mark.parametrize("dims", RAGGED + [(24, 20, 16)])
def test_spill_mesh_is_the_numpy_rule(dims):
    rng = np.random.default_rng(11 * sum(dims))
    o = _mixed_volume(rng, dims)
    inten, _ = o.surface_intensity()
    nrm, _ = o.surface_normals()
    mv, mt = o.mesh()
    ds = [tuple(int(sg * m) for sg, m in zip(sign, (2, 1, 3))) for sign in SIGNS] + \
         [(dims[0], 0, 0), (0, -dims[1], 0), (0, 0, dims[2] + 4), (-1, 40, 0)]
    n_seam = 0
    for d in ds:
        vertex, tri_mask, pts, ids, tris = _np_spill_mesh(o, d)
        got, gt, keys, nv, nt = o.spill_mesh(d, smo.POINTS)
        remap = np.cumsum(vertex) - 1
        assert nv == vertex.sum() and np.array_equal(got.view(u32), pts[vertex].view(u32)), d
        assert nt == tri_mask.sum() and np.array_equal(gt, remap[tris[tri_mask]]), d
        assert np.array_equal(smo.keys_to_ids(keys, o.dims, o.D), ids[vertex]), d
        got_i = o.spill_mesh(d, smo.INTENSITY)[0]
        got_n = o.spill_mesh(d, smo.NORMALS)[0]
        assert np.array_equal(got_i.view(u32), inten[vertex].view(u32))
        assert np.array_equal(got_n.view(u32), nrm[vertex].view(u32))
        n_seam += int(vertex.sum() - o.spill(d, smo.POINTS)[1])
        if d == (0, 0, 0):
            assert nv == nt == 0
        if any(abs(x) >= m for x, m in zip(d, dims)):   # everything leaves: the spill mesh is mesh()
            assert np.array_equal(got.view(u32), mv.view(u32)) and np.array_equal(gt, mt)
        if nt:   # capacities below both counts
            part_v, part_t, part_k, nv2, nt2 = o.spill_mesh(d, smo.POINTS, nv // 2, nt // 3)
            assert (nv2, nt2) == (nv, nt) and np.array_equal(part_t, gt[:nt // 3])
            assert np.array_equal(part_v.view(u32), got[:nv // 2].view(u32)) and np.array_equal(part_k, keys[:nv // 2])
    if min(dims) >= 9:
        assert len(mt) > 20 and n_seam > 0    # the grid has a mesh, and seam vertices occur


def _mesh_with_ids(o):
    verts, tris = o.mesh()
    ids = o.surfaceIds()
    return verts, tris, ids


@pytest.mark.parametrize("d", [(2, 0, 0), (-3, 1, 0), (0, -2, 4), (5, 5, -5), (1, -1, 1), (0, 0, -1)])
def test_mesh_before_is_spill_plus_mesh_after(d):
    rng = np.random.default_rng(abs(hash(d)) % 2 ** 32)
    o = _exact_volume(rng, (20, 18, 16))
    bv, bt, bids = _mesh_with_ids(o)
    bi = o.surfaceIntensity()
    sv, st, sids = o.spillMesh(d)
    si = o.spillMeshIntensity(d)
    o.shift(d)
    av, at, aids = _mesh_with_ids(o)
    ai = o.surfaceIntensity()
    assert len(st) > 0 and len(at) > 0
    fails = _identity_failures((bids, _ids_of_triangles(bt, bids)), (sids, _ids_of_triangles(st, sids)),
                               (aids, _ids_of_triangles(at, aids)))
    assert not fails, fails
    # positions, weights and intensities bit for bit by id (the seam vertices on both sides)
    by_id = {tuple(r): q for q, r in enumerate(bids)}
    for verts, inten, ids in ((sv, si, sids), (av, ai, aids)):
        q = np.array([by_id[tuple(r)] for r in ids])
        assert np.array_equal(verts.view(u32), bv[q].view(u32)) and np.array_equal(inten.view(u32), bi[q].view(u32))
    seam = {tuple(r) for r in sids} & {tuple(r) for r in aids}
    assert seam   # seam vertices are shared


@pytest.mark.parametrize("bug", ["cube_ignores_x", "no_seam", "k_off_by_one"])
def test_planted_bugs_break_the_identity(bug):
    """The numpy rule passes the identity and each planted bug fails it, on grids where the correct rule's seam
    vertices, x-leaving cubes and K's faces all matter."""
    caught = 0
    for seed, d in enumerate([(2, 0, 0), (-3, 1, 0), (0, -2, 4), (5, 5, -5)]):
        o = _exact_volume(np.random.default_rng(100 + seed), (20, 18, 16))
        _, bt, bids = _mesh_with_ids(o)
        before = (bids, _ids_of_triangles(bt, bids))
        spills = []
        for b in (None, bug):
            vertex, tri_mask, _, ids, tris = _np_spill_mesh(o, d, b)
            spills.append((ids[vertex], _ids_of_triangles(tris[tri_mask], ids)))
        o.shift(d)
        _, at, aids = _mesh_with_ids(o)
        after = (aids, _ids_of_triangles(at, aids))
        assert not _identity_failures(before, spills[0], after)
        fails = _identity_failures(before, spills[1], after)
        caught += bool(fails)
        print(f"{bug} d={d}: {fails}")
    assert caught >= 3, caught


def _scene_reproduces(o, shifts, intensity=True):
    """Add the spill mesh of every shift to a SceneMesh, then compare its mesh with o's mesh before the shifts."""
    bv, bt, bids = _mesh_with_ids(o)
    bi = o.surfaceIntensity()
    scene = SceneMesh(intensity=intensity, normals=True)
    seen = []   # every chunk's ids in order: the scene's vertices are their first occurrences, if welding is right
    for d in shifts:
        seen.append(o.spillMesh(d)[2])
        scene.addSpill(o, d)
        o.shift(d)
    seen.append(o.surfaceIds())
    V, T, I, N = scene.mesh(o)
    V2, T2, I2, N2 = scene.mesh(o)   # repeatable, the state unchanged
    assert np.array_equal(V2.view(u32), V.view(u32)) and np.array_equal(T2, T) and np.array_equal(I2, I)
    allids = np.concatenate(seen)
    _, first = np.unique(allids, axis=0, return_index=True)
    vids = allids[np.sort(first)]
    assert len(V) == len(vids) == len(bids), (len(V), len(vids), len(bids))   # each vertex once
    assert {tuple(r) for r in vids} == {tuple(r) for r in bids}
    assert T.min(initial=0) >= 0 and T.max(initial=-1) < len(V) and N.shape == (len(V), 3)
    assert sorted(_ids_of_triangles(T, vids)) == sorted(_ids_of_triangles(bt, bids))
    by_id = {tuple(r): q for q, r in enumerate(bids)}
    q = np.array([by_id[tuple(r)] for r in vids])
    assert np.array_equal(V.view(u32), bv[q].view(u32))
    assert (I is None) != intensity and (I is None or np.array_equal(I.view(u32), bi[q].view(u32)))
    return len(seen) - 1


@pytest.mark.parametrize("seed", [0, 1, 2])
def test_scene_mesh_without_integration_reproduces_the_mesh(seed):
    rng = np.random.default_rng(500 + seed)
    o = _exact_volume(rng, (20, 18, 16))
    shifts = [tuple(int(x) for x in rng.integers(-4, 5, 3)) for _ in range(4)]
    shifts += [tuple(-x for x in shifts[0]), (3, -2, 1), (-3, 2, -1)]   # back into unknown space
    assert _scene_reproduces(o, shifts) == len(shifts)


def test_scene_mesh_on_ragged_grids_and_whole_grid_shifts():
    for dims in RAGGED[3:]:
        rng = np.random.default_rng(sum(dims))
        o = _exact_volume(rng, dims)
        _scene_reproduces(o, [(1, 0, -1), (0, 0, 0), (-2, 1, 1), (dims[0], 0, 0)], intensity=False)


def test_scene_mesh_does_not_weld_a_surface_that_re_enters():
    """A voxel that leaves and comes back starts new vertices: integrate the same records again after the shift back
    (here: upload them) and the scene has two copies of what re-entered."""
    rng = np.random.default_rng(9)
    o = _exact_volume(rng, (20, 18, 16))
    t, w = o.tsdf.copy(), o.weight.copy()
    scene = SceneMesh()
    scene.addSpill(o, (5, 0, 0))
    o.shift((5, 0, 0))
    scene.addSpill(o, (-5, 0, 0))
    o.shift((-5, 0, 0))
    o.tsdf, o.weight = t, w          # the same surface, seen again
    V, T, _, _ = scene.mesh(o)
    n_before = len(o.surfaceIds())
    assert len(V) > n_before    # what re-entered is a second, unwelded surface
