"""The brick-store model (tests/volume_store_oracle.py) pinned without a GPU.

  * on shift sequences that never bring a stored voxel back, the model's window equals the shift oracle's bit for bit;
  * the stored-brick set and records follow the eviction rule, checked voxel by voxel;
  * shift(d) then shift(-d) gives back the window, for any d;
  * api.TsdfVolume.mapMesh run on the model: its triangles, as vertex ids, are those of the whole map meshed as one
    dense grid, no directed edge is used twice, and the model is unchanged afterwards.
"""
import numpy as np
import pytest

import mesh_checks
import spill_mesh_oracle as smo
import volume_shift_oracle as vso
from volume_store_oracle import StoreModel, kept_box, moving

u32 = np.uint32


def world(u, centre=(20.0, 14.0, 11.0), radius=9.0):
    """Sphere TSDF at unbounded voxels u [..., 3] (x, y, z), in units of 3 voxels."""
    r = np.sqrt(((u - np.asarray(centre)) ** 2).sum(-1))
    return np.clip((r - radius) / 3.0, -1.0, 1.0).astype(np.float32)


def paint(v, rng, p=0.8, intensity=True):
    """Observe the world in the window: a random p of its voxels get the world's tsdf (weight + 1, colour)."""
    nx, ny, nz = v.dims
    k, j, i = np.meshgrid(np.arange(nz), np.arange(ny), np.arange(nx), indexing="ij")
    u = np.stack([i, j, k], -1) + v.D
    m = rng.random((nz, ny, nx)) < p
    v.tsdf[m] = world(u)[m]
    v.weight[m] += 1.0
    if intensity:
        v.cint[m] = rng.random(int(m.sum())).astype(np.float32)
        v.cw[m] += 1.0


def _model(dims):
    return StoreModel(dims, 0.05, (-1.0, -0.5, 0.25), 0.15, 64.0)


def _window(v):
    return [x.copy() for x in (v.tsdf, v.weight, v.cint, v.cw)]


def _same_window(a, b):
    return all(np.array_equal(x.view(u32), y.view(u32)) for x, y in zip(a, b))


def test_model_equals_shift_oracle_without_reentry():
    rng = np.random.default_rng(0x5701)
    dims = (37, 20, 29)
    m = _model(dims)
    o = vso.OracleVolume(dims, 0.05, (-1.0, -0.5, 0.25), 0.15, 64.0)
    for d in [(5, 3, 0), (9, 0, 2), (1, 1, 1), (40, 0, 0), (0, 7, 30), (3, 2, 1)]:   # every component >= 0
        paint(m, rng)
        o.tsdf, o.weight, o.cint, o.cw = _window(m)
        m.shift(d)
        o.shift(d)
        assert m.restored == 0
        assert _same_window(_window(m), [o.tsdf, o.weight, o.cint, o.cw]), d
        assert np.array_equal(m.origin.view(u32), o.origin.view(u32))
    assert len(m.bricks) > 0


def test_stored_bricks_follow_the_eviction_rule():
    rng = np.random.default_rng(0x5702)
    dims = (21, 16, 11)
    m = _model(dims)
    for d in [(3, 0, 0), (-5, 2, 0), (0, 0, -11), (7, -9, 4), (-3, 0, 0), (30, 30, 30), (-30, -30, -30)]:
        paint(m, rng, p=0.1)
        before = dict((c, r.copy()) for c, r in m.bricks.items())
        win, D = _window(m), m.D.copy()
        lo, hi = kept_box(dims, d)
        leave = moving(dims, lo, hi)
        want = set(before)
        expect = {}
        for k, j, i in zip(*np.nonzero(leave)):
            u = np.array([i, j, k], np.int64) + D
            c = tuple(int(x) for x in u // 8)
            if win[1][k, j, i] > 0:
                want.add(c)
            expect.setdefault(c, []).append((tuple(int(x) for x in u % 8), [w[k, j, i] for w in win]))
        m.shift(d)
        assert set(m.bricks) == want, d
        for c, vox in expect.items():
            if c not in want:
                continue
            r = m.bricks[c]
            for (lx, ly, lz), vals in vox:
                assert all(np.float32(r[q, lz, ly, lx]).view(u32) == np.float32(vals[q]).view(u32) for q in range(4))
            if c not in before:   # a new brick: its voxels that did not leave are (0, 0)
                left = np.zeros((8, 8, 8), bool)
                for (lx, ly, lz), _ in vox:
                    left[lz, ly, lx] = True
                assert not r[:, ~left].any()


@pytest.mark.parametrize("dims", [(21, 16, 11), (1, 9, 17)])
def test_round_trip_is_lossless(dims):
    rng = np.random.default_rng(0x5703 + dims[0])
    m = _model(dims)
    for _ in range(12):
        paint(m, rng, p=0.3)
        d = rng.integers(-2 * np.asarray(dims), 2 * np.asarray(dims) + 1)
        win = _window(m)
        m.shift(d)
        m.shift(-d)
        assert _same_window(win, _window(m)), d


def test_map_mesh_on_the_model_equals_the_dense_map():
    from rpg_open_remode_b200.api import TsdfVolume
    rng = np.random.default_rng(0x5704)
    dims = (17, 14, 12)
    m = _model(dims)
    for d in [(0, 0, 0), (9, 0, 0), (8, 5, 0), (-4, 3, 6), (-20, -8, 0), (6, 2, -5)]:
        m.shift(d)
        paint(m, rng, p=0.95, intensity=False)
    m.shift((2, 1, 0))
    win, D, (coords, rec) = _window(m), m.D.copy(), m.download_store()
    verts, tris, inten, nrm = TsdfVolume.mapMesh(m, intensity=True, normals=True)
    assert len(tris) > 100 and len(inten) == len(verts) == len(nrm)
    assert np.array_equal(m.D, D) and _same_window(win, _window(m))
    # the store keeps what it held; the bricks the sweep added hold nothing outside the window
    coords2, rec2 = m.download_store()
    old = np.array([tuple(c) in set(map(tuple, coords.tolist())) for c in coords2.tolist()], bool)
    assert np.array_equal(coords2[old], coords) and np.array_equal(rec2[old].view(u32), rec.view(u32))
    assert not rec2[~old].any()
    mesh_checks.open_edges(tris, len(verts))
    # the whole map as one dense grid
    lo, t, w = m.dense_map()
    g = smo.OracleVolume(t.shape[::-1], 0.05, (0.0, 0.0, 0.0), 0.15, 64.0)
    g.tsdf, g.weight = t, w
    g.cint, g.cw = np.zeros_like(t), np.zeros_like(w)
    dv, dt = g.mesh()
    dids = g.surfaceIds()
    dids[:, :3] += lo
    # mapMesh's ids, recomputed the same way: each vertex's id from the tile that first had it
    ids = _map_ids(m)
    assert len(ids) == len(verts) == len(dv)
    got = sorted(tuple(map(tuple, ids[t_])) for t_ in tris)
    want = sorted(tuple(map(tuple, dids[t_])) for t_ in dt)
    assert got == want


def _map_ids(m):
    """The ids of mapMesh's vertices in its order: the same sweep, keeping the ids."""
    from rpg_open_remode_b200.api import TsdfVolume
    ids = []
    real_mesh = m.mesh

    def mesh_with_ids():
        ids.append(m.surfaceIds())
        return real_mesh()

    m.mesh = mesh_with_ids
    try:
        TsdfVolume.mapMesh(m)
    finally:
        del m.mesh
    allids = np.concatenate(ids)
    _, first = np.unique(allids, axis=0, return_index=True)
    return allids[np.sort(first)]
