"""The ESDF oracle (oracle/rmd_oracle_volume_esdf.c) pinned on the CPU (DESIGN.md 4.8):

  * the snapshot against brute force (min over all sites, int64) on small grids: ragged sizes, nx = 1, a single site,
    empty O, empty F, all unknown, a checkerboard, -0.0 and NaN tsdf;
  * against scipy.ndimage.distance_transform_edt, squared and rounded, on a 64^3 grid fused from ground-truth frames by
    the volume oracle;
  * the query against a float64 trilinear function and its derivative, and the NaN / +-inf / outside rules.
"""
import numpy as np
import pytest

import volume_esdf_oracle as veo
import volume_oracle as vo
from test_volume import _grid

F = np.float32
u32 = np.uint32


def _brute_d2(occ):
    """Per voxel, the squared distance to the nearest voxel of the other set (int64; -1 when that set is empty)."""
    idx = np.argwhere(np.ones(occ.shape, bool))
    out = np.full(occ.shape, -1, np.int64)
    for want in (True, False):
        sites = np.argwhere(occ == want)
        mine = idx[(occ != want).reshape(-1)]
        if not len(sites) or not len(mine):
            continue
        d2 = ((mine[:, None, :] - sites[None, :, :]) ** 2).sum(-1).min(1)
        out[tuple(mine.T)] = d2
    return out


def _expected(tsdf, weight, s):
    occ = veo.occupied(tsdf, weight)
    d2 = _brute_d2(occ)
    dist = (np.sqrt(np.maximum(d2, 0).astype(F)) * F(s)).astype(F)
    dist[d2 < 0] = np.inf
    return np.where(occ, -dist, dist).astype(F)


def _grids():
    rng = np.random.default_rng(0x5EED0E5D)
    return veo.adversarial_grids(rng)


@pytest.mark.parametrize("name,tsdf,weight", _grids(), ids=[g[0] for g in _grids()])
def test_snapshot_equals_brute_force(name, tsdf, weight):
    s = F(0.05)
    dist, w = veo.esdf(tsdf, weight, s)
    want = _expected(tsdf, weight, s)
    assert np.array_equal(dist.view(u32), want.view(u32)), f"{name}: {(dist != want).sum()} voxels differ"
    assert np.array_equal(w.view(u32), weight.view(u32))
    occ = veo.occupied(tsdf, weight)
    if not occ.any():
        assert np.all(dist == np.inf)
    if occ.all():
        assert np.all(dist == -np.inf)


def test_random_grids_equal_brute_force():
    rng = np.random.default_rng(7)
    for _ in range(20):
        shape = tuple(int(x) for x in rng.integers(1, 12, 3))
        t = rng.uniform(-1, 1, shape).astype(F)
        w = (rng.random(shape) < rng.uniform(0.2, 1.0)).astype(F)
        t[rng.random(shape) < rng.uniform(0.0, 0.95)] = 1.0
        dist, _ = veo.esdf(t, w, F(0.1))
        want = _expected(t, w, F(0.1))
        assert np.array_equal(dist.view(u32), want.view(u32)), shape


def test_size_limit():
    with pytest.raises(ValueError):
        veo.esdf(np.ones((1, 4096, 4096), F), np.zeros((1, 4096, 4096), F), 0.1)
    # 4096 x 1 x 1: (nx - 1)^2 = 4095^2 < 2^24 is within it
    d, _ = veo.esdf(np.ones((1, 1, 4096), F), np.ones((1, 1, 4096), F), 0.1)
    assert np.all(d == np.inf)


def test_fused_grid_equals_scipy():
    from scipy import ndimage
    from rpg_open_remode_b200 import synth
    seq = synth.SyntheticSequence(160, 120, seed=0x5EED0E50)
    frames = [seq.frame(k) for k in (0, 20, 40)]
    s, origin, tau = _grid(seq, frames, 64)
    o = vo.OracleVolume((64, 64, 64), s, origin, tau, 64.0)
    for fr in frames:
        o.integrate(fr.depth, seq.camera, fr.T_cam_world)
    occ = veo.occupied(o.tsdf, o.weight)
    assert 0 < occ.sum() < occ.size // 2 and (o.weight == 0).any()
    dist, w = veo.esdf(o.tsdf, o.weight, s)
    d2 = np.where(occ, np.rint(ndimage.distance_transform_edt(occ) ** 2),
                  np.rint(ndimage.distance_transform_edt(~occ) ** 2)).astype(np.int64)
    want = (np.sqrt(d2.astype(F)) * F(s)).astype(F)
    want = np.where(occ, -want, want)
    assert np.array_equal(dist.view(u32), want.view(u32)), f"{(dist != want).sum()} voxels differ"
    assert np.array_equal(w.view(u32), o.weight.view(u32))


def _trilinear64(dist, s, origin, p):
    """float64 trilinear value and gradient (per metre) at points p inside the grid."""
    u = (p.astype(np.float64) - origin.astype(np.float64)) / float(s)
    c = np.floor(u).astype(np.int64)
    f = u - c
    e = np.empty((len(p), 2, 2, 2))   # [z][y][x]
    for dz in (0, 1):
        for dy in (0, 1):
            for dx in (0, 1):
                e[:, dz, dy, dx] = dist[c[:, 2] + dz, c[:, 1] + dy, c[:, 0] + dx]
    fx, fy, fz = f[:, 0, None, None], f[:, 1, None], f[:, 2]
    ex = e[:, :, :, 0] * (1 - fx[..., 0:1]) + e[:, :, :, 1] * fx[..., 0:1]   # [z][y]
    ey = ex[:, :, 0] * (1 - fy) + ex[:, :, 1] * fy                             # [z]
    val = ey[:, 0] * (1 - fz) + ey[:, 1] * fz
    gx = ((e[:, :, :, 1] - e[:, :, :, 0])[:, :, 0] * (1 - fy) + (e[:, :, :, 1] - e[:, :, :, 0])[:, :, 1] * fy)
    gx = gx[:, 0] * (1 - fz) + gx[:, 1] * fz
    fxx = f[:, 0, None]
    gy = (e[:, :, 1, :] - e[:, :, 0, :])[:, :, 0] * (1 - fxx) + (e[:, :, 1, :] - e[:, :, 0, :])[:, :, 1] * fxx
    gy = gy[:, 0] * (1 - fz) + gy[:, 1] * fz
    gz = (e[:, 1] - e[:, 0])[:, :, 0] * (1 - fxx) + (e[:, 1] - e[:, 0])[:, :, 1] * fxx
    gz = gz[:, 0] * (1 - f[:, 1]) + gz[:, 1] * f[:, 1]
    return val, np.stack([gx, gy, gz], 1) / float(s)


def test_query_against_float64():
    rng = np.random.default_rng(11)
    shape = (9, 13, 17)
    t = np.ones(shape, F)
    t[rng.random(shape) < 0.08] = -0.5
    w = rng.integers(1, 9, shape).astype(F)
    w[0, 0, 0] = 0
    s, origin = F(0.07), np.array([-0.4, 0.3, 1.1], F)
    dist, ww = veo.esdf(t, w, s)
    n = np.array(shape[::-1])
    p = (origin + rng.uniform(0, 1, (5000, 3)) * (n - 1) * s).astype(F)
    dg, wq = veo.query(dist, ww, s, origin, p)
    inside = np.isfinite(dg[:, 0])
    assert inside.mean() > 0.99
    val, grad = _trilinear64(dist, s, origin, p[inside])
    scale = float(np.abs(dist).max())
    assert np.abs(dg[inside, 0] - val).max() <= 8 * np.finfo(F).eps * scale
    assert np.abs(dg[inside, 1:] - grad).max() <= 32 * np.finfo(F).eps * scale / float(s)
    # weight: min of the 8 corners
    u = np.floor((p[inside].astype(np.float64) - origin) / float(s)).astype(np.int64)
    wm = np.full(len(u), np.inf)
    for dz in (0, 1):
        for dy in (0, 1):
            for dx in (0, 1):
                wm = np.minimum(wm, ww[u[:, 2] + dz, u[:, 1] + dy, u[:, 0] + dx])
    assert np.array_equal(wq[inside], wm.astype(F))
    assert (wq == 0).any()


def test_query_rules():
    shape = (4, 5, 6)
    s, origin = F(0.25), np.array([1.0, -2.0, 0.5], F)
    t = np.ones(shape, F)
    t[2, 2, 2] = -1
    dist, w = veo.esdf(t, np.ones(shape, F), s)
    n = np.array(shape[::-1])
    last = origin + (n - 1) * s            # exactly on the last voxel plane of every axis
    mid = origin + 1.5 * s
    pts = np.array([mid, last, [last[0], mid[1], mid[2]], origin, [np.nan, mid[1], mid[2]],
                    [np.inf, mid[1], mid[2]], origin - F(0.01)], F)
    dg, wq = veo.query(dist, w, s, origin, pts)
    assert np.isfinite(dg[0]).all() and wq[0] == 1
    for q in (1, 2, 4, 5, 6):             # outside: NaN (the kernels' 0x7fffffff), gradient 0, weight 0
        assert dg[q].view(u32)[0] == 0x7fffffff and not dg[q, 1:].any() and wq[q] == 0, q
    assert np.isfinite(dg[3, 0])           # the first voxel centre is inside
    # +-inf snapshots: the corner's value, gradient 0
    for sign, tt in ((1, np.ones(shape, F)), (-1, -np.ones(shape, F))):
        d, ww = veo.esdf(tt, np.ones(shape, F), s)
        g, _ = veo.query(d, ww, s, origin, pts[:1])
        assert g[0, 0] == sign * np.inf and not g[0, 1:].any()
