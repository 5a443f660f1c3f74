"""The moving-volume oracle (oracle/rmd_oracle_volume_shift.c, DESIGN.md 4.8) pinned against numpy, on the CPU.

  * a shift is slicing with unknown fill, on random ragged grids (down to nx = 1) with the intensity channel, for
    every sign pattern of d, d = 0 and |d| >= n;
  * the spill is the numpy surface points filtered by the rule "voxel a or neighbour b outside the kept box", bit
    for bit, and so are its intensities and normals (filtered from the surface oracles);
  * on an exact grid (power-of-two voxel, origin a small multiple of it): surface after the shift + spill = surface
    before, bit for bit and in order; and integrate, shift, integrate = a large fixed volume's window;
  * many small shifts give the same origin as one large shift.
"""
import itertools

import numpy as np
import pytest

import volume_shift_oracle as vso

F = np.float32
u32 = np.uint32


def _np_shift(a, d):
    """numpy slicing: out[k, j, i] = a[k + dz, j + dy, i + dx] where inside, else 0."""
    out = np.zeros_like(a)
    src, dst = [], []
    for n, dd in zip(a.shape[::-1], d):   # x, y, z
        lo, hi = max(0, dd), min(n, n + dd)
        if lo >= hi:
            return out
        src.append(slice(lo, hi))
        dst.append(slice(lo - dd, hi - dd))
    out[dst[2], dst[1], dst[0]] = a[src[2], src[1], src[0]]
    return out


def _np_surface(tsdf, weight, s, origin):
    """Surface points (float32 numpy, one rounding per operation) in voxel order then axis, with their voxel a
    (i, j, k) and axis."""
    nz, ny, nx = tsdf.shape
    near = (weight > 0) & (np.abs(tsdf) < 1)
    keys, pts, vox, axes = [], [], [], []
    kk, jj, ii = np.meshgrid(np.arange(nz), np.arange(ny), np.arange(nx), indexing="ij")
    for axis in range(3):
        sl_a = [slice(None)] * 3
        sl_b = [slice(None)] * 3
        sl_a[2 - axis] = slice(0, -1)
        sl_b[2 - axis] = slice(1, None)
        ta, tb = tsdf[tuple(sl_a)], tsdf[tuple(sl_b)]
        ok = near[tuple(sl_a)] & near[tuple(sl_b)] & (((ta > 0) & (tb <= 0)) | ((ta <= 0) & (tb > 0)))
        i, j, k = ii[tuple(sl_a)][ok], jj[tuple(sl_a)][ok], kk[tuple(sl_a)][ok]
        p = np.stack([F(origin[0]) + i.astype(F) * F(s), F(origin[1]) + j.astype(F) * F(s),
                      F(origin[2]) + k.astype(F) * F(s)], 1).astype(F)
        p[:, axis] = p[:, axis] + (ta[ok] / (ta[ok] - tb[ok])) * F(s)
        w = np.minimum(weight[tuple(sl_a)][ok], weight[tuple(sl_b)][ok])
        pts.append(np.concatenate([p, w[:, None]], 1))
        keys.append(3 * ((k.astype(np.int64) * ny + j) * nx + i) + axis)
        vox.append(np.stack([i, j, k], 1))
        axes.append(np.full(len(i), axis))
    keys = np.concatenate(keys)
    order = np.argsort(keys, kind="stable")
    return np.concatenate(pts)[order], np.concatenate(vox)[order], np.concatenate(axes)[order]


def _spill_mask(vox, axes, dims, d):
    n, d = np.array(dims), np.asarray(d)
    lo, hi = np.maximum(0, d), np.minimum(n, n + d)
    b = vox + np.eye(3, dtype=np.int64)[axes]
    return ~(np.all((vox >= lo) & (vox < hi), 1) & np.all((b >= lo) & (b < hi), 1))


def _random_volume(rng, dims, s=0.05, origin=(0.3, -0.7, 1.1)):
    """An oracle volume with random records: a noisy band around a tilted plane, unknown patches and free space, and
    a random intensity channel."""
    o = vso.OracleVolume(dims, s, origin, 4 * s, 64.0)
    nx, ny, nz = dims
    k, j, i = np.meshgrid(np.arange(nz), np.arange(ny), np.arange(nx), indexing="ij")
    t = np.clip((0.6 * i + 0.5 * j + 0.7 * k - 0.3 * (nx + ny + nz)) / 3.0 + rng.normal(0, 0.3, i.shape), -1.2, 1.2)
    o.tsdf = np.ascontiguousarray(t.astype(F))
    o.weight = np.where(rng.random(i.shape) < 0.85, rng.integers(1, 20, i.shape), 0).astype(F)
    o.cint = rng.random(i.shape).astype(F)
    o.cw = np.where(rng.random(i.shape) < 0.8, rng.integers(1, 20, i.shape), 0).astype(F)
    return o


RAGGED = [(1, 7, 5), (9, 1, 6), (5, 6, 1), (13, 11, 9), (17, 3, 12)]
SIGNS = list(itertools.product((-1, 0, 1), repeat=3))


@pytest.mark.parametrize("dims", RAGGED)
def test_shift_is_slicing(dims):
    rng = np.random.default_rng(sum(dims))
    o = _random_volume(rng, dims)
    for sign in SIGNS:
        for mag in (1, 2):
            d = tuple(int(sg * min(mag, n)) for sg, n in zip(sign, dims))
            for a in (o.tsdf, o.weight, o.cint, o.cw):
                got, _ = vso.shift_records(a, a, d)
                assert np.array_equal(got.view(u32), _np_shift(a, d).view(u32)), (dims, d)
    for d in ((0, 0, 0), (dims[0], 0, 0), (0, -dims[1], 0), (0, 0, dims[2] + 5), (-3 * dims[0], 2, -1)):
        got_t, got_w = vso.shift_records(o.tsdf, o.weight, d)
        assert np.array_equal(got_t.view(u32), _np_shift(o.tsdf, d).view(u32)), d
        assert np.array_equal(got_w, _np_shift(o.weight, d)), d
        if d == (0, 0, 0):
            assert np.array_equal(got_t.view(u32), o.tsdf.view(u32))
        else:
            assert not got_w.any()   # |d| >= n on an axis: everything leaves


@pytest.mark.parametrize("dims", RAGGED[3:] + [(24, 20, 16)])
def test_spill_is_the_filtered_surface(dims):
    rng = np.random.default_rng(7 * sum(dims))
    o = _random_volume(rng, dims)
    pts, vox, axes = _np_surface(o.tsdf, o.weight, o.s, o.origin)
    want_pts, n = o.surface_points()
    assert n == len(pts) > 50 and np.array_equal(want_pts.view(u32), pts.view(u32))
    inten, _ = o.surface_intensity()
    nrm, _ = o.surface_normals()
    ds = [tuple(int(sg * m) for sg, m in zip(sign, (2, 1, 3))) for sign in SIGNS] + \
         [(dims[0], 0, 0), (0, 0, -dims[2]), (-1, 40, 0)]
    for d in ds:
        m = _spill_mask(vox, axes, dims, d)
        got, cnt = o.spill(d, vso.POINTS)
        assert cnt == m.sum() and np.array_equal(got.view(u32), pts[m].view(u32)), d
        got, cnt = o.spill(d, vso.INTENSITY)
        assert cnt == m.sum() and np.array_equal(got.view(u32), inten[m].view(u32)), d
        got, cnt = o.spill(d, vso.NORMALS)
        assert cnt == m.sum() and np.array_equal(got.view(u32), nrm[m].view(u32)), d
        if d == (0, 0, 0):
            assert cnt == 0
        cap = cnt // 3
        part, cnt2 = o.spill(d, vso.POINTS, capacity=cap)
        assert cnt2 == cnt and np.array_equal(part.view(u32), pts[m][:cap].view(u32))


def _exact_volume(rng, dims):
    """Voxel 2^-4 m and an origin of small multiples of it: o + i s is exact, so positions survive a shift."""
    s = F(2.0 ** -4)
    o = _random_volume(rng, dims, s=s, origin=(F(-3) * s, F(5) * s, F(16) * s))
    return o


@pytest.mark.parametrize("d", [(2, 0, 0), (-3, 1, 0), (0, -2, 4), (5, 5, -5), (1, -1, 1)])
def test_exact_grid_partition(d):
    rng = np.random.default_rng(abs(hash(d)) % 2**32)
    o = _exact_volume(rng, (20, 18, 16))
    before, n = o.surface_points()
    before_i, _ = o.surface_intensity()
    _, vox, axes = _np_surface(o.tsdf, o.weight, o.s, o.origin)
    m = _spill_mask(vox, axes, o.dims, d)
    spill, ns = o.spill(d, vso.POINTS)
    spill_i, _ = o.spill(d, vso.INTENSITY)
    o.shift(d)
    after, na = o.surface_points()
    after_i, _ = o.surface_intensity()
    assert ns + na == n and ns > 0 and na > 0
    # the spill and the shifted grid's points interleave back into the points before, in order
    assert np.array_equal(before[m].view(u32), spill.view(u32))
    assert np.array_equal(before[~m].view(u32), after.view(u32))
    assert np.array_equal(before_i[m].view(u32), spill_i.view(u32))
    assert np.array_equal(before_i[~m].view(u32), after_i.view(u32))


def _plane_depth(cam, T_cam_world, w, h, z0):
    """Distance along each ray to the tilted plane z = z0 + 0.1 x - 0.05 y (world; camera at the world origin,
    looking down +z), float32."""
    fx, fy, cx, cy = cam
    yy, xx = np.mgrid[0:h, 0:w].astype(np.float64)
    r = np.stack([(xx - cx) / fx, (yy - cy) / fy, np.ones_like(xx)], -1)
    r /= np.linalg.norm(r, axis=-1, keepdims=True)
    T = np.asarray(T_cam_world, np.float64).reshape(3, 4)
    R, t = T[:, :3].T, -T[:, :3].T @ T[:, 3]    # camera -> world
    dw = r @ R.T
    # t + l dw on the plane: (t_z + l dw_z) = z0 + 0.1 (t_x + l dw_x) - 0.05 (t_y + l dw_y)
    num = z0 + 0.1 * t[0] - 0.05 * t[1] - t[2]
    den = dw[..., 2] - 0.1 * dw[..., 0] + 0.05 * dw[..., 1]
    return (num / den).astype(F)


def _pose(tx):
    T = np.zeros((3, 4), F)
    T[:, :3] = np.eye(3, dtype=F)
    T[0, 3] = F(-tx)   # world -> camera of a camera at (tx, 0, 0)
    return T


def test_integrate_shift_integrate_is_a_window_of_a_fixed_volume():
    s = F(2.0 ** -5)
    cam = (60.0, 60.0, 39.5, 29.5)
    W, H = 80, 60
    big_dims, dims, off = (96, 40, 48), (40, 40, 48), np.array([10, 0, 0])
    o_big = F(-48) * s, F(-20) * s, F(16) * s
    later_only = vso.OracleVolume(big_dims, s, o_big, 4 * s, 64.0)
    big = vso.OracleVolume(big_dims, s, o_big, 4 * s, 64.0)
    small_origin = [F(o_big[a] + F(off[a]) * s) for a in range(3)]
    small = vso.OracleVolume(dims, s, small_origin, 4 * s, 64.0)
    d1 = np.array([7, 0, 0])
    T1, T2 = _pose(0.0), _pose(0.25)
    D1, D2 = _plane_depth(cam, T1, W, H, 1.0), _plane_depth(cam, T2, W, H, 1.05)
    I1, I2 = np.full((H, W), 0.25, F), np.full((H, W), 0.75, F)
    for v in (big, small):
        v.integrate(D1, cam, T1, None, I1)
    small.shift(d1)
    for v in (big, small, later_only):
        v.integrate(D2, cam, T2, None, I2)
    assert np.array_equal(small.origin, [F(o_big[a] + F((off + d1)[a]) * s) for a in range(3)])
    lo = off + d1
    win = tuple(slice(lo[a], lo[a] + dims[a]) for a in (2, 1, 0))
    # voxels in both windows (pre-shift x in [off + d1, off + n)): the big volume's records
    n_old = dims[0] - d1[0]
    for mine, ref_all, ref_later in ((small.tsdf, big.tsdf, later_only.tsdf),
                                     (small.weight, big.weight, later_only.weight),
                                     (small.cint, big.cint, later_only.cint), (small.cw, big.cw, later_only.cw)):
        ref, ref2 = ref_all[win], ref_later[win]
        assert np.array_equal(mine[..., :n_old].view(u32), ref[..., :n_old].view(u32))
        assert np.array_equal(mine[..., n_old:].view(u32), ref2[..., n_old:].view(u32))
    assert (small.weight[..., :n_old] > 1).any() and (small.weight[..., n_old:] > 0).any()
    assert len(small.surface_points()[0]) > 100


def test_many_small_shifts_give_the_origin_of_one():
    s, o0 = F(0.0137), (F(0.123), F(-4.56), F(7.89))
    rng = np.random.default_rng(3)
    steps = rng.integers(-9, 10, (200, 3))
    D = np.zeros(3, np.int64)
    for st in steps:
        D += st
    want = vso.shift_origin(o0, D, s)
    assert np.array_equal(want, (np.array(o0, F) + D.astype(F) * s).astype(F))
    a = vso.OracleVolume((6, 5, 4), s, o0, 4 * s, 64.0)
    b = vso.OracleVolume((6, 5, 4), s, o0, 4 * s, 64.0)
    for st in steps:
        a.shift(st)
    b.shift(D)
    assert np.array_equal(a.origin.view(u32), b.origin.view(u32)) and np.array_equal(a.origin, want)
    # accumulating the steps in float instead drifts
    acc = np.array(o0, F)
    for st in steps:
        acc = (acc + st.astype(F) * s).astype(F)
    assert not np.array_equal(acc, want)
