"""The checker of the TSDF volume's normals (oracle/rmd_oracle_volume_normals.c, bound by volume_normals_oracle.py;
DESIGN.md 4.8), on the CPU.

As for the volume oracle: pinned against an independent numpy float32 evaluation (correctly rounded, so equality is
exact) on random ragged grids whose records mix unknown voxels, truncated +-1 voxels and exact zeros, and against
known answers (a linear field, an analytic sphere, the sphere's mesh).  Then what the normals give is measured on the
synthetic sequence's ground truth: a view that was not fused, against normals of the frame's true depth.  Also the
PLY writer's normals.
"""
import numpy as np
import pytest

import mesh_checks as mc
import mesh_oracle as mo
import volume_normals_oracle as vno
from test_volume_oracle import SPHERE, _pose, _random_case, _rot, _sphere, ground_truth_points, scene_grid

F = np.float32
u32 = np.uint32


# ------------------------------------------------------------------ numpy float32 restatement
def _numpy_gradients(tsdf, weight):
    """float32 (nz, ny, nx, 3): the gradient rule of every voxel."""
    g = np.zeros(tsdf.shape + (3,), F)
    for axis in range(3):
        ax = 2 - axis
        lo, hi = [slice(None)] * 3, [slice(None)] * 3
        lo[ax], hi[ax] = slice(0, -1), slice(1, None)
        lo, hi = tuple(lo), tuple(hi)
        tp, tm = np.zeros_like(tsdf), np.zeros_like(tsdf)
        up, dn = np.zeros(tsdf.shape, bool), np.zeros(tsdf.shape, bool)
        tp[lo], up[lo] = tsdf[hi], weight[hi] > 0
        tm[hi], dn[hi] = tsdf[lo], weight[lo] > 0
        with np.errstate(invalid="ignore", over="ignore"):
            g[..., axis] = np.where(up & dn, (tp - tm) * F(0.5),
                                    np.where(up, tp - tsdf, np.where(dn, tsdf - tm, F(0))))
    return g


def _numpy_unit(g):
    """g [..., 3] -> [..., 4] (g / len, 0), zero where len is 0 or not finite."""
    with np.errstate(invalid="ignore", over="ignore", divide="ignore"):
        ln = np.sqrt((g[..., 0] * g[..., 0] + g[..., 1] * g[..., 1]) + g[..., 2] * g[..., 2])
        ok = (ln > 0) & np.isfinite(ln)
        out = np.zeros(g.shape[:-1] + (4,), F)
        out[..., :3] = np.where(ok[..., None], g / np.where(ok, ln, F(1))[..., None], F(0))
    return out


def _numpy_surface_normals(tsdf, weight):
    nz, ny, nx = tsdf.shape
    G = _numpy_gradients(tsdf, weight)
    k, j, i = np.meshgrid(np.arange(nz), np.arange(ny), np.arange(nx), indexing="ij")
    lin = ((k * ny + j) * nx + i).astype(np.int64)
    near = (weight > 0) & (np.abs(tsdf) < 1)
    keys, vals = [], []
    for axis in range(3):
        a, b = [slice(None)] * 3, [slice(None)] * 3
        a[2 - axis], b[2 - axis] = slice(0, -1), slice(1, None)
        a, b = tuple(a), tuple(b)
        ta, tb = tsdf[a], tsdf[b]
        sel = near[a] & near[b] & (((ta > 0) & (tb <= 0)) | ((ta <= 0) & (tb > 0)))
        f = (ta[sel] / (ta[sel] - tb[sel]))[:, None]
        ga, gb = G[a][sel], G[b][sel]
        vals.append(_numpy_unit(ga + f * (gb - ga)))
        keys.append(lin[a][sel] * 3 + axis)
    keys, vals = np.concatenate(keys), np.concatenate(vals)
    return vals[np.argsort(keys, kind="stable")]


def _hit_grid_coords(s, origin, cam, T_curr_world, depth):
    """Grid coordinates of every pixel's org + depth * dir, in the march's form (float32)."""
    h, w = depth.shape
    fx, fy, cx, cy = (F(c) for c in cam)
    T = np.asarray(vno.vo.pose_inverse(T_curr_world), F)
    yy, xx = np.mgrid[0:h, 0:w].astype(F)
    vx, vy = (xx - cx) / fx, (yy - cy) / fy
    inv_len = F(1) / np.sqrt((vx * vx + vy * vy) + F(1))
    q = (vx * inv_len, vy * inv_len, F(1) * inv_len)
    dirs = [(T[r, 0] * q[0] + T[r, 1] * q[1]) + T[r, 2] * q[2] for r in range(3)]
    o = np.asarray(origin, F)
    return [((T[r, 3] + depth * dirs[r]) - o[r]) / F(s) for r in range(3)], np.stack(dirs, -1)


def _numpy_raycast_normals(tsdf, weight, s, origin, cam, T_curr_world, depth):
    """(normals [h, w, 4] at every hit of `depth` (the volume oracle's raycast), mask of hits whose cell has a corner
    outside the grid or unknown), in numpy float32."""
    nz, ny, nx = tsdf.shape
    h, w = depth.shape
    g, _ = _hit_grid_coords(s, origin, cam, T_curr_world, depth)
    x0, y0, z0 = (np.floor(c) for c in g)
    hit = depth > 0
    with np.errstate(invalid="ignore"):
        ok = hit & (x0 >= 0) & (y0 >= 0) & (z0 >= 0) & (x0 + 1 < nx) & (y0 + 1 < ny) & (z0 + 1 < nz)
    in_grid = ok.copy()
    i0, j0, k0 = (np.where(ok, c, 0).astype(np.int64) for c in (x0, y0, z0))
    G = _numpy_gradients(tsdf, weight)
    c = {}
    for dz in (0, 1):
        for dy in (0, 1):
            for dx in (0, 1):
                idx = (np.minimum(k0 + dz, nz - 1), np.minimum(j0 + dy, ny - 1), np.minimum(i0 + dx, nx - 1))
                ok &= weight[idx] != 0
                c[dx, dy, dz] = G[idx]
    fxx, fyy, fzz = ((g[0] - x0)[..., None], (g[1] - y0)[..., None], (g[2] - z0)[..., None])

    def lerp(a, b, f):
        return a + f * (b - a)
    with np.errstate(invalid="ignore", over="ignore"):
        c00, c10 = lerp(c[0, 0, 0], c[1, 0, 0], fxx), lerp(c[0, 1, 0], c[1, 1, 0], fxx)
        c01, c11 = lerp(c[0, 0, 1], c[1, 0, 1], fxx), lerp(c[0, 1, 1], c[1, 1, 1], fxx)
        v = lerp(lerp(c00, c10, fyy), lerp(c01, c11, fyy), fzz)
    out = np.zeros((h, w, 4), F)
    out[ok] = _numpy_unit(v[ok])
    return out, in_grid & ~ok


def _usable(weight, axis):
    """(+ neighbour usable, - neighbour usable) of every voxel along axis (0 = x)."""
    ax = 2 - axis
    lo, hi = [slice(None)] * 3, [slice(None)] * 3
    lo[ax], hi[ax] = slice(0, -1), slice(1, None)
    up, dn = np.zeros(weight.shape, bool), np.zeros(weight.shape, bool)
    up[tuple(lo)], dn[tuple(hi)] = weight[tuple(hi)] > 0, weight[tuple(lo)] > 0
    return up, dn


def _perturb(rng, o):
    """Mix unknown voxels, truncated +-1 voxels and exact zeros into an integrated grid."""
    known = o.weight > 0
    r = rng.random(o.tsdf.shape)
    o.weight[known & (r < 0.04)] = 0
    o.tsdf[known & (r >= 0.04) & (r < 0.07)] = 1
    o.tsdf[known & (r >= 0.07) & (r < 0.09)] = -1
    o.tsdf[known & (r >= 0.09) & (r < 0.11)] = 0
    o.tsdf[known & (r >= 0.11) & (r < 0.12)] = -0.0


@pytest.mark.parametrize("dims,size,seed", [((37, 29, 23), (61, 47), 1), ((64, 48, 40), (160, 120), 2),
                                            ((97, 64, 71), (96, 72), 3), ((1, 50, 33), (40, 30), 4),
                                            ((45, 1, 30), (40, 30), 5)])
def test_oracle_normals_equal_numpy_float32(dims, size, seed):
    rng = np.random.default_rng(0x90C0 + seed)
    s, origin, cam, T, depth, _ = _random_case(rng, dims, size)
    # a smooth surface (so that rays find crossings) with the random case's invalid pixels
    w, h = size
    yy, xx = np.mgrid[0:h, 0:w]
    smooth = F(1.2 * dims[2] * s) * (1 + 0.15 * np.sin(xx / 7.0 + rng.uniform(0, 6)) * np.cos(yy / 5.0))
    depth = np.where(np.isfinite(depth) & (depth > 0), smooth, depth).astype(F)
    o = vno.OracleVolume(dims, s, origin, F(3.0) * s, 5.0)
    for rep in range(4):
        if rep:
            depth = (depth * F(rng.uniform(0.97, 1.03))).astype(F)
        o.integrate(depth, cam, T)
    _perturb(rng, o)
    G = _numpy_gradients(o.tsdf, o.weight)
    assert np.array_equal(o.gradients().view(u32), G.view(u32))
    # every branch of the rule is taken on known voxels: both, only +, only - and no usable neighbour
    for axis in range(3):
        if dims[axis] > 2:
            up, dn = _usable(o.weight, axis)
            known = o.weight > 0
            for sel in (up & dn, up & ~dn, ~up & dn, ~up & ~dn):
                assert (known & sel).sum() > 0
    got, n = o.surface_normals()
    want = _numpy_surface_normals(o.tsdf, o.weight)
    assert n == len(want) == len(o.surface_points()[0]) > 0
    assert np.array_equal(got.view(u32), want.view(u32))
    nonzero = np.abs(got[:, :3]).sum(1) > 0
    assert nonzero.mean() > 0.9
    assert np.allclose(np.linalg.norm(got[nonzero, :3].astype(np.float64), axis=1), 1, atol=1e-6)
    assert np.all(got[:, 3] == 0)
    part, n2 = o.surface_normals(capacity=n // 3)
    assert n2 == n and np.array_equal(part.view(u32), want[:n // 3].view(u32))
    w, h = size
    d_o, n_o = o.raycast_normals(cam, T, w, h)
    assert np.array_equal(d_o.view(u32), o.raycast(cam, T, w, h).view(u32))
    want, unknown_corner = _numpy_raycast_normals(o.tsdf, o.weight, s, origin, cam, T, d_o)
    assert np.array_equal(n_o.view(u32), want.view(u32))
    assert not n_o[d_o == 0].any()                     # no hit: (0, 0, 0, 0)
    assert not n_o[unknown_corner].any()               # a hit whose cell has an unknown corner: (0, 0, 0, 0)
    if min(dims[0], dims[1]) > 1:
        assert (d_o > 0).sum() > 20 and (np.abs(n_o[..., :3]).sum(-1) > 0).sum() > 10


# ------------------------------------------------------------------ known answers
ULP1 = 2.0 ** -23
LINEAR_MAX_ULPS = 4      # measured: at most 0.7 ulp


@pytest.mark.parametrize("seed", [1, 2, 3])
def test_known_answer_linear_field(seed):
    """t = n.(p - p0) / tau: every surface normal and every raycast normal is n within a few ulp."""
    rng = np.random.default_rng(0x11E0 + seed)
    n = rng.normal(size=3)
    n /= np.linalg.norm(n)
    dims, s, origin = (24, 22, 20), 0.05, np.array([-0.6, -0.55, 1.0], F)
    tau = 8 * s                                        # no clamping within 8 voxels of the plane
    p0 = origin.astype(np.float64) + np.array(dims) * s / 2 + rng.uniform(-0.02, 0.02, 3)
    (x, y, z) = np.meshgrid(*(origin[a] + np.arange(dims[a]) * np.float64(np.float32(s)) for a in range(3)),
                            indexing="ij")
    t = ((x - p0[0]) * n[0] + (y - p0[1]) * n[1] + (z - p0[2]) * n[2]) / tau
    o = vno.OracleVolume(dims, s, origin, tau, 64.0)
    o.tsdf[...] = np.clip(t, -1, 1).transpose(2, 1, 0).astype(F)
    o.weight[...] = 1
    got, cnt = o.surface_normals()
    assert cnt > 300
    err = np.abs(got[:, :3] - n).max() / ULP1
    cam = (60.0, 60.0, 31.5, 23.5)
    R = _rot(rng, 0.1)
    cam_pos = p0 + n * 1.0                             # on the free side (t > 0), looking at p0
    zc = (p0 - cam_pos) / np.linalg.norm(p0 - cam_pos)
    xc = np.cross(R[1], zc)
    xc /= np.linalg.norm(xc)
    Rw = np.stack([xc, np.cross(zc, xc), zc])          # rows: the camera axes in the world
    depth, nr = o.raycast_normals(cam, _pose(Rw, -Rw @ cam_pos), 64, 48)
    hit = np.abs(nr[..., :3]).sum(-1) > 0
    assert hit.sum() > 1000 and hit.sum() >= 0.95 * (depth > 0).sum()
    err_r = np.abs(nr[hit][:, :3] - n).max() / ULP1
    print(f"\nlinear field: max |normal - n| = {err:.1f} ulp (surface), {err_r:.1f} ulp (raycast)")
    assert err <= LINEAR_MAX_ULPS and err_r <= LINEAR_MAX_ULPS


# The analytic sphere of test_volume_oracle (R = 10 m, s = 1 cm).  Measured, away from the grid's faces: the largest
# angle between a normal and the radial direction is 1.27e-6 rad for the surface points and 1.14e-6 rad for the
# raycast, while voxel a's gradient alone is 1.0e-3 rad off (the normal turns by s / R = 1e-3 rad per voxel).  At the
# faces, where differences are one-sided, 7.1e-4 rad.
SPHERE_MAX_ANGLE = 2e-5
SPHERE_MAX_ANGLE_FACES = 1e-3


def _angles(a, b):
    a = np.asarray(a, np.float64)[..., :3]
    b = np.asarray(b, np.float64)[..., :3]
    a = a / np.linalg.norm(a, axis=-1, keepdims=True)
    b = b / np.linalg.norm(b, axis=-1, keepdims=True)
    return np.arccos(np.clip((a * b).sum(-1), -1, 1))


def test_known_answer_sphere_is_radial():
    S = SPHERE
    o = vno.OracleVolume(S["dims"], S["s"], S["origin"], S["tau"], 10.0)
    o.tsdf[...], o.weight[...] = _sphere(S["dims"], S["s"], S["origin"], S["centre"], S["radius"], S["tau"])
    pts, n = o.surface_points()
    nrm, n2 = o.surface_normals()
    assert n == n2 > 1000
    radial = pts[:, :3].astype(np.float64) - np.asarray(S["centre"])
    ang = _angles(nrm, radial)
    # away from the grid's faces every gradient is a central difference (one-sided ones are first order there)
    ijk, axis = mc.surface_point_edges(o.tsdf, o.weight)
    hi = np.array(S["dims"]) - 2
    inner = np.all((ijk >= 1) & (ijk + np.eye(3, dtype=int)[axis] <= hi), axis=1)
    # the rejected variant: voxel a's gradient alone, no interpolation towards b
    ga = o.gradients()[ijk[:, 2], ijk[:, 1], ijk[:, 0]]
    ang_a = _angles(ga, radial)
    cam = (80.0, 80.0, 23.5, 19.5)
    T_world_cam = _pose(_rot(np.random.default_rng(5), 0.02), [0.01, -0.02, 0.0])
    T_cam_world = vno.vo.pose_inverse(T_world_cam)
    depth, nr = o.raycast_normals(cam, T_cam_world, 48, 40)
    hit = depth > 0
    g, dirs = _hit_grid_coords(S["s"], S["origin"], cam, T_cam_world, depth)
    p = np.stack([S["origin"][a] + g[a].astype(np.float64) * np.float32(S["s"]) for a in range(3)], -1)
    ang_r = _angles(nr[hit], p[hit] - np.asarray(S["centre"]))
    cell = np.stack([np.floor(c[hit]) for c in g], -1)
    inner_r = np.all((cell >= 1) & (cell + 2 <= np.array(S["dims"]) - 1), axis=1)
    print(f"\nsphere: max angle to radial {ang[inner].max():.2e} rad inside / {ang.max():.2e} rad at the faces "
          f"(surface, {inner.sum()} / {n} points), {ang_r[inner_r].max():.2e} / {ang_r.max():.2e} rad (raycast, "
          f"{inner_r.sum()} / {hit.sum()} hits); voxel a's gradient alone {ang_a[inner].max():.2e} rad inside")
    assert hit.mean() > 0.9 and np.all(np.abs(nr[hit][:, :3]).sum(-1) > 0)
    assert inner.sum() > 1000 and inner_r.sum() > 1000
    assert ang[inner].max() <= SPHERE_MAX_ANGLE and ang_r[inner_r].max() <= SPHERE_MAX_ANGLE
    assert ang.max() <= SPHERE_MAX_ANGLE_FACES and ang_r.max() <= SPHERE_MAX_ANGLE_FACES
    assert ang_a[inner].max() > 5 * SPHERE_MAX_ANGLE
    # outward: towards the camera, which is outside the sphere
    assert np.all((nr[hit][:, :3] * dirs[hit]).sum(-1) < 0)


def test_known_answer_mesh_faces_agree_with_vertex_normals():
    """Every triangle of the closed sphere's mesh faces the same side as its three vertex normals."""
    from test_volume_mesh_oracle import SPHERE as MS
    for tau_voxels in (2.0, 5.0):
        tsdf, weight = mc.sphere_field(MS["dims"], MS["s"], MS["origin"], MS["centre"], MS["radius"],
                                       tau_voxels * MS["s"])
        o = mo.OracleVolume(MS["dims"], MS["s"], MS["origin"], tau_voxels * MS["s"], 64.0)
        o.tsdf[...], o.weight[...] = tsdf, weight
        verts, tris = o.mesh()
        on = vno.OracleVolume(MS["dims"], MS["s"], MS["origin"], tau_voxels * MS["s"], 64.0)
        on.tsdf[...], on.weight[...] = tsdf, weight
        nrm, n = on.surface_normals()
        assert n == len(verts) and len(tris) > 1000
        face, _ = mc.normals(verts, tris)
        dots = np.stack([(face * nrm[tris[:, c], :3]).sum(1) for c in range(3)], 1)
        assert np.all(dots > 0), (dots <= 0).sum()
        radial = verts[:, :3].astype(np.float64) - np.asarray(MS["centre"])
        print(f"\nclosed sphere, tau = {tau_voxels} voxels: {len(tris)} triangles, max vertex-normal angle to radial "
              f"{_angles(nrm, radial).max():.4f} rad")


def test_trilinear_field_on_an_edge_is_the_vertex_normal():
    """On a cube edge the trilinear field reduces to the edge's linear interpolation: a raycast hit exactly on an
    x edge (y and z grid coordinates integral) gets the normal of the surface point of that edge."""
    dims, s, origin = (16, 16, 24), 0.0625, (-0.5, -0.5, 0.25)
    o = vno.OracleVolume(dims, s, origin, 0.25, 10.0)
    # a curved field, positive towards the camera (small z), so that the gradients of an edge's two voxels differ
    k, j, i = np.meshgrid(np.arange(dims[2]), np.arange(dims[1]), np.arange(dims[0]), indexing="ij")
    o.tsdf[...] = np.clip((12.3 - k - 0.04 * (i - 8.0) ** 2 - 0.03 * (j - 9.0) ** 2 + 0.08 * (k - 12.0) ** 2
                            + 0.05 * (i - 7.0) * (k - 12.0)) / 4.0, -1, 1).astype(F)
    o.weight[...] = np.random.default_rng(3).integers(1, 5, o.weight.shape).astype(F)
    pts, _ = o.surface_points()
    nrm, _ = o.surface_normals()
    # the camera at (x, y) of voxel column (8, 7), z = 0, looking along +z: the centre pixel's ray is that column
    # (dyadic grid: its grid coordinates x = 8, y = 7 are exact) and its samples lie on the voxel centres
    cam = (40.0, 40.0, 32.0, 32.0)
    T = np.array([[1, 0, 0, -(origin[0] + 8 * s)], [0, 1, 0, -(origin[1] + 7 * s)], [0, 0, 1, 0]], F)
    depth, nr = o.raycast_normals(cam, T, 65, 65)
    d = float(depth[32, 32])
    assert d > 0
    ijk, axis = mc.surface_point_edges(o.tsdf, o.weight)
    sel = (ijk[:, 0] == 8) & (ijk[:, 1] == 7) & (axis == 2)
    assert sel.sum() == 1
    assert abs(float(pts[sel][0, 2]) - d) <= 1e-6      # the hit is that z edge's surface point
    ga, gb = (o.gradients()[ijk[sel][0, 2] + q, 7, 8] for q in (0, 1))
    assert np.abs(ga - gb).max() > 1e-3                # the edge's gradients differ: the interpolation matters
    assert np.abs(nr[32, 32, :3] - nrm[sel][0, :3]).max() <= 4 * ULP1


# ------------------------------------------------------------------ what the normals give on ground truth
def frame_normals(points, depth, dirs, max_jump=0.02):
    """Normals of an organised world point map [h, w, 3] by central finite differences, oriented towards the
    camera (n . dir < 0); NaN at the border, where depth is 0, and at depth discontinuities (a neighbour whose
    depth differs by more than max_jump of the pixel's)."""
    P = np.asarray(points, np.float64)
    d = np.asarray(depth, np.float64)
    h, w = d.shape
    n = np.full((h, w, 3), np.nan)
    c = (slice(1, -1), slice(1, -1))
    dx = P[1:-1, 2:] - P[1:-1, :-2]
    dy = P[2:, 1:-1] - P[:-2, 1:-1]
    m = np.cross(dx, dy)
    m /= np.maximum(np.linalg.norm(m, axis=-1, keepdims=True), 1e-300)
    m *= -np.sign((m * dirs[c]).sum(-1, keepdims=True))
    ok = d[c] > 0
    for nb in (d[1:-1, 2:], d[1:-1, :-2], d[2:, 1:-1], d[:-2, 1:-1]):
        ok &= (nb > 0) & (np.abs(nb - d[c]) <= max_jump * d[c])
    n[c] = np.where(ok[..., None], m, np.nan)
    return n


def normal_quality(depth, normals, truth_points, truth_depth, cam, T_world_cam):
    """(median angle of the raycast normals, median angle of finite differences of the raycast depth, share of hits
    with a normal, share of those facing the camera) against the true normals, over pixels where all are defined."""
    h, w = depth.shape
    fx, fy, cx, cy = cam
    yy, xx = np.mgrid[0:h, 0:w].astype(np.float64)
    d = np.stack([(xx - cx) / fx, (yy - cy) / fy, np.ones_like(xx)], -1)
    d /= np.linalg.norm(d, axis=-1, keepdims=True)
    T = np.asarray(T_world_cam, np.float64)
    dirs = d @ T[:, :3].T
    truth = frame_normals(truth_points, truth_depth, dirs)
    fd = frame_normals(dirs * depth[..., None] + T[:, 3], depth, dirs)
    hit = depth > 0
    has = hit & (np.abs(normals[..., :3]).sum(-1) > 0)
    facing = (np.asarray(normals[..., :3], np.float64)[has] * dirs[has]).sum(-1) < 0
    ok = has & np.isfinite(truth[..., 0]) & np.isfinite(fd[..., 0])
    return (float(np.median(_angles(normals[ok], truth[ok]))), float(np.median(_angles(fd[ok], truth[ok]))),
            float(has.sum() / max(1, hit.sum())), float(facing.mean()))


# Setup of test_volume_intensity_oracle.test_ground_truth_novel_view: QVGA frames 0, 20, ..., 100 fused into 256^3,
# frame 10 raycast.  Measured: median angle to the true normals 0.98 deg for the raycast normals against 1.27 deg
# for finite differences of the raycast depth (ratio 0.77); 99.91 % of the hits have a normal, 100.00 % of those face
# the camera.
GT_MEDIAN_DEG = 1.5
GT_OVER_DEPTH_FD = 0.9
GT_NORMAL_SHARE = 0.99
GT_FACING_SHARE = 0.99


def test_ground_truth_novel_view_normals():
    from rpg_open_remode_b200 import synth
    seq = synth.SyntheticSequence(320, 240, seed=0x5EED0001)
    cam = seq.camera
    used = [seq.frame(k) for k in range(0, 101, 20)]
    n, tau_vox = 256, 4.0
    s, origin = scene_grid(np.concatenate([ground_truth_points(fr, cam).reshape(-1, 3) for fr in used]), n, tau_vox)
    o = vno.OracleVolume((n, n, n), s, origin, F(tau_vox) * s, 64.0)
    for fr in used:
        o.integrate(fr.depth, cam, fr.T_cam_world)
    f10 = seq.frame(10)
    depth, nr = o.raycast_normals(cam, f10.T_cam_world, 320, 240)
    want, _ = _numpy_raycast_normals(o.tsdf, o.weight, s, origin, cam, f10.T_cam_world, depth)
    assert np.array_equal(nr.view(u32), want.view(u32))
    med, med_fd, share, facing = normal_quality(depth, nr, ground_truth_points(f10, cam), f10.depth, cam,
                                                f10.T_world_cam)
    print(f"\nnovel view (frame 10), QVGA, 256^3: median angle to the true normals {np.degrees(med):.2f} deg "
          f"(finite differences of the raycast depth: {np.degrees(med_fd):.2f} deg); {100 * share:.2f} % of the hits "
          f"have a normal, {100 * facing:.2f} % of those face the camera")
    assert np.degrees(med) <= GT_MEDIAN_DEG
    assert med <= GT_OVER_DEPTH_FD * med_fd
    assert share >= GT_NORMAL_SHARE and facing >= GT_FACING_SHARE


# ------------------------------------------------------------------ PLY normals
def _read_ply(path):
    data = open(path, "rb").read()
    end = data.index(b"end_header\n") + len(b"end_header\n")
    return data[:end].decode("ascii"), data[end:]


def test_write_ply_normals(tmp_path):
    from rpg_open_remode_b200 import write_ply
    rng = np.random.default_rng(8)
    v = rng.normal(size=(6, 4)).astype(F)
    t = np.array([[0, 1, 2], [3, 4, 5]], np.int32)
    nrm = rng.normal(size=(6, 3)).astype(F)
    inten = np.array([-1, 0.0, 0.5, 1.0, 1.7, 0.2], F)
    plain, with_n, both, grey = (tmp_path / f"{k}.ply" for k in ("plain", "n", "both", "grey"))
    write_ply(str(plain), v, t)
    write_ply(str(with_n), v, t, normals=nrm)
    write_ply(str(both), v, t, inten, nrm)
    write_ply(str(grey), v, t, inten)
    h0, b0 = _read_ply(plain)
    normal_props = "property float nx\nproperty float ny\nproperty float nz\n"
    colour_props = "property uchar red\nproperty uchar green\nproperty uchar blue\n"
    h1, b1 = _read_ply(with_n)
    assert h1 == h0.replace("property float weight\n", "property float weight\n" + normal_props)
    rec = np.frombuffer(b1[:6 * 28], np.dtype([("p", "<f4", 4), ("n", "<f4", 3)]))
    assert np.array_equal(rec["p"], v) and np.array_equal(rec["n"], nrm)
    assert b1[6 * 28:] == b0[6 * 16:]
    h2, b2 = _read_ply(both)
    assert h2 == h0.replace("property float weight\n", "property float weight\n" + normal_props + colour_props)
    rec = np.frombuffer(b2[:6 * 31], np.dtype([("p", "<f4", 4), ("n", "<f4", 3), ("c", "u1", 3)]))
    hg, bg = _read_ply(grey)
    grey_rec = np.frombuffer(bg[:6 * 19], np.dtype([("p", "<f4", 4), ("c", "u1", 3)]))
    assert np.array_equal(rec["p"], v) and np.array_equal(rec["n"], nrm) and np.array_equal(rec["c"], grey_rec["c"])
    assert b2[6 * 31:] == b0[6 * 16:]
    with pytest.raises(ValueError):
        write_ply(str(with_n), v, t, normals=nrm[:5])
