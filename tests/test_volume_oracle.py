"""The checker of the TSDF volume (oracle/rmd_oracle_volume.c, bound by volume_oracle.py; DESIGN.md 4.8), on the CPU.

The reference has no such step, so the oracle is pinned the way the prior's is: against an independent numpy
float32 evaluation (every numpy float32 operation is correctly rounded, so equality is exact) on random grids,
poses, state maps and ragged sizes, and against known answers.  Then the fusion itself is checked against the
synthetic sequence's ground truth.
"""
import numpy as np
import pytest

import oracle_binding as ob
import volume_oracle as vo

F = np.float32


def _rot(rng, angle):
    axis = rng.normal(size=3)
    axis /= np.linalg.norm(axis)
    K = np.array([[0, -axis[2], axis[1]], [axis[2], 0, -axis[0]], [-axis[1], axis[0], 0]])
    return np.eye(3) + np.sin(angle) * K + (1 - np.cos(angle)) * K @ K


def _pose(R, t):
    return np.concatenate([np.asarray(R, F), np.asarray(t, F).reshape(3, 1)], axis=1).astype(F)


def _voxel_centres(dims, s, origin):
    nx, ny, nz = dims
    k, j, i = np.meshgrid(np.arange(nz), np.arange(ny), np.arange(nx), indexing="ij")
    o = np.asarray(origin, F)
    return (o[0] + i.astype(F) * F(s), o[1] + j.astype(F) * F(s), o[2] + k.astype(F) * F(s)), (i, j, k)


def _numpy_integrate(tsdf, weight, dims, s, origin, depth, cam, T, conv, trunc, wmax):
    """One integration in numpy float32, in the kernel's operation order.  Updates in place; returns the count."""
    (wx, wy, wz), _ = _voxel_centres(dims, s, origin)
    T = np.asarray(T, F).reshape(3, 4)
    p = [((T[r, 0] * wx + T[r, 1] * wy) + T[r, 2] * wz) + T[r, 3] for r in range(3)]
    fx, fy, cx, cy = (F(c) for c in cam)
    h, w = depth.shape
    with np.errstate(invalid="ignore", divide="ignore", over="ignore"):
        tu = np.floor(((fx * p[0]) / p[2] + cx) + F(0.5))
        tv = np.floor(((fy * p[1]) / p[2] + cy) + F(0.5))
        ok = (p[2] > 0) & (tu >= 0) & (tu < w) & (tv >= 0) & (tv < h)
        x, y = np.where(ok, tu, 0).astype(np.int64), np.where(ok, tv, 0).astype(np.int64)
        if conv is not None:
            ok &= conv[y, x] == 1
        d = depth[y, x]
        ok &= (d > 0) & np.isfinite(d)
        r = np.sqrt((p[0] * p[0] + p[1] * p[1]) + p[2] * p[2])
        sdf = d - r
        ok &= sdf >= -F(trunc)
        o = np.minimum(F(1), sdf / F(trunc))
    w1 = weight[ok] + F(1)
    tsdf[ok] = (tsdf[ok] * weight[ok] + o[ok]) / w1
    weight[ok] = np.minimum(w1, F(wmax))
    return int(ok.sum())


def _numpy_surface(tsdf, weight, s, origin):
    nz, ny, nx = tsdf.shape
    (px, py, pz), (i, j, k) = _voxel_centres((nx, ny, nz), s, origin)
    lin = ((k * ny + j) * nx + i).astype(np.int64)
    near = (weight > 0) & (np.abs(tsdf) < 1)
    keys, pts = [], []
    for axis in range(3):
        a = [slice(None)] * 3
        b = [slice(None)] * 3
        a[2 - axis], b[2 - axis] = slice(0, -1), slice(1, None)
        a, b = tuple(a), tuple(b)
        ta, tb = tsdf[a], tsdf[b]
        sel = near[a] & near[b] & (((ta > 0) & (tb <= 0)) | ((ta <= 0) & (tb > 0)))
        c = [px[a][sel], py[a][sel], pz[a][sel]]
        c[axis] = c[axis] + (ta[sel] / (ta[sel] - tb[sel])) * F(s)
        pts.append(np.stack(c + [np.minimum(weight[a][sel], weight[b][sel])], axis=1))
        keys.append(lin[a][sel] * 3 + axis)
    keys, pts = np.concatenate(keys), np.concatenate(pts)
    return pts[np.argsort(keys, kind="stable")].astype(F)


def _random_case(rng, dims, size):
    nx, ny, nz = dims
    w, h = size
    s = F(rng.uniform(0.02, 0.05))
    cam = tuple(float(F(c)) for c in (0.75 * w, -0.75 * w, (w - 1) / 2, (h - 1) / 2))
    # the camera looks at the grid's centre from a few voxels' worth of distance, slightly rotated
    centre = np.array([nx, ny, nz], np.float64) * s / 2
    origin = (rng.normal(size=3) * 0.1).astype(F)
    R = _rot(rng, 0.15)
    cam_pos = origin + centre - R[2] * (1.2 * nz * s)
    T = _pose(R, -R @ cam_pos)   # world -> camera: rows of R are the camera axes in the world
    depth = rng.uniform(0.6 * nz * s, 1.8 * nz * s, (h, w)).astype(F)
    depth[rng.random((h, w)) < 0.03] = np.nan
    depth[rng.random((h, w)) < 0.02] = np.inf
    depth[rng.random((h, w)) < 0.02] = -1.0
    depth[rng.random((h, w)) < 0.02] = 0.0
    conv = rng.integers(0, 6, (h, w)).astype(np.int32)
    conv[rng.random((h, w)) < 0.5] = 1
    return s, origin, cam, T, depth, conv


@pytest.mark.parametrize("dims,size,seed,with_conv", [((37, 29, 23), (61, 47), 1, True),
                                                      ((64, 48, 40), (160, 120), 2, True),
                                                      ((97, 64, 71), (96, 72), 3, False),
                                                      ((1, 50, 33), (40, 30), 4, True)])
def test_oracle_integrate_and_surface_equal_numpy_float32(dims, size, seed, with_conv):
    rng = np.random.default_rng(0x70C0 + seed)
    s, origin, cam, T, depth, conv = _random_case(rng, dims, size)
    trunc, wmax = F(3.0) * s, 5.0
    conv = conv if with_conv else None
    o = vo.OracleVolume(dims, s, origin, trunc, wmax)
    t_np, w_np = np.zeros_like(o.tsdf), np.zeros_like(o.weight)
    for rep in range(7):    # repeated views: running averages and the weight cap
        if rep:
            depth = (depth * F(rng.uniform(0.97, 1.03))).astype(F)
        n_o = o.integrate(depth, cam, T, conv)
        n_np = _numpy_integrate(t_np, w_np, dims, s, origin, depth, cam, T, conv, trunc, wmax)
        assert n_o == n_np > 0.01 * np.prod(dims)
        assert np.array_equal(o.tsdf.view(np.uint32), t_np.view(np.uint32))
        assert np.array_equal(o.weight, w_np)
    assert w_np.max() == F(wmax) and (w_np == 0).any()
    got, n = o.surface_points()
    want = _numpy_surface(t_np, w_np, s, origin)
    assert n == len(want) > 0
    assert np.array_equal(got.view(np.uint32), want.view(np.uint32))
    part, n2 = o.surface_points(capacity=n // 3)
    assert n2 == n and np.array_equal(part, want[:n // 3])


def _plane_setup():
    W = H = 65
    cam = (40.0, 40.0, 32.0, 32.0)        # pixel (32, 32) is the optical axis
    s, origin, dims = 0.0625, (-0.5, -0.5, 0.25), (17, 17, 48)     # voxel (8, 8, k) lies on the optical axis
    D, tau = F(1.53125), F(0.25)    # half-way between two voxel centres on the axis
    yy, xx = np.mgrid[0:H, 0:W].astype(F)
    vx, vy = (xx - F(cam[2])) / F(cam[0]), (yy - F(cam[3])) / F(cam[1])
    depth = (D * np.sqrt(vx * vx + vy * vy + F(1))).astype(F)     # fronto-parallel plane z = D
    return W, H, cam, s, origin, dims, D, tau, depth


def test_oracle_known_answers_plane():
    W, H, cam, s, origin, dims, D, tau, depth = _plane_setup()
    I = np.eye(4, dtype=F)[:3]
    o = vo.OracleVolume(dims, s, origin, tau, 10.0)
    assert o.integrate(depth, cam, I) > 0
    z = F(origin[2]) + np.arange(dims[2]).astype(F) * F(s)
    axis_t, axis_w = o.tsdf[:, 8, 8], o.weight[:, 8, 8]
    sdf = D - z
    front = sdf >= -tau
    assert np.array_equal(axis_t[front], np.minimum(F(1), sdf[front] / tau))
    assert np.all(axis_w[front] == 1)
    assert np.all(axis_t[~front] == 0) and np.all(axis_w[~front] == 0) and (~front).sum() > 10
    # twice: unchanged tsdf, weight 2
    t1 = o.tsdf.copy()
    o.integrate(depth, cam, I)
    assert np.array_equal(o.tsdf, t1) and np.all(o.weight[:, 8, 8][front] == 2)
    # saturation at w_max
    o2 = vo.OracleVolume(dims, s, origin, tau, 3.0)
    for _ in range(6):
        o2.integrate(depth, cam, I)
    assert o2.weight.max() == 3 and np.all(o2.weight[:, 8, 8][front] == 3)
    # the surface points of the plane lie at z = D on the axis column
    pts, n = o.surface_points()
    on_axis = pts[(pts[:, 0] == 0) & (pts[:, 1] == 0)]
    assert len(on_axis) == 1 and abs(on_axis[0, 2] - D) <= 1e-6 and on_axis[0, 3] == 2


def test_oracle_known_answers_untouched():
    W, H, cam, s, origin, dims, D, tau, depth = _plane_setup()
    I = np.eye(4, dtype=F)[:3]

    def fresh():
        return vo.OracleVolume(dims, s, origin, tau, 10.0)

    behind = _pose(np.diag([-1.0, 1.0, -1.0]), [0, 0, 0])      # the camera turned around: the grid is behind it
    assert fresh().integrate(depth, cam, behind) == 0
    aside = _pose(np.eye(3), [-100.0, 0, 0])                     # the grid projects outside the image
    assert fresh().integrate(depth, cam, aside) == 0
    assert fresh().integrate(depth, cam, I, np.zeros((H, W), np.int32)) == 0      # no CONVERGED pixel
    for bad in (np.nan, np.inf, -np.inf, 0.0, -1.0):
        o = fresh()
        assert o.integrate(np.full((H, W), bad, F), cam, I) == 0
        assert not o.weight.any() and not o.tsdf.any()
    # one CONVERGED pixel: only the voxels that project onto it change
    conv = np.zeros((H, W), np.int32)
    conv[32, 32] = 1
    o = fresh()
    n = o.integrate(depth, cam, I, conv)
    assert n > 0 and (o.weight > 0).sum() == n and np.all(o.weight[:, 8, 8][o.weight[:, 8, 8] > 0] == 1)
    full = fresh()
    full.integrate(depth, cam, I)
    assert np.array_equal(o.tsdf[o.weight > 0], full.tsdf[o.weight > 0])


def _sphere(dims, s, origin, centre, radius, tau):
    (x, y, z), _ = _voxel_centres(dims, s, origin)
    d = np.sqrt((x.astype(np.float64) - centre[0]) ** 2 + (y - centre[1]) ** 2 + (z - centre[2]) ** 2) - radius
    return np.clip(d / tau, -1, 1).astype(F), np.ones(d.shape, F)


SPHERE = dict(dims=(61, 61, 31), s=0.01, origin=(-0.3, -0.3, 0.85), centre=(0.0, 0.0, 11.0), radius=10.0, tau=0.05)


def _ray_sphere(cam, T_world_cam, w, h, centre, radius):
    """Exact distance along each pixel's ray to the sphere (float64), nan on a miss."""
    yy, xx = np.mgrid[0:h, 0:w].astype(np.float64)
    fx, fy, cx, cy = cam
    d = np.stack([(xx - cx) / fx, (yy - cy) / fy, np.ones_like(xx)], -1)
    d /= np.linalg.norm(d, axis=-1, keepdims=True)
    R, c = np.asarray(T_world_cam, np.float64)[:, :3], np.asarray(T_world_cam, np.float64)[:, 3]
    d = d @ R.T
    oc = c - np.asarray(centre)
    b = (d * oc).sum(-1)
    disc = b * b - (oc @ oc - radius ** 2)
    with np.errstate(invalid="ignore"):
        return -b - np.sqrt(disc)


def test_oracle_known_answers_sphere_and_miss():
    S = SPHERE
    o = vo.OracleVolume(S["dims"], S["s"], S["origin"], S["tau"], 10.0)
    o.tsdf[...], o.weight[...] = _sphere(S["dims"], S["s"], S["origin"], S["centre"], S["radius"], S["tau"])
    w, h = 48, 40
    cam = (80.0, 80.0, 23.5, 19.5)
    T_world_cam = _pose(_rot(np.random.default_rng(5), 0.02), [0.01, -0.02, 0.0])
    T_cam_world = ob.se3_inv(T_world_cam)
    got = o.raycast(cam, T_cam_world, w, h)
    want = _ray_sphere(cam, vo.pose_inverse(T_cam_world), w, h, S["centre"], S["radius"])
    hit = got > 0
    assert hit.mean() > 0.9
    assert np.abs(got[hit] - want[hit]).max() <= 1e-3 * S["s"]
    pts, n = o.surface_points()
    assert n > 1000
    r = np.linalg.norm(pts[:, :3].astype(np.float64) - np.asarray(S["centre"]), axis=1)
    assert np.abs(r - S["radius"]).max() <= 1e-3 * S["s"]
    assert np.all(pts[:, 3] == 1)
    # looking away from the box, and from beside it: every ray misses
    away = ob.se3_inv(_pose(np.diag([1.0, -1.0, -1.0]), [0, 0, 0]))
    assert not o.raycast(cam, away, w, h).any()
    beside = ob.se3_inv(_pose(np.eye(3), [5.0, 0, 0]))
    assert not o.raycast(cam, beside, w, h).any()
    # the host pose inverse is the library's (api.SE3.inv mirrors it)
    from rpg_open_remode_b200 import SE3
    assert np.array_equal(vo.pose_inverse(T_cam_world).reshape(-1), SE3(T_cam_world.reshape(-1)).inv().data)


# ------------------------------------------------------------------ what fusion gives on ground truth
# Bars of the ground-truth fusion (DESIGN.md 5.3): QVGA, 256^3, tau = 4 voxels, six integrated views.
GT_HIT_SHARE = 0.90
GT_MEDIAN_ERROR_VOXELS = 0.5


def scene_grid(points, n, tau_voxels):
    """(voxel size, origin) of an n^3 grid over `points`, padded by 2 tau on every side (tau = tau_voxels * s)."""
    lo, hi = points.min(0), points.max(0)
    s = F((hi - lo).max() / (n - 1 - 4 * tau_voxels))
    return s, (lo - 2 * tau_voxels * float(s)).astype(F)


def ground_truth_points(fr, cam):
    """World points of a frame's ground-truth depth (float64), shape (h, w, 3)."""
    h, w = fr.depth.shape
    fx, fy, cx, cy = cam
    yy, xx = np.mgrid[0:h, 0:w].astype(np.float64)
    d = np.stack([(xx - cx) / fx, (yy - cy) / fy, np.ones_like(xx)], -1)
    d /= np.linalg.norm(d, axis=-1, keepdims=True)
    p = d * fr.depth[..., None]
    T = fr.T_world_cam.astype(np.float64)
    return (p @ T[:, :3].T + T[:, 3]).reshape(h, w, 3)


def test_ground_truth_fusion_accuracy():
    from rpg_open_remode_b200 import synth
    seq = synth.SyntheticSequence(320, 240, seed=0x5EED0001)
    cam = seq.camera
    used = [seq.frame(k) for k in range(0, 101, 20)]
    n, tau_vox = 256, 4.0
    s, origin = scene_grid(np.concatenate([ground_truth_points(fr, cam).reshape(-1, 3) for fr in used]), n, tau_vox)
    o = vo.OracleVolume((n, n, n), s, origin, F(tau_vox) * s, 64.0)
    for fr in used:
        o.integrate(fr.depth, cam, fr.T_cam_world)
    f10 = seq.frame(10)
    got = o.raycast(cam, f10.T_cam_world, 320, 240)
    p10 = ground_truth_points(f10, cam)
    box_hi = origin.astype(np.float64) + (n - 1) * float(s)
    inside = np.all((p10 >= origin) & (p10 <= box_hi), axis=-1)
    hit = inside & (got > 0)
    share = hit.sum() / inside.sum()
    err = np.median(np.abs(got[hit] - f10.depth[hit])) / float(s)
    print(f"\nground-truth fusion, QVGA, 256^3 (s = {float(s):.5f} m): {100 * share:.2f} % of the in-grid pixels hit, "
          f"median |raycast - truth| = {err:.3f} voxels")
    assert share >= GT_HIT_SHARE
    assert err <= GT_MEDIAN_ERROR_VOXELS
