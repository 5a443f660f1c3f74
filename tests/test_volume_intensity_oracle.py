"""The checker of the TSDF volume's intensity channel (oracle/rmd_oracle_volume_intensity.c, bound by
volume_intensity_oracle.py; DESIGN.md 4.8), on the CPU.

As for the volume oracle: pinned against an independent numpy float32 evaluation (correctly rounded, so equality is
exact) on random ragged grids, poses, depth and intensity images with NaN / inf / 0 / negative entries and state
maps, and against known answers.  Then what the channel gives is measured on the synthetic sequence's ground truth:
a view that was not fused, shaded from the volume, against the real frame.  Also the PLY writer's colour.
"""
import numpy as np
import pytest

import volume_intensity_oracle as vio
from test_volume_oracle import _numpy_integrate, _numpy_surface, _plane_setup, _random_case, _voxel_centres
from test_volume_oracle import ground_truth_points, scene_grid

F = np.float32


def _numpy_integrate_intensity(cint, cw, dims, s, origin, depth, cam, T, conv, inten, trunc, wmax):
    """The intensity half of one integration in numpy float32, in the kernel's order.  In place; returns the count."""
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
        I = inten[y, x]
        ok &= (sdf >= -F(trunc)) & (sdf < F(trunc)) & np.isfinite(I)
    w1 = cw[ok] + F(1)
    cint[ok] = (cint[ok] * cw[ok] + I[ok]) / w1
    cw[ok] = np.minimum(w1, F(wmax))
    return int(ok.sum())


def _numpy_surface_intensity(tsdf, weight, cint, cw):
    nz, ny, nx = tsdf.shape
    k, j, i = np.meshgrid(np.arange(nz), np.arange(ny), np.arange(nx), indexing="ij")
    lin = ((k * ny + j) * nx + i).astype(np.int64)
    near = (weight > 0) & (np.abs(tsdf) < 1)
    keys, vals = [], []
    for axis in range(3):
        a = [slice(None)] * 3
        b = [slice(None)] * 3
        a[2 - axis], b[2 - axis] = slice(0, -1), slice(1, None)
        a, b = tuple(a), tuple(b)
        ta, tb = tsdf[a], tsdf[b]
        sel = near[a] & near[b] & (((ta > 0) & (tb <= 0)) | ((ta <= 0) & (tb > 0)))
        ca, cb, wa, wb = cint[a][sel], cint[b][sel], cw[a][sel], cw[b][sel]
        f = ta[sel] / (ta[sel] - tb[sel])
        v = np.where((wa > 0) & (wb > 0), ca + f * (cb - ca), np.where(wa > 0, ca, np.where(wb > 0, cb, F(-1))))
        vals.append(v.astype(F))
        keys.append(lin[a][sel] * 3 + axis)
    keys, vals = np.concatenate(keys), np.concatenate(vals)
    return vals[np.argsort(keys, kind="stable")]


def _numpy_raycast_intensity(cint, cw, s, origin, cam, T_curr_world, depth):
    """The intensity at every hit of `depth` (the volume oracle's raycast), in numpy float32."""
    nz, ny, nx = cint.shape
    h, w = depth.shape
    fx, fy, cx, cy = (F(c) for c in cam)
    T = np.asarray(vio.vo.pose_inverse(T_curr_world), F)
    yy, xx = np.mgrid[0:h, 0:w].astype(F)
    vx, vy = (xx - cx) / fx, (yy - cy) / fy
    inv_len = F(1) / np.sqrt((vx * vx + vy * vy) + F(1))
    q = (vx * inv_len, vy * inv_len, F(1) * inv_len)
    dirs = [(T[r, 0] * q[0] + T[r, 1] * q[1]) + T[r, 2] * q[2] for r in range(3)]
    o = np.asarray(origin, F)
    g = [((T[r, 3] + depth * dirs[r]) - o[r]) / F(s) for r in range(3)]
    x0, y0, z0 = (np.floor(c) for c in g)
    out = np.full((h, w), F(-1))
    hit = depth > 0
    with np.errstate(invalid="ignore"):
        ok = hit & (x0 >= 0) & (y0 >= 0) & (z0 >= 0) & (x0 + 1 < nx) & (y0 + 1 < ny) & (z0 + 1 < nz)
    i0, j0, k0 = (np.where(ok, c, 0).astype(np.int64) for c in (x0, y0, z0))
    corner = {}
    for dz in (0, 1):
        for dy in (0, 1):
            for dx in (0, 1):
                corner[dx, dy, dz] = (np.minimum(k0 + dz, nz - 1), np.minimum(j0 + dy, ny - 1),
                                      np.minimum(i0 + dx, nx - 1))   # clamped where ok is already false
                ok &= cw[corner[dx, dy, dz]] != 0
    c = {key: cint[idx] for key, idx in corner.items()}
    fxx, fyy, fzz = g[0] - x0, g[1] - y0, g[2] - z0

    def lerp(a, b, f):
        return a + f * (b - a)
    c00, c10 = lerp(c[0, 0, 0], c[1, 0, 0], fxx), lerp(c[0, 1, 0], c[1, 1, 0], fxx)
    c01, c11 = lerp(c[0, 0, 1], c[1, 0, 1], fxx), lerp(c[0, 1, 1], c[1, 1, 1], fxx)
    v = lerp(lerp(c00, c10, fyy), lerp(c01, c11, fyy), fzz)
    out[ok] = v[ok]
    return out


def _random_intensity(rng, size):
    w, h = size
    I = rng.uniform(0, 1, (h, w)).astype(F)
    I[rng.random((h, w)) < 0.03] = np.nan
    I[rng.random((h, w)) < 0.02] = np.inf
    I[rng.random((h, w)) < 0.02] = -np.inf
    I[rng.random((h, w)) < 0.03] = 0.0
    I[rng.random((h, w)) < 0.03] = -0.5
    return I


@pytest.mark.parametrize("dims,size,seed,with_conv", [((37, 29, 23), (61, 47), 1, True),
                                                      ((64, 48, 40), (160, 120), 2, True),
                                                      ((97, 64, 71), (96, 72), 3, False),
                                                      ((1, 50, 33), (40, 30), 4, True)])
def test_oracle_intensity_equals_numpy_float32(dims, size, seed, with_conv):
    rng = np.random.default_rng(0x1C0 + seed)
    s, origin, cam, T, depth, conv = _random_case(rng, dims, size)
    trunc, wmax = F(3.0) * s, 5.0
    conv = conv if with_conv else None
    o = vio.OracleVolume(dims, s, origin, trunc, wmax)
    t_np, w_np = np.zeros_like(o.tsdf), np.zeros_like(o.weight)
    c_np, cw_np = np.zeros_like(o.tsdf), np.zeros_like(o.weight)
    for rep in range(7):    # repeated views: running averages and the weight cap
        if rep:
            depth = (depth * F(rng.uniform(0.97, 1.03))).astype(F)
        inten = _random_intensity(rng, size)
        o.integrate(depth, cam, T, conv, inten)
        _numpy_integrate(t_np, w_np, dims, s, origin, depth, cam, T, conv, trunc, wmax)
        n_np = _numpy_integrate_intensity(c_np, cw_np, dims, s, origin, depth, cam, T, conv, inten, trunc, wmax)
        assert n_np > 0.002 * np.prod(dims)
        # the tsdf is the plain volume oracle's
        assert np.array_equal(o.tsdf.view(np.uint32), t_np.view(np.uint32)) and np.array_equal(o.weight, w_np)
        assert np.array_equal(o.cint.view(np.uint32), c_np.view(np.uint32))
        assert np.array_equal(o.cw, cw_np)
    assert cw_np.max() == F(wmax) and ((w_np > 0) & (cw_np == 0)).any()
    assert not ((cw_np > 0) & (w_np == 0)).any()
    got, n = o.surface_intensity()
    want = _numpy_surface_intensity(t_np, w_np, c_np, cw_np)
    assert n == len(want) == len(_numpy_surface(t_np, w_np, s, origin)) > 0
    assert np.array_equal(got.view(np.uint32), want.view(np.uint32))
    part, n2 = o.surface_intensity(capacity=n // 3)
    assert n2 == n and np.array_equal(part.view(np.uint32), want[:n // 3].view(np.uint32))
    w, h = size
    d_o, i_o = o.raycast_intensity(cam, T, w, h)
    assert np.array_equal(d_o.view(np.uint32), o.raycast(cam, T, w, h).view(np.uint32))
    want = _numpy_raycast_intensity(c_np, cw_np, s, origin, cam, T, d_o)
    assert np.array_equal(i_o.view(np.uint32), want.view(np.uint32))
    assert np.all(i_o[d_o == 0] == -1)   # shaded hits are pinned on a real scene in test_ground_truth_novel_view


def _plane(wmax=10.0, value=0.375, reps=1):
    W, H, cam, s, origin, dims, D, tau, depth = _plane_setup()
    I = np.eye(4, dtype=F)[:3]
    o = vio.OracleVolume(dims, s, origin, tau, wmax)
    for _ in range(reps):
        o.integrate(depth, cam, I, None, np.full((H, W), value, F))
    return o, W, H, cam, s, origin, dims, D, tau, I


def test_known_answers_constant_intensity():
    """A constant dyadic intensity fuses, extracts and renders to exactly that value."""
    o, W, H, cam, *_, I = _plane(reps=3)
    assert (o.cw > 0).sum() > 100 and np.all(o.cint[o.cw > 0] == F(0.375))
    got, n = o.surface_intensity()
    assert n > 100 and np.all(got == F(0.375))
    depth, inten = o.raycast_intensity(cam, I, W, H)
    hit = depth > 0
    assert hit.sum() > 400 and np.all(inten[hit] == F(0.375)) and np.all(inten[~hit] == -1)


def test_known_answers_band_and_saturation():
    o, W, H, cam, s, origin, dims, D, tau, I = _plane()
    z = F(origin[2]) + np.arange(dims[2]).astype(F) * F(s)
    sdf = D - z
    axis_w, axis_cw = o.weight[:, 8, 8], o.cw[:, 8, 8]
    band = (sdf >= -tau) & (sdf < tau)
    assert np.all(axis_cw[band] == 1) and band.sum() >= 4
    # free space (sdf >= tau) is carved but takes no colour
    free = sdf >= tau
    assert free.sum() > 5 and np.all(axis_w[free] == 1) and np.all(axis_cw[free] == 0)
    assert not ((o.cw > 0) & (o.weight == 0)).any()
    # the colour weight saturates at max_weight, the running average goes on
    o2, *_ = _plane(wmax=3.0, value=0.5, reps=6)
    assert o2.cw.max() == 3 and np.all(o2.cw[o2.weight > 0][o2.cw[o2.weight > 0] > 0] == 3)
    # a plain integration (no intensity image) leaves the channel alone
    c0, w0 = o.cint.copy(), o.cw.copy()
    depth = _plane_setup()[-1]
    o.integrate(depth, cam, I)
    assert np.array_equal(o.cint, c0) and np.array_equal(o.cw, w0)
    # non-finite intensities are skipped, zero and negative ones are fused
    for bad in (np.nan, np.inf, -np.inf):
        o3 = vio.OracleVolume(dims, s, origin, tau, 10.0)
        assert o3.integrate_intensity_only(depth, cam, I, None, np.full((H, W), bad, F)) == 0
    o3 = vio.OracleVolume(dims, s, origin, tau, 10.0)
    assert o3.integrate_intensity_only(depth, cam, I, None, np.full((H, W), -0.25, F)) > 0
    assert np.all(o3.cint[o3.cw > 0] == F(-0.25))


def test_known_answers_surface_rules():
    """Both voxels known: interpolated; one known: its value; neither: -1."""
    dims = (4, 3, 3)
    o = vio.OracleVolume(dims, 0.1, (0, 0, 0), 0.3, 10.0)
    o.weight[...] = 1
    o.tsdf[...] = 0.5
    o.tsdf[:, :, 2:] = -0.25          # one crossing per row between i = 1 and i = 2, factor 0.5 / 0.75
    rows = [(k, j) for k in range(3) for j in range(3)]
    for q, (k, j) in enumerate(rows):
        mode = q % 4
        if mode in (0, 1):
            o.cint[k, j, 1], o.cw[k, j, 1] = 0.25, 1
        if mode in (0, 2):
            o.cint[k, j, 2], o.cw[k, j, 2] = 0.75, 2
    got, n = o.surface_intensity()
    assert n == len(rows)
    f = F(0.5) / (F(0.5) - F(-0.25))
    want = [F(0.25) + f * (F(0.75) - F(0.25)), F(0.25), F(0.75), F(-1)]
    assert [float(g) for g in got] == [float(want[q % 4]) for q in range(len(rows))]


# ------------------------------------------------------------------ what the channel gives on ground truth
# The setup of test_volume_oracle.test_ground_truth_fusion_accuracy, fusing each view's image as well: the view of
# frame 10 (not fused) is rendered from the volume and compared with frame 10's image.  Measured (DESIGN.md 5.3):
# 99.39 % of the hits shaded, median |rendered - frame| 8.82 grey levels against 22.51 for the frame's mean,
# correlation 0.904.
GT_SHADED_SHARE = 0.95
GT_ERROR_OVER_CONSTANT = 0.5
GT_CORRELATION = 0.8


def test_ground_truth_novel_view():
    from rpg_open_remode_b200 import synth
    seq = synth.SyntheticSequence(320, 240, seed=0x5EED0001)
    cam = seq.camera
    used = [seq.frame(k) for k in range(0, 101, 20)]
    n, tau_vox = 256, 4.0
    s, origin = scene_grid(np.concatenate([ground_truth_points(fr, cam).reshape(-1, 3) for fr in used]), n, tau_vox)
    o = vio.OracleVolume((n, n, n), s, origin, F(tau_vox) * s, 64.0)
    for fr in used:
        o.integrate(fr.depth, cam, fr.T_cam_world, None, fr.image)
    f10 = seq.frame(10)
    depth, inten = o.raycast_intensity(cam, f10.T_cam_world, 320, 240)
    assert np.array_equal(inten.view(np.uint32), _numpy_raycast_intensity(o.cint, o.cw, s, origin, cam,
                                                                          f10.T_cam_world, depth).view(np.uint32))
    hit = depth > 0
    shaded = hit & (inten >= 0)
    share = shaded.sum() / hit.sum()
    truth = f10.image[shaded].astype(np.float64)
    got = inten[shaded].astype(np.float64)
    err = np.median(np.abs(got - truth)) * 255
    const = np.median(np.abs(truth.mean() - truth)) * 255
    corr = np.corrcoef(got, truth)[0, 1]
    print(f"\nnovel view (frame 10), QVGA, 256^3: {100 * share:.2f} % of the hits shaded, median |rendered - frame| "
          f"= {err:.2f} grey levels vs {const:.2f} for the frame's mean, correlation {corr:.3f}")
    assert share >= GT_SHADED_SHARE
    assert err <= GT_ERROR_OVER_CONSTANT * const
    assert corr >= GT_CORRELATION


# ------------------------------------------------------------------ PLY colour
def _read_ply(path):
    data = open(path, "rb").read()
    end = data.index(b"end_header\n") + len(b"end_header\n")
    return data[:end].decode("ascii"), data[end:]


def test_write_ply_intensity(tmp_path):
    from rpg_open_remode_b200 import write_ply
    rng = np.random.default_rng(7)
    v = rng.normal(size=(6, 4)).astype(F)
    t = np.array([[0, 1, 2], [3, 4, 5]], np.int32)
    inten = np.array([-1, 0.0, 0.5, 1.0, 1.7, 0.2], F)
    plain, shaded = tmp_path / "plain.ply", tmp_path / "shaded.ply"
    write_ply(str(plain), v, t)
    write_ply(str(shaded), v, t, inten)
    h0, b0 = _read_ply(plain)
    assert "red" not in h0
    h1, b1 = _read_ply(shaded)
    assert h1 == h0.replace("property float weight\n", "property float weight\nproperty uchar red\n"
                                                      "property uchar green\nproperty uchar blue\n")
    rec = np.frombuffer(b1[:6 * 19], np.dtype([("p", "<f4", 4), ("c", "u1", 3)]))
    assert np.array_equal(rec["p"], v)
    grey = np.array([0, 0, 128, 255, 255, 51], np.uint8)   # clip(rint(255 i)); -1 -> 0
    assert np.array_equal(rec["c"], np.repeat(grey[:, None], 3, 1))
    assert b1[6 * 19:] == b0[6 * 16:]   # the faces are unchanged
    with pytest.raises(ValueError):
        write_ply(str(shaded), v, t, inten[:5])
