"""The moving TSDF volume on the GPU (csrc/volume.cu: volume_shift_kernel and the spill passes; rmd_volume_shift,
rmd_volume_spill_*, api.TsdfVolume.shift / spill*, DepthmapNode(follow_volume=); DESIGN.md 4.8).

  * the product against the oracle (oracle/rmd_oracle_volume_shift.c) bit for bit: records (tsdf, weight, intensity),
    origin and the spill's points, intensities and normals across shifts -- ground truth at QVGA and VGA, the ragged
    97 x 64 x 71 grid, real filter output (mu and denoised), the 1024 x 1024 x 320 grid (records beyond 2^31 bytes and
    the second array), capacities below the count and the count-only call;
  * stream ordering without host syncs against the same calls with a sync between each;
  * every error code;
  * the node: follow_volume=False publishes and fuses bit-identically; on bench.py's c2 sequence a following volume (256^3, or smaller
    until it shifts three times) created at the origin against the fixed 512^3 volume placed from ground truth.
"""
import ctypes
import gc

import numpy as np
import pytest

import volume_shift_oracle as vso
from test_volume import _grid
from test_volume_oracle import ground_truth_points

F = np.float32
u32 = np.uint32
INVALID, NOT_INITIALISED = -1, -2


def _pair(dims, s, origin, tau, intensity=True):
    import rpg_open_remode_b200 as rmd
    return (rmd.TsdfVolume(dims, s, origin, tau, 64.0, device=0, intensity=intensity),
            vso.OracleVolume(dims, s, origin, tau, 64.0))


def _same_records(v, o, what):
    t, w = v.download()
    assert np.array_equal(w.view(u32), o.weight.view(u32)), f"{what}: weight differs at {(w != o.weight).sum()}"
    assert np.array_equal(t.view(u32), o.tsdf.view(u32)), f"{what}: tsdf differs"
    if v.intensity:
        c, cw = v.downloadIntensity()
        assert np.array_equal(c.view(u32), o.cint.view(u32)) and np.array_equal(cw.view(u32), o.cw.view(u32)), what
    assert np.array_equal(v.origin.view(u32), o.origin.view(u32)), f"{what}: origin {v.origin} != {o.origin}"


def _same_spill(v, o, d, what, min_points=1):
    got, (want, n) = v.spillPoints(d), o.spill(d, vso.POINTS)
    assert len(got) == n >= min_points, f"{what}: {len(got)} / {n} spilled points"
    assert np.array_equal(got.view(u32), want.view(u32)), f"{what}: spilled points differ"
    got, (want, _) = v.spillNormals(d), o.spill(d, vso.NORMALS)
    assert np.array_equal(got.view(u32), want[:, :3].view(u32)), f"{what}: spilled normals differ"
    if v.intensity:
        got, (want, _) = v.spillIntensity(d), o.spill(d, vso.INTENSITY)
        assert np.array_equal(got.view(u32), want.view(u32)), f"{what}: spilled intensities differ"
    return n


def _shift(v, o, d, what, min_points=1):
    n = _same_spill(v, o, d, what, min_points)
    before = len(v.surfacePoints())
    v.shift(d)
    o.shift(d)
    _same_records(v, o, f"{what} after shift {d}")
    assert len(v.surfacePoints()) + n == before, what   # every point either spilled or stayed
    return n


# ------------------------------------------------------------------ product == oracle
@pytest.mark.gpu
@pytest.mark.parametrize("size,dims", [((320, 240), (256, 256, 256)), ((640, 480), (256, 256, 256)),
                                       ((320, 240), (97, 64, 71))])
def test_ground_truth_equals_oracle(size, dims):
    import rpg_open_remode_b200 as rmd
    from rpg_open_remode_b200 import synth
    W, H = size
    seq = synth.SyntheticSequence(W, H, seed=0x5EED0800 + W)
    frames = [seq.frame(k) for k in (0, 25, 50)]
    s, origin, tau = _grid(seq, frames, max(dims))
    v, o = _pair(dims, s, origin, tau)
    cam = rmd.PinholeCamera(*seq.camera)
    n = np.array(dims)
    steps = [tuple(int(x) for x in n // q) for q in (np.array([5, -7, 9]), np.array([-4, 6, -11]))] + [(0, 0, 0)]
    spilled = 0
    for fr, d in zip(frames, steps):
        v.integrateDepth(fr.depth, cam, fr.T_cam_world, None, fr.image)
        o.integrate(fr.depth, seq.camera, fr.T_cam_world, None, fr.image)
        _same_records(v, o, f"{size} {dims}")
        spilled += _shift(v, o, d, f"{size} {dims}", min_points=0)
    assert spilled > 0
    # a shift by the whole grid: the spill is every point, the grid is reset, the origin moves
    d = (0, 0, -dims[2])
    _shift(v, o, (1, 1, 1), "small", min_points=0)
    n_all = len(v.surfacePoints())
    assert _shift(v, o, d, "whole grid", min_points=n_all) == n_all
    assert not v.download()[1].any()


@pytest.mark.gpu
@pytest.mark.parametrize("size,patch,n", [((320, 240), 5, 40), ((640, 480), 5, 30)])
def test_filter_output_equals_oracle(size, patch, n):
    """Keyframes of the real depth filter, fused with their reference images, shifted between keyframes: mu and the
    denoised image."""
    import rpg_open_remode_b200 as rmd
    from rpg_open_remode_b200 import synth
    W, H = size
    seq = synth.SyntheticSequence(W, H, seed=0x5EED0810 + W + patch)
    cam = rmd.PinholeCamera(*seq.camera)
    f0 = seq.frame(0)
    dmin, dmax = float(f0.depth.min()), float(f0.depth.max())
    s, origin, tau = _grid(seq, [f0], 160)
    v_mu, o_mu = _pair((160, 160, 160), s, origin, tau)
    v_dn, o_dn = _pair((160, 160, 160), s, origin, tau)
    den = rmd.DepthmapDenoiser(W, H, device=0)
    den.setLargeSigmaSq(dmax - dmin)
    img = rmd.DeviceImage(W, H, "float32")
    spilled = 0
    for ref, d in ((0, (40, -30, 50)), (n + 1, (-60, 20, -30))):
        g = rmd.SeedMatrix(W, H, cam, patch_side=patch, device=0)
        fr = seq.frame(ref)
        g.setReferenceImage(fr.image_u8, fr.T_cam_world, dmin, dmax)
        for k in range(ref + 1, ref + n + 1):
            g.update(seq.frame(k, want_depth=False).image_u8, seq.frame(k, want_depth=False).T_cam_world)
        conv, mu, ref_img = g.downloadConvergence(), g.downloadDepthmap(), g._download(rmd.FIELD_REF_IMG)
        v_mu.integrate(g)
        o_mu.integrate(mu, seq.camera, fr.T_cam_world, conv, ref_img)
        den.denoiseSeedsToDevice(g, img.data, img.pitch, 0.5, 100)
        v_dn.integrate(g, img)
        den.sync()
        o_dn.integrate(img.getDevData(), seq.camera, fr.T_cam_world, conv, ref_img)
        _same_records(v_mu, o_mu, f"mu {size}")
        _same_records(v_dn, o_dn, f"denoised {size}")
        spilled += _shift(v_mu, o_mu, d, f"mu {size}", min_points=0)
        spilled += _shift(v_dn, o_dn, d, f"denoised {size}", min_points=0)
    assert spilled > 0


@pytest.mark.gpu
def test_grid_beyond_2gb_and_capacity():
    """1024 x 1024 x 320 voxels with the intensity channel: 2.7 GB per record array, and the second arrays of the
    first shift.  Then capacities smaller than the count and the count-only call."""
    import rpg_open_remode_b200 as rmd
    from rpg_open_remode_b200 import _native, synth
    W, H = 640, 480
    seq = synth.SyntheticSequence(W, H, seed=0x5EED0830)
    f0 = seq.frame(0)
    pts = ground_truth_points(f0, seq.camera).reshape(-1, 3)
    dims = (1024, 1024, 320)
    lo, hi = pts.min(0), pts.max(0)
    s = F(((hi - lo) / (np.array(dims) - 1 - 16)).max())
    origin = (lo - 8 * float(s)).astype(F)
    origin[2] = F(hi[2] - (dims[2] - 1 - 8) * float(s))   # the farthest surface in the last planes, beyond 2^31 B
    v, o = _pair(dims, s, origin, F(4) * s)
    cam = rmd.PinholeCamera(*seq.camera)
    v.integrateDepth(f0.depth, cam, f0.T_cam_world, None, f0.image)
    o.integrate(f0.depth, seq.camera, f0.T_cam_world, None, f0.image)
    assert (o.weight.reshape(-1)[2 ** 28:] > 0).any()     # records beyond the first 2^31 bytes are reached
    d = (300, -200, 40)
    want, n = o.spill(d, vso.POINTS)
    assert n > 1000
    L, cnt = _native.lib(), ctypes.c_size_t()
    dd = np.array(d, np.int32)
    cap = n // 7
    for fn, kind, per in ((L.rmd_volume_spill_points, vso.POINTS, 4), (L.rmd_volume_spill_normals, vso.NORMALS, 4),
                          (L.rmd_volume_spill_intensity, vso.INTENSITY, 1)):
        w_all, _ = o.spill(d, kind)
        part = np.empty((cap, per), F)
        assert fn(v.handle, dd.ctypes.data, part.ctypes.data, cap, ctypes.byref(cnt)) == 0
        assert cnt.value == n and np.array_equal(part.reshape(w_all[:cap].shape).view(u32), w_all[:cap].view(u32))
        assert fn(v.handle, dd.ctypes.data, None, 0, ctypes.byref(cnt)) == 0 and cnt.value == n
    assert len(v.spillPoints(d, capacity=cap)) == cap
    _shift(v, o, d, "2.7 GB grid")
    f1 = seq.frame(20)
    v.integrateDepth(f1.depth, cam, f1.T_cam_world, None, f1.image)
    o.integrate(f1.depth, seq.camera, f1.T_cam_world, None, f1.image)
    _shift(v, o, (-100, 50, -20), "2.7 GB grid, second shift", min_points=0)   # writes the first arrays again


# ------------------------------------------------------------------ stream ordering
@pytest.mark.gpu
def test_stream_ordering_without_syncs():
    """integrate -> shift -> integrate -> priorFromVolume -> shift with no host sync equals the same calls with a
    sync between each; and a shift right after the prior leaves the prior of the unshifted model."""
    import rpg_open_remode_b200 as rmd
    from rpg_open_remode_b200 import synth
    W, H = 640, 480
    seq = synth.SyntheticSequence(W, H, seed=0x5EED0840)
    f0, f1, f2 = seq.frame(0), seq.frame(20), seq.frame(30)
    dmin, dmax = float(f0.depth.min()), float(f0.depth.max())
    s, origin, tau = _grid(seq, [f0, f1], 320)
    cam = rmd.PinholeCamera(*seq.camera)
    imgs = []
    for fr in (f0, f1):
        dimg, iimg = rmd.DeviceImage(W, H, "float32"), rmd.DeviceImage(W, H, "float32")
        dimg.setDevData(fr.depth)
        iimg.setDevData(fr.image)
        imgs.append((dimg, iimg, fr.T_cam_world))

    def run(sync):
        v = rmd.TsdfVolume((320, 320, 320), s, origin, tau, 64.0, device=0, intensity=True)
        g = rmd.SeedMatrix(W, H, cam, device=0)
        g.setReferenceImage(f2.image_u8, f2.T_cam_world, dmin, dmax)
        g.sync()
        steps = [lambda: v.integrateDepth(imgs[0][0], cam, imgs[0][2], None, imgs[0][1]),
                 lambda: v.shift((9, -4, 6)),
                 lambda: v.integrateDepth(imgs[1][0], cam, imgs[1][2], None, imgs[1][1]),
                 lambda: g.priorFromVolume(v, 0.25),
                 lambda: v.shift((-70, 30, 150))]   # overwrites the array the prior's rays read
        for st in steps:
            st()
            if sync:
                v.sync()
                g.sync()
        g.sync()
        return v, g.downloadDepthmap()

    v_a, mu_a = run(False)
    v_b, mu_b = run(True)
    for a, b in zip(v_a.download() + v_a.downloadIntensity(), v_b.download() + v_b.downloadIntensity()):
        assert np.array_equal(a.view(u32), b.view(u32))
    assert np.array_equal(mu_a.view(u32), mu_b.view(u32)) and np.array_equal(v_a.origin, v_b.origin)
    # the prior is the unshifted model's: the same seeds from a volume that never took the last shift
    v_c = rmd.TsdfVolume((320, 320, 320), s, origin, tau, 64.0, device=0, intensity=True)
    v_c.integrateDepth(imgs[0][0], cam, imgs[0][2], None, imgs[0][1])
    v_c.shift((9, -4, 6))
    v_c.integrateDepth(imgs[1][0], cam, imgs[1][2], None, imgs[1][1])
    g = rmd.SeedMatrix(W, H, cam, device=0)
    g.setReferenceImage(f2.image_u8, f2.T_cam_world, dmin, dmax)
    g.priorFromVolume(v_c, 0.25)
    g.sync()
    mu_c = g.downloadDepthmap()
    assert np.array_equal(mu_a.view(u32), mu_c.view(u32))
    g0 = rmd.SeedMatrix(W, H, cam, device=0)
    g0.setReferenceImage(f2.image_u8, f2.T_cam_world, dmin, dmax)
    assert (mu_c != g0.downloadDepthmap()).mean() > 0.05    # the prior did hit


# ------------------------------------------------------------------ error codes
@pytest.mark.gpu
def test_error_codes():
    import rpg_open_remode_b200 as rmd
    from rpg_open_remode_b200 import _native
    L = _native.lib()
    v = rmd.TsdfVolume((16, 16, 16), 0.1, (-0.8, -0.8, 0.5), 0.3, 10.0, device=0)
    d = np.array([1, 2, 3], np.int32)
    n = ctypes.c_size_t()
    out = np.empty((4, 4), F)
    assert L.rmd_volume_shift(None, d.ctypes.data) == INVALID
    assert L.rmd_volume_shift(v.handle, None) == INVALID
    for fn in (L.rmd_volume_spill_points, L.rmd_volume_spill_normals):
        assert fn(None, d.ctypes.data, out.ctypes.data, 4, ctypes.byref(n)) == INVALID
        assert fn(v.handle, None, out.ctypes.data, 4, ctypes.byref(n)) == INVALID
        assert fn(v.handle, d.ctypes.data, out.ctypes.data, 4, None) == INVALID
        assert fn(v.handle, d.ctypes.data, None, 4, ctypes.byref(n)) == INVALID
        assert fn(v.handle, d.ctypes.data, None, 0, ctypes.byref(n)) == 0 and n.value == 0
    assert L.rmd_volume_spill_intensity(v.handle, d.ctypes.data, None, 0, ctypes.byref(n)) == NOT_INITIALISED
    with pytest.raises(ValueError):
        v.shift((1.5, 0, 0))
    # an origin that would not be finite: refused, the volume unchanged (the 64-bit total itself cannot overflow
    # from int32 steps within 2^32 calls)
    big = np.array([2 ** 31 - 1, 0, 0], np.int32)
    o = np.empty(3, F)
    huge = rmd.TsdfVolume((4, 4, 4), 1e29, (0, 0, 0), 1e29, 10.0, device=0)
    assert L.rmd_volume_shift(huge.handle, big.ctypes.data) == 0       # (2^31 - 1) * 1e29 < 3.4e38
    before = np.empty(3, F)
    assert L.rmd_volume_size(huge.handle, None, None, None, None, before.ctypes.data) == 0
    assert np.isfinite(before).all() and before[0] > 1e38
    assert L.rmd_volume_shift(huge.handle, big.ctypes.data) == INVALID
    assert L.rmd_volume_size(huge.handle, None, None, None, None, o.ctypes.data) == 0
    assert np.array_equal(o, before)
    # d = 0 is a no-op, and the volume still works after refused calls
    assert L.rmd_volume_shift(v.handle, np.zeros(3, np.int32).ctypes.data) == 0
    v.sync()


# ------------------------------------------------------------------ the node
def _node_run(seq, n_frames, volume, **kw):
    import rpg_open_remode_b200 as rmd
    from rpg_open_remode_b200 import node
    W, H = seq.width, seq.height
    fx, fy, cx, cy = seq.camera
    f0 = seq.frame(0)
    dmin, dmax = float(f0.depth.min()), float(f0.depth.max())
    dm = rmd.Depthmap(W, H, fx, cx, fy, cy, device=0)
    published = []

    def publisher(kind, d):
        if kind == "depthmap_and_pointcloud":
            published.append((kind, d.getDepthmap().copy(), d.getConvergenceMap().copy()))
        elif kind == "volume_spill":
            published.append((kind,) + tuple(d))

    nd = node.DepthmapNode(dm, publisher=publisher, volume=volume, **kw)
    views = {}
    for k in range(n_frames):
        fr = seq.frame(k, want_depth=False)
        nd.denseInputCallback(fr.image_u8, rmd.SE3(fr.T_world_cam.reshape(12)), dmin, dmax)
        if k in (50, 100, 150, 199):
            views[k] = volume.raycast(rmd.PinholeCamera(*seq.camera), fr.T_cam_world, W, H)
    return published, views


@pytest.mark.gpu
def test_node_follow_volume_off_is_bit_identical():
    import rpg_open_remode_b200 as rmd
    from rpg_open_remode_b200 import synth
    seq = synth.SyntheticSequence(320, 240, seed=0x5EED0850)
    s, origin, tau = _grid(seq, [seq.frame(k) for k in (0, 30, 59)], 192)
    va = rmd.TsdfVolume((192, 192, 192), s, origin, tau, 64.0, device=0)
    vb = rmd.TsdfVolume((192, 192, 192), s, origin, tau, 64.0, device=0)
    pa, _ = _node_run(seq, 60, va)
    pb, _ = _node_run(seq, 60, vb, follow_volume=False)
    assert len(pa) == len(pb) >= 2
    for a, b in zip(pa, pb):
        assert a[0] == b[0] == "depthmap_and_pointcloud"
        assert np.array_equal(a[1].view(u32), b[1].view(u32)) and np.array_equal(a[2], b[2])
    for a, b in zip(va.download(), vb.download()):
        assert np.array_equal(a.view(u32), b.view(u32))
    with pytest.raises(ValueError):
        from rpg_open_remode_b200 import node
        node.DepthmapNode(rmd.Depthmap(32, 24, 30, 15.5, 30, 11.5, device=0), follow_volume=True)


# Measured on an H100 80 GB HBM3 at 400 W (DESIGN.md 5.3): bench.py's c2 sequence (VGA, 200 frames) through the node; a
# following volume created at the origin with the 512^3 volume's voxel size -- 256^3, or the next smaller power of two
# if 256^3 shifts fewer than three times -- against the fixed 512^3 volume placed from ground truth.  Measured: 256^3
# shifts once (the first keyframe's placement), 128^3 three times; at frames 50 / 100 / 150 / 199 the raycast median
# |depth - truth| is 1.26 / 1.16 / 1.13 / 1.18x the fixed volume's and it hits 0.64 / 0.62 / 0.57 / 0.51x its pixels;
# spills + final points 23489 against 36730 (0.64x), at a median / p95 distance of 0.49 / 0.58 voxels from the fixed
# volume's points.
FOLLOW_MIN_SHIFTS = 3
FOLLOW_MEDIAN_OVER_FIXED = 1.5    # raycast median |depth - truth| of the following volume over the fixed one's
FOLLOW_HIT_OVER_FIXED = 0.4       # pixels hit, over the fixed volume's
FOLLOW_POINTS_OVER_FIXED = 0.5    # spills + final surface points, over the fixed volume's points
FOLLOW_P95_VOXELS = 1.0           # p95 distance of those points to the fixed volume's points, in voxels


@pytest.mark.gpu
def test_follow_volume_on_c2():
    import torch
    from scipy.spatial import cKDTree
    import rpg_open_remode_b200 as rmd
    from rpg_open_remode_b200 import multi_gpu, synth
    W, H, N = 640, 480, 200
    seq = synth.SyntheticSequence(W, H, seed=multi_gpu.keyframe_seed(0))    # bench.py's c2 sequence
    s, origin, tau = _grid(seq, [seq.frame(k) for k in range(0, N, 25)] + [seq.frame(N - 1)], 512)
    fixed = rmd.TsdfVolume((512, 512, 512), s, origin, tau, 64.0, device=0)
    pf, vf = _node_run(seq, N, fixed)
    for n in (256, 128, 64, 32):
        gc.collect()
        torch.cuda.synchronize()
        m0 = torch.cuda.mem_get_info()[0]
        follow = rmd.TsdfVolume((n, n, n), s, (0.0, 0.0, 0.0), tau, 64.0, device=0)
        pm, vm = _node_run(seq, N, follow, follow_volume=True)
        gc.collect()
        follow_bytes = m0 - torch.cuda.mem_get_info()[0]   # the volume's records, second arrays and staging
        spills = [p for p in pm if p[0] == "volume_spill"]
        print(f"\nc2 follow {n}^3: {len(spills)} shifts")
        if len(spills) >= FOLLOW_MIN_SHIFTS:
            break
        del follow
    maps_f = [p for p in pf if p[0] == "depthmap_and_pointcloud"]
    maps_m = [p for p in pm if p[0] == "depthmap_and_pointcloud"]
    assert len(maps_f) == len(maps_m) and all(np.array_equal(a[1].view(u32), b[1].view(u32))
                                              for a, b in zip(maps_f, maps_m))   # the filter is untouched
    pts = np.concatenate([sp[1][:, :3] for sp in spills] + [follow.surfacePoints()[:, :3]])
    ref = fixed.surfacePoints()[:, :3]
    dist = cKDTree(ref).query(pts)[0] / float(s)
    rows = []
    for k in (50, 100, 150, 199):
        truth = seq.frame(k).depth
        row = []
        for v in (vf[k], vm[k]):
            hit = (v > 0) & np.isfinite(truth)
            row += [float(np.median(np.abs(v[hit] - truth[hit]))) if hit.any() else float("inf"), int(hit.sum())]
        rows.append(row)
    print(f"c2 follow {n}^3: {len(spills)} shifts; per view (50, 100, 150, 199) [fixed 512^3 median |d - truth| m, "
          f"hits, following median, hits]: {rows}; points: {len(pts)} (spills + final) vs {len(ref)} fixed, distance to "
          f"the fixed points median {np.median(dist):.3f} p95 {np.percentile(dist, 95):.3f} voxels; device memory: "
          f"fixed records {512 ** 3 * 8 / 2 ** 20:.0f} MiB, following volume {follow_bytes / 2 ** 20:.1f} MiB measured "
          f"({2 * n ** 3 * 8 / 2 ** 20:.1f} MiB of records)")
    assert len(spills) >= FOLLOW_MIN_SHIFTS
    for mf, hf, mm, hm in rows:
        assert mm <= FOLLOW_MEDIAN_OVER_FIXED * mf and hm >= FOLLOW_HIT_OVER_FIXED * hf
    assert len(pts) >= FOLLOW_POINTS_OVER_FIXED * len(ref)
    assert np.percentile(dist, 95) <= FOLLOW_P95_VOXELS
