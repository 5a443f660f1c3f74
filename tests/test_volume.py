"""TSDF volume on the GPU (csrc/volume.cu, rmd_volume_*, api.TsdfVolume; DESIGN.md 4.8).

  * the product against the oracle (oracle/rmd_oracle_volume.c) bit for bit: every voxel's tsdf and weight, the
    surface points (count, order, bits) and the raycast depth -- ground-truth depth and real filter output at QVGA
    and VGA, seeds' mu and the denoised device image, 5x5 and 7x7 handles, a ragged grid, a grid of more than 2^31
    bytes, a capacity smaller than the count;
  * device-side ordering of integrate_seeds against a following update of the seeds;
  * every error code;
  * the node: unchanged without a volume, the same published map with one, the fused volume == the oracle's;
  * what fusion buys on bench.py's c2 sequence.
"""
import ctypes

import numpy as np
import pytest

import volume_oracle as vo
from test_volume_oracle import ground_truth_points, scene_grid

F = np.float32
INVALID, NOT_INIT = -1, -2


def _grid(seq, frames, n, tau_vox=4.0):
    pts = np.concatenate([ground_truth_points(fr, seq.camera).reshape(-1, 3) for fr in frames])
    s, origin = scene_grid(pts, n, tau_vox)
    return s, origin, F(tau_vox) * s


def _pair(dims, s, origin, tau, wmax=64.0):
    import rpg_open_remode_b200 as rmd
    return rmd.TsdfVolume(dims, s, origin, tau, wmax, device=0), vo.OracleVolume(dims, s, origin, tau, wmax)


def _same(v, o, what, cam=None, poses=(), size=None, check_points=True):
    t, w = v.download()
    assert np.array_equal(w, o.weight), f"{what}: weight differs at {(w != o.weight).sum()} voxels"
    assert np.array_equal(t.view(np.uint32), o.tsdf.view(np.uint32)), \
        f"{what}: tsdf differs at {(t.view(np.uint32) != o.tsdf.view(np.uint32)).sum()} voxels"
    assert (w > 0).sum() > 0
    if check_points:
        got = v.surfacePoints()
        want, n = o.surface_points()
        assert len(got) == n > 0, f"{what}: {len(got)} / {n} points"
        assert np.array_equal(got.view(np.uint32), want.view(np.uint32)), f"{what}: points differ"
    import rpg_open_remode_b200 as rmd
    for T in poses:
        got = v.raycast(rmd.PinholeCamera(*cam), T, *size)
        want = o.raycast(cam, T, *size)
        assert np.array_equal(got.view(np.uint32), want.view(np.uint32)), \
            f"{what}: raycast differs at {(got != want).sum()} pixels"
        assert (got > 0).mean() > 0.05, what


# ------------------------------------------------------------------ product == oracle
@pytest.mark.gpu
@pytest.mark.parametrize("size,dims,with_conv", [((320, 240), (256, 256, 256), False),
                                                 ((640, 480), (256, 256, 256), True),
                                                 ((320, 240), (97, 64, 71), True)])
def test_ground_truth_depth_equals_oracle(size, dims, with_conv):
    import rpg_open_remode_b200 as rmd
    from rpg_open_remode_b200 import synth
    W, H = size
    seq = synth.SyntheticSequence(W, H, seed=0x5EED0500 + W)
    frames = [seq.frame(k) for k in (0, 25, 50)]
    s, origin, tau = _grid(seq, frames, max(dims))
    v, o = _pair(dims, s, origin, tau)
    cam = rmd.PinholeCamera(*seq.camera)
    rng = np.random.default_rng(W)
    for fr in frames:
        # 90 % CONVERGED: enough for rays to find 8 known corners; the rest masks voxels out
        conv = np.where(rng.random((H, W)) < 0.9, 1, rng.integers(2, 6, (H, W))).astype(np.int32) \
            if with_conv else None
        depth = fr.depth.copy()
        depth[rng.random((H, W)) < 0.01] = np.nan
        v.integrateDepth(depth, cam, fr.T_cam_world, conv)
        o.integrate(depth, seq.camera, fr.T_cam_world, conv)
    _same(v, o, f"{size} {dims}", seq.camera, [seq.frame(12, want_depth=False).T_cam_world], (W, H))


@pytest.mark.gpu
@pytest.mark.parametrize("size,patch,n", [((320, 240), 5, 40), ((320, 240), 7, 40), ((640, 480), 5, 30)])
def test_filter_output_equals_oracle(size, patch, n):
    """Keyframes of the real depth filter: the seeds' mu and the denoised device image as the depth."""
    import rpg_open_remode_b200 as rmd
    from rpg_open_remode_b200 import synth
    W, H = size
    seq = synth.SyntheticSequence(W, H, seed=0x5EED0510 + W + patch)
    cam = rmd.PinholeCamera(*seq.camera)
    f0 = seq.frame(0)
    dmin, dmax = float(f0.depth.min()), float(f0.depth.max())
    s, origin, tau = _grid(seq, [f0], 160)
    v_mu, o_mu = _pair((160, 160, 160), s, origin, tau)
    v_dn, o_dn = _pair((160, 160, 160), s, origin, tau)
    den = rmd.DepthmapDenoiser(W, H, device=0)
    den.setLargeSigmaSq(dmax - dmin)
    img = rmd.DeviceImage(W, H, "float32")
    for ref in (0, n + 1):     # two keyframes
        g = rmd.SeedMatrix(W, H, cam, patch_side=patch, device=0)
        fr = seq.frame(ref)
        g.setReferenceImage(fr.image, fr.T_cam_world, dmin, dmax)
        for k in range(ref + 1, ref + n + 1):
            fk = seq.frame(k, want_depth=False)
            g.update(fk.image, fk.T_cam_world)
        conv, mu = g.downloadConvergence(), g.downloadDepthmap()
        assert (conv == 1).sum() > 0.02 * W * H
        v_mu.integrate(g)
        o_mu.integrate(mu, seq.camera, fr.T_cam_world, conv)
        den.denoiseSeedsToDevice(g, img.data, img.pitch, 0.5, 100)
        v_dn.integrate(g, img)
        den.sync()
        o_dn.integrate(img.getDevData(), seq.camera, fr.T_cam_world, conv)
    view = [seq.frame(n // 2, want_depth=False).T_cam_world]
    _same(v_mu, o_mu, f"mu {size} p{patch}", seq.camera, view, (W, H))
    _same(v_dn, o_dn, f"denoised {size} p{patch}", seq.camera, view, (W, H))


@pytest.mark.gpu
def test_grid_beyond_2gb_and_capacity():
    """1024 x 1024 x 320 voxels = 2.7 GB of records: 64-bit addressing end to end.  Then a capacity smaller than
    the number of points, on the host and the device variant."""
    import rpg_open_remode_b200 as rmd
    from rpg_open_remode_b200 import _native, synth
    W, H = 640, 480
    seq = synth.SyntheticSequence(W, H, seed=0x5EED0520)
    f0 = seq.frame(0)
    pts = ground_truth_points(f0, seq.camera).reshape(-1, 3)
    dims = (1024, 1024, 320)
    lo, hi = pts.min(0), pts.max(0)
    s = F(((hi - lo) / (np.array(dims) - 1 - 16)).max())
    origin = (lo - 8 * float(s)).astype(F)
    v, o = _pair(dims, s, origin, F(4) * s)
    v.integrateDepth(f0.depth, rmd.PinholeCamera(*seq.camera), f0.T_cam_world)
    o.integrate(f0.depth, seq.camera, f0.T_cam_world)
    t, w = v.download()
    assert np.array_equal(w, o.weight) and np.array_equal(t.view(np.uint32), o.tsdf.view(np.uint32))
    assert (w.reshape(-1)[2 ** 28:] > 0).any()     # voxels beyond the first 2^31 bytes are reached
    del t, w
    want, n = o.surface_points()
    got = v.surfacePoints()
    assert len(got) == n > 0 and np.array_equal(got.view(np.uint32), want.view(np.uint32))
    L, cnt = _native.lib(), ctypes.c_size_t()
    cap = n // 7
    part = np.empty((cap, 4), F)
    assert L.rmd_volume_surface_points(v.handle, part.ctypes.data, cap, ctypes.byref(cnt)) == 0
    assert cnt.value == n and np.array_equal(part, want[:cap])
    dev = rmd.DeviceImage(4 * cap, 1, "float32")
    assert L.rmd_volume_surface_points_device(v.handle, dev.data, cap, ctypes.byref(cnt)) == 0
    assert cnt.value == n and np.array_equal(dev.getDevData().reshape(cap, 4), want[:cap])
    assert L.rmd_volume_surface_points(v.handle, None, 0, ctypes.byref(cnt)) == 0 and cnt.value == n
    T = seq.frame(5, want_depth=False).T_cam_world
    assert np.array_equal(v.raycast(rmd.PinholeCamera(*seq.camera), T, 160, 120).view(np.uint32),
                          o.raycast(seq.camera, T, 160, 120).view(np.uint32))
    v.reset()
    assert not v.download()[1].any()


# ------------------------------------------------------------------ ordering
@pytest.mark.gpu
@pytest.mark.parametrize("source", ["mu", "denoised"])
def test_integrate_is_ordered_before_the_next_update(source):
    """integrate(seeds) and update(seeds) back to back, no host sync: the volume holds the state from before the
    update."""
    import rpg_open_remode_b200 as rmd
    from rpg_open_remode_b200 import synth
    W, H, n = 640, 480, 30
    seq = synth.SyntheticSequence(W, H, seed=0x5EED0530)
    cam = rmd.PinholeCamera(*seq.camera)
    f0 = seq.frame(0)
    dmin, dmax = float(f0.depth.min()), float(f0.depth.max())
    g = rmd.SeedMatrix(W, H, cam, device=0)
    g.setReferenceImage(f0.image, f0.T_cam_world, dmin, dmax)
    later = [seq.frame(k, want_depth=False) for k in range(1, n + 8)]
    for fr in later[:n]:
        g.update(fr.image, fr.T_cam_world)
    conv, mu = g.downloadConvergence(), g.downloadDepthmap()
    s, origin, tau = _grid(seq, [f0], 384)
    v, o = _pair((384, 384, 384), s, origin, tau)
    if source == "denoised":
        den = rmd.DepthmapDenoiser(W, H, device=0)
        den.setLargeSigmaSq(dmax - dmin)
        want_img = den.denoiseSeeds(g, 0.5, 200)
        img = rmd.DeviceImage(W, H, "float32")
        den.denoiseSeedsToDevice(g, img.data, img.pitch, 0.5, 200)
        v.integrate(g, img)
        o.integrate(want_img, seq.camera, f0.T_cam_world, conv)
    else:
        v.integrate(g)
        o.integrate(mu, seq.camera, f0.T_cam_world, conv)
    for fr in later[n:]:            # immediately: these overwrite mu and the convergence map
        g.update(fr.image, fr.T_cam_world)
    g.sync()
    assert not np.array_equal(g.downloadDepthmap(), mu)
    _same(v, o, f"ordering ({source})", check_points=False)


# ------------------------------------------------------------------ error codes
@pytest.mark.gpu
def test_error_codes():
    import rpg_open_remode_b200 as rmd
    from rpg_open_remode_b200 import _native, synth
    L = _native.lib()
    W, H = 160, 120
    seq = synth.SyntheticSequence(W, H, seed=0x5EED0540)
    cam = rmd.PinholeCamera(*seq.camera)
    o3 = np.zeros(3, F)
    h = ctypes.c_void_p()

    def create(nx=8, ny=8, nz=8, s=0.1, origin=o3, tau=0.3, wmax=10.0, out=True):
        return L.rmd_volume_create(nx, ny, nz, s, origin.ctypes.data if origin is not None else None, tau, wmax, 0,
                                   ctypes.byref(h) if out else None)

    assert create() == 0 and L.rmd_volume_destroy(h) == 0
    for bad in (dict(nx=0), dict(ny=-1), dict(nz=0), dict(s=0.0), dict(s=-0.1), dict(s=float("nan")),
                dict(tau=0.0), dict(tau=-1.0), dict(wmax=0.5), dict(wmax=float("nan")), dict(origin=None),
                dict(out=False), dict(nx=65536, ny=65536, nz=1), dict(nx=2048, ny=1024, nz=1025)):
        assert create(**bad) == INVALID, bad
    assert create(nx=2048, ny=1024, nz=1, s=0.1) == 0 and L.rmd_volume_destroy(h) == 0
    v = rmd.TsdfVolume((16, 16, 16), 0.1, (-0.8, -0.8, 0.5), 0.3, 10.0, device=0)
    f0 = seq.frame(0)
    T = np.ascontiguousarray(f0.T_cam_world.reshape(12))
    img = rmd.DeviceImage(W, H, "float32")
    conv = rmd.DeviceImage(W, H, "int32")
    img.setDevData(f0.depth)
    c = ctypes.c_float

    def integ(width=W, height=H, depth=img.data, pitch=img.pitch, conv_ptr=None, conv_pitch=0, pose=T.ctypes.data,
              handle=v.handle):
        return L.rmd_volume_integrate_depth(handle, width, height, c(cam.fx), c(cam.fy), c(cam.cx), c(cam.cy), pose,
                                            depth, pitch, conv_ptr, conv_pitch)

    assert integ() == 0
    assert integ(conv_ptr=conv.data, conv_pitch=conv.pitch) == 0
    for bad in (dict(width=0), dict(height=-1), dict(depth=None), dict(pose=None), dict(handle=None),
                dict(pitch=4 * W - 4), dict(pitch=4 * W + 2), dict(conv_ptr=conv.data, conv_pitch=4 * W - 4),
                dict(conv_ptr=conv.data, conv_pitch=4 * W + 2)):
        assert integ(**bad) == INVALID, bad
    g = rmd.SeedMatrix(W, H, cam, device=0)
    assert L.rmd_volume_integrate_seeds(v.handle, g.handle, None, 0) == NOT_INIT
    g.setReferenceImage(f0.image, f0.T_cam_world, float(f0.depth.min()), float(f0.depth.max()))
    assert L.rmd_volume_integrate_seeds(v.handle, g.handle, None, 0) == 0
    assert L.rmd_volume_integrate_seeds(v.handle, g.handle, img.data, img.pitch) == 0
    assert L.rmd_volume_integrate_seeds(v.handle, g.handle, img.data, 4 * W - 4) == INVALID
    assert L.rmd_volume_integrate_seeds(v.handle, None, None, 0) == INVALID
    assert L.rmd_volume_integrate_seeds(None, g.handle, None, 0) == INVALID
    n = ctypes.c_size_t()
    assert L.rmd_volume_surface_points(v.handle, None, 5, ctypes.byref(n)) == INVALID
    assert L.rmd_volume_surface_points(v.handle, None, 0, None) == INVALID
    assert L.rmd_volume_surface_points_device(v.handle, img.data + 4, 1, ctypes.byref(n)) == INVALID
    out = rmd.DeviceImage(W, H, "float32")
    assert L.rmd_volume_raycast(v.handle, W, H, c(cam.fx), c(cam.fy), c(cam.cx), c(cam.cy), T.ctypes.data, out.data,
                                4 * W - 4) == INVALID
    assert L.rmd_volume_raycast(v.handle, 0, H, c(cam.fx), c(cam.fy), c(cam.cx), c(cam.cy), T.ctypes.data, out.data,
                                out.pitch) == INVALID
    assert L.rmd_volume_download(v.handle, None, None) == INVALID
    assert L.rmd_volume_upload(v.handle, None, None) == INVALID
    for fn in (L.rmd_volume_reset, L.rmd_volume_sync):
        assert fn(None) == INVALID
    assert L.rmd_volume_size(None, None, None, None, None, None) == INVALID
    nx, s_, org = ctypes.c_int(), ctypes.c_float(), np.zeros(3, F)
    assert L.rmd_volume_size(v.handle, ctypes.byref(nx), None, None, ctypes.byref(s_), org.ctypes.data) == 0
    assert nx.value == 16 and s_.value == F(0.1) and np.array_equal(org, np.array([-0.8, -0.8, 0.5], F))
    assert L.rmd_volume_destroy(None) == 0
    if rmd.device_count() >= 2:
        other = rmd.SeedMatrix(W, H, cam, device=1)
        other.setReferenceImage(f0.image, f0.T_cam_world, 0.5, 2.0)
        assert L.rmd_volume_integrate_seeds(v.handle, other.handle, None, 0) == INVALID


# ------------------------------------------------------------------ the node
def _run_node(seq, n_frames, volume=None):
    """DepthmapNode over the sequence's 8-bit frames; returns what it published and, per finished keyframe, the
    reference frame's T_curr_world (computed as the node computes it), the converged mu and the convergence map."""
    import rpg_open_remode_b200 as rmd
    from rpg_open_remode_b200 import node
    W, H = seq.width, seq.height
    fx, fy, cx, cy = seq.camera
    f0 = seq.frame(0)
    dmin, dmax = float(f0.depth.min()), float(f0.depth.max())
    dm = rmd.Depthmap(W, H, fx, cx, fy, cy, device=0)
    published, keyframes, ref = [], [], {}

    def publisher(kind, d):
        if kind == "depthmap_and_pointcloud":
            published.append((d.getDepthmap().copy(), d.getConvergenceMap().copy()))
            keyframes.append((ref["k"], ref["T"], d.seeds_.downloadDepthmap()))

    nd = node.DepthmapNode(dm, publisher=publisher, volume=volume)
    for k in range(n_frames):
        fr = seq.frame(k, want_depth=False)
        T_world_curr = rmd.SE3(fr.T_world_cam.reshape(12))
        if nd.state_ == node.TAKE_REFERENCE_FRAME:
            ref["k"], ref["T"] = k, T_world_curr.inv().data.copy()
        nd.denseInputCallback(fr.image_u8, T_world_curr, dmin, dmax)
    return published, keyframes


@pytest.mark.gpu
def test_node_with_and_without_a_volume():
    import rpg_open_remode_b200 as rmd
    from rpg_open_remode_b200 import synth
    W, H, N = 320, 240, 90
    seq = synth.SyntheticSequence(W, H, seed=0x5EED0001)
    plain, _ = _run_node(seq, N)
    s, origin, tau = _grid(seq, [seq.frame(0), seq.frame(N - 1)], 160)
    v, o = _pair((160, 160, 160), s, origin, tau)
    fused, keyframes = _run_node(seq, N, v)
    assert len(plain) == len(fused) >= 2
    for (d0, c0), (d1, c1) in zip(plain, fused):       # the published maps do not change
        assert np.array_equal(d0.view(np.uint32), d1.view(np.uint32)) and np.array_equal(c0, c1)
    for (depth, conv), (_, T, _) in zip(fused, keyframes):
        o.integrate(depth, seq.camera, T, conv)
    _same(v, o, "node", seq.camera, [seq.frame(N // 2, want_depth=False).T_cam_world], (W, H))
    # fuseDenoisedInto's host map is downloadDenoisedDepthmap's
    fx, fy, cx, cy = seq.camera
    dm = rmd.Depthmap(W, H, fx, cx, fy, cy, device=0)
    f0 = seq.frame(0)
    dm.setReferenceImage(f0.image_u8, f0.T_cam_world, float(f0.depth.min()), float(f0.depth.max()))
    for k in range(1, 30):
        fr = seq.frame(k, want_depth=False)
        dm.update(fr.image_u8, fr.T_cam_world)
    dm.downloadDenoisedDepthmap(0.5, 200)
    a = dm.getDepthmap().copy()
    v.reset()
    dm.fuseDenoisedInto(v, 0.5, 200)
    assert np.array_equal(a.view(np.uint32), dm.getDepthmap().view(np.uint32))
    assert v.download()[1].any()


# ------------------------------------------------------------------ what fusion buys
# Measured on an H100 SXM 80 GB (DESIGN.md 5.3): bench.py's c2 sequence (VGA, 200 frames) through the node with a
# 512^3 volume, raycast at frames 50, 100, 150 and 199.
# Measured: 9 keyframes fused, error ratio 0.361 (2.36 mm against 6.55 mm), coverage ratio 4.73 (182 754 pixels hit
# against 38 612 converged seeds).
RAYCAST_ERROR_RATIO = 0.5      # median |raycast - truth| over hit pixels <= this x median |mu - truth| (published)
COVERAGE_RATIO = 3.0           # pixels hit at frame 199 > this x converged seeds of the last published keyframe


@pytest.mark.gpu
def test_what_fusion_buys_on_c2():
    import rpg_open_remode_b200 as rmd
    from rpg_open_remode_b200 import multi_gpu, synth
    W, H, N = 640, 480, 200
    seq = synth.SyntheticSequence(W, H, seed=multi_gpu.keyframe_seed(0))    # bench.py's c2 sequence
    s, origin, tau = _grid(seq, [seq.frame(k) for k in range(0, N, 25)] + [seq.frame(N - 1)], 512)
    v = rmd.TsdfVolume((512, 512, 512), s, origin, tau, 64.0, device=0)
    published, keyframes = _run_node(seq, N, v)
    assert len(keyframes) >= 3
    # the published converged seeds: |mu - truth| of each keyframe's CONVERGED pixels at its reference frame
    seed_err = np.concatenate([np.abs(mu - seq.frame(k).depth)[conv == 1]
                               for (_, conv), (k, _, mu) in zip(published, keyframes)])
    last_converged = int((published[-1][1] == 1).sum())
    cam = rmd.PinholeCamera(*seq.camera)
    ray_err, hits = [], {}
    for k in (50, 100, 150, 199):
        fr = seq.frame(k)
        d = v.raycast(cam, fr.T_cam_world, W, H)
        hit = d > 0
        hits[k] = int(hit.sum())
        ray_err.append(np.abs(d - fr.depth)[hit])
    e_ray, e_seed = float(np.median(np.concatenate(ray_err))), float(np.median(seed_err))
    print(f"\nc2 + 512^3 volume (s = {float(s) * 1000:.2f} mm): {len(keyframes)} keyframes fused; median |raycast - truth| "
          f"= {e_ray:.5f} m vs median |mu - truth| of the published converged seeds = {e_seed:.5f} m (ratio "
          f"{e_ray / e_seed:.3f}); pixels hit {hits} vs {last_converged} converged seeds in the last published keyframe "
          f"(ratio {hits[199] / max(1, last_converged):.2f})")
    assert e_ray <= RAYCAST_ERROR_RATIO * e_seed
    assert hits[199] > COVERAGE_RATIO * last_converged
