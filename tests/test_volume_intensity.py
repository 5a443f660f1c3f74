"""The TSDF volume's intensity channel on the GPU (csrc/volume.cu INTENSITY instances, rmd_volume_*intensity*,
api.TsdfVolume(intensity=True); DESIGN.md 4.8).

  * the product against the oracle (oracle/rmd_oracle_volume_intensity.c) bit for bit: every voxel's intensity
    record, the surface intensities (count, order, bits) and the raycast intensity -- ground truth at QVGA and VGA,
    real filter output (mu and denoised, 5x5 and 7x7), 8-bit reference frames with undistortion, a ragged grid, a
    grid of more than 2^31 bytes, capacities smaller than the count;
  * an enabled volume's tsdf, weight, surface points, mesh and raycast depth equal a plain volume's bit for bit;
  * device-side ordering of integrate_seeds against a following set_reference of the seeds;
  * every error code;
  * the node with an enabled volume on bench.py's c2 sequence: rendered views against the frames.
"""
import ctypes

import numpy as np
import pytest

import volume_intensity_oracle as vio
from test_volume import _grid, _run_node
from test_volume_oracle import ground_truth_points

F = np.float32
INVALID, NOT_INIT = -1, -2
u32 = np.uint32


def _trio(dims, s, origin, tau, wmax=64.0):
    """(plain volume, enabled volume, oracle)."""
    import rpg_open_remode_b200 as rmd
    return (rmd.TsdfVolume(dims, s, origin, tau, wmax, device=0),
            rmd.TsdfVolume(dims, s, origin, tau, wmax, device=0, intensity=True),
            vio.OracleVolume(dims, s, origin, tau, wmax))


def _same(plain, v, o, what, cam=None, poses=(), size=None, mesh=True):
    import rpg_open_remode_b200 as rmd
    t0, w0 = plain.download()
    t, w = v.download()
    assert np.array_equal(t.view(u32), t0.view(u32)) and np.array_equal(w.view(u32), w0.view(u32)), what
    assert np.array_equal(t.view(u32), o.tsdf.view(u32)) and np.array_equal(w, o.weight), what
    c, cw = v.downloadIntensity()
    assert np.array_equal(cw, o.cw), f"{what}: intensity weight differs at {(cw != o.cw).sum()} voxels"
    assert np.array_equal(c.view(u32), o.cint.view(u32)), \
        f"{what}: intensity differs at {(c.view(u32) != o.cint.view(u32)).sum()} voxels"
    assert (cw > 0).sum() > 0
    got, want = v.surfaceIntensity(), o.surface_intensity()[0]
    assert len(got) == len(want) > 0 and np.array_equal(got.view(u32), want.view(u32)), f"{what}: surface intensity"
    assert (got >= 0).mean() > 0.5, what
    if mesh:
        (pv, pt), (ev, et) = plain.mesh(), v.mesh()
        assert np.array_equal(pv.view(u32), ev.view(u32)) and np.array_equal(pt, et), f"{what}: mesh"
        assert len(ev) == len(got)
    for T in poses:
        cam_ = rmd.PinholeCamera(*cam)
        d0 = plain.raycast(cam_, T, *size)
        d, i = v.raycastIntensity(cam_, T, *size)
        dw, iw = o.raycast_intensity(cam, T, *size)
        assert np.array_equal(d.view(u32), d0.view(u32)) and np.array_equal(d.view(u32), dw.view(u32)), what
        assert np.array_equal(i.view(u32), iw.view(u32)), f"{what}: raycast intensity differs at {(i != iw).sum()}"
        assert (i >= 0).mean() > 0.02, what


# ------------------------------------------------------------------ product == oracle
@pytest.mark.gpu
@pytest.mark.parametrize("size,dims,with_conv", [((320, 240), (256, 256, 256), False),
                                                 ((320, 240), (256, 256, 256), True),
                                                 ((640, 480), (256, 256, 256), True),
                                                 ((640, 480), (256, 256, 256), False),
                                                 ((320, 240), (97, 64, 71), True)])
def test_ground_truth_equals_oracle(size, dims, with_conv):
    import rpg_open_remode_b200 as rmd
    from rpg_open_remode_b200 import synth
    W, H = size
    seq = synth.SyntheticSequence(W, H, seed=0x5EED0600 + W)
    frames = [seq.frame(k) for k in (0, 25, 50)]
    s, origin, tau = _grid(seq, frames, max(dims))
    plain, v, o = _trio(dims, s, origin, tau)
    cam = rmd.PinholeCamera(*seq.camera)
    rng = np.random.default_rng(W + 7)
    for fr in frames:
        conv = np.where(rng.random((H, W)) < 0.9, 1, rng.integers(2, 6, (H, W))).astype(np.int32) \
            if with_conv else None
        depth = fr.depth.copy()
        depth[rng.random((H, W)) < 0.01] = np.nan
        inten = fr.image.copy()
        inten[rng.random((H, W)) < 0.01] = np.nan
        inten[rng.random((H, W)) < 0.005] = np.inf
        plain.integrateDepth(depth, cam, fr.T_cam_world, conv)
        v.integrateDepth(depth, cam, fr.T_cam_world, conv, inten)
        o.integrate(depth, seq.camera, fr.T_cam_world, conv, inten)
    # a plain integration into the enabled volume leaves the channel alone
    fr = seq.frame(60)
    plain.integrateDepth(fr.depth, cam, fr.T_cam_world)
    v.integrateDepth(fr.depth, cam, fr.T_cam_world)
    o.integrate(fr.depth, seq.camera, fr.T_cam_world)
    _same(plain, v, o, f"{size} {dims}", seq.camera, [seq.frame(12, want_depth=False).T_cam_world], (W, H))


@pytest.mark.gpu
@pytest.mark.parametrize("size,patch,n", [((320, 240), 5, 40), ((320, 240), 7, 40), ((640, 480), 5, 30)])
def test_filter_output_equals_oracle(size, patch, n):
    """Keyframes of the real depth filter, fused with their float reference images: mu and the denoised image."""
    import rpg_open_remode_b200 as rmd
    from rpg_open_remode_b200 import synth
    W, H = size
    seq = synth.SyntheticSequence(W, H, seed=0x5EED0610 + W + patch)
    cam = rmd.PinholeCamera(*seq.camera)
    f0 = seq.frame(0)
    dmin, dmax = float(f0.depth.min()), float(f0.depth.max())
    s, origin, tau = _grid(seq, [f0], 160)
    p_mu, v_mu, o_mu = _trio((160, 160, 160), s, origin, tau)
    p_dn, v_dn, o_dn = _trio((160, 160, 160), s, origin, tau)
    den = rmd.DepthmapDenoiser(W, H, device=0)
    den.setLargeSigmaSq(dmax - dmin)
    img = rmd.DeviceImage(W, H, "float32")
    for ref in (0, n + 1):
        g = rmd.SeedMatrix(W, H, cam, patch_side=patch, device=0)
        fr = seq.frame(ref)
        g.setReferenceImage(fr.image, fr.T_cam_world, dmin, dmax)
        for k in range(ref + 1, ref + n + 1):
            fk = seq.frame(k, want_depth=False)
            g.update(fk.image, fk.T_cam_world)
        conv, mu = g.downloadConvergence(), g.downloadDepthmap()
        p_mu.integrate(g)
        v_mu.integrate(g)
        o_mu.integrate(mu, seq.camera, fr.T_cam_world, conv, fr.image)
        den.denoiseSeedsToDevice(g, img.data, img.pitch, 0.5, 100)
        p_dn.integrate(g, img)
        v_dn.integrate(g, img)
        den.sync()
        o_dn.integrate(img.getDevData(), seq.camera, fr.T_cam_world, conv, fr.image)
    view = [seq.frame(n // 2, want_depth=False).T_cam_world]
    _same(p_mu, v_mu, o_mu, f"mu {size} p{patch}", seq.camera, view, (W, H))
    _same(p_dn, v_dn, o_dn, f"denoised {size} p{patch}", seq.camera, view, (W, H))


@pytest.mark.gpu
def test_u8_reference_with_undistortion_equals_oracle():
    """8-bit reference frames through the undistortion map: the fused image is the seeds' own (undistorted,
    x 1/255) reference."""
    import rpg_open_remode_b200 as rmd
    from rpg_open_remode_b200 import synth
    W, H, n = 320, 240, 30
    seq = synth.SyntheticSequence(W, H, seed=0x5EED0620)
    cam = rmd.PinholeCamera(*seq.camera)
    f0 = seq.frame(0)
    dmin, dmax = float(f0.depth.min()), float(f0.depth.max())
    s, origin, tau = _grid(seq, [f0], 160)
    plain, v, o = _trio((160, 160, 160), s, origin, tau)
    g = rmd.SeedMatrix(W, H, cam, device=0)
    g.initUndistortionMap(-0.05, 0.01, 0.001, -0.001)
    g.setReferenceImage(f0.image_u8, f0.T_cam_world, dmin, dmax)
    for k in range(1, n + 1):
        fk = seq.frame(k, want_depth=False)
        g.update(fk.image_u8, fk.T_cam_world)
    conv, mu, ref = g.downloadConvergence(), g.downloadDepthmap(), g._download(rmd.FIELD_REF_IMG)
    want = (g.undistort(f0.image_u8).astype(F) * F(1.0 / 255.0)).astype(F)
    assert np.abs(ref - want).max() <= 1e-6 and not np.array_equal(g.undistort(f0.image_u8), f0.image_u8)
    plain.integrate(g)
    v.integrate(g)
    o.integrate(mu, seq.camera, f0.T_cam_world, conv, ref)
    _same(plain, v, o, "u8 + undistortion", seq.camera, [seq.frame(n // 2, want_depth=False).T_cam_world], (W, H))


@pytest.mark.gpu
def test_grid_beyond_2gb_and_capacity():
    """1024 x 1024 x 320 voxels: 2.7 GB of intensity records, 64-bit indexing of the colour array.  Then capacities
    smaller than the count on the host and the device variant."""
    import rpg_open_remode_b200 as rmd
    from rpg_open_remode_b200 import _native, synth
    W, H = 640, 480
    seq = synth.SyntheticSequence(W, H, seed=0x5EED0630)
    f0 = seq.frame(0)
    pts = ground_truth_points(f0, seq.camera).reshape(-1, 3)
    dims = (1024, 1024, 320)
    lo, hi = pts.min(0), pts.max(0)
    s = F(((hi - lo) / (np.array(dims) - 1 - 16)).max())
    origin = (lo - 8 * float(s)).astype(F)
    origin[2] = F(hi[2] - (dims[2] - 1 - 8) * float(s))   # the farthest surface in the last planes, beyond 2^31 B
    v = rmd.TsdfVolume(dims, s, origin, F(4) * s, 64.0, device=0, intensity=True)
    o = vio.OracleVolume(dims, s, origin, F(4) * s, 64.0)
    cam = rmd.PinholeCamera(*seq.camera)
    v.integrateDepth(f0.depth, cam, f0.T_cam_world, None, f0.image)
    o.integrate(f0.depth, seq.camera, f0.T_cam_world, None, f0.image)
    c, cw = v.downloadIntensity()
    assert np.array_equal(cw, o.cw) and np.array_equal(c.view(u32), o.cint.view(u32))
    assert (cw.reshape(-1)[2 ** 28:] > 0).any()     # records beyond the first 2^31 bytes are reached
    del c, cw
    want, n = o.surface_intensity()
    got = v.surfaceIntensity()
    assert len(got) == n > 0 and np.array_equal(got.view(u32), want.view(u32))
    L, cnt = _native.lib(), ctypes.c_size_t()
    cap = n // 7
    part = np.empty(cap, F)
    assert L.rmd_volume_surface_intensity(v.handle, part.ctypes.data, cap, ctypes.byref(cnt)) == 0
    assert cnt.value == n and np.array_equal(part.view(u32), want[:cap].view(u32))
    dev = rmd.DeviceImage(cap, 1, "float32")
    assert L.rmd_volume_surface_intensity_device(v.handle, dev.data, cap, ctypes.byref(cnt)) == 0
    assert cnt.value == n and np.array_equal(dev.getDevData().reshape(cap).view(u32), want[:cap].view(u32))
    assert L.rmd_volume_surface_intensity(v.handle, None, 0, ctypes.byref(cnt)) == 0 and cnt.value == n
    assert np.array_equal(v.surfacePoints().view(u32), o.surface_points()[0].view(u32))
    T = seq.frame(5, want_depth=False).T_cam_world
    d, i = v.raycastIntensity(cam, T, 160, 120)
    dw, iw = o.raycast_intensity(seq.camera, T, 160, 120)
    assert np.array_equal(d.view(u32), dw.view(u32)) and np.array_equal(i.view(u32), iw.view(u32))
    v.reset()
    assert not v.downloadIntensity()[1].any()


# ------------------------------------------------------------------ ordering
@pytest.mark.gpu
@pytest.mark.parametrize("how", ["host", "device", "u8"])
def test_integrate_is_ordered_before_the_next_set_reference(how):
    """integrate(seeds) and set_reference*(seeds) back to back, no host sync: the volume fuses the OLD reference
    image."""
    import rpg_open_remode_b200 as rmd
    from rpg_open_remode_b200 import synth
    W, H, n = 640, 480, 20
    seq = synth.SyntheticSequence(W, H, seed=0x5EED0640)
    cam = rmd.PinholeCamera(*seq.camera)
    f0 = seq.frame(0)
    dmin, dmax = float(f0.depth.min()), float(f0.depth.max())
    g = rmd.SeedMatrix(W, H, cam, device=0)
    g.setReferenceImage(f0.image, f0.T_cam_world, dmin, dmax)
    for k in range(1, n + 1):
        fk = seq.frame(k, want_depth=False)
        g.update(fk.image, fk.T_cam_world)
    conv, mu = g.downloadConvergence(), g.downloadDepthmap()
    s, origin, tau = _grid(seq, [f0], 384)
    plain, v, o = _trio((384, 384, 384), s, origin, tau)
    nxt = seq.frame(n + 1)
    new_img = rmd.DeviceImage(W, H, "float32")
    new_img.setDevData(np.ascontiguousarray(1.0 - nxt.image, F))
    g.sync()
    plain.integrate(g)
    plain.sync()          # the seeds order themselves after the last volume that read them: v
    v.integrate(g)
    if how == "host":
        g.setReferenceImage(1.0 - nxt.image, nxt.T_cam_world, dmin, dmax)
    elif how == "device":
        g.setReferenceImageDevice(new_img.data, new_img.pitch, nxt.T_cam_world, dmin, dmax)
    else:
        g.setReferenceImage(255 - nxt.image_u8, nxt.T_cam_world, dmin, dmax)
    g.sync()
    assert not np.array_equal(g._download(rmd.FIELD_REF_IMG), f0.image)
    o.integrate(mu, seq.camera, f0.T_cam_world, conv, f0.image)
    _same(plain, v, o, f"ordering ({how})", mesh=False)


# ------------------------------------------------------------------ error codes
@pytest.mark.gpu
def test_error_codes():
    import torch
    import rpg_open_remode_b200 as rmd
    from rpg_open_remode_b200 import _native, synth
    L = _native.lib()
    W, H = 160, 120
    seq = synth.SyntheticSequence(W, H, seed=0x5EED0650)
    cam = rmd.PinholeCamera(*seq.camera)
    c = ctypes.c_float
    f0 = seq.frame(0)
    T = np.ascontiguousarray(f0.T_cam_world.reshape(12))
    img, inten, out, out2 = (rmd.DeviceImage(W, H, "float32") for _ in range(4))
    img.setDevData(f0.depth)
    inten.setDevData(f0.image)
    conv = rmd.DeviceImage(W, H, "int32")
    plain = rmd.TsdfVolume((16, 16, 16), 0.1, (-0.8, -0.8, 0.5), 0.3, 10.0, device=0)
    v = rmd.TsdfVolume((16, 16, 16), 0.1, (-0.8, -0.8, 0.5), 0.3, 10.0, device=0, intensity=True)
    n = ctypes.c_size_t()
    buf = np.zeros(16 ** 3, F)

    def integ(handle=v.handle, width=W, height=H, depth=img.data, pitch=img.pitch, conv_ptr=None, conv_pitch=0,
              pose=T.ctypes.data, ip=inten.data, ipitch=inten.pitch):
        return L.rmd_volume_integrate_depth_intensity(handle, width, height, c(cam.fx), c(cam.fy), c(cam.cx),
                                                      c(cam.cy), pose, depth, pitch, conv_ptr, conv_pitch, ip, ipitch)

    def ray(handle=v.handle, width=W, height=H, pose=T.ctypes.data, dp=out.data, dpitch=out.pitch, ip=out2.data,
            ipitch=out2.pitch):
        return L.rmd_volume_raycast_intensity(handle, width, height, c(cam.fx), c(cam.fy), c(cam.cx), c(cam.cy), pose,
                                              dp, dpitch, ip, ipitch)

    assert integ() == 0 and integ(conv_ptr=conv.data, conv_pitch=conv.pitch) == 0 and ray() == 0
    for bad in (dict(handle=None), dict(width=0), dict(height=-1), dict(depth=None), dict(pose=None), dict(ip=None),
                dict(pitch=4 * W - 4), dict(ipitch=4 * W - 4), dict(ipitch=4 * W + 2),
                dict(conv_ptr=conv.data, conv_pitch=4 * W - 4)):
        assert integ(**bad) == INVALID, bad
    for bad in (dict(handle=None), dict(width=0), dict(pose=None), dict(dp=None), dict(ip=None),
                dict(dpitch=4 * W - 4), dict(ipitch=4 * W - 4), dict(ipitch=4 * W + 2)):
        assert ray(**bad) == INVALID, bad
    assert L.rmd_volume_surface_intensity(v.handle, None, 5, ctypes.byref(n)) == INVALID
    assert L.rmd_volume_surface_intensity(v.handle, None, 0, None) == INVALID
    assert L.rmd_volume_surface_intensity(None, None, 0, ctypes.byref(n)) == INVALID
    assert L.rmd_volume_surface_intensity_device(v.handle, img.data + 2, 1, ctypes.byref(n)) == INVALID
    assert L.rmd_volume_surface_intensity_device(v.handle, None, 3, ctypes.byref(n)) == INVALID
    assert L.rmd_volume_download_intensity(v.handle, None, None) == INVALID
    assert L.rmd_volume_upload_intensity(v.handle, buf.ctypes.data, None) == INVALID
    assert L.rmd_volume_enable_intensity(None) == INVALID
    assert L.rmd_volume_download_intensity(None, buf.ctypes.data, buf.ctypes.data) == INVALID
    # a volume without the channel
    assert integ(handle=plain.handle) == NOT_INIT
    assert ray(handle=plain.handle) == NOT_INIT
    assert L.rmd_volume_surface_intensity(plain.handle, None, 0, ctypes.byref(n)) == NOT_INIT
    assert L.rmd_volume_surface_intensity_device(plain.handle, None, 0, ctypes.byref(n)) == NOT_INIT
    assert L.rmd_volume_download_intensity(plain.handle, buf.ctypes.data, buf.ctypes.data) == NOT_INIT
    assert L.rmd_volume_upload_intensity(plain.handle, buf.ctypes.data, buf.ctypes.data) == NOT_INIT
    with pytest.raises(rmd.RmdError):
        plain.surfaceIntensity()
    # upload / download round trip; enable is idempotent (a second call keeps the records); reset clears the channel
    vals = np.random.default_rng(1).random(16 ** 3).astype(F)
    v.uploadIntensity(vals, vals * 2)
    assert L.rmd_volume_enable_intensity(v.handle) == 0
    got = v.downloadIntensity()
    assert np.array_equal(got[0].reshape(-1), vals) and np.array_equal(got[1].reshape(-1), vals * 2)
    v.reset()
    assert not v.downloadIntensity()[1].any() and not v.download()[1].any()
    # the channel does not fit: cudaErrorMemoryAllocation, and the volume stays usable without it
    big = rmd.TsdfVolume((1024, 1024, 256), 0.01, (0, 0, 0), 0.03, 10.0, device=0)   # 2 GB; channel 2 GB
    torch.cuda.set_device(0)
    free, _ = torch.cuda.mem_get_info(0)
    filler = torch.empty(int(free - (1 << 30)), dtype=torch.uint8, device="cuda:0")   # leaves 1 GB
    try:
        assert L.rmd_volume_enable_intensity(big.handle) == 2      # cudaErrorMemoryAllocation
        assert L.rmd_volume_surface_intensity(big.handle, None, 0, ctypes.byref(n)) == NOT_INIT
    finally:
        del filler
        torch.cuda.empty_cache()
    assert L.rmd_volume_enable_intensity(big.handle) == 0
    assert not big.downloadIntensity()[1].any()


# ------------------------------------------------------------------ the node
# Measured on an H100 80 GB HBM3 at 400 W (DESIGN.md 5.3): bench.py's c2 sequence (VGA, 200 frames) through the node
# with a 512^3 volume with the intensity channel, rendered at frames 50, 100, 150 and 199 against the frames.
# Measured: 9 keyframes fused; shaded share 0.9942 / 0.9931 / 0.9947 / 0.9939; median |rendered - frame| 9.35 / 9.37 /
# 9.56 / 9.34 grey levels against 22.66 / 22.52 / 22.68 / 23.41 for the frame's mean (ratio <= 0.42); correlation
# 0.890 / 0.891 / 0.887 / 0.890.
NODE_SHADED_SHARE = 0.97       # hits with an intensity, over all hits
NODE_ERROR_OVER_CONSTANT = 0.5   # median |rendered - frame| <= this x median |frame mean - frame| over shaded hits
NODE_CORRELATION = 0.8


@pytest.mark.gpu
def test_node_with_an_intensity_volume_on_c2():
    import rpg_open_remode_b200 as rmd
    from rpg_open_remode_b200 import multi_gpu, synth
    W, H, N = 640, 480, 200
    seq = synth.SyntheticSequence(W, H, seed=multi_gpu.keyframe_seed(0))    # bench.py's c2 sequence
    s, origin, tau = _grid(seq, [seq.frame(k) for k in range(0, N, 25)] + [seq.frame(N - 1)], 512)
    v = rmd.TsdfVolume((512, 512, 512), s, origin, tau, 64.0, device=0, intensity=True)
    published, keyframes = _run_node(seq, N, v)
    assert len(keyframes) >= 3
    cam = rmd.PinholeCamera(*seq.camera)
    shares, errs, consts, corrs = [], [], [], []
    for k in (50, 100, 150, 199):
        fr = seq.frame(k)
        d, i = v.raycastIntensity(cam, fr.T_cam_world, W, H)
        assert np.array_equal(d.view(u32), v.raycast(cam, fr.T_cam_world, W, H).view(u32))
        hit = d > 0
        shaded = hit & (i >= 0)
        truth, got = fr.image[shaded].astype(np.float64), i[shaded].astype(np.float64)
        shares.append(shaded.sum() / max(1, hit.sum()))
        errs.append(np.median(np.abs(got - truth)) * 255)
        consts.append(np.median(np.abs(truth.mean() - truth)) * 255)
        corrs.append(np.corrcoef(got, truth)[0, 1])
    print(f"\nc2 + 512^3 intensity volume: {len(keyframes)} keyframes; per view (50, 100, 150, 199): shaded share "
          f"{np.round(shares, 4).tolist()}, median |rendered - frame| {np.round(errs, 2).tolist()} grey levels vs "
          f"{np.round(consts, 2).tolist()} for the frame's mean, correlation {np.round(corrs, 3).tolist()}")
    for sh, e, c0, r in zip(shares, errs, consts, corrs):
        assert sh >= NODE_SHADED_SHARE
        assert e <= NODE_ERROR_OVER_CONSTANT * c0
        assert r >= NODE_CORRELATION
    # the shaded mesh: one intensity per vertex
    verts, tris = v.mesh()
    inten = v.surfaceIntensity()
    assert len(inten) == len(verts) and len(tris) > 0 and (inten >= 0).mean() > 0.9
