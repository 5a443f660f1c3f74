"""The TSDF volume's normals on the GPU (csrc/volume.cu: the NORMALS surface write instance and
volume_raycast_normals_kernel; rmd_volume_surface_normals[_device], rmd_volume_raycast_normals,
api.TsdfVolume.surfaceNormals / raycastNormals; DESIGN.md 4.8).

  * the product against the oracle (oracle/rmd_oracle_volume_normals.c) bit for bit: the surface normals (count,
    order, bits) and the raycast normals, with a raycast depth identical to rmd_volume_raycast's -- ground truth at
    QVGA and VGA with and without a state map, real filter output (mu and denoised, 5x5 and 7x7), a ragged grid, a
    grid of more than 2^31 bytes, capacities smaller than the count, a volume with the intensity channel;
  * one normal per mesh vertex;
  * every error code;
  * the node on bench.py's c2 sequence: raycast normals against normals of the frames' true depth.
"""
import ctypes

import numpy as np
import pytest

import volume_normals_oracle as vno
from test_volume import _grid, _run_node
from test_volume_normals_oracle import normal_quality
from test_volume_oracle import ground_truth_points

F = np.float32
INVALID = -1
u32 = np.uint32


def _pair(dims, s, origin, tau, wmax=64.0, intensity=False):
    import rpg_open_remode_b200 as rmd
    return (rmd.TsdfVolume(dims, s, origin, tau, wmax, device=0, intensity=intensity),
            vno.OracleVolume(dims, s, origin, tau, wmax))


def _same(v, o, what, cam, poses, size, mesh=True):
    import rpg_open_remode_b200 as rmd
    t, w = v.download()
    assert np.array_equal(t.view(u32), o.tsdf.view(u32)) and np.array_equal(w, o.weight), what
    got, (want, n) = v.surfaceNormals(), o.surface_normals()
    assert len(got) == n > 0, what
    assert np.array_equal(got.view(u32), want[:, :3].view(u32)), \
        f"{what}: surface normals differ at {(got.view(u32) != want[:, :3].view(u32)).any(1).sum()} of {n} points"
    assert (np.abs(got).sum(1) > 0).mean() > 0.9, what
    if mesh:
        verts, _ = v.mesh()
        assert len(verts) == len(got), what
    for T in poses:
        cam_ = rmd.PinholeCamera(*cam)
        d0 = v.raycast(cam_, T, *size)
        d, nr = v.raycastNormals(cam_, T, *size)
        dw, nw = o.raycast_normals(cam, T, *size)
        assert np.array_equal(d.view(u32), d0.view(u32)) and np.array_equal(d.view(u32), dw.view(u32)), what
        assert np.array_equal(nr.view(u32), nw[..., :3].view(u32)), \
            f"{what}: raycast normals differ at {(nr.view(u32) != nw[..., :3].view(u32)).any(-1).sum()} pixels"
        assert (np.abs(nr).sum(-1) > 0).sum() > 0.5 * (d > 0).sum() > 0, what


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
    seq = synth.SyntheticSequence(W, H, seed=0x5EED0700 + W)
    frames = [seq.frame(k) for k in (0, 25, 50)]
    s, origin, tau = _grid(seq, frames, max(dims))
    v, o = _pair(dims, s, origin, tau)
    cam = rmd.PinholeCamera(*seq.camera)
    rng = np.random.default_rng(W + 11)
    for fr in frames:
        conv = np.where(rng.random((H, W)) < 0.9, 1, rng.integers(2, 6, (H, W))).astype(np.int32) \
            if with_conv else None
        depth = fr.depth.copy()
        depth[rng.random((H, W)) < 0.01] = np.nan
        v.integrateDepth(depth, cam, fr.T_cam_world, conv)
        o.integrate(depth, seq.camera, fr.T_cam_world, conv)
    poses = [seq.frame(k, want_depth=False).T_cam_world for k in (12, 40)]
    _same(v, o, f"{size} {dims}", seq.camera, poses, (W, H))


@pytest.mark.gpu
@pytest.mark.parametrize("size,patch,n", [((320, 240), 5, 40), ((320, 240), 7, 40), ((640, 480), 5, 30)])
def test_filter_output_equals_oracle(size, patch, n):
    """Keyframes of the real depth filter: mu and the denoised image."""
    import rpg_open_remode_b200 as rmd
    from rpg_open_remode_b200 import synth
    W, H = size
    seq = synth.SyntheticSequence(W, H, seed=0x5EED0710 + W + patch)
    cam = rmd.PinholeCamera(*seq.camera)
    f0 = seq.frame(0)
    dmin, dmax = float(f0.depth.min()), float(f0.depth.max())
    s, origin, tau = _grid(seq, [f0], 160)
    v_mu, o_mu = _pair((160, 160, 160), s, origin, tau)
    v_dn, o_dn = _pair((160, 160, 160), s, origin, tau)
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
def test_intensity_volume_equals_oracle():
    """The normals read the tsdf records only: a volume with the intensity channel gives the same bits."""
    import rpg_open_remode_b200 as rmd
    from rpg_open_remode_b200 import synth
    W, H = 320, 240
    seq = synth.SyntheticSequence(W, H, seed=0x5EED0720)
    frames = [seq.frame(k) for k in (0, 30)]
    s, origin, tau = _grid(seq, frames, 192)
    v, o = _pair((192, 192, 192), s, origin, tau, intensity=True)
    plain = rmd.TsdfVolume((192, 192, 192), s, origin, tau, 64.0, device=0)
    cam = rmd.PinholeCamera(*seq.camera)
    for fr in frames:
        v.integrateDepth(fr.depth, cam, fr.T_cam_world, None, fr.image)
        plain.integrateDepth(fr.depth, cam, fr.T_cam_world)
        o.integrate(fr.depth, seq.camera, fr.T_cam_world)
    T = seq.frame(15, want_depth=False).T_cam_world
    _same(v, o, "intensity volume", seq.camera, [T], (W, H))
    assert np.array_equal(v.surfaceNormals().view(u32), plain.surfaceNormals().view(u32))
    assert np.array_equal(v.raycastNormals(cam, T, W, H)[1].view(u32), plain.raycastNormals(cam, T, W, H)[1].view(u32))


@pytest.mark.gpu
def test_grid_beyond_2gb_and_capacity():
    """1024 x 1024 x 320 voxels: 2.7 GB of records, 64-bit indexing of the neighbour loads.  Then capacities
    smaller than the count on the host and the device variant, and the count-only call."""
    import rpg_open_remode_b200 as rmd
    from rpg_open_remode_b200 import _native, synth
    W, H = 640, 480
    seq = synth.SyntheticSequence(W, H, seed=0x5EED0730)
    f0 = seq.frame(0)
    pts = ground_truth_points(f0, seq.camera).reshape(-1, 3)
    dims = (1024, 1024, 320)
    lo, hi = pts.min(0), pts.max(0)
    s = F(((hi - lo) / (np.array(dims) - 1 - 16)).max())
    origin = (lo - 8 * float(s)).astype(F)
    origin[2] = F(hi[2] - (dims[2] - 1 - 8) * float(s))   # the farthest surface in the last planes, beyond 2^31 B
    v, o = _pair(dims, s, origin, F(4) * s)
    cam = rmd.PinholeCamera(*seq.camera)
    v.integrateDepth(f0.depth, cam, f0.T_cam_world)
    o.integrate(f0.depth, seq.camera, f0.T_cam_world)
    want, n = o.surface_normals()
    got = v.surfaceNormals()
    assert len(got) == n > 0 and np.array_equal(got.view(u32), want[:, :3].view(u32))
    assert (o.weight.reshape(-1)[2 ** 28:] > 0).any()     # records beyond the first 2^31 bytes are reached
    L, cnt = _native.lib(), ctypes.c_size_t()
    cap = n // 7
    part = np.empty((cap, 4), F)
    assert L.rmd_volume_surface_normals(v.handle, part.ctypes.data, cap, ctypes.byref(cnt)) == 0
    assert cnt.value == n and np.array_equal(part.view(u32), want[:cap].view(u32))     # (nx, ny, nz, 0)
    dev = rmd.DeviceImage(4 * cap, 1, "float32")
    assert L.rmd_volume_surface_normals_device(v.handle, dev.data, cap, ctypes.byref(cnt)) == 0
    assert cnt.value == n and np.array_equal(dev.getDevData().reshape(cap, 4).view(u32), want[:cap].view(u32))
    assert L.rmd_volume_surface_normals(v.handle, None, 0, ctypes.byref(cnt)) == 0 and cnt.value == n
    assert L.rmd_volume_surface_normals_device(v.handle, None, 0, ctypes.byref(cnt)) == 0 and cnt.value == n
    assert len(v.surfaceNormals(capacity=cap)) == cap
    T = seq.frame(5, want_depth=False).T_cam_world
    d, nr = v.raycastNormals(cam, T, 160, 120)
    dw, nw = o.raycast_normals(seq.camera, T, 160, 120)
    assert np.array_equal(d.view(u32), dw.view(u32)) and np.array_equal(nr.view(u32), nw[..., :3].view(u32))
    assert (d > 0).sum() > 1000


# ------------------------------------------------------------------ error codes
@pytest.mark.gpu
def test_error_codes():
    import rpg_open_remode_b200 as rmd
    from rpg_open_remode_b200 import _native, synth
    L = _native.lib()
    W, H = 160, 120
    seq = synth.SyntheticSequence(W, H, seed=0x5EED0740)
    cam = rmd.PinholeCamera(*seq.camera)
    c = ctypes.c_float
    f0 = seq.frame(0)
    T = np.ascontiguousarray(f0.T_cam_world.reshape(12))
    out = rmd.DeviceImage(W, H, "float32")
    nrm = rmd.DeviceImage(4 * W, H, "float32")
    assert nrm.pitch % 16 == 0 and nrm.data % 16 == 0
    v = rmd.TsdfVolume((16, 16, 16), 0.1, (-0.8, -0.8, 0.5), 0.3, 10.0, device=0)
    v.integrateDepth(f0.depth, cam, f0.T_cam_world)
    n = ctypes.c_size_t()

    def ray(handle=v.handle, width=W, height=H, pose=T.ctypes.data, dp=out.data, dpitch=out.pitch, np_=nrm.data,
            npitch=nrm.pitch):
        return L.rmd_volume_raycast_normals(handle, width, height, c(cam.fx), c(cam.fy), c(cam.cx), c(cam.cy), pose,
                                            dp, dpitch, np_, npitch)

    assert ray() == 0 and ray(npitch=16 * W) == 0
    for bad in (dict(handle=None), dict(width=0), dict(height=-1), dict(pose=None), dict(dp=None), dict(np_=None),
                dict(dpitch=4 * W - 4), dict(dpitch=4 * W + 2), dict(npitch=16 * W - 16), dict(npitch=16 * W + 4),
                dict(npitch=16 * W + 8), dict(np_=nrm.data + 4), dict(np_=nrm.data + 8)):
        assert ray(**bad) == INVALID, bad
    assert L.rmd_volume_surface_normals(v.handle, None, 5, ctypes.byref(n)) == INVALID
    assert L.rmd_volume_surface_normals(v.handle, None, 0, None) == INVALID
    assert L.rmd_volume_surface_normals(None, None, 0, ctypes.byref(n)) == INVALID
    assert L.rmd_volume_surface_normals_device(v.handle, nrm.data + 4, 1, ctypes.byref(n)) == INVALID
    assert L.rmd_volume_surface_normals_device(v.handle, nrm.data + 8, 1, ctypes.byref(n)) == INVALID
    assert L.rmd_volume_surface_normals_device(v.handle, None, 3, ctypes.byref(n)) == INVALID
    assert L.rmd_volume_surface_normals_device(v.handle, None, 0, None) == INVALID
    assert L.rmd_volume_surface_normals_device(None, None, 0, ctypes.byref(n)) == INVALID
    # a refused call leaves the volume usable
    assert L.rmd_volume_surface_normals(v.handle, None, 0, ctypes.byref(n)) == 0
    assert L.rmd_volume_surface_normals_device(v.handle, nrm.data, 1, ctypes.byref(n)) == 0
    # an empty volume: no points, no hits, every normal (0, 0, 0)
    e = rmd.TsdfVolume((16, 16, 16), 0.1, (-0.8, -0.8, 0.5), 0.3, 10.0, device=0)
    assert len(e.surfaceNormals()) == 0
    d, nr = e.raycastNormals(cam, f0.T_cam_world, W, H)
    assert not d.any() and not nr.any()


# ------------------------------------------------------------------ the node
# Measured on an H100 80 GB HBM3 at 400 W (DESIGN.md 5.3): bench.py's c2 sequence (VGA, 200 frames) through the node
# into a 512^3 volume, raycast at frames 50, 100, 150 and 199 against normals of the frames' ground-truth depth.
# Measured: 9 keyframes fused; median angle 6.14 / 6.17 / 6.12 / 6.09 deg against 9.33 / 9.19 / 9.28 / 9.13 deg for
# finite differences of the raycast depth (ratio <= 0.66); share of hits with a normal 0.9978 / 0.9969 / 0.9980 /
# 0.9975; facing the camera 0.9999 / 1.0 / 1.0 / 0.9999.
NODE_MEDIAN_DEG = 8.0            # median angle of the raycast normals to the true normals
NODE_OVER_DEPTH_FD = 0.8         # ... over that of finite differences of the raycast depth
NODE_NORMAL_SHARE = 0.99         # hits with a normal, over all hits
NODE_FACING_SHARE = 0.99         # normals with n . dir < 0, over the hits with a normal


@pytest.mark.gpu
def test_normals_on_c2():
    import rpg_open_remode_b200 as rmd
    from rpg_open_remode_b200 import multi_gpu, synth
    W, H, N = 640, 480, 200
    seq = synth.SyntheticSequence(W, H, seed=multi_gpu.keyframe_seed(0))    # bench.py's c2 sequence
    s, origin, tau = _grid(seq, [seq.frame(k) for k in range(0, N, 25)] + [seq.frame(N - 1)], 512)
    v = rmd.TsdfVolume((512, 512, 512), s, origin, tau, 64.0, device=0)
    published, keyframes = _run_node(seq, N, v)
    assert len(keyframes) >= 3
    cam = rmd.PinholeCamera(*seq.camera)
    meds, fds, shares, facings = [], [], [], []
    for k in (50, 100, 150, 199):
        fr = seq.frame(k)
        d, nr = v.raycastNormals(cam, fr.T_cam_world, W, H)
        assert np.array_equal(d.view(u32), v.raycast(cam, fr.T_cam_world, W, H).view(u32))
        med, med_fd, share, facing = normal_quality(d, nr, ground_truth_points(fr, seq.camera), fr.depth, seq.camera,
                                                    fr.T_world_cam)
        meds.append(np.degrees(med))
        fds.append(np.degrees(med_fd))
        shares.append(share)
        facings.append(facing)
    print(f"\nc2 + 512^3 volume: {len(keyframes)} keyframes; per view (50, 100, 150, 199): median angle to the true "
          f"normals {np.round(meds, 2).tolist()} deg vs {np.round(fds, 2).tolist()} deg for finite differences of the "
          f"raycast depth; share of hits with a normal {np.round(shares, 4).tolist()}, facing the camera "
          f"{np.round(facings, 4).tolist()}")
    for m, f, sh, fa in zip(meds, fds, shares, facings):
        assert m <= NODE_MEDIAN_DEG
        assert m <= NODE_OVER_DEPTH_FD * f
        assert sh >= NODE_NORMAL_SHARE and fa >= NODE_FACING_SHARE
    verts, tris = v.mesh()
    nrm = v.surfaceNormals()
    assert len(nrm) == len(verts) and len(tris) > 0 and (np.abs(nrm).sum(1) > 0).mean() > 0.99
