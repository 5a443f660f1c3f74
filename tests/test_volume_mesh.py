"""The TSDF volume's triangle mesh on the GPU (volume_mesh_{count,write}_kernel, rmd_volume_mesh[_device],
api.TsdfVolume.mesh; DESIGN.md 4.8).

  * the product against the oracle (oracle/rmd_oracle_mesh.c) bit for bit -- vertices and triangles -- on the fusion
    cases of test_volume.py: ground-truth depth at QVGA and VGA into 256^3 and the ragged 97x64x71 grid, real filter
    output with mu and the denoised image (5x5, 7x7), and the 1024x1024x320 grid with capacities smaller than both
    counts on the host and device variants and the count-only call;
  * an uploaded analytic sphere: the oracle's mesh, closed, genus 0, outward;
  * every error code, RMD_ERR_UNSUPPORTED on a 3-D checkerboard with more than 2^31 vertices;
  * the node's fusion of bench.py's c2 sequence meshes to a manifold with valid indices.
"""
import ctypes

import numpy as np
import pytest

import mesh_checks as mc
import mesh_oracle as mo
from test_volume import _grid, _pair, _run_node
from test_volume_oracle import ground_truth_points

F = np.float32
INVALID, UNSUPPORTED = -1, -3


def _same_mesh(v, o, what):
    got_v, got_t = v.mesh()
    want_v, want_t = mo.mesh(o)
    assert len(got_v) == len(want_v) > 0, f"{what}: {len(got_v)} / {len(want_v)} vertices"
    assert np.array_equal(got_v.view(np.uint32), want_v.view(np.uint32)), f"{what}: vertices differ"
    assert len(got_t) == len(want_t) > 0, f"{what}: {len(got_t)} / {len(want_t)} triangles"
    assert np.array_equal(got_t, want_t), f"{what}: triangles differ at {(got_t != want_t).any(1).sum()}"
    assert np.array_equal(got_v.view(np.uint32), v.surfacePoints().view(np.uint32))
    mc.open_edges(got_t, len(got_v))       # no directed edge twice
    return got_v, got_t


@pytest.mark.gpu
@pytest.mark.parametrize("size,dims,with_conv", [((320, 240), (256, 256, 256), False),
                                                 ((640, 480), (256, 256, 256), True),
                                                 ((320, 240), (97, 64, 71), True)])
def test_ground_truth_mesh_equals_oracle(size, dims, with_conv):
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
        conv = np.where(rng.random((H, W)) < 0.9, 1, rng.integers(2, 6, (H, W))).astype(np.int32) \
            if with_conv else None
        depth = fr.depth.copy()
        depth[rng.random((H, W)) < 0.01] = np.nan
        v.integrateDepth(depth, cam, fr.T_cam_world, conv)
        o.integrate(depth, seq.camera, fr.T_cam_world, conv)
    _same_mesh(v, o, f"{size} {dims}")


@pytest.mark.gpu
@pytest.mark.parametrize("size,patch,n", [((320, 240), 5, 40), ((320, 240), 7, 40), ((640, 480), 5, 30)])
def test_filter_output_mesh_equals_oracle(size, patch, n):
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
    _same_mesh(v_mu, o_mu, f"mu {size} p{patch}")
    _same_mesh(v_dn, o_dn, f"denoised {size} p{patch}")


@pytest.mark.gpu
def test_grid_beyond_2gb_capacities_and_count_only():
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
    want_v, want_t = mo.mesh(o)
    _same_mesh(v, o, "1024x1024x320")
    L = _native.lib()
    nv, nt = ctypes.c_size_t(), ctypes.c_size_t()
    assert L.rmd_volume_mesh(v.handle, None, 0, None, 0, ctypes.byref(nv), ctypes.byref(nt)) == 0
    assert (nv.value, nt.value) == (len(want_v), len(want_t))
    assert L.rmd_volume_mesh_device(v.handle, None, 0, None, 0, ctypes.byref(nv), ctypes.byref(nt)) == 0
    assert (nv.value, nt.value) == (len(want_v), len(want_t))
    cv, ct = len(want_v) // 7, len(want_t) // 5
    pv, pt = np.full((cv + 3, 4), -7, F), np.full((ct + 3, 3), -7, np.int32)
    assert L.rmd_volume_mesh(v.handle, pv.ctypes.data, cv, pt.ctypes.data, ct, ctypes.byref(nv),
                             ctypes.byref(nt)) == 0
    assert (nv.value, nt.value) == (len(want_v), len(want_t))
    assert np.array_equal(pv[:cv], want_v[:cv]) and np.all(pv[cv:] == -7)
    assert np.array_equal(pt[:ct], want_t[:ct]) and np.all(pt[ct:] == -7)
    assert pt[:ct].max() >= cv           # triangles index vertices beyond the vertex capacity
    dv, dt = rmd.DeviceImage(4 * (cv + 3), 1, "float32"), rmd.DeviceImage(3 * (ct + 3), 1, "int32")
    dv.setDevData(np.full((1, 4 * (cv + 3)), -7, F))
    dt.setDevData(np.full((1, 3 * (ct + 3)), -7, np.int32))
    assert L.rmd_volume_mesh_device(v.handle, dv.data, cv, dt.data, ct, ctypes.byref(nv), ctypes.byref(nt)) == 0
    assert (nv.value, nt.value) == (len(want_v), len(want_t))
    gv, gt = dv.getDevData().reshape(-1, 4), dt.getDevData().reshape(-1, 3)
    assert np.array_equal(gv[:cv], want_v[:cv]) and np.all(gv[cv:] == -7)
    assert np.array_equal(gt[:ct], want_t[:ct]) and np.all(gt[ct:] == -7)
    # vertices only, triangles only
    got = v.mesh(vertex_capacity=cv, triangle_capacity=0)
    assert np.array_equal(got[0], want_v[:cv]) and len(got[1]) == 0
    got = v.mesh(vertex_capacity=0, triangle_capacity=ct)
    assert len(got[0]) == 0 and np.array_equal(got[1], want_t[:ct])


@pytest.mark.gpu
def test_uploaded_sphere():
    import rpg_open_remode_b200 as rmd
    S = dict(dims=(90, 80, 70), s=0.025, origin=(-1.1, -0.98, -0.85), centre=(0.02, 0.01, 0.03), radius=0.75)
    tau = 3 * S["s"]
    tsdf, weight = mc.sphere_field(S["dims"], S["s"], S["origin"], S["centre"], S["radius"], tau)
    v = rmd.TsdfVolume(S["dims"], S["s"], S["origin"], tau, 64.0, device=0)
    o = mo.OracleVolume(S["dims"], S["s"], S["origin"], tau, 64.0)
    v.upload(tsdf, weight)
    o.tsdf[...], o.weight[...] = tsdf, weight
    verts, tris = _same_mesh(v, o, "sphere")
    mc.assert_sphere_mesh(verts, tris, S["centre"], S["radius"])


def _checkerboard_plane(nx, ny):
    j, i = np.mgrid[0:ny, 0:nx]
    return np.where((i + j) & 1, F(-0.5), F(0.5)).astype(F)


@pytest.mark.gpu
def test_error_codes():
    import rpg_open_remode_b200 as rmd
    from rpg_open_remode_b200 import _native
    L = _native.lib()
    dims = (12, 10, 9)
    tsdf, weight = mc.sphere_field(dims, 0.1, (-0.55, -0.45, -0.4), (0, 0, 0), 0.3, 0.2)
    v = rmd.TsdfVolume(dims, 0.1, (-0.55, -0.45, -0.4), 0.2, 10.0, device=0)
    v.upload(tsdf, weight)
    nv, nt = ctypes.c_size_t(), ctypes.c_size_t()
    buf_v, buf_t = np.zeros((64, 4), F), np.zeros((64, 3), np.int32)
    dv, dt = rmd.DeviceImage(256, 1, "float32"), rmd.DeviceImage(192, 1, "int32")
    for fn, (pv, pt) in ((L.rmd_volume_mesh, (buf_v.ctypes.data, buf_t.ctypes.data)),
                         (L.rmd_volume_mesh_device, (dv.data, dt.data))):
        assert fn(v.handle, pv, 64, pt, 64, ctypes.byref(nv), ctypes.byref(nt)) == 0 and nv.value > 0
        for bad in ((None, pv, 64, pt, 64, ctypes.byref(nv), ctypes.byref(nt)),
                    (v.handle, pv, 64, pt, 64, None, ctypes.byref(nt)),
                    (v.handle, pv, 64, pt, 64, ctypes.byref(nv), None),
                    (v.handle, None, 1, pt, 64, ctypes.byref(nv), ctypes.byref(nt)),
                    (v.handle, pv, 64, None, 1, ctypes.byref(nv), ctypes.byref(nt))):
            assert fn(*bad) == INVALID, (fn, bad)
    assert L.rmd_volume_mesh_device(v.handle, dv.data + 4, 8, dt.data, 8, ctypes.byref(nv), ctypes.byref(nt)) \
        == INVALID
    assert L.rmd_volume_mesh_device(v.handle, dv.data, 8, dt.data + 2, 8, ctypes.byref(nv), ctypes.byref(nt)) \
        == INVALID
    assert L.rmd_volume_mesh_device(v.handle, dv.data, 8, dt.data + 4, 8, ctypes.byref(nv), ctypes.byref(nt)) == 0
    del v
    # a 3-D checkerboard of +-0.5, weight 1: a point on every edge of the grid, more than 2^31 of them
    nx, ny, nz = 1024, 1024, 684
    n_points = (nx - 1) * ny * nz + nx * (ny - 1) * nz + nx * ny * (nz - 1)
    assert n_points >= 2 ** 31
    big = rmd.TsdfVolume((nx, ny, nz), 0.01, (0, 0, 0), 0.04, 64.0, device=0)
    plane = _checkerboard_plane(nx, ny)
    t = np.empty((nz, ny, nx), F)
    t[0::2], t[1::2] = plane, -plane
    big.upload(t, np.ones((nz, ny, nx), F))
    del t, plane
    nv.value, nt.value = 0, 0
    assert L.rmd_volume_mesh(big.handle, None, 0, None, 0, ctypes.byref(nv), ctypes.byref(nt)) == UNSUPPORTED
    assert nv.value == n_points
    assert nt.value == 4 * (nx - 1) * (ny - 1) * (nz - 1)   # every cube: four inside corners cut off
    sentinel_v, sentinel_t = np.full((4, 4), -7, F), np.full((4, 3), -7, np.int32)
    assert L.rmd_volume_mesh(big.handle, sentinel_v.ctypes.data, 4, sentinel_t.ctypes.data, 4, ctypes.byref(nv),
                             ctypes.byref(nt)) == UNSUPPORTED
    assert nv.value == n_points and np.all(sentinel_v == -7) and np.all(sentinel_t == -7)
    with pytest.raises(rmd.RmdError):
        big.mesh()


@pytest.mark.gpu
def test_fused_c2_scene_is_a_manifold():
    import rpg_open_remode_b200 as rmd
    from rpg_open_remode_b200 import multi_gpu, synth
    W, H, N = 640, 480, 200
    seq = synth.SyntheticSequence(W, H, seed=multi_gpu.keyframe_seed(0))    # bench.py's c2 sequence
    s, origin, tau = _grid(seq, [seq.frame(k) for k in range(0, N, 25)] + [seq.frame(N - 1)], 512)
    v = rmd.TsdfVolume((512, 512, 512), s, origin, tau, 64.0, device=0)
    _, keyframes = _run_node(seq, N, v)
    assert len(keyframes) >= 3
    verts, tris = v.mesh()
    assert len(tris) > 10000 and tris.min() >= 0 and tris.max() < len(verts)
    assert np.array_equal(verts.view(np.uint32), v.surfacePoints().view(np.uint32))
    e = mc.open_edges(tris, len(verts))     # every edge in at most two triangles, in opposite directions
    area, _ = mc.area_and_volume(verts, tris)
    print(f"\nc2 + 512^3: {len(verts)} vertices, {len(tris)} triangles, {len(e)} open edges, area {area:.3f} m^2")
