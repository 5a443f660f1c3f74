"""The TSDF volume's Euclidean signed distance field on the GPU (csrc/volume.cu: volume_esdf_kernel and
volume_esdf_query_kernel; rmd_volume_esdf*, api.TsdfVolume.computeEsdf / downloadEsdf / esdfQuery*,
DepthmapNode(esdf=True); DESIGN.md 4.8).

  * the product against the oracle (oracle/rmd_oracle_volume_esdf.c) bit for bit, snapshot (distance and weight) and
    query (distance, gradient, weight): ground truth at QVGA and VGA on 256^3 and 97 x 64 x 71, real filter output,
    uploaded adversarial grids, a grid after shifts, the 1024 x 1024 x 320 grid;
  * the size limit, the error codes, snapshot semantics without host syncs, the device query against the host query;
  * the node on bench.py's c2 sequence.
"""
import ctypes
import gc

import numpy as np
import pytest

import volume_esdf_oracle as veo
import volume_shift_oracle as vso
from test_volume import _grid
from test_volume_oracle import ground_truth_points

F = np.float32
u32 = np.uint32
INVALID, NOT_INITIALISED, UNSUPPORTED = -1, -2, -3


def _points(v, rng, n_random=20000):
    """Query points: the surface points, random points in and slightly around the window, and the window's corners."""
    n = np.array(v.dims)
    lo = v.origin.astype(np.float64)
    hi = lo + (n - 1) * v.voxel_size
    pad = 2 * v.voxel_size
    rnd = rng.uniform(lo - pad, hi + pad, (n_random, 3)).astype(F)
    corners = np.array([[lo[0], lo[1], lo[2]], [hi[0], hi[1], hi[2]], [hi[0], lo[1], lo[2]]], F)
    pts = [rnd, corners]
    sp = v.surfacePoints()
    if len(sp):
        pts.append(sp[:, :3])
    return np.concatenate(pts).astype(F)


def _same_esdf(v, tsdf, weight, what, rng, origin=None):
    """v's snapshot and queries against the oracle on records (tsdf, weight) at origin (default: v's)."""
    want_d, want_w = veo.esdf(tsdf, weight, v.voxel_size)
    got_d, got_w = v.downloadEsdf()
    assert np.array_equal(got_w.view(u32), want_w.view(u32)), f"{what}: ESDF weight differs"
    bad = got_d.view(u32) != want_d.view(u32)
    assert not bad.any(), f"{what}: distance differs at {bad.sum()} voxels, first {np.argwhere(bad)[:3]}"
    origin = v.origin if origin is None else origin
    pts = _points(v, rng)
    dg, w = v.esdfQuery(pts)
    want_dg, want_wq = veo.query(want_d, want_w, v.voxel_size, origin, pts)
    assert np.array_equal(dg.view(u32), want_dg.view(u32)), \
        f"{what}: query differs at {(dg.view(u32) != want_dg.view(u32)).any(1).sum()} points"
    assert np.array_equal(w.view(u32), want_wq.view(u32)), f"{what}: query weight differs"
    return want_d


# ------------------------------------------------------------------ product == oracle
@pytest.mark.gpu
@pytest.mark.parametrize("size,dims", [((320, 240), (256, 256, 256)), ((640, 480), (256, 256, 256)),
                                       ((320, 240), (97, 64, 71))])
def test_ground_truth_equals_oracle(size, dims):
    import rpg_open_remode_b200 as rmd
    from rpg_open_remode_b200 import synth
    W, H = size
    seq = synth.SyntheticSequence(W, H, seed=0x5EED0E00 + W)
    frames = [seq.frame(k) for k in (0, 25, 50)]
    s, origin, tau = _grid(seq, frames, max(dims))
    v = rmd.TsdfVolume(dims, s, origin, tau, 64.0, device=0)
    cam = rmd.PinholeCamera(*seq.camera)
    rng = np.random.default_rng(W)
    for fr in frames:
        v.integrateDepth(fr.depth, cam, fr.T_cam_world)
        v.computeEsdf()
        t, w = v.download()
        d = _same_esdf(v, t, w, f"{size} {dims}", rng)
    occ = veo.occupied(t, w)
    assert occ.any() and (~occ).any() and np.isfinite(d).all()


@pytest.mark.gpu
def test_filter_output_equals_oracle():
    import rpg_open_remode_b200 as rmd
    from rpg_open_remode_b200 import synth
    W, H = 320, 240
    seq = synth.SyntheticSequence(W, H, seed=0x5EED0E10)
    cam = rmd.PinholeCamera(*seq.camera)
    f0 = seq.frame(0)
    dmin, dmax = float(f0.depth.min()), float(f0.depth.max())
    s, origin, tau = _grid(seq, [f0], 160)
    v = rmd.TsdfVolume((160, 160, 160), s, origin, tau, 64.0, device=0)
    g = rmd.SeedMatrix(W, H, cam, device=0)
    g.setReferenceImage(f0.image_u8, f0.T_cam_world, dmin, dmax)
    for k in range(1, 41):
        fr = seq.frame(k, want_depth=False)
        g.update(fr.image_u8, fr.T_cam_world)
    v.integrate(g)
    v.computeEsdf()
    t, w = v.download()
    assert veo.occupied(t, w).sum() > 1000
    _same_esdf(v, t, w, "filter output", np.random.default_rng(1))


@pytest.mark.gpu
def test_adversarial_grids_equal_oracle():
    import rpg_open_remode_b200 as rmd
    rng = np.random.default_rng(0x5EED0E5D)
    for name, t, w in veo.adversarial_grids(rng):
        nz, ny, nx = t.shape
        v = rmd.TsdfVolume((nx, ny, nz), 0.05, (0.25, -0.5, 1.0), 0.2, 64.0, device=0)
        v.upload(t, w)
        v.computeEsdf()
        _same_esdf(v, t, w, name, rng)


@pytest.mark.gpu
def test_after_shifts_equals_oracle():
    import rpg_open_remode_b200 as rmd
    from rpg_open_remode_b200 import synth
    W, H = 320, 240
    seq = synth.SyntheticSequence(W, H, seed=0x5EED0E20)
    frames = [seq.frame(k) for k in (0, 30, 60)]
    s, origin, tau = _grid(seq, frames, 128)
    v = rmd.TsdfVolume((128, 128, 128), s, origin, tau, 64.0, device=0)
    o = vso.OracleVolume((128, 128, 128), s, origin, tau, 64.0)
    cam = rmd.PinholeCamera(*seq.camera)
    rng = np.random.default_rng(2)
    for fr, d in zip(frames, ((17, -9, 23), (-30, 12, -5), (0, 0, 0))):
        v.integrateDepth(fr.depth, cam, fr.T_cam_world)
        o.integrate(fr.depth, seq.camera, fr.T_cam_world)
        v.shift(d)
        o.shift(d)
        v.computeEsdf()
        assert np.array_equal(v.origin.view(u32), o.origin.view(u32))
        _same_esdf(v, o.tsdf, o.weight, f"after shift {d}", rng)


@pytest.mark.gpu
def test_grid_beyond_2gb():
    """1024 x 1024 x 320: long columns, records and snapshot past 2^31 bytes."""
    import rpg_open_remode_b200 as rmd
    from rpg_open_remode_b200 import synth
    W, H = 640, 480
    seq = synth.SyntheticSequence(W, H, seed=0x5EED0E30)
    f0 = seq.frame(0)
    pts = ground_truth_points(f0, seq.camera).reshape(-1, 3)
    dims = (1024, 1024, 320)
    lo, hi = pts.min(0), pts.max(0)
    s = F(((hi - lo) / (np.array(dims) - 1 - 16)).max())
    origin = (lo - 8 * float(s)).astype(F)
    origin[2] = F(hi[2] - (dims[2] - 1 - 8) * float(s))   # the farthest surface in the last planes
    v = rmd.TsdfVolume(dims, s, origin, F(4) * s, 64.0, device=0)
    v.integrateDepth(f0.depth, rmd.PinholeCamera(*seq.camera), f0.T_cam_world)
    v.computeEsdf()
    t, w = v.download()
    assert (w.reshape(-1)[2 ** 28:] > 0).any()
    _same_esdf(v, t, w, "1024 x 1024 x 320", np.random.default_rng(3))
    del t, w
    gc.collect()


# ------------------------------------------------------------------ limits, errors, semantics
@pytest.mark.gpu
def test_size_limit_and_error_codes():
    import rpg_open_remode_b200 as rmd
    from rpg_open_remode_b200 import _native
    L = _native.lib()
    big = rmd.TsdfVolume((4096, 4096, 1), 0.1, (0, 0, 0), 0.3, 10.0, device=0)
    assert L.rmd_volume_esdf(big.handle) == UNSUPPORTED
    with pytest.raises(rmd.RmdError):
        big.computeEsdf()
    del big
    v = rmd.TsdfVolume((16, 12, 8), 0.1, (-0.8, -0.6, 0.5), 0.3, 10.0, device=0)
    a = np.zeros(16 * 12 * 8, F)
    p = np.zeros((4, 4), F)
    assert L.rmd_volume_esdf(None) == INVALID
    assert L.rmd_volume_download_esdf(v.handle, a.ctypes.data, a.ctypes.data) == NOT_INITIALISED
    assert L.rmd_volume_esdf_query(v.handle, p.ctypes.data, 4, p.ctypes.data, None) == NOT_INITIALISED
    assert L.rmd_volume_esdf_query_device(v.handle, None, 0, None, None) == NOT_INITIALISED
    v.computeEsdf()
    assert L.rmd_volume_download_esdf(v.handle, None, a.ctypes.data) == INVALID
    assert L.rmd_volume_download_esdf(None, a.ctypes.data, a.ctypes.data) == INVALID
    assert L.rmd_volume_esdf_query(v.handle, None, 4, p.ctypes.data, None) == INVALID
    assert L.rmd_volume_esdf_query(v.handle, p.ctypes.data, 4, None, None) == INVALID
    assert L.rmd_volume_esdf_query(v.handle, None, 0, None, None) == 0
    assert L.rmd_volume_esdf_query_device(v.handle, None, 4, None, None) == INVALID
    with pytest.raises(ValueError):
        v.esdfQuery(np.zeros((3, 2), F))
    d, w = v.downloadEsdf()   # an unknown volume: O is empty
    assert np.all(d == np.inf) and not w.any()


@pytest.mark.gpu
def test_snapshot_semantics_without_syncs():
    """compute, then integrate and shift with no host sync: queries and download give the snapshot of the grid before
    the changes (at its origin); a recompute gives the new grid's."""
    import rpg_open_remode_b200 as rmd
    from rpg_open_remode_b200 import synth
    W, H = 640, 480
    seq = synth.SyntheticSequence(W, H, seed=0x5EED0E40)
    f0, f1 = seq.frame(0), seq.frame(30)
    s, origin, tau = _grid(seq, [f0, f1], 192)
    cam = rmd.PinholeCamera(*seq.camera)
    imgs = []
    for fr in (f0, f1):
        dimg = rmd.DeviceImage(W, H, "float32")
        dimg.setDevData(fr.depth)
        imgs.append(dimg)
    v = rmd.TsdfVolume((192, 192, 192), s, origin, tau, 64.0, device=0)
    o = vso.OracleVolume((192, 192, 192), s, origin, tau, 64.0)
    o.integrate(f0.depth, seq.camera, f0.T_cam_world)
    t0, w0, origin0 = o.tsdf.copy(), o.weight.copy(), o.origin.copy()
    v.integrateDepth(imgs[0], cam, f0.T_cam_world)
    v.computeEsdf()
    v.integrateDepth(imgs[1], cam, f1.T_cam_world)
    v.shift((11, -7, 5))
    rng = np.random.default_rng(4)
    _same_esdf(v, t0, w0, "before the changes", rng, origin=origin0)
    o.integrate(f1.depth, seq.camera, f1.T_cam_world)
    o.shift((11, -7, 5))
    v.computeEsdf()
    _same_esdf(v, o.tsdf, o.weight, "recomputed", rng)
    v.reset()
    d_after_reset = v.downloadEsdf()[0]
    assert np.isfinite(d_after_reset).all()   # reset leaves the snapshot


@pytest.mark.gpu
def test_device_query_equals_host_query():
    import torch
    import rpg_open_remode_b200 as rmd
    from rpg_open_remode_b200 import synth
    seq = synth.SyntheticSequence(320, 240, seed=0x5EED0E60)
    fr = seq.frame(0)
    s, origin, tau = _grid(seq, [fr], 128)
    v = rmd.TsdfVolume((128, 128, 128), s, origin, tau, 64.0, device=0)
    v.integrateDepth(fr.depth, rmd.PinholeCamera(*seq.camera), fr.T_cam_world)
    v.computeEsdf()
    pts = _points(v, np.random.default_rng(5), 100000)
    xyzw = np.zeros((len(pts), 4), F)
    xyzw[:, :3] = pts
    dg, w = v.esdfQuery(xyzw)
    d_p = torch.from_numpy(xyzw).cuda()
    d_dg = torch.empty((len(pts), 4), dtype=torch.float32, device="cuda")
    d_w = torch.empty(len(pts), dtype=torch.float32, device="cuda")
    torch.cuda.synchronize()
    v.esdfQueryDevice(d_p.data_ptr(), len(pts), d_dg.data_ptr(), d_w.data_ptr())
    v.sync()
    assert np.array_equal(d_dg.cpu().numpy().view(u32), dg.view(u32))
    assert np.array_equal(d_w.cpu().numpy().view(u32), w.view(u32))
    v.esdfQueryDevice(d_p.data_ptr(), len(pts), d_dg.data_ptr())   # without weights
    v.sync()
    assert np.array_equal(d_dg.cpu().numpy().view(u32), dg.view(u32))


# ------------------------------------------------------------------ the node
@pytest.mark.gpu
def test_node_esdf_on_c2():
    """bench.py's c2 sequence through the node with a following 128^3 volume: esdf=True publishes the same depth maps
    and spills as esdf=False, plus one volume_esdf per keyframe that equals the oracle on the records fused so far."""
    import rpg_open_remode_b200 as rmd
    from rpg_open_remode_b200 import multi_gpu, node, synth
    W, H, N = 640, 480, 200
    seq = synth.SyntheticSequence(W, H, seed=multi_gpu.keyframe_seed(0))
    s, origin, tau = _grid(seq, [seq.frame(k) for k in range(0, N, 25)] + [seq.frame(N - 1)], 512)
    fx, fy, cx, cy = seq.camera
    f0 = seq.frame(0)
    dmin, dmax = float(f0.depth.min()), float(f0.depth.max())

    def run(esdf):
        vol = rmd.TsdfVolume((128, 128, 128), s, (0.0, 0.0, 0.0), tau, 64.0, device=0)
        dm = rmd.Depthmap(W, H, fx, cx, fy, cy, device=0)
        out, checked = [], []

        def publisher(kind, d):
            if kind == "depthmap_and_pointcloud":
                out.append((kind, d.getDepthmap().copy(), d.getConvergenceMap().copy()))
            elif kind == "volume_spill":
                out.append((kind,) + tuple(x for x in d if x is not None))
            elif kind == "volume_esdf":
                t, w = d.download()
                want_d, _ = veo.esdf(t, w, d.voxel_size)
                got_d, got_w = d.downloadEsdf()
                checked.append(np.array_equal(got_d.view(u32), want_d.view(u32)) and
                               np.array_equal(got_w.view(u32), w.view(u32)) and bool(veo.occupied(t, w).any()))

        nd = node.DepthmapNode(dm, publisher=publisher, volume=vol, follow_volume=True, esdf=esdf)
        for k in range(N):
            fr = seq.frame(k, want_depth=False)
            nd.denseInputCallback(fr.image_u8, rmd.SE3(fr.T_world_cam.reshape(12)), dmin, dmax)
        return out, checked

    plain, none = run(False)
    with_esdf, checked = run(True)
    assert not none
    keyframes = [p for p in plain if p[0] == "depthmap_and_pointcloud"]
    assert len(plain) == len(with_esdf) and len(checked) == len(keyframes) >= 2
    assert any(p[0] == "volume_spill" for p in plain)
    for a, b in zip(plain, with_esdf):
        assert a[0] == b[0] and len(a) == len(b)
        for x, y in zip(a[1:], b[1:]):
            assert np.array_equal(np.asarray(x).view(np.uint8), np.asarray(y).view(np.uint8)), a[0]
    assert all(checked)
    with pytest.raises(ValueError):
        node.DepthmapNode(rmd.Depthmap(32, 24, 30, 15.5, 30, 11.5, device=0), esdf=True)
