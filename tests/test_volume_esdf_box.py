"""The ESDF of a box of the map on the GPU (csrc/volume.cu: volume_esdf_gather_kernel, then volume_esdf_kernel<0, 1, 2>;
rmd_volume_esdf_box / _esdf_info, api.TsdfVolume.computeEsdf(lo, dims) / esdfBox, DepthmapNode(esdf_camera_margin=r);
DESIGN.md 4.8).

Every comparison is bit for bit: the snapshot (distance and weight), queries at points in and around the box, and
esdfBox().  The reference is the ESDF oracle (tests/volume_esdf_oracle.py) run on the box's records
(tests/volume_esdf_box_oracle.py) at the box's origin.

  * the box (0, n) against computeEsdf(), with and without the store;
  * grown, asymmetric, inner, disjoint and one-voxel-thick boxes against the oracle;
  * a store walk with evictions and restores against the brick-store model, where stored obstacles come closer;
  * a snapshot past 2^31 bytes; error codes and limits; snapshot semantics without host syncs; the device query;
  * the node on bench.py's c2 sequence: the camera, outside the following window, gets a finite distance.
"""
import gc

import numpy as np
import pytest

import volume_esdf_box_oracle as veb
import volume_esdf_oracle as veo
from test_volume import _grid
from test_volume_store import _steps
from volume_store_oracle import StoreModel

F = np.float32
u32 = np.uint32
INVALID, NOT_INITIALISED, UNSUPPORTED = -1, -2, -3


def _bits(a, b):
    return np.array_equal(np.asarray(a).view(u32), np.asarray(b).view(u32))


def _box_points(origin, dims, s, rng, n_random=20000, extra=None):
    """Random points in and slightly around the box, its corners and, when given, extra points [N, 3]."""
    lo = np.asarray(origin, np.float64)
    hi = lo + (np.asarray(dims) - 1) * float(s)
    pad = 2 * float(s)
    pts = [rng.uniform(lo - pad, hi + pad, (n_random, 3)),
           np.array([lo, hi, [hi[0], lo[1], lo[2]], [lo[0], hi[1], hi[2]]])]
    if extra is not None and len(extra):
        pts.append(np.asarray(extra)[:, :3])
    return np.concatenate(pts).astype(F)


def _expected_origin(v, o0, lo):
    """The box origin: o0 + (float)(D + lo) * s per axis, the window's origin itself where lo = 0."""
    lo = np.asarray(lo, np.int64)
    return np.where(lo == 0, v.origin, veb.box_origin(o0, v.offset + lo, v.voxel_size)).astype(F)


def _volume_box_records(v, lo, dims):
    """The box records of a volume from download() and, with the store, downloadStore()."""
    t, w = v.download()
    bricks = None
    if v.store:
        coords, st, sw = v.downloadStore()[:3]
        bricks = veb.downloaded_bricks(coords, st, sw)
    return veb.box_records(v.offset + np.asarray(lo, np.int64), dims, v.offset, t, w, bricks)


def _same_box(v, lo, dims, t, w, origin, what, rng, extra_points=None):
    """v's snapshot, esdfBox() and queries against the oracle on box records (t, w) at origin."""
    lo_u, m, o = v.esdfBox()
    assert list(lo_u) == list(v.offset + np.asarray(lo, np.int64)) and m == tuple(dims), f"{what}: box"
    assert _bits(o, origin), f"{what}: origin {o} / {origin}"
    want_d, want_w = veo.esdf(t, w, v.voxel_size)
    got_d, got_w = v.downloadEsdf()
    assert got_d.shape == tuple(dims[::-1])
    assert _bits(got_w, want_w), f"{what}: weight differs"
    bad = got_d.view(u32) != want_d.view(u32)
    assert not bad.any(), f"{what}: distance differs at {bad.sum()} voxels, first {np.argwhere(bad)[:3]}"
    pts = _box_points(origin, dims, v.voxel_size, rng, extra=extra_points)
    dg, wq = v.esdfQuery(pts)
    want_dg, want_wq = veo.query(want_d, want_w, v.voxel_size, origin, pts)
    assert _bits(dg, want_dg), f"{what}: query differs at {(dg.view(u32) != want_dg.view(u32)).any(1).sum()} points"
    assert _bits(wq, want_wq), f"{what}: query weight differs"
    return want_d


def _scene(W, H, seed, n, ks=(0, 30, 60)):
    import rpg_open_remode_b200 as rmd
    from rpg_open_remode_b200 import synth
    seq = synth.SyntheticSequence(W, H, seed=seed)
    frames = [seq.frame(k) for k in ks]
    s, origin, tau = _grid(seq, frames, n)
    return seq, frames, rmd.PinholeCamera(*seq.camera), s, origin, tau


# ------------------------------------------------------------------ the window's box
@pytest.mark.gpu
@pytest.mark.parametrize("dims,store", [((256, 256, 256), False), ((256, 256, 256), True),
                                        ((97, 64, 71), False), ((97, 64, 71), True)])
def test_window_box_equals_compute(dims, store):
    import rpg_open_remode_b200 as rmd
    seq, frames, cam, s, origin, tau = _scene(320, 240, 0x5EEDB000 + dims[0], max(dims))
    v = rmd.TsdfVolume(dims, s, origin, tau, 64.0, device=0, store=store)
    rng = np.random.default_rng(dims[0])
    n = np.array(dims)
    for fr, d in zip(frames, ((n[0] // 3, -5, 7), (-(n[0] // 3), 5, -7), (0, 0, 0))):
        v.integrateDepth(fr.depth, cam, fr.T_cam_world)
        v.shift(d)
        v.computeEsdf()
        d0, w0 = v.downloadEsdf()
        box0 = v.esdfBox()
        pts = _box_points(v.origin, dims, s, rng, extra=v.surfacePoints())
        q0 = v.esdfQuery(pts)
        v.computeEsdf((0, 0, 0), dims)
        d1, w1 = v.downloadEsdf()
        box1 = v.esdfBox()
        q1 = v.esdfQuery(pts)
        assert _bits(d0, d1) and _bits(w0, w1), f"{dims} store={store} d={d}"
        assert list(box0[0]) == list(box1[0]) == list(v.offset) and box0[1] == box1[1] == tuple(dims)
        assert _bits(box0[2], v.origin) and _bits(box1[2], v.origin)
        assert _bits(q0[0], q1[0]) and _bits(q0[1], q1[1])
    assert np.isfinite(d1).all() and (d1 < 0).any()
    if store:
        assert v.storeInfo()[0] > 0


# ------------------------------------------------------------------ boxes against the oracle
def _boxes(n):
    n = np.asarray(n)
    return {"grown": ((-16, -16, -16), tuple(n + 32)),
            "asymmetric": ((-37, 5, -11), (n[0] + 50, n[1] - 20, 40)),
            "inside": ((10, 20, 5), (50, 30, 40)),
            "disjoint": ((n[0] + 30, -100, 10), (40, 50, 30)),
            "one voxel thick": ((-5, 7, -3), (n[0] + 10, 1, n[2] + 6))}


@pytest.mark.gpu
@pytest.mark.parametrize("store", [False, True])
def test_boxes_equal_oracle(store):
    import rpg_open_remode_b200 as rmd
    dims = (97, 64, 71)
    seq, frames, cam, s, origin, tau = _scene(320, 240, 0x5EEDB100, max(dims))
    v = rmd.TsdfVolume(dims, s, origin, tau, 64.0, device=0, store=store)
    o0 = v.origin.copy()
    rng = np.random.default_rng(7)
    for fr, d in zip(frames, ((40, -20, 25), (-15, 30, -40), (5, 0, 0))):
        v.integrateDepth(fr.depth, cam, fr.T_cam_world)
        v.shift(d)
        for name, (lo, m) in _boxes(dims).items():
            v.computeEsdf(lo, m)
            t, w = _volume_box_records(v, lo, m)
            _same_box(v, lo, m, t, w, _expected_origin(v, o0, lo), f"{name} store={store} d={d}", rng)
    if store:
        assert v.storeInfo()[0] > 0


@pytest.mark.gpu
def test_store_walk_equals_model():
    """test_volume_store.py's schedule of shifts and returns: each box equals the oracle on the brick-store model's box
    records, and some voxel of the window is strictly closer to an obstacle than the window alone says."""
    import rpg_open_remode_b200 as rmd
    dims = (97, 64, 71)
    seq, frames, cam, s, origin, tau = _scene(320, 240, 0x5EEDB200, max(dims))
    v = rmd.TsdfVolume(dims, s, origin, tau, 64.0, device=0, store=True)
    m = StoreModel(dims, s, origin, tau, 64.0)
    o0 = v.origin.copy()
    rng, steps_rng = np.random.default_rng(9), np.random.default_rng(dims[0] + 320)
    closer = False
    n = np.array(dims)
    lo, mm = (-48, -40, -44), tuple(n + 96)
    for q, fr in enumerate(frames):
        v.integrateDepth(fr.depth, cam, fr.T_cam_world)
        m.integrate(fr.depth, seq.camera, fr.T_cam_world)
        for d in _steps(dims, steps_rng, q == len(frames) - 1):
            v.shift(d)
            m.shift(d)
            lo_u = m.D + np.asarray(lo, np.int64)
            t, w = veb.box_records(lo_u, mm, m.D, m.tsdf, m.weight, veb.model_bricks(m))
            v.computeEsdf(lo, mm)
            d_box = _same_box(v, lo, mm, t, w, _expected_origin(v, o0, lo), f"walk d={d}", rng)
            d_win, _ = veo.esdf(m.tsdf, m.weight, s)
            inner = d_box[-lo[2]:-lo[2] + n[2], -lo[1]:-lo[1] + n[1], -lo[0]:-lo[0] + n[0]]
            fin = np.isfinite(inner) & np.isfinite(d_win)
            closer = closer or bool(np.any(np.abs(inner[fin]) < np.abs(d_win[fin])) or
                                    np.any(np.isfinite(inner) & ~np.isfinite(d_win)))
    assert closer and len(m.bricks) > 0


@pytest.mark.gpu
def test_box_beyond_2gb():
    """A 512^3 window with the store in a 768 x 768 x 640 box: records, snapshot and scratch past 2^31 bytes each
    (about 9 GB in all).  The reference is a second volume whose window holds the box's records at the box's origin:
    its window compute, which test_volume_esdf.py checks against the oracle past 2^31 bytes, must give the same snapshot
    and queries bit for bit (the oracle itself would take half a minute on the CPU at this size)."""
    import rpg_open_remode_b200 as rmd
    seq, frames, cam, s, origin, tau = _scene(640, 480, 0x5EEDB300, 512, ks=(0,))
    v = rmd.TsdfVolume((512, 512, 512), s, origin, tau, 64.0, device=0, store=True)
    o0 = v.origin.copy()
    v.integrateDepth(frames[0].depth, cam, frames[0].T_cam_world)
    v.shift((96, 0, -40))   # part of the surface goes to the store
    assert v.storeInfo()[0] > 0
    lo, m = (-160, -128, -64), (768, 768, 640)
    v.computeEsdf(lo, m)
    origin_box = _expected_origin(v, o0, lo)
    lo_u, dims, o = v.esdfBox()
    assert list(lo_u) == list(v.offset + np.asarray(lo)) and dims == m and _bits(o, origin_box)
    t, w = _volume_box_records(v, lo, m)
    assert (w[:, :, :160] > 0).any()   # stored records beyond the window's low x face
    ref = rmd.TsdfVolume(m, s, origin_box, tau, 64.0, device=0)
    ref.upload(t, w)
    del t, w
    ref.computeEsdf()
    got, want = v.downloadEsdf(), ref.downloadEsdf()
    assert _bits(got[1], want[1]), "768 x 768 x 640: weight differs"
    assert _bits(got[0], want[0]), "768 x 768 x 640: distance differs"
    assert np.isfinite(got[0]).all() and (got[0] < 0).any()
    del got, want
    gc.collect()
    pts = _box_points(origin_box, m, s, np.random.default_rng(3))
    dg, wq = v.esdfQuery(pts)
    want_dg, want_wq = ref.esdfQuery(pts)
    assert _bits(dg, want_dg) and _bits(wq, want_wq)
    assert np.isfinite(dg[:, 0]).sum() > len(pts) // 2


# ------------------------------------------------------------------ limits, errors, semantics
@pytest.mark.gpu
def test_limits_and_error_codes():
    import rpg_open_remode_b200 as rmd
    from rpg_open_remode_b200 import _native
    L = _native.lib()
    v = rmd.TsdfVolume((16, 12, 8), 0.1, (-0.8, -0.6, 0.5), 0.3, 10.0, device=0, store=True)

    def box(lo, dims, h=v.handle):
        a = np.array(lo, np.int64)
        m = np.array(dims, np.int32)
        return L.rmd_volume_esdf_box(h, a.ctypes.data, m.ctypes.data)

    lo3, m3, o3 = np.zeros(3, np.int64), np.zeros(3, np.int32), np.zeros(3, F)
    assert L.rmd_volume_esdf_info(v.handle, lo3.ctypes.data, m3.ctypes.data, o3.ctypes.data) == NOT_INITIALISED
    with pytest.raises(rmd.RmdError):
        v.esdfBox()
    assert box((0, 0, 0), (4096, 4096, 2)) == UNSUPPORTED
    with pytest.raises(rmd.RmdError):
        v.computeEsdf((0, 0, 0), (4096, 4096, 2))
    assert L.rmd_volume_esdf_info(v.handle, None, None, None) == NOT_INITIALISED   # nothing computed by a failure

    t = np.ones((8, 12, 16), F)
    t[4, 6, 8] = -1.0
    v.upload(t, np.ones_like(t))
    v.computeEsdf((-3, 2, -1), (20, 7, 9))
    d_ok, w_ok = v.downloadEsdf()
    a = np.zeros(3, np.int64)
    m = np.array((4, 4, 4), np.int32)
    big, small = 2 ** 63 - 1, -2 ** 63
    for lo, dims in [((0, 0, 0), (0, 4, 4)), ((0, 0, 0), (4, -1, 4)), ((0, 0, 0), (4, 4, 0)),
                     ((big - 3, 0, 0), (4, 4, 4)), ((0, big, 0), (4, 4, 4)), ((0, 0, big - 10), (1, 1, 16))]:
        assert box(lo, dims) == INVALID, (lo, dims)
    assert box((0, 0, 0), (4, 4, 4), None) == INVALID
    assert L.rmd_volume_esdf_box(v.handle, None, m.ctypes.data) == INVALID
    assert L.rmd_volume_esdf_box(v.handle, a.ctypes.data, None) == INVALID
    assert L.rmd_volume_esdf_info(None, None, None, None) == INVALID
    with pytest.raises(ValueError):
        v.computeEsdf((0, 0, 0))
    with pytest.raises(ValueError):
        v.computeEsdf((0.5, 0, 0), (4, 4, 4))
    # D cannot come near the limit (shifts take int steps), but D + lo can pass it from below: D = -1
    v.shift((-1, 0, 0))
    assert box((small, 0, 0), (4, 4, 4)) == INVALID
    assert box((small + 1, 0, 0), (4, 4, 4)) == 0   # D + lo = INT64_MIN itself is fine: a box of unknown space
    d, w = v.downloadEsdf()
    assert np.all(d == np.inf) and not w.any()
    assert list(v.esdfBox()[0]) == [small, 0, 0]
    v.shift((1, 0, 0))
    assert box((big - 4, 0, 0), (4, 4, 4)) == 0     # D + lo + m = INT64_MAX: the last box that fits
    assert L.rmd_volume_esdf_info(v.handle, lo3.ctypes.data, m3.ctypes.data, o3.ctypes.data) == 0
    assert list(lo3) == [big - 4, 0, 0] and list(m3) == [4, 4, 4] and np.isfinite(o3).all()
    # the largest box the limit allows along one axis
    assert box((0, 0, 0), (4096, 1, 1)) == 0
    assert box((0, 0, 0), (4097, 1, 1)) == UNSUPPORTED
    assert v.esdfBox()[1] == (4096, 1, 1)
    # a failed call leaves the snapshot as it was
    v.computeEsdf((-3, 2, -1), (20, 7, 9))
    assert box((0, 0, 0), (0, 1, 1)) == INVALID and box((0, 0, 0), (4096, 4096, 2)) == UNSUPPORTED
    d2, w2 = v.downloadEsdf()
    assert _bits(d2, d_ok) and _bits(w2, w_ok)


@pytest.mark.gpu
def test_snapshot_semantics_without_syncs():
    """compute a box, then integrate and shift (evicting and restoring) with no host sync: download and queries give
    the box of the map before the changes; a recompute gives the new one."""
    import rpg_open_remode_b200 as rmd
    W, H = 320, 240
    seq, frames, cam, s, origin, tau = _scene(W, H, 0x5EEDB400, 128, ks=(0, 30))
    imgs = []
    for fr in frames:
        dimg = rmd.DeviceImage(W, H, "float32")
        dimg.setDevData(fr.depth)
        imgs.append(dimg)
    v = rmd.TsdfVolume((128, 128, 128), s, origin, tau, 64.0, device=0, store=True)
    m = StoreModel((128, 128, 128), s, origin, tau, 64.0)
    o0 = v.origin.copy()
    v.integrateDepth(imgs[0], cam, frames[0].T_cam_world)
    m.integrate(frames[0].depth, seq.camera, frames[0].T_cam_world)
    v.shift((40, -16, 24))
    m.shift((40, -16, 24))
    v.sync()
    lo, mm = (-56, -8, -32), (208, 152, 176)
    want0 = veb.box_records(m.D + np.asarray(lo), mm, m.D, m.tsdf, m.weight, veb.model_bricks(m))
    origin0 = _expected_origin(v, o0, lo)
    D0 = v.offset.copy()
    v.computeEsdf(lo, mm)
    v.integrateDepth(imgs[1], cam, frames[1].T_cam_world)
    v.shift((-40, 16, -24))   # restores what the box read from the store
    v.shift((11, -7, 5))
    rng = np.random.default_rng(4)
    lo_u, m_box, o_box = v.esdfBox()
    assert list(lo_u) == list(D0 + np.asarray(lo)) and m_box == mm and _bits(o_box, origin0)
    want_d, want_w = veo.esdf(*want0, s)
    got_d, got_w = v.downloadEsdf()
    assert _bits(got_d, want_d) and _bits(got_w, want_w), "before the changes"
    pts = _box_points(origin0, mm, s, rng)
    dg, wq = v.esdfQuery(pts)
    want_dg, want_wq = veo.query(want_d, want_w, s, origin0, pts)
    assert _bits(dg, want_dg) and _bits(wq, want_wq)
    m.integrate(frames[1].depth, seq.camera, frames[1].T_cam_world)
    m.shift((-40, 16, -24))
    m.shift((11, -7, 5))
    v.computeEsdf(lo, mm)
    t, w = veb.box_records(m.D + np.asarray(lo), mm, m.D, m.tsdf, m.weight, veb.model_bricks(m))
    _same_box(v, lo, mm, t, w, _expected_origin(v, o0, lo), "recomputed", rng)
    v.reset()
    assert _bits(v.downloadEsdf()[0], veo.esdf(t, w, s)[0])   # reset leaves the snapshot


@pytest.mark.gpu
def test_device_query_equals_host_query():
    import torch
    import rpg_open_remode_b200 as rmd
    seq, frames, cam, s, origin, tau = _scene(320, 240, 0x5EEDB600, 128, ks=(0,))
    v = rmd.TsdfVolume((128, 128, 128), s, origin, tau, 64.0, device=0, store=True)
    v.integrateDepth(frames[0].depth, cam, frames[0].T_cam_world)
    v.shift((40, 0, 0))
    v.computeEsdf((-60, -10, -20), (200, 150, 170))
    _, dims, o = v.esdfBox()
    pts = _box_points(o, dims, s, np.random.default_rng(5), 100000)
    xyzw = np.zeros((len(pts), 4), F)
    xyzw[:, :3] = pts
    dg, w = v.esdfQuery(xyzw)
    assert np.isfinite(dg[:, 0]).sum() > len(pts) // 2
    d_p = torch.from_numpy(xyzw).cuda()
    d_dg = torch.empty((len(pts), 4), dtype=torch.float32, device="cuda")
    d_w = torch.empty(len(pts), dtype=torch.float32, device="cuda")
    torch.cuda.synchronize()
    v.esdfQueryDevice(d_p.data_ptr(), len(pts), d_dg.data_ptr(), d_w.data_ptr())
    v.sync()
    assert _bits(d_dg.cpu().numpy(), dg) and _bits(d_w.cpu().numpy(), w)


# ------------------------------------------------------------------ the node
@pytest.mark.gpu
def test_node_camera_box_on_c2():
    """bench.py's c2 sequence (its first 120 frames) through the node with a following 128^3 volume with the store:
    esdf_camera_margin=32 publishes the same depth maps and spills as esdf=False; each snapshot equals the oracle on its
    box's records; the keyframe camera's centre gets a finite distance, where the window-only snapshot of the same
    volume gives NaN."""
    import rpg_open_remode_b200 as rmd
    from rpg_open_remode_b200 import multi_gpu, node, synth
    W, H, N, N_RUN = 640, 480, 200, 120
    seq = synth.SyntheticSequence(W, H, seed=multi_gpu.keyframe_seed(0))
    s, origin, tau = _grid(seq, [seq.frame(k) for k in range(0, N, 25)] + [seq.frame(N - 1)], 512)
    fx, fy, cx, cy = seq.camera
    f0 = seq.frame(0)
    dmin, dmax = float(f0.depth.min()), float(f0.depth.max())
    rng = np.random.default_rng(8)

    def run(margin):
        vol = rmd.TsdfVolume((128, 128, 128), s, (0.0, 0.0, 0.0), tau, 64.0, device=0, store=True)
        o0 = vol.origin.copy()
        dm = rmd.Depthmap(W, H, fx, cx, fy, cy, device=0)
        out, checked, at_camera, at_camera_window, pose = [], [], [], [], []

        def publisher(kind, d):
            if kind == "depthmap_and_pointcloud":
                out.append((kind, d.getDepthmap().copy(), d.getConvergenceMap().copy()))
                pose.append(np.asarray(d.getT_world_ref().data, np.float32).reshape(3, 4))
            elif kind == "volume_spill":
                out.append((kind,) + tuple(x for x in d if x is not None))
            elif kind == "volume_esdf":
                cam_c = pose[-1][:, 3].astype(F)[None]
                lo_u, dims, o = d.esdfBox()
                lo = lo_u - d.offset
                t, w = _volume_box_records(d, lo, dims)
                _same_box(d, lo, dims, t, w, _expected_origin(d, o0, lo), f"keyframe {len(checked)}", rng,
                          extra_points=cam_c)
                checked.append(bool(veo.occupied(t, w).any()))
                at_camera.append(d.esdfQuery(cam_c)[0][0, 0])
                # the window-only snapshot of the same records, then the node's box again
                d.computeEsdf()
                at_camera_window.append(d.esdfQuery(cam_c)[0][0, 0])
                d.computeEsdf(lo, dims)

        nd = node.DepthmapNode(dm, publisher=publisher, volume=vol, follow_volume=True, esdf=bool(margin),
                               esdf_camera_margin=margin)
        for k in range(N_RUN):
            fr = seq.frame(k, want_depth=False)
            nd.denseInputCallback(fr.image_u8, rmd.SE3(fr.T_world_cam.reshape(12)), dmin, dmax)
        return out, checked, at_camera, at_camera_window

    plain, none, _, _ = run(0)
    boxed, checked, at_cam, at_cam_window = run(32)
    assert not none
    keyframes = [p for p in plain if p[0] == "depthmap_and_pointcloud"]
    assert len(plain) == len(boxed) and len(checked) == len(keyframes) >= 2 and all(checked)
    assert any(p[0] == "volume_spill" for p in plain)
    for a, b in zip(plain, boxed):
        assert a[0] == b[0] and len(a) == len(b)
        for x, y in zip(a[1:], b[1:]):
            assert np.array_equal(np.asarray(x).view(np.uint8), np.asarray(y).view(np.uint8)), a[0]
    assert np.all(np.isfinite(at_cam)), at_cam
    assert len(at_cam_window) == len(at_cam) and np.all(np.isnan(at_cam_window)), at_cam_window
    with pytest.raises(ValueError):
        node.DepthmapNode(rmd.Depthmap(32, 24, 30, 15.5, 30, 11.5, device=0), esdf_camera_margin=4)
