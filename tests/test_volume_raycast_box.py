"""Raycasts and the keyframe prior over a box of the map on the GPU (rmd_volume_raycast_box, rmd_volume_prior_seeds_box;
api.TsdfVolume.raycast / raycastIntensity / raycastNormals (lo, dims), SeedMatrix.priorFromVolume(..., lo, dims),
DepthmapNode(prior_view_box=True); DESIGN.md 4.8).

The box's records are gathered by the ESDF box's kernel and marched by the existing raycast and prior kernels, so
every comparison is bit for bit against the same call on a second, plain volume created with dims m at the box's
origin (volume_esdf_box_oracle.box_origin) and holding the box's records (box_records on download() and
downloadStore()):

  * the window box (0, n) against the window entry points, with and without the store and the intensity channel;
  * grown, asymmetric, inner, disjoint, one-voxel-thick and store-only boxes, cameras inside and outside the box, and
    on small grids the CPU raycast, intensity, normals and prior oracles on the box's records;
  * a revisit: a surface that lives only in the store is hit by the box calls and missed by the window calls;
  * ordering without host syncs against the shared scratch and a following shift or integrate;
  * error codes and limits;
  * the node on bench.py's c2 sequence: prior_view_box=False is today's node, True takes each keyframe's prior from
    its view box's records.
"""
import gc

import numpy as np
import pytest

import volume_esdf_box_oracle as veb
import volume_intensity_oracle as vio
import volume_normals_oracle as vno
import volume_oracle as vo
from test_volume import _grid
from test_volume_prior import _expect, _same, _snap

F = np.float32
u32 = np.uint32
INVALID, NOT_INITIALISED, UNSUPPORTED = -1, -2, -3
F_PRIOR = 1.0 / 16.0
PATCH = 5


def _bits(a, b):
    return np.array_equal(np.asarray(a).view(u32), np.asarray(b).view(u32))


def _box_records(v, lo, dims):
    """(tsdf, weight, intensity, intensity weight) of the box from download[Intensity]() and downloadStore(); the
    intensity pair is None without the channel."""
    lo_u = v.offset + np.asarray(lo, np.int64)
    t, w = v.download()
    ci = cw = None
    bricks = cbricks = None
    if v.store:
        st = v.downloadStore()
        bricks = veb.downloaded_bricks(st[0], st[1], st[2])
        if v.intensity:
            cbricks = veb.downloaded_bricks(st[0], st[3], st[4])
    rt, rw = veb.box_records(lo_u, dims, v.offset, t, w, bricks)
    if v.intensity:
        a, b = v.downloadIntensity()
        ci, cw = veb.box_records(lo_u, dims, v.offset, a, b, cbricks)
    return rt, rw, ci, cw


def _box_origin(v, o0, lo):
    lo = np.asarray(lo, np.int64)
    return np.where(lo == 0, v.origin, veb.box_origin(o0, v.offset + lo, v.voxel_size)).astype(F)


def _twin(v, o0, lo, dims):
    """A plain volume of dims m at the box's origin holding the box's records, and those records."""
    import rpg_open_remode_b200 as rmd
    rec = _box_records(v, lo, dims)
    tw = rmd.TsdfVolume(tuple(int(x) for x in dims), v.voxel_size, _box_origin(v, o0, lo), v.truncation,
                        v.max_weight, device=0, intensity=v.intensity)
    tw.upload(rec[0], rec[1])
    if v.intensity:
        tw.uploadIntensity(rec[2], rec[3])
    return tw, rec


def _views(v, cam, T, size, lo=None, dims=None):
    """depth, (depth, intensity) or None, (depth, normals) of the three raycasts."""
    W, H = size
    d = v.raycast(cam, T, W, H, lo, dims)
    di = v.raycastIntensity(cam, T, W, H, lo, dims) if v.intensity else None
    dn = v.raycastNormals(cam, T, W, H, lo, dims)
    return d, di, dn


def _same_views(a, b, what):
    assert _bits(a[0], b[0]), f"{what}: depth differs at {(a[0].view(u32) != b[0].view(u32)).sum()} pixels"
    assert (a[1] is None) == (b[1] is None)
    if a[1] is not None:
        assert _bits(a[1][0], b[1][0]) and _bits(a[1][1], b[1][1]), f"{what}: intensity view differs"
        assert _bits(a[1][0], a[0])
    assert _bits(a[2][0], b[2][0]) and _bits(a[2][1], b[2][1]), f"{what}: normals view differs"
    assert _bits(a[2][0], a[0])


def _prior(v, cam, frame, size, dmin, dmax, lo=None, dims=None):
    import rpg_open_remode_b200 as rmd
    g = rmd.SeedMatrix(*size, cam, PATCH, device=0)
    g.setReferenceImage(frame.image, frame.T_cam_world, dmin, dmax)
    g.priorFromVolume(v, F_PRIOR, lo, dims)
    return _snap(g)


def _scene(dims, intensity, store, seed, size=(320, 240)):
    """A following volume of the synthetic scene: three frames fused, with shifts between them, so that with the
    store part of the surface lives only there.  Returns (volume, o0, seq, cam, frames, dmin, dmax)."""
    import rpg_open_remode_b200 as rmd
    from rpg_open_remode_b200 import synth
    W, H = size
    seq = synth.SyntheticSequence(W, H, seed=seed)
    frames = [seq.frame(k) for k in (0, 30, 60)]
    s, origin, tau = _grid(seq, frames, max(dims))
    v = rmd.TsdfVolume(dims, s, origin, tau, 64.0, device=0, intensity=intensity, store=store)
    o0 = v.origin.copy()
    cam = rmd.PinholeCamera(*seq.camera)
    n = np.asarray(dims)
    for q, fr in enumerate(frames):
        v.integrateDepth(fr.depth, cam, fr.T_cam_world, None, fr.image if intensity else None)
        if q == 0:
            v.shift(n // 4)
        elif q == 1:
            v.shift(-(n // 2))
    f0 = frames[0]
    return v, o0, seq, cam, frames, float(f0.depth.min()), float(f0.depth.max())


def _store_only_box(v):
    """(lo, dims) of a box that lies wholly outside the window, around the stored voxel nearest the surface: its
    records come from the store alone."""
    coords, t, w = v.downloadStore()[:3]   # voxels inside the window come back as (0, 0)
    q = np.argwhere(w > 0)
    assert len(q)
    best = q[np.argmin(np.abs(t[tuple(q.T)]))]
    u = coords[best[0]] * 8 + best[1:][::-1]   # (z, y, x) within the brick
    x = u - v.offset
    n = np.asarray(v.dims)
    a = int(np.argmax((x < 0) | (x >= n)))
    lo, m = x - 4, np.full(3, 9)
    if x[a] >= n[a]:
        lo[a], m[a] = n[a], x[a] - n[a] + 5
    else:
        m[a] = -lo[a]
    return tuple(int(c) for c in lo), m


def _camera_box(v, T_cam_world, pad=3):
    """A box that holds the window and the camera's voxel with `pad` voxels around it."""
    T = np.asarray(T_cam_world, np.float64).reshape(3, 4)
    R, t = T[:, :3], T[:, 3]
    c = -R.T @ t
    g = np.floor((c - v.origin.astype(np.float64)) / v.voxel_size).astype(np.int64)
    lo = np.minimum(0, g - pad)
    return lo, np.maximum(np.asarray(v.dims), g + pad + 1) - lo


# ------------------------------------------------------------------ the window box
@pytest.mark.gpu
@pytest.mark.parametrize("store,intensity", [(False, False), (False, True), (True, False), (True, True)])
def test_window_box_is_the_window(store, intensity):
    dims = (96, 80, 72)
    v, o0, seq, cam, frames, dmin, dmax = _scene(dims, intensity, store, 0x5EED0A00 + 2 * store + intensity)
    size = (seq.width, seq.height)
    zero = (0, 0, 0)
    for fr in frames:
        _same_views(_views(v, cam, fr.T_cam_world, size, zero, dims), _views(v, cam, fr.T_cam_world, size),
                    "window box")
        _same(_prior(v, cam, fr, size, dmin, dmax, zero, dims), _prior(v, cam, fr, size, dmin, dmax), "window prior")
    assert (v.raycast(cam, frames[-1].T_cam_world, *size) > 0).mean() > 0.05


# ------------------------------------------------------------------ box shapes against a plain volume
@pytest.mark.gpu
@pytest.mark.parametrize("intensity", [False, True])
def test_box_shapes_equal_a_plain_volume(intensity):
    dims = (64, 56, 48)
    v, o0, seq, cam, frames, dmin, dmax = _scene(dims, intensity, True, 0x5EED0A10 + intensity, (160, 120))
    size = (seq.width, seq.height)
    n = np.asarray(dims)
    v.shift((n[0] // 2, 0, 0))   # the observed low-x half leaves: the store then holds voxels outside the window
    assert v.storeInfo()[0] > 0
    D = v.offset
    boxes = {"grown": ((-8, -8, -8), n + 16),
             "asymmetric": ((-21, 3, -5), (n[0] + 7, n[1] - 10, n[2] + 30)),
             "inner": ((10, 9, 8), n - 20),
             "disjoint": ((n[0] + 3, -4, 0), (30, n[1] + 8, n[2])),
             "store only": _store_only_box(v),
             "thin x": ((5, -6, -6), (1, n[1] + 12, n[2] + 12)),
             "thin z": ((-6, -6, 17), (n[0] + 12, n[1] + 12, 1)),
             "one voxel": ((3, 4, 5), (1, 1, 1)),
             # where the window stood before its last shift: the store, and what the window still covers of it
             "store": (tuple(int(x) for x in n // 2), n)}
    for name, (lo, m) in boxes.items():
        m = np.asarray(m)
        tw, rec = _twin(v, o0, lo, m)
        o = _box_origin(v, o0, lo)
        small = np.prod(m) <= 200000
        if name == "store only":
            assert (rec[1] > 0).any() and (np.any(np.asarray(lo) >= n) or np.any(np.asarray(lo) + m <= 0))
        for q, fr in enumerate(frames):
            what = f"{name} box, frame {q}"
            got = _views(v, cam, fr.T_cam_world, size, lo, m)
            _same_views(got, _views(tw, cam, fr.T_cam_world, size), what)
            _same(_prior(v, cam, fr, size, dmin, dmax, lo, m), _prior(tw, cam, fr, size, dmin, dmax), what + " prior")
            if small:   # the CPU oracles on the box's records
                ob = vno.OracleVolume(m, v.voxel_size, o, v.truncation, v.max_weight)
                ob.tsdf, ob.weight = np.ascontiguousarray(rec[0]), np.ascontiguousarray(rec[1])
                assert _bits(got[0], ob.raycast(seq.camera, fr.T_cam_world, *size)), what + ": oracle depth"
                od, on = ob.raycast_normals(seq.camera, fr.T_cam_world, *size)
                assert _bits(got[2][0], od) and _bits(got[2][1], on[..., :3]), what + ": oracle normals"
                if intensity:
                    oi = vio.OracleVolume(m, v.voxel_size, o, v.truncation, v.max_weight)
                    oi.tsdf, oi.weight = ob.tsdf, ob.weight
                    oi.cint, oi.cw = np.ascontiguousarray(rec[2]), np.ascontiguousarray(rec[3])
                    di, ii = oi.raycast_intensity(seq.camera, fr.T_cam_world, *size)
                    assert _bits(got[1][0], di) and _bits(got[1][1], ii), what + ": oracle intensity"
                want = _expect(ob, seq.camera, fr.T_cam_world, size, PATCH, dmin, dmax, F_PRIOR)[0]
                _same(_prior(v, cam, fr, size, dmin, dmax, lo, m), want, what + ": oracle prior")
        del tw
    # cameras inside the box: the window and each camera's voxel
    for q, fr in enumerate(frames):
        lo, m = _camera_box(v, fr.T_cam_world)
        tw, _ = _twin(v, o0, lo, m)
        got = _views(v, cam, fr.T_cam_world, size, lo, m)
        _same_views(got, _views(tw, cam, fr.T_cam_world, size), f"camera box {q}")
        _same(_prior(v, cam, fr, size, dmin, dmax, lo, m), _prior(tw, cam, fr, size, dmin, dmax), f"camera box {q}")
        assert (got[0] > 0).mean() > 0.05
    assert np.array_equal(v.offset, D)


# ------------------------------------------------------------------ a revisit
@pytest.mark.gpu
def test_revisit_hits_the_surface_in_the_store():
    import rpg_open_remode_b200 as rmd
    from rpg_open_remode_b200 import synth
    W, H, n = 320, 240, 96
    seq = synth.SyntheticSequence(W, H, seed=0x5EED0A20)
    fr = seq.frame(0)
    s, origin, tau = _grid(seq, [fr], n)
    v = rmd.TsdfVolume((n, n, n), s, origin, tau, 64.0, device=0, intensity=True, store=True)
    o0 = v.origin.copy()
    cam = rmd.PinholeCamera(*seq.camera)
    v.integrateDepth(fr.depth, cam, fr.T_cam_world, None, fr.image)
    dmin, dmax = float(fr.depth.min()), float(fr.depth.max())
    before = _views(v, cam, fr.T_cam_world, (W, H))
    v.shift((n + 5, 0, 0))   # the whole window leaves: the surface lives in the store only
    lo, m = (-(n + 5), 0, 0), (n, n, n)
    tw, _ = _twin(v, o0, lo, m)
    got = _views(v, cam, fr.T_cam_world, (W, H), lo, m)
    _same_views(got, _views(tw, cam, fr.T_cam_world, (W, H)), "revisit")
    _same_views(got, before, "revisit against the window before the shift")
    assert (got[0] > 0).mean() > 0.2
    window = _views(v, cam, fr.T_cam_world, (W, H))
    assert not window[0].any() and np.all(window[1][1] == -1.0)
    boxed = _prior(v, cam, fr, (W, H), dmin, dmax, lo, m)
    _same(boxed, _prior(tw, cam, fr, (W, H), dmin, dmax), "revisit prior")
    fresh = _prior(v, cam, fr, (W, H), dmin, dmax)
    applied = boxed["sigma_sq"] != fresh["sigma_sq"]
    assert applied.mean() > 0.2 and np.all(fresh["sigma_sq"] == fresh["sigma_sq"].max())
    assert _bits(boxed["mu"][applied], got[0][applied])


# ------------------------------------------------------------------ ordering
@pytest.mark.gpu
@pytest.mark.parametrize("then", ["shift", "integrate"])
def test_box_prior_reads_the_map_before_a_following_write(then):
    """prior_seeds_box then at once a shift or an integration, no host sync: the rays saw the map before it."""
    import rpg_open_remode_b200 as rmd
    dims = (128, 128, 128)
    v0, o0, seq, cam, frames, dmin, dmax = _scene(dims, False, True, 0x5EED0A30, (640, 480))
    lo, m = (-32, -32, -32), (192, 192, 192)
    fr = frames[1]
    results = []
    for sync in (True, False):
        v, _, _, _, _, _, _ = _scene(dims, False, True, 0x5EED0A30, (640, 480))
        g = rmd.SeedMatrix(seq.width, seq.height, cam, PATCH, device=0)
        g.setReferenceImage(fr.image, fr.T_cam_world, dmin, dmax)
        g.priorFromVolume(v, F_PRIOR, lo, m)
        if sync:
            g.sync()
        if then == "shift":
            v.shift((40, -30, 20))
        else:
            v.integrateDepth(np.full_like(fr.depth, 0.5 * (dmin + dmax)), cam, fr.T_cam_world)
        results.append(_snap(g))
    _same(results[1], results[0], then)
    _same(results[0], _prior(v0, cam, fr, (seq.width, seq.height), dmin, dmax, lo, m), then + " against the map")


@pytest.mark.gpu
def test_box_raycast_then_esdf_box_on_the_shared_scratch():
    """raycast_box then at once computeEsdf(lo, dims) over another box, no host sync: both equal a synchronised
    run's."""
    import rpg_open_remode_b200 as rmd
    from rpg_open_remode_b200 import _native
    L = _native.lib()
    dims = (128, 128, 128)
    lo1, m1 = np.array([-40, -20, -30], np.int64), np.array([200, 170, 190], np.int32)
    lo2, m2 = (-10, -10, -10), (150, 150, 150)
    out = []
    for sync in (True, False):
        v, o0, seq, cam, frames, dmin, dmax = _scene(dims, True, True, 0x5EED0A40, (640, 480))
        W, H = seq.width, seq.height
        T = np.ascontiguousarray(np.asarray(frames[2].T_cam_world, F).reshape(12))
        d, i = rmd.DeviceImage(W, H, "float32"), rmd.DeviceImage(W, H, "float32")
        assert L.rmd_volume_raycast_box(v.handle, lo1.ctypes.data, m1.ctypes.data, W, H, cam.fx, cam.fy, cam.cx,
                                        cam.cy, T.ctypes.data, d.data, d.pitch, i.data, i.pitch, None, 0) == 0
        if sync:
            v.sync()
        v.computeEsdf(lo2, m2)
        v.sync()
        out.append((d.getDevData(), i.getDevData(), v.downloadEsdf()))
    (d0, i0, (e0, w0)), (d1, i1, (e1, w1)) = out
    assert _bits(d0, d1) and _bits(i0, i1) and _bits(e0, e1) and _bits(w0, w1)
    assert (d0 > 0).mean() > 0.05
    want = v.raycastIntensity(cam, frames[2].T_cam_world, W, H, lo1, m1)
    assert _bits(want[0], d0) and _bits(want[1], i0)


# ------------------------------------------------------------------ error codes and limits
@pytest.mark.gpu
def test_error_codes_and_limits():
    import rpg_open_remode_b200 as rmd
    from rpg_open_remode_b200 import _native
    L = _native.lib()
    W, H = 64, 48
    v = rmd.TsdfVolume((32, 32, 32), 0.05, (-0.8, -0.8, 0.2), 0.2, 16.0, device=0, store=True)
    cam = rmd.PinholeCamera(50.0, 50.0, 31.5, 23.5)
    v.integrateDepth(np.full((H, W), 1.0, F), cam, np.eye(3, 4, dtype=F))
    v.computeEsdf((-2, -2, -2), (36, 36, 36))
    esdf_before = v.downloadEsdf()
    T = np.ascontiguousarray(np.eye(3, 4, dtype=F).reshape(12))
    d, i = rmd.DeviceImage(W, H, "float32"), rmd.DeviceImage(W, H, "float32")
    nrm = rmd.DeviceImage(4 * W, H, "float32")

    def box(lo, m, h=v.handle, depth=d.data, pitch=d.pitch, inten=None, ipitch=0, normals=None, npitch=0, pose=None):
        a = None if lo is None else np.ascontiguousarray(lo, np.int64)
        b = None if m is None else np.ascontiguousarray(m, np.int32)
        return L.rmd_volume_raycast_box(h, a.ctypes.data if a is not None else None,
                                        b.ctypes.data if b is not None else None, W, H, cam.fx, cam.fy, cam.cx,
                                        cam.cy, T.ctypes.data if pose is None else pose, depth, pitch, inten, ipitch,
                                        normals, npitch)

    assert box((0, 0, 0), (32, 32, 32)) == 0
    assert box((0, 0, 0), (32, 32, 32), normals=nrm.data, npitch=nrm.pitch) == 0
    assert box((0, 0, 0), (32, 32, 32), h=None) == INVALID
    assert box(None, (32, 32, 32)) == INVALID and box((0, 0, 0), None) == INVALID
    assert box((0, 0, 0), (32, 32, 32), depth=None) == INVALID
    assert box((0, 0, 0), (0, 32, 32)) == INVALID and box((0, 0, 0), (32, -1, 32)) == INVALID
    assert box((2 ** 63 - 20, 0, 0), (32, 32, 32)) == INVALID
    assert box((0, 0, 0), (32, 32, 32), pitch=4 * W - 4) == INVALID
    assert box((0, 0, 0), (32, 32, 32), normals=nrm.data, npitch=16 * W - 16) == INVALID
    assert box((0, 0, 0), (32, 32, 32), normals=nrm.data + 4, npitch=nrm.pitch) == INVALID
    assert box((0, 0, 0), (32, 32, 32), inten=i.data, ipitch=i.pitch) == NOT_INITIALISED
    # a 65536-voxel dimension is refused before anything is allocated or enqueued; so is a box whose records could
    # never fit the device
    for m in ((65536, 1, 1), (1, 65536, 1), (1, 1, 65536)):
        assert box((0, 0, 0), m) == UNSUPPORTED
    assert box((0, 0, 0), (65535, 65535, 65535)) == 2   # cudaErrorMemoryAllocation
    v.enableIntensity()
    assert box((0, 0, 0), (32, 32, 32), inten=i.data, ipitch=4 * W - 4) == INVALID
    assert box((0, 0, 0), (32, 32, 32), inten=i.data, ipitch=i.pitch) == 0
    v.sync()
    # the ESDF snapshot is untouched by the box calls that share its scratch
    e, w = v.downloadEsdf()
    assert _bits(e, esdf_before[0]) and _bits(w, esdf_before[1])
    assert v.esdfBox()[1] == (36, 36, 36)

    g = rmd.SeedMatrix(W, H, cam, PATCH, device=0)
    a64, m32 = np.zeros(3, np.int64), np.array([32, 32, 32], np.int32)
    assert L.rmd_volume_prior_seeds_box(v.handle, g.handle, F_PRIOR, a64.ctypes.data, m32.ctypes.data) \
        == NOT_INITIALISED
    g.setReferenceImage(np.full((H, W), 0.5, F), np.eye(3, 4, dtype=F), 0.5, 2.0)
    assert L.rmd_volume_prior_seeds_box(None, g.handle, F_PRIOR, a64.ctypes.data, m32.ctypes.data) == INVALID
    assert L.rmd_volume_prior_seeds_box(v.handle, None, F_PRIOR, a64.ctypes.data, m32.ctypes.data) == INVALID
    assert L.rmd_volume_prior_seeds_box(v.handle, g.handle, 0.0, a64.ctypes.data, m32.ctypes.data) == INVALID
    assert L.rmd_volume_prior_seeds_box(v.handle, g.handle, F_PRIOR, None, m32.ctypes.data) == INVALID
    assert L.rmd_volume_prior_seeds_box(v.handle, g.handle, F_PRIOR, a64.ctypes.data, None) == INVALID
    big = np.array([1, 65536, 1], np.int32)
    assert L.rmd_volume_prior_seeds_box(v.handle, g.handle, F_PRIOR, a64.ctypes.data, big.ctypes.data) == UNSUPPORTED
    assert L.rmd_volume_prior_seeds_box(v.handle, g.handle, F_PRIOR, a64.ctypes.data, m32.ctypes.data) == 0
    with pytest.raises(ValueError):
        v.raycast(cam, np.eye(3, 4), W, H, (0, 0, 0), None)
    with pytest.raises(ValueError):
        g.priorFromVolume(v, F_PRIOR, (0, 0), (1, 1, 1))
    with pytest.raises(rmd.RmdError):
        v.raycastNormals(cam, np.eye(3, 4), W, H, (0, 0, 0), (70000, 1, 1))


# ------------------------------------------------------------------ the node
@pytest.mark.gpu
def test_node_view_box_prior_on_c2():
    """bench.py's c2 sequence (first 120 frames) through the node with a following 128^3 volume with the store and the
    volume prior: with prior_view_box=True each keyframe's prior is the reference composition -- the CPU raycast oracle
    on its view box's records, then prior_apply -- and the run publishes depth maps and spills.  That False makes the
    node's calls of a node without the option is checked on the CPU (test_volume_view_box.py); the window prior's
    output is checked by test_volume_prior.py."""
    import rpg_open_remode_b200 as rmd
    from rpg_open_remode_b200 import multi_gpu, node, synth
    W, H, N, N_RUN = 640, 480, 200, 120
    seq = synth.SyntheticSequence(W, H, seed=multi_gpu.keyframe_seed(0))
    s, origin, tau = _grid(seq, [seq.frame(k) for k in range(0, N, 25)] + [seq.frame(N - 1)], 512)
    fx, fy, cx, cy = seq.camera
    f0 = seq.frame(0)
    dmin, dmax = float(f0.depth.min()), float(f0.depth.max())

    def run(**kw):
        vol = rmd.TsdfVolume((128, 128, 128), s, (0.0, 0.0, 0.0), tau, 64.0, device=0, store=True)
        o0 = vol.origin.copy()
        dm = rmd.Depthmap(W, H, fx, cx, fy, cy, device=0)
        out, checked = [], []
        ref_pose = []

        def publisher(kind, d):
            if kind == "depthmap_and_pointcloud":
                out.append((kind, d.getDepthmap().copy(), d.getConvergenceMap().copy()))
            elif kind == "volume_spill":
                out.append((kind,) + tuple(x for x in d if x is not None))

        if kw.get("prior_view_box"):
            set_ref, prior = dm.setReferenceImage, dm.priorFromVolume

            def set_reference(img, T_curr_world, mn, mx):
                ref_pose.append(T_curr_world)
                return set_ref(img, T_curr_world, mn, mx)

            def prior_from_volume(volume, f, lo=None, dims=None):
                assert lo is not None and dims is not None
                T = ref_pose[-1].data if hasattr(ref_pose[-1], "data") else ref_pose[-1]
                rt, rw, _, _ = _box_records(volume, lo, dims)
                o = vo.OracleVolume(dims, volume.voxel_size, _box_origin(volume, o0, lo), volume.truncation,
                                    volume.max_weight)
                o.tsdf, o.weight = np.ascontiguousarray(rt), np.ascontiguousarray(rw)
                want = _expect(o, seq.camera, T, (W, H), PATCH, dmin, dmax, f)[0]
                del o, rt, rw
                prior(volume, f, lo, dims)
                _same(_snap(dm.seeds_), want, f"keyframe {len(checked)}")
                interior = want["conv"] != rmd.ConvergenceStates.BORDER
                checked.append(int((want["sigma_sq"][interior] != want["sigma_sq"][interior].max()).sum()))

            dm.setReferenceImage, dm.priorFromVolume = set_reference, prior_from_volume
        nd = node.DepthmapNode(dm, publisher=publisher, volume=vol, follow_volume=True, prior_from_volume=F_PRIOR,
                               **kw)
        for k in range(N_RUN):
            fr = seq.frame(k, want_depth=False)
            nd.denseInputCallback(fr.image_u8, rmd.SE3(fr.T_world_cam.reshape(12)), dmin, dmax)
        if kw.get("prior_view_box"):
            del dm.setReferenceImage, dm.priorFromVolume   # the wrappers refer to dm: no cycle outlives the run
        return out, checked

    boxed, checked = run(prior_view_box=True)
    keyframes = [p for p in boxed if p[0] == "depthmap_and_pointcloud"]
    assert len(keyframes) >= 2 and any(p[0] == "volume_spill" for p in boxed)
    assert len(checked) >= len(keyframes)
    print("keyframe priors from the view box:", checked)
    assert sum(checked[1:]) > 0
    del boxed
    gc.collect()
