"""The brick store of the moving TSDF volume on the GPU (csrc/volume.cu: the store kernels; rmd_volume_enable_store,
rmd_volume_shift with the store, rmd_volume_store_info, rmd_volume_download_store / upload_store;
api.TsdfVolume(store=True), mapMesh; DESIGN.md 4.8).

  * the product against the numpy model (tests/volume_store_oracle.py) bit for bit: window records, the stored bricks'
    coordinates and records and their number, across integrations of ground truth (QVGA and VGA) and real filter
    output, and shifts with returns and |d| >= n, on 256^3 and the ragged 97 x 64 x 71 grid, with and without
    intensity;
  * shift(d) then shift(-d) is lossless, and a revisited region raycasts, meshes and seeds the prior as before it left
    (without the store: no hits);
  * mapMesh against the model's sweep and the dense map, and the volume unchanged afterwards;
  * stream ordering without host syncs, the 1024 x 1024 x 320 grid, capacities, upload / download, error codes;
  * the node on bench.py's c2 sequence: a following volume with the store publishes bit-identically to one without.
"""
import ctypes
import gc

import numpy as np
import pytest

import mesh_checks
from test_volume import _grid
from test_volume_shift import _node_run
from volume_store_oracle import StoreModel, kept_box, moving

F = np.float32
u32 = np.uint32
INVALID, NOT_INITIALISED = -1, -2


def _pair(dims, s, origin, tau, intensity=True):
    import rpg_open_remode_b200 as rmd
    return (rmd.TsdfVolume(dims, s, origin, tau, 64.0, device=0, intensity=intensity, store=True),
            StoreModel(dims, s, origin, tau, 64.0))


def _same(v, m, what):
    t, w = v.download()
    assert np.array_equal(w.view(u32), m.weight.view(u32)), f"{what}: weight differs at {(w != m.weight).sum()}"
    assert np.array_equal(t.view(u32), m.tsdf.view(u32)), f"{what}: tsdf differs"
    if v.intensity:
        c, cw = v.downloadIntensity()
        assert np.array_equal(c.view(u32), m.cint.view(u32)) and np.array_equal(cw.view(u32), m.cw.view(u32)), what
    assert np.array_equal(v.origin.view(u32), m.origin.view(u32)) and np.array_equal(v.offset, m.D), what
    coords, rec = m.download_store()
    got = v.downloadStore()
    assert v.storeInfo()[0] == len(coords) == len(got[0]), f"{what}: {len(got[0])} / {len(coords)} bricks"
    assert np.array_equal(got[0], coords), f"{what}: brick coordinates differ"
    for q, a in enumerate(got[1:]):
        assert np.array_equal(a.view(u32), rec[:, q].view(u32)), f"{what}: stored records {q} differ"


def _steps(dims, rng, last):
    """A shift and, half of the time, its return; after the last frame also |d| >= n and back."""
    n = np.asarray(dims)
    d = rng.integers(-(n // 3), n // 3 + 1)
    out = [d, -d] if rng.random() < 0.5 else [d]
    return out + ([n * np.array([1, 0, 0]) + 3, -(n * np.array([1, 0, 0]) + 3)] if last else [])


@pytest.mark.gpu
@pytest.mark.parametrize("size,dims,intensity", [((320, 240), (256, 256, 256), True),
                                                 ((640, 480), (256, 256, 256), False),
                                                 ((320, 240), (97, 64, 71), True),
                                                 ((320, 240), (97, 64, 71), False)])
def test_ground_truth_equals_model(size, dims, intensity):
    import rpg_open_remode_b200 as rmd
    from rpg_open_remode_b200 import synth
    W, H = size
    seq = synth.SyntheticSequence(W, H, seed=0x5EED0900 + W + dims[0])
    frames = [seq.frame(k) for k in (0, 30, 60)]
    s, origin, tau = _grid(seq, frames, max(dims))
    v, m = _pair(dims, s, origin, tau, intensity)
    cam = rmd.PinholeCamera(*seq.camera)
    rng = np.random.default_rng(dims[0] + W)
    restored = 0
    for q, fr in enumerate(frames):
        v.integrateDepth(fr.depth, cam, fr.T_cam_world, None, fr.image if intensity else None)
        m.integrate(fr.depth, seq.camera, fr.T_cam_world, None, fr.image if intensity else None)
        if not intensity:
            m.cint[:], m.cw[:] = 0, 0
        for d in _steps(dims, rng, q == len(frames) - 1):
            v.shift(d)
            m.shift(d)
            restored += m.restored
            _same(v, m, f"{size} {dims} d={d}")
    assert restored > 0 and len(m.bricks) > 0


@pytest.mark.gpu
def test_filter_output_equals_model():
    """Keyframes of the real depth filter, fused as mu and as the denoised map, with shifts that come back."""
    import rpg_open_remode_b200 as rmd
    from rpg_open_remode_b200 import synth
    W, H = 320, 240
    seq = synth.SyntheticSequence(W, H, seed=0x5EED0910)
    cam = rmd.PinholeCamera(*seq.camera)
    f0 = seq.frame(0)
    dmin, dmax = float(f0.depth.min()), float(f0.depth.max())
    s, origin, tau = _grid(seq, [f0], 160)
    v_mu, m_mu = _pair((160, 160, 160), s, origin, tau)
    v_dn, m_dn = _pair((160, 160, 160), s, origin, tau)
    den = rmd.DepthmapDenoiser(W, H, device=0)
    den.setLargeSigmaSq(dmax - dmin)
    img = rmd.DeviceImage(W, H, "float32")
    for ref, ds in ((0, [(40, -30, 50), (-40, 30, -50)]), (31, [(-60, 20, -30), (200, 0, 0), (-200, 0, 0)])):
        g = rmd.SeedMatrix(W, H, cam, device=0)
        fr = seq.frame(ref)
        g.setReferenceImage(fr.image_u8, fr.T_cam_world, dmin, dmax)
        for k in range(ref + 1, ref + 31):
            f = seq.frame(k, want_depth=False)
            g.update(f.image_u8, f.T_cam_world)
        conv, mu, ref_img = g.downloadConvergence(), g.downloadDepthmap(), g._download(rmd.FIELD_REF_IMG)
        v_mu.integrate(g)
        m_mu.integrate(mu, seq.camera, fr.T_cam_world, conv, ref_img)
        den.denoiseSeedsToDevice(g, img.data, img.pitch, 0.5, 100)
        v_dn.integrate(g, img)
        den.sync()
        m_dn.integrate(img.getDevData(), seq.camera, fr.T_cam_world, conv, ref_img)
        for d in ds:
            for v, m in ((v_mu, m_mu), (v_dn, m_dn)):
                v.shift(d)
                m.shift(d)
                _same(v, m, f"filter output d={d}")


# ------------------------------------------------------------------ round trip and revisit
@pytest.mark.gpu
def test_round_trip_and_revisit():
    import rpg_open_remode_b200 as rmd
    from rpg_open_remode_b200 import synth
    W, H = 320, 240
    seq = synth.SyntheticSequence(W, H, seed=0x5EED0920)
    f0, f1 = seq.frame(0), seq.frame(15)
    s, origin, tau = _grid(seq, [f0, f1], 128)
    cam = rmd.PinholeCamera(*seq.camera)
    dmin, dmax = float(f0.depth.min()), float(f0.depth.max())

    def views(v):
        g = rmd.SeedMatrix(W, H, cam, device=0)
        g.setReferenceImage(f1.image_u8, f1.T_cam_world, dmin, dmax)
        g.priorFromVolume(v, 0.25)
        g.sync()
        verts, tris = v.mesh()
        return [v.raycast(cam, f1.T_cam_world, W, H), *v.raycastIntensity(cam, f1.T_cam_world, W, H),
                *v.raycastNormals(cam, f1.T_cam_world, W, H), v.surfacePoints(), verts, tris, g.downloadDepthmap()]

    out = {}
    for store in (True, False):
        v = rmd.TsdfVolume((128, 128, 128), s, origin, tau, 64.0, device=0, intensity=True, store=store)
        v.integrateDepth(f0.depth, cam, f0.T_cam_world, None, f0.image)
        rng = np.random.default_rng(7)
        for _ in range(6 if store else 0):   # shift(d); shift(-d) is lossless for any d
            win = v.download() + v.downloadIntensity()
            d = rng.integers(-200, 201, 3)
            v.shift(d)
            v.shift(-d)
            assert all(np.array_equal(a.view(u32), b.view(u32))
                       for a, b in zip(win, v.download() + v.downloadIntensity())), d
        before = views(v)
        v.shift((0, 0, 300))   # away by more than n, then back
        v.shift((0, 0, -300))
        after = views(v)
        out[store] = before, after
    before, after = out[True]
    for a, b in zip(before, after):
        assert np.array_equal(np.asarray(a).view(np.uint8), np.asarray(b).view(np.uint8))
    assert (before[0] > 0).mean() > 0.3
    assert not (out[False][1][0] > 0).any()       # without the store the revisit sees nothing
    assert len(out[False][1][5]) == 0


# ------------------------------------------------------------------ mapMesh
@pytest.mark.gpu
@pytest.mark.parametrize("dims", [(64, 64, 64), (41, 30, 37)])
def test_map_mesh_equals_model(dims):
    import rpg_open_remode_b200 as rmd
    from rpg_open_remode_b200 import synth
    from rpg_open_remode_b200.api import TsdfVolume
    W, H = 320, 240
    seq = synth.SyntheticSequence(W, H, seed=0x5EED0930 + dims[0])
    frames = [seq.frame(k) for k in (0, 30, 60, 90)]
    # an exact grid: voxel size and origin powers of two, so that positions match across tiles
    s0, o0, _ = _grid(seq, frames, 2 * max(dims))
    s = F(2.0 ** np.ceil(np.log2(float(s0))))
    origin = (np.floor(np.asarray(o0, np.float64) / s) * s).astype(F)
    v, m = _pair(dims, s, origin, F(4) * s)
    cam = rmd.PinholeCamera(*seq.camera)
    n = np.asarray(dims)
    for q, fr in enumerate(frames):
        v.integrateDepth(fr.depth, cam, fr.T_cam_world, None, fr.image)
        m.integrate(fr.depth, seq.camera, fr.T_cam_world, None, fr.image)
        d = (n // 2) * np.array([1, 1, 0]) if q % 2 == 0 else (n // 2) * np.array([0, -1, 1])
        v.shift(d)
        m.shift(d)
    state = v.download() + v.downloadIntensity() + v.downloadStore()
    D = v.offset
    got = v.mapMesh(intensity=True, normals=True)
    want = TsdfVolume.mapMesh(m, intensity=True, normals=True)
    assert len(got[1]) > 1000
    for a, b in zip(got, want):
        assert np.array_equal(a.view(u32), b.view(u32))
    mesh_checks.open_edges(got[1], len(got[0]))
    # the volume is unchanged, apart from the bricks the sweep stored from the window
    assert np.array_equal(v.offset, D)
    after = v.download() + v.downloadIntensity()
    assert all(np.array_equal(a.view(u32), b.view(u32)) for a, b in zip(state[:4], after))
    coords = v.downloadStore()
    old = np.array([tuple(c) in set(map(tuple, state[4].tolist())) for c in coords[0].tolist()], bool)
    assert np.array_equal(coords[0][old], state[4])
    assert all(np.array_equal(a[old].view(u32), b.view(u32)) for a, b in zip(coords[1:], state[5:]))
    assert not any(a[~old].any() for a in coords[1:])
    # id triangles against the dense map meshed as one grid (the model's, pinned on the CPU)
    from test_volume_store_oracle import _map_ids
    import spill_mesh_oracle as smo
    lo, t, w = m.dense_map()
    g = smo.OracleVolume(t.shape[::-1], s, origin, F(4) * s, 64.0)
    g.tsdf, g.weight, g.cint, g.cw = t, w, np.zeros_like(t), np.zeros_like(w)
    dv, dt = g.mesh()
    dids = g.surfaceIds()
    dids[:, :3] += lo
    ids = _map_ids(m)
    assert sorted(tuple(map(tuple, ids[x])) for x in got[1]) == sorted(tuple(map(tuple, dids[x])) for x in dt)
    assert got[2].shape == (len(got[0]),) and got[3].shape == (len(got[0]), 3)


# ------------------------------------------------------------------ ordering and limits
@pytest.mark.gpu
def test_stream_ordering_without_syncs():
    import rpg_open_remode_b200 as rmd
    from rpg_open_remode_b200 import synth
    W, H = 640, 480
    seq = synth.SyntheticSequence(W, H, seed=0x5EED0940)
    f0, f1, f2 = seq.frame(0), seq.frame(20), seq.frame(30)
    dmin, dmax = float(f0.depth.min()), float(f0.depth.max())
    s, origin, tau = _grid(seq, [f0, f1], 256)
    cam = rmd.PinholeCamera(*seq.camera)
    imgs = []
    for fr in (f0, f1):
        dimg, iimg = rmd.DeviceImage(W, H, "float32"), rmd.DeviceImage(W, H, "float32")
        dimg.setDevData(fr.depth)
        iimg.setDevData(fr.image)
        imgs.append((dimg, iimg, fr.T_cam_world))

    def run(sync):
        v = rmd.TsdfVolume((256, 256, 256), s, origin, tau, 64.0, device=0, intensity=True, store=True)
        g = rmd.SeedMatrix(W, H, cam, device=0)
        g.setReferenceImage(f2.image_u8, f2.T_cam_world, dmin, dmax)
        g.sync()
        steps = [lambda: v.integrateDepth(imgs[0][0], cam, imgs[0][2], None, imgs[0][1]),
                 lambda: v.shift((90, -40, 60)),
                 lambda: v.integrateDepth(imgs[1][0], cam, imgs[1][2], None, imgs[1][1]),
                 lambda: v.shift((-90, 40, -60)),
                 lambda: g.priorFromVolume(v, 0.25),
                 lambda: v.shift((-70, 30, 150))]
        for st in steps:
            st()
            if sync:
                v.sync()
                g.sync()
        g.sync()
        return v, g.downloadDepthmap()

    (v_a, mu_a), (v_b, mu_b) = run(False), run(True)
    for a, b in zip(v_a.download() + v_a.downloadIntensity() + v_a.downloadStore(),
                    v_b.download() + v_b.downloadIntensity() + v_b.downloadStore()):
        assert np.array_equal(a.view(u32), b.view(u32))
    assert np.array_equal(mu_a.view(u32), mu_b.view(u32))


@pytest.mark.gpu
def test_grid_beyond_2gb_capacity_upload_and_errors():
    import rpg_open_remode_b200 as rmd
    from rpg_open_remode_b200 import _native, synth
    from test_volume_oracle import ground_truth_points
    W, H = 640, 480
    seq = synth.SyntheticSequence(W, H, seed=0x5EED0950)
    f0 = seq.frame(0)
    pts = ground_truth_points(f0, seq.camera).reshape(-1, 3)
    dims = (1024, 1024, 320)
    lo, hi = pts.min(0), pts.max(0)
    s = F(((hi - lo) / (np.array(dims) - 1 - 16)).max())
    origin = (lo - 8 * float(s)).astype(F)
    origin[2] = F(hi[2] - (dims[2] - 1 - 8) * float(s))
    v = rmd.TsdfVolume(dims, s, origin, F(4) * s, 64.0, device=0, intensity=True, store=True)
    cam = rmd.PinholeCamera(*seq.camera)
    v.integrateDepth(f0.depth, cam, f0.T_cam_world, None, f0.image)
    win = v.download() + v.downloadIntensity()
    v.shift((300, -200, 200))
    n1 = v.storeInfo()[0]
    v.shift((-300, 200, -200))
    assert all(np.array_equal(a.view(u32), b.view(u32)) for a, b in zip(win, v.download() + v.downloadIntensity()))
    del win
    bricks, nbytes = v.storeInfo()
    print(f"\n1024x1024x320 with the store: {bricks} bricks ({n1} after the first shift), {nbytes / 2 ** 20:.1f} MiB")
    assert bricks == n1 > 1000 and nbytes >= bricks * 8192
    # capacities and the count-only call
    L, cnt = _native.lib(), ctypes.c_size_t()
    full = v.downloadStore()
    cap = bricks // 7
    part = v.downloadStore(capacity=cap)
    assert len(part[0]) == cap and all(np.array_equal(a.view(u32), b[:cap].view(u32)) for a, b in zip(part, full))
    assert L.rmd_volume_download_store(v.handle, None, None, None, None, None, 0, ctypes.byref(cnt)) == 0
    assert cnt.value == bricks
    del v, full, part
    gc.collect()

    # upload / download round trip on a small volume, and the error codes
    v = rmd.TsdfVolume((20, 16, 12), 0.1, (0, 0, 0), 0.3, 10.0, device=0, store=True)
    rng = np.random.default_rng(3)
    coords = np.array([[-3, 0, 1], [5, -2, 0], [0, 0, 0], [1, 1, -1]], np.int64)
    t, w = rng.random((4, 8, 8, 8)).astype(F), rng.random((4, 8, 8, 8)).astype(F)
    v.uploadStore(coords, t, w)
    got = v.downloadStore()
    order = np.lexsort(coords.T)   # ascending (z, y, x)
    assert np.array_equal(got[0], coords[order])
    # brick (0, 0, 0) lies inside the 20 x 16 x 12 window: returned as (0, 0)
    assert not got[1][got[0][:, 0] == 0].any() and not got[2][got[0][:, 0] == 0].any()
    assert np.array_equal(got[1][got[0][:, 0] == -3], t[:1]) and np.array_equal(got[2][got[0][:, 0] == 5], w[1:2])
    v.enableIntensity()            # bricks already stored get zeroed colour records
    assert not any(a.any() for a in v.downloadStore()[3:])
    v.reset()
    assert v.storeInfo()[0] == 0 and v.storeInfo()[1] > 0
    h, d3 = v.handle, np.array([1, 2, 3], np.int32)
    z = ctypes.c_size_t()
    assert L.rmd_volume_enable_store(None) == INVALID
    assert L.rmd_volume_store_info(None, None, None) == INVALID
    assert L.rmd_volume_download_store(h, None, None, None, None, None, 4, ctypes.byref(z)) == INVALID
    assert L.rmd_volume_download_store(h, None, None, None, None, None, 0, None) == INVALID
    assert L.rmd_volume_upload_store(h, None, None, None, None, None, 2) == INVALID
    c2 = np.zeros((2, 3), np.int64)
    r2 = np.zeros((2, 512), F)
    assert L.rmd_volume_upload_store(h, c2.ctypes.data, r2.ctypes.data, r2.ctypes.data, None, None, 2) == INVALID
    c2[1, 0] = 2 ** 61
    assert L.rmd_volume_upload_store(h, c2.ctypes.data, r2.ctypes.data, r2.ctypes.data, None, None, 2) == INVALID
    c2[1, 0] = 1
    assert L.rmd_volume_upload_store(h, c2.ctypes.data, r2.ctypes.data, r2.ctypes.data, r2.ctypes.data, None,
                                     2) == INVALID
    with pytest.raises(ValueError):
        v.uploadStore(c2, r2[:1], r2)
    plain = rmd.TsdfVolume((8, 8, 8), 0.1, (0, 0, 0), 0.3, 10.0, device=0, store=True)
    assert L.rmd_volume_download_store(plain.handle, None, None, None, r2.ctypes.data, None, 0,
                                       ctypes.byref(z)) == NOT_INITIALISED
    assert L.rmd_volume_upload_store(plain.handle, c2.ctypes.data, r2.ctypes.data, r2.ctypes.data, r2.ctypes.data,
                                     r2.ctypes.data, 2) == NOT_INITIALISED
    none = rmd.TsdfVolume((8, 8, 8), 0.1, (0, 0, 0), 0.3, 10.0, device=0)
    assert L.rmd_volume_store_info(none.handle, ctypes.byref(z), None) == NOT_INITIALISED
    assert L.rmd_volume_download_store(none.handle, None, None, None, None, None, 0, ctypes.byref(z)) == NOT_INITIALISED
    with pytest.raises(rmd.RmdError):
        none.mapMesh()
    # the volume still shifts after refused calls
    assert L.rmd_volume_shift(h, d3.ctypes.data) == 0 and np.array_equal(v.offset, [1, 2, 3])
    # a node with the store cannot take a SceneMesh
    from rpg_open_remode_b200 import node
    with pytest.raises(ValueError):
        node.DepthmapNode(rmd.Depthmap(32, 24, 30, 15.5, 30, 11.5, device=0), volume=v, follow_volume=True,
                          scene_mesh=rmd.SceneMesh())


# ------------------------------------------------------------------ the node on c2
def _bits_equal(x, y):
    """Publications equal bit for bit: arrays by their bytes, tuples and lists element by element."""
    if isinstance(x, (tuple, list)) or isinstance(y, (tuple, list)):
        return type(x) is type(y) and len(x) == len(y) and all(_bits_equal(p, q) for p, q in zip(x, y))
    if isinstance(x, np.ndarray) or isinstance(y, np.ndarray):
        a, b = np.asarray(x), np.asarray(y)
        return a.dtype == b.dtype and a.shape == b.shape and a.tobytes() == b.tobytes()
    return x == y


# Measured on an H100 80 GB HBM3 at 700 W (DESIGN.md 5.3): 128^3 shifts 3 times and 64^3 7 times on c2, and neither
# brings a known stored voxel back.  mapMesh: 128^3 23489 vertices (0.640x the fixed 512^3 mesh's 36730, as SceneMesh),
# 1.63 % open directed edges, median / p95 distance 0.494 / 0.576 voxels, store 1078 bricks in 8 MiB; 64^3 5712
# vertices (0.156x), 2.84 % open, 0.507 / 0.592 voxels, 156 bricks in 1 MiB.
STORE_C2_MIN_VERTEX_RATIO = {128: 0.5, 64: 0.1}   # mapMesh vertices over the fixed 512^3 mesh's
STORE_C2_P95_VOXELS = 1.0           # p95 distance of mapMesh vertices to the fixed mesh's vertices, in voxels


@pytest.mark.gpu
def test_store_on_c2():
    from scipy.spatial import cKDTree
    import rpg_open_remode_b200 as rmd
    from rpg_open_remode_b200 import multi_gpu, synth
    W, H, N = 640, 480, 200
    seq = synth.SyntheticSequence(W, H, seed=multi_gpu.keyframe_seed(0))    # bench.py's c2 sequence
    s, origin, tau = _grid(seq, [seq.frame(k) for k in range(0, N, 25)] + [seq.frame(N - 1)], 512)
    fixed = rmd.TsdfVolume((512, 512, 512), s, origin, tau, 64.0, device=0)
    _node_run(seq, N, fixed)
    fv, ft = fixed.mesh()
    del fixed
    gc.collect()
    for n in (128, 64):
        plain = rmd.TsdfVolume((n, n, n), s, (0.0, 0.0, 0.0), tau, 64.0, device=0)
        pa, _ = _node_run(seq, N, plain, follow_volume=True)
        del plain
        vol = rmd.TsdfVolume((n, n, n), s, (0.0, 0.0, 0.0), tau, 64.0, device=0, store=True)
        restored, shift = [], vol.shift

        def counting_shift(d, vol=vol, shift=shift, restored=restored):
            shift(d)
            lo, hi = kept_box(vol.dims, -np.asarray(d, np.int64))
            restored.append(int((vol.download()[1][moving(vol.dims, lo, hi)] > 0).sum()))

        vol.shift = counting_shift
        pb, _ = _node_run(seq, N, vol, follow_volume=True)
        assert len(pa) == len(pb)
        for a, b in zip(pa, pb):
            assert a[0] == b[0]
            if a[0] == "depthmap_and_pointcloud":
                assert np.array_equal(a[1].view(u32), b[1].view(u32)) and np.array_equal(a[2], b[2])
            else:
                assert _bits_equal(a[1:], b[1:])
        del vol.shift
        mv, mt, _, _ = vol.mapMesh()
        dist = cKDTree(fv[:, :3]).query(mv[:, :3])[0] / float(s)
        opened = len(mesh_checks.open_edges(mt, len(mv))) / max(3 * len(mt), 1)
        bricks, nbytes = vol.storeInfo()
        print(f"\nc2 {n}^3 with the store: {len(restored)} shifts, known voxels restored per shift {restored}; "
              f"mapMesh {len(mv)} vertices, {len(mt)} triangles vs fixed 512^3 {len(fv)} vertices "
              f"(ratio {len(mv) / len(fv):.3f}), distance median {np.median(dist):.3f} p95 "
              f"{np.percentile(dist, 95):.3f} voxels, open directed edges {100 * opened:.2f} %; store {bricks} bricks, "
              f"{nbytes / 2 ** 20:.1f} MiB")
        assert len(mv) >= STORE_C2_MIN_VERTEX_RATIO[n] * len(fv) and np.percentile(dist, 95) <= STORE_C2_P95_VOXELS
        del vol
        gc.collect()
