"""The spill mesh of a moving TSDF volume on the GPU (csrc/volume.cu: volume_spill_mesh_* and volume_spill_tri_*;
rmd_volume_spill_mesh[_intensity|_normals], rmd_volume_surface_ids, rmd_volume_offset; api.TsdfVolume.spillMesh,
api.SceneMesh, DepthmapNode(scene_mesh=); DESIGN.md 4.8).

  * the product against the oracle (oracle/rmd_oracle_volume_spill_mesh.c) bit for bit: vertices, triangles, ids,
    intensities and normals across shifts -- ground truth at QVGA and VGA into 256^3, the ragged 97 x 64 x 71 grid,
    real filter output (mu and denoised), the 1024 x 1024 x 320 grid (records beyond 2^31 bytes, also after a shift),
    capacities below both counts and the count-only call, d = 0 and |d| >= n;
  * mesh before a shift == spill mesh + mesh after it, by ids; SceneMesh without integration reproduces mesh();
  * every error code;
  * the node on bench.py's c2 sequence with scene_mesh: bit-identical publications and volume, and the scene mesh
    measured against the fixed 512^3 volume's.
"""
import ctypes

import numpy as np
import pytest

import spill_mesh_oracle as smo
from test_volume import _grid
from test_volume_shift import _node_run
from test_volume_spill_mesh_oracle import _identity_failures, _ids_of_triangles, _scene_reproduces

F = np.float32
u32 = np.uint32
INVALID, NOT_INITIALISED = -1, -2


def _pair(dims, s, origin, tau, intensity=True):
    import rpg_open_remode_b200 as rmd
    return (rmd.TsdfVolume(dims, s, origin, tau, 64.0, device=0, intensity=intensity),
            smo.OracleVolume(dims, s, origin, tau, 64.0))


def _same_spill_mesh(v, o, d, what, values=True):
    """spillMesh (and with values its intensities and normals) == the oracle's, bit for bit; returns (n vertices,
    n triangles)."""
    gv, gt, gids = v.spillMesh(d)
    wv, wt, wk, nv, nt = o.spill_mesh(d, smo.POINTS)
    assert len(gv) == nv and len(gt) == nt, f"{what}: {len(gv)} / {nv} vertices, {len(gt)} / {nt} triangles"
    assert np.array_equal(gv.view(u32), wv.view(u32)), f"{what}: vertices differ"
    assert np.array_equal(gt, wt), f"{what}: triangles differ"
    assert np.array_equal(gids, smo.keys_to_ids(wk, o.dims, o.D)), f"{what}: ids differ"
    assert np.array_equal(v.offset, o.D)
    if not values:
        return nv, nt
    got, want = v.spillMeshNormals(d), o.spill_mesh(d, smo.NORMALS, nv, 0)[0]
    assert np.array_equal(got.view(u32), want[:, :3].view(u32)), f"{what}: normals differ"
    if v.intensity:
        got, want = v.spillMeshIntensity(d), o.spill_mesh(d, smo.INTENSITY, nv, 0)[0]
        assert np.array_equal(got.view(u32), want.view(u32)), f"{what}: intensities differ"
    return nv, nt


def _mesh_ids(v):
    verts, tris = v.mesh()
    ids = v.surfaceIds()
    assert len(ids) == len(verts)
    return ids, _ids_of_triangles(tris, ids)


def _shift(v, o, d, what, values=True):
    """Compare the spill mesh, check before == spill + after by ids on the GPU, then shift both."""
    nv, nt = _same_spill_mesh(v, o, d, what, values)
    before = _mesh_ids(v)
    sv, st, sids = v.spillMesh(d)
    v.shift(d)
    o.shift(d)
    after = _mesh_ids(v)
    fails = _identity_failures(before, (sids, _ids_of_triangles(st, sids)), after)
    assert not fails, f"{what} d={d}: {fails}"
    return nt


# ------------------------------------------------------------------ product == oracle
@pytest.mark.gpu
@pytest.mark.parametrize("size,dims", [((320, 240), (256, 256, 256)), ((640, 480), (256, 256, 256)),
                                       ((320, 240), (97, 64, 71))])
def test_ground_truth_equals_oracle(size, dims):
    import rpg_open_remode_b200 as rmd
    from rpg_open_remode_b200 import synth
    W, H = size
    seq = synth.SyntheticSequence(W, H, seed=0x5EED0A00 + W)
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
        spilled += _shift(v, o, d, f"{size} {dims}")
    assert spilled > 0
    assert _same_spill_mesh(v, o, (0, 0, 0), "d = 0") == (0, 0)
    # |d| >= n: the spill mesh is mesh()
    mv, mt = v.mesh()
    gv, gt, _ = v.spillMesh((0, -dims[1], 3))
    assert len(mt) > 0 and np.array_equal(gv.view(u32), mv.view(u32)) and np.array_equal(gt, mt)
    _same_spill_mesh(v, o, (dims[0] + 1, 0, 0), "whole grid")


@pytest.mark.gpu
@pytest.mark.parametrize("size,n", [((320, 240), 40), ((640, 480), 30)])
def test_filter_output_equals_oracle(size, n):
    """Keyframes of the real depth filter, fused with their reference images, mu and the denoised image."""
    import rpg_open_remode_b200 as rmd
    from rpg_open_remode_b200 import synth
    W, H = size
    seq = synth.SyntheticSequence(W, H, seed=0x5EED0A10 + W)
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
        g = rmd.SeedMatrix(W, H, cam, device=0)
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
        spilled += _shift(v_mu, o_mu, d, f"mu {size}")
        spilled += _shift(v_dn, o_dn, d, f"denoised {size}")
    assert spilled > 0


@pytest.mark.gpu
def test_grid_beyond_2gb_and_capacity():
    """1024 x 1024 x 320 voxels with the intensity channel: records beyond 2^31 bytes, before and after a shift (the
    second arrays); capacities below both counts and the count-only call."""
    import rpg_open_remode_b200 as rmd
    from rpg_open_remode_b200 import _native, synth
    from test_volume_oracle import ground_truth_points
    W, H = 640, 480
    seq = synth.SyntheticSequence(W, H, seed=0x5EED0A30)
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
    assert (o.weight.reshape(-1)[2 ** 28:] > 0).any()
    d = (300, -200, 40)
    wv, wt, wk, nv, nt = o.spill_mesh(d)
    assert nv > 1000 and nt > 1000
    L, cv, ct = _native.lib(), ctypes.c_size_t(), ctypes.c_size_t()
    dd = np.array(d, np.int32)
    assert L.rmd_volume_spill_mesh(v.handle, dd.ctypes.data, None, 0, None, 0, None, ctypes.byref(cv),
                                   ctypes.byref(ct)) == 0 and (cv.value, ct.value) == (nv, nt)
    for mv, mt in ((nv // 7, nt // 5), (0, nt // 3), (nv // 3, 0)):
        xyzw, tri, ids = np.empty((max(mv, 1), 4), F), np.empty((max(mt, 1), 3), np.int32), np.empty((max(mv, 1), 4),
                                                                                                      np.int64)
        assert L.rmd_volume_spill_mesh(v.handle, dd.ctypes.data, xyzw.ctypes.data, mv, tri.ctypes.data, mt,
                                       ids.ctypes.data, ctypes.byref(cv), ctypes.byref(ct)) == 0
        assert (cv.value, ct.value) == (nv, nt)
        assert np.array_equal(xyzw[:mv].view(u32), wv[:mv].view(u32)) and np.array_equal(tri[:mt], wt[:mt])
        assert np.array_equal(ids[:mv], smo.keys_to_ids(wk[:mv], dims, o.D))
    for fn, kind, per in ((L.rmd_volume_spill_mesh_normals, smo.NORMALS, 4),
                          (L.rmd_volume_spill_mesh_intensity, smo.INTENSITY, 1)):
        w_all = o.spill_mesh(d, kind, nv, 0)[0]
        cap = nv // 7
        part = np.empty((cap, per), F)
        assert fn(v.handle, dd.ctypes.data, part.ctypes.data, cap, ctypes.byref(cv)) == 0 and cv.value == nv
        assert np.array_equal(part.reshape(w_all[:cap].shape).view(u32), w_all[:cap].view(u32))
        assert fn(v.handle, dd.ctypes.data, None, 0, ctypes.byref(cv)) == 0 and cv.value == nv
    ids_all = v.surfaceIds()
    assert np.array_equal(v.surfaceIds(capacity=len(ids_all) // 3), ids_all[:len(ids_all) // 3])
    _shift(v, o, d, "2.7 GB grid", values=False)   # the values were compared above
    f1 = seq.frame(20)
    v.integrateDepth(f1.depth, cam, f1.T_cam_world, None, f1.image)
    o.integrate(f1.depth, seq.camera, f1.T_cam_world, None, f1.image)
    _shift(v, o, (-100, 50, -20), "2.7 GB grid, second shift", values=False)


# ------------------------------------------------------------------ the welder
@pytest.mark.gpu
def test_scene_mesh_without_integration_reproduces_the_mesh():
    """Ground truth fused into an exact grid (power-of-two voxel, origin a multiple of it), then shifts with no
    integration between them, back into unknown space included: the scene mesh is the mesh before the shifts."""
    import rpg_open_remode_b200 as rmd
    from rpg_open_remode_b200 import synth
    seq = synth.SyntheticSequence(640, 480, seed=0x5EED0A40)
    frames = [seq.frame(k) for k in (0, 30)]
    s0, origin0, _ = _grid(seq, frames, 256)
    s = F(2.0 ** np.round(np.log2(float(s0))))
    origin = (np.round(np.asarray(origin0, np.float64) / float(s)) * float(s)).astype(F)
    v = rmd.TsdfVolume((256, 256, 256), s, origin, F(4) * s, 64.0, device=0, intensity=True)
    cam = rmd.PinholeCamera(*seq.camera)
    for fr in frames:
        v.integrateDepth(fr.depth, cam, fr.T_cam_world, None, fr.image)
    shifts = [(40, -30, 20), (-25, 60, 0), (-40, 30, -20), (0, 0, 90), (0, 0, -90)]
    assert _scene_reproduces(v, shifts) == len(shifts)


# ------------------------------------------------------------------ error codes
@pytest.mark.gpu
def test_error_codes():
    import rpg_open_remode_b200 as rmd
    from rpg_open_remode_b200 import _native
    L = _native.lib()
    v = rmd.TsdfVolume((16, 16, 16), 0.1, (-0.8, -0.8, 0.5), 0.3, 10.0, device=0)
    d = np.array([1, 2, 3], np.int32)
    nv, nt, n = ctypes.c_size_t(), ctypes.c_size_t(), ctypes.c_size_t()
    out, tri, ids = np.empty((4, 4), F), np.empty((4, 3), np.int32), np.empty((4, 4), np.int64)
    ok = (v.handle, d.ctypes.data, out.ctypes.data, 4, tri.ctypes.data, 4, ids.ctypes.data, ctypes.byref(nv),
          ctypes.byref(nt))
    for q in (0, 1, 7, 8):
        bad = list(ok)
        bad[q] = None
        assert L.rmd_volume_spill_mesh(*bad) == INVALID, q
    bad = list(ok)
    bad[2] = None
    assert L.rmd_volume_spill_mesh(*bad) == INVALID
    bad = list(ok)
    bad[4] = None
    assert L.rmd_volume_spill_mesh(*bad) == INVALID
    bad = list(ok)
    bad[6] = None   # ids may be NULL
    assert L.rmd_volume_spill_mesh(*bad) == 0 and nv.value == nt.value == 0
    for fn in (L.rmd_volume_spill_mesh_normals, L.rmd_volume_spill_mesh_intensity):
        assert fn(None, d.ctypes.data, out.ctypes.data, 4, ctypes.byref(n)) == INVALID
        assert fn(v.handle, None, out.ctypes.data, 4, ctypes.byref(n)) == INVALID
        assert fn(v.handle, d.ctypes.data, out.ctypes.data, 4, None) == INVALID
        assert fn(v.handle, d.ctypes.data, None, 4, ctypes.byref(n)) == INVALID
    assert L.rmd_volume_spill_mesh_normals(v.handle, d.ctypes.data, None, 0, ctypes.byref(n)) == 0 and n.value == 0
    assert L.rmd_volume_spill_mesh_intensity(v.handle, d.ctypes.data, None, 0, ctypes.byref(n)) == NOT_INITIALISED
    assert L.rmd_volume_surface_ids(None, ids.ctypes.data, 4, ctypes.byref(n)) == INVALID
    assert L.rmd_volume_surface_ids(v.handle, None, 4, ctypes.byref(n)) == INVALID
    assert L.rmd_volume_surface_ids(v.handle, ids.ctypes.data, 4, None) == INVALID
    assert L.rmd_volume_surface_ids(v.handle, None, 0, ctypes.byref(n)) == 0 and n.value == 0
    D = np.empty(3, np.int64)
    assert L.rmd_volume_offset(None, D.ctypes.data) == INVALID and L.rmd_volume_offset(v.handle, None) == INVALID
    v.shift((3, -2, 1))
    v.shift((1, 1, 1))
    assert np.array_equal(v.offset, [4, -1, 2])
    with pytest.raises(ValueError):
        v.spillMesh((0.5, 0, 0))
    v.sync()


# ------------------------------------------------------------------ the node
@pytest.mark.gpu
def test_node_scene_mesh_off_and_argument():
    import rpg_open_remode_b200 as rmd
    from rpg_open_remode_b200 import node
    dm = rmd.Depthmap(32, 24, 30, 15.5, 30, 11.5, device=0)
    v = rmd.TsdfVolume((8, 8, 8), 0.1, (0, 0, 0), 0.3, device=0)
    with pytest.raises(ValueError):
        node.DepthmapNode(dm, volume=v, scene_mesh=rmd.SceneMesh())
    node.DepthmapNode(dm, volume=v, follow_volume=True, scene_mesh=rmd.SceneMesh())


def _edges(T):
    """Directed edges of the triangles [m, 3] as one int64 per edge, and the count of those used twice and of those
    whose reverse is missing (open edges)."""
    T = T.astype(np.int64)
    a = np.concatenate([T[:, 0], T[:, 1], T[:, 2]])
    b = np.concatenate([T[:, 1], T[:, 2], T[:, 0]])
    key, rev = a * 2 ** 31 + b, b * 2 ** 31 + a
    uniq, cnt = np.unique(key, return_counts=True)
    return int((cnt > 1).sum()), int((~np.isin(rev, key)).sum())


# Measured on an H100 80 GB HBM3 at 700 W (DESIGN.md 5.3): bench.py's c2 sequence (VGA, 200 frames) through the node, a
# 128^3 volume following from the origin with the fixed 512^3 volume's voxel size (it shifts three times), with
# scene_mesh: 23489 vertices (the spills' points plus the final window's), 44341 triangles -- all of them the final
# window's: the spill meshes of this run hold vertices but no meshed cube -- 2173 open directed edges (0.0163 of
# them), none used twice; distance of the vertices to the fixed volume's mesh vertices median 0.494, p95 0.576
# voxels.  The run is deterministic; the bars leave a margin.
SCENE_MIN_SHIFTS = 3
SCENE_MIN_VERTICES = 20000
SCENE_MAX_OPEN_EDGE_FRACTION = 0.05   # open directed edges over all directed edges
SCENE_MEDIAN_VOXELS = 0.75            # median distance of the scene's vertices to the fixed mesh's vertices, in voxels
SCENE_P95_VOXELS = 1.0                # p95 of that distance


@pytest.mark.gpu
def test_scene_mesh_on_c2():
    from scipy.spatial import cKDTree
    import rpg_open_remode_b200 as rmd
    from rpg_open_remode_b200 import multi_gpu, synth
    W, H, N = 640, 480, 200
    seq = synth.SyntheticSequence(W, H, seed=multi_gpu.keyframe_seed(0))    # bench.py's c2 sequence
    s, origin, tau = _grid(seq, [seq.frame(k) for k in range(0, N, 25)] + [seq.frame(N - 1)], 512)
    fixed = rmd.TsdfVolume((512, 512, 512), s, origin, tau, 64.0, device=0)
    _node_run(seq, N, fixed)
    ref = fixed.mesh()[0][:, :3]
    del fixed
    n = 128
    plain = rmd.TsdfVolume((n, n, n), s, (0.0, 0.0, 0.0), tau, 64.0, device=0)
    p_plain, _ = _node_run(seq, N, plain, follow_volume=True)
    follow = rmd.TsdfVolume((n, n, n), s, (0.0, 0.0, 0.0), tau, 64.0, device=0)
    scene = rmd.SceneMesh(normals=True)
    p_scene, _ = _node_run(seq, N, follow, follow_volume=True, scene_mesh=scene)
    # the publications and the volume are those of the same run without scene_mesh
    assert len(p_plain) == len(p_scene)
    for a, b in zip(p_plain, p_scene):
        assert a[0] == b[0]
        for x, y in zip(a[1:], b[1:]):
            assert (x is None and y is None) or np.array_equal(np.asarray(x).view(u32), np.asarray(y).view(u32))
    for a, b in zip(plain.download(), follow.download()):
        assert np.array_equal(a.view(u32), b.view(u32))
    shifts = sum(p[0] == "volume_spill" for p in p_scene)
    V, T, _, Nrm = scene.mesh(follow)
    assert T.min() >= 0 and T.max() < len(V) and len(Nrm) == len(V)
    twice, open_edges = _edges(T)
    dist = cKDTree(ref).query(V[:, :3])[0] / float(s)
    med, p95 = float(np.median(dist)), float(np.percentile(dist, 95))
    print(f"\nc2 scene mesh, following {n}^3 ({shifts} shifts): {len(V)} vertices, {len(T)} triangles, {open_edges} "
          f"open edges ({open_edges / (3 * len(T)):.4f} of the directed edges), {twice} directed edges used twice; "
          f"window alone {len(follow.mesh()[1])} triangles; fixed 512^3 mesh {len(ref)} vertices; distance to its "
          f"vertices median {med:.3f} p95 {p95:.3f} voxels")
    assert shifts >= SCENE_MIN_SHIFTS
    assert twice == 0
    assert len(V) >= SCENE_MIN_VERTICES
    assert open_edges <= SCENE_MAX_OPEN_EDGE_FRACTION * 3 * len(T)
    assert med <= SCENE_MEDIAN_VOXELS and p95 <= SCENE_P95_VOXELS
