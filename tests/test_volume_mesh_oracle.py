"""The TSDF mesh's checker (oracle/rmd_oracle_mesh.c, bound as mesh_oracle.OracleVolume.mesh; DESIGN.md 4.8) and
the PLY writer, on the CPU: known answers (a plane, an analytic sphere), watertightness on random sign fields, the
rules for unknown and truncated voxels, and the vertex array = the surface points bit for bit."""
import numpy as np
import pytest

import mesh_checks as mc
import mesh_oracle as mo

F = np.float32


def _oracle(tsdf, weight, s=0.05, origin=(0.0, 0.0, 0.0)):
    nz, ny, nx = tsdf.shape
    o = mo.OracleVolume((nx, ny, nz), s, origin, 4 * s, 64.0)
    o.tsdf[...], o.weight[...] = tsdf, weight
    return o


def test_plane_gives_two_triangles_per_column_and_its_area():
    nx, ny, nz, s = 23, 17, 12, 0.05
    z0, tau = 0.2625, 0.15                    # between voxel layers 5 and 6, tau = 3 voxels
    z = np.arange(nz, dtype=F) * F(s)
    t = np.clip((z - F(z0)) / F(tau), -1, 1).astype(F)
    tsdf = np.broadcast_to(t[:, None, None], (nz, ny, nx)).copy()
    o = _oracle(tsdf, np.ones_like(tsdf), s)
    verts, tris = o.mesh()
    assert len(verts) == nx * ny and len(tris) == 2 * (nx - 1) * (ny - 1)
    assert np.allclose(verts[:, 2], z0, atol=1e-6)
    area, _ = mc.area_and_volume(verts, tris)
    assert abs(area - (nx - 1) * (ny - 1) * s * s) <= 1e-5 * area
    n, _ = mc.normals(verts, tris)
    assert np.all(n[:, 2] > 0) and np.allclose(n[:, :2], 0, atol=1e-9)     # towards tsdf > 0 (+z)
    e = mc.open_edges(tris, len(verts))
    assert mc.on_grid_boundary(tsdf, o.weight, e).all()


SPHERE = dict(dims=(56, 52, 50), s=0.05, origin=(-1.3, -1.25, -1.2), centre=(0.05, 0.02, 0.03), radius=1.0)


@pytest.mark.parametrize("tau_voxels", [2.0, 5.0])
def test_analytic_sphere_is_closed_outward_and_measures_right(tau_voxels):
    S = SPHERE
    tsdf, weight = mc.sphere_field(S["dims"], S["s"], S["origin"], S["centre"], S["radius"], tau_voxels * S["s"])
    o = mo.OracleVolume(S["dims"], S["s"], S["origin"], tau_voxels * S["s"], 64.0)
    o.tsdf[...], o.weight[...] = tsdf, weight
    verts, tris = o.mesh()
    pts, n = o.surface_points()
    assert n == len(verts) and np.array_equal(verts.view(np.uint32), pts.view(np.uint32))
    assert len(np.unique(tris)) == n           # every crossing is used: no cube of the band is rejected
    mc.assert_sphere_mesh(verts, tris, S["centre"], S["radius"])


def _random_field(rng, dims, p_zero=0.05):
    nx, ny, nz = dims
    t = rng.uniform(-0.999, 0.999, (nz, ny, nx)).astype(F)
    t[rng.random(t.shape) < p_zero] = 0.0
    t[rng.random(t.shape) < p_zero] = -0.0
    return t


@pytest.mark.parametrize("dims,seed", [((9, 7, 5), 1), ((16, 11, 13), 2), ((2, 2, 2), 3), ((1, 6, 7), 4),
                                       ((31, 3, 17), 5), ((24, 24, 24), 6)])
def test_random_fields_are_watertight_inside_the_grid(dims, seed):
    rng = np.random.default_rng(0x3E5 + seed)
    for rep in range(8 if np.prod(dims) < 5000 else 2):
        tsdf = _random_field(rng, dims, p_zero=[0.0, 0.05, 0.3][rep % 3])
        o = _oracle(tsdf, np.ones_like(tsdf))
        verts, tris = o.mesh()
        pts, n = o.surface_points()
        assert np.array_equal(verts.view(np.uint32), pts.view(np.uint32))
        if min(dims) < 2:
            assert len(tris) == 0
            continue
        assert (len(tris) > 0) == (n > 0)   # a 2x2x2 grid may hold one sign only
        if n == 0:
            continue
        assert tris.min() >= 0 and tris.max() < n
        e = mc.open_edges(tris, n)          # no directed edge twice
        assert mc.on_grid_boundary(tsdf, o.weight, e).all(), "an open edge inside the grid"
        # every interior crossing is used (all weights 1, |tsdf| < 1: no cube is rejected)
        assert len(np.unique(tris)) == n


def test_unknown_and_truncated_voxels():
    rng = np.random.default_rng(0x3E50)
    dims = (21, 18, 15)
    for rep in range(6):
        tsdf = _random_field(rng, dims)
        tsdf[rng.random(tsdf.shape) < 0.15] = 1.0
        tsdf[rng.random(tsdf.shape) < 0.05] = -1.0
        tsdf[rng.random(tsdf.shape) < 0.02] = 1.5
        weight = rng.integers(1, 5, tsdf.shape).astype(F)
        weight[rng.random(tsdf.shape) < 0.1] = 0.0
        o = _oracle(tsdf, weight)
        verts, tris = o.mesh()
        pts, n = o.surface_points()
        assert np.array_equal(verts.view(np.uint32), pts.view(np.uint32))
        assert len(tris) > 0 and tris.min() >= 0 and tris.max() < n
        mc.open_edges(tris, n)              # asserts no directed edge is used twice
        # a triangle's corner cube had 8 known corners: its vertices carry weight > 0
        assert np.all(verts[tris.reshape(-1), 3] > 0)
    # all unknown / all free space: nothing
    for t, w in ((np.zeros(dims[::-1], F), np.zeros(dims[::-1], F)), (np.ones(dims[::-1], F), np.ones(dims[::-1], F))):
        verts, tris = _oracle(t, w).mesh()
        assert len(verts) == 0 and len(tris) == 0


def test_truncated_crossing_rejects_the_cube():
    """One cube: corner 0 inside at -0.5, the rest outside; replacing one outside value by 1.0 (truncated) on a
    crossing edge removes the triangle, on a non-crossing edge keeps it."""
    t = np.full((2, 2, 2), 0.5, F)
    t[0, 0, 0] = -0.5
    w = np.ones_like(t)
    verts, tris = _oracle(t, w).mesh()
    assert len(verts) == 3 and tris.tolist() == [[0, 1, 2]]
    t2 = t.copy()
    t2[0, 0, 1] = 1.0                        # corner 1 = +x neighbour of the inside corner
    verts, tris = _oracle(t2, w).mesh()
    assert len(verts) == 2 and len(tris) == 0
    t3 = t.copy()
    t3[1, 1, 1] = 1.0                        # corner 7: no crossing touches it
    verts, tris = _oracle(t3, w).mesh()
    assert len(verts) == 3 and len(tris) == 1
    w4 = w.copy()
    w4[1, 1, 1] = 0.0                        # an unknown corner
    verts, tris = _oracle(t, w4).mesh()
    assert len(verts) == 3 and len(tris) == 0


def test_ply_round_trip(tmp_path):
    from rpg_open_remode_b200 import write_ply
    rng = np.random.default_rng(7)
    verts = rng.normal(size=(57, 4)).astype(F)
    tris = rng.integers(0, 57, (31, 3)).astype(np.int32)
    for v, t in ((verts, tris), (verts[:0], tris[:0])):
        path = tmp_path / "mesh.ply"
        write_ply(str(path), v, t)
        data = path.read_bytes()
        end = data.index(b"end_header\n") + len(b"end_header\n")
        header = data[:end].decode("ascii").splitlines()
        assert header[:2] == ["ply", "format binary_little_endian 1.0"]
        assert "element vertex %d" % len(v) in header and "element face %d" % len(t) in header
        assert "property list uchar int vertex_indices" in header
        body = np.frombuffer(data, np.uint8, offset=end)
        got_v = np.frombuffer(body[:16 * len(v)].tobytes(), "<f4").reshape(-1, 4)
        faces = np.frombuffer(body[16 * len(v):].tobytes(), np.dtype([("n", "u1"), ("i", "<i4", 3)]))
        assert len(faces) == len(t) and np.all(faces["n"] == 3)
        assert np.array_equal(got_v.view(np.uint32), v.view(np.uint32)) and np.array_equal(faces["i"], t)
