"""Properties of a TSDF triangle mesh (DESIGN.md 4.8), shared by the oracle's CPU tests and the GPU tests.

Triangles are int32 [m, 3] vertex indices; vertices are float32 [n, 4] (x, y, z, weight).  Nothing here knows the
case table: the checks are on the mesh as any consumer would see it.
"""
import numpy as np


def directed_edges(tris):
    """[3m, 2] int64: (a, b), (b, c), (c, a) of every triangle."""
    t = np.asarray(tris, np.int64)
    return np.concatenate([t[:, [0, 1]], t[:, [1, 2]], t[:, [2, 0]]])


def _codes(e, n):
    return e[:, 0] * n + e[:, 1]


def edge_use(tris, n_vertices):
    """(uses of each directed edge, uses of its reverse), one entry per directed edge occurrence."""
    e = directed_edges(tris)
    codes, rev = _codes(e, n_vertices), _codes(e[:, ::-1], n_vertices)
    uniq, counts = np.unique(codes, return_counts=True)
    fwd = counts[np.searchsorted(uniq, codes)]
    pos = np.clip(np.searchsorted(uniq, rev), 0, len(uniq) - 1)
    back = np.where(uniq[pos] == rev, counts[pos], 0)
    return e, fwd, back


def open_edges(tris, n_vertices):
    """Directed edges whose reverse no triangle uses, [k, 2]; asserts no directed edge is used twice."""
    e, fwd, back = edge_use(tris, n_vertices)
    assert fwd.max(initial=1) == 1, "a directed edge is used by two triangles"
    return e[back == 0]


def assert_closed(tris, n_vertices):
    """Every directed edge once, and its reverse once."""
    e, fwd, back = edge_use(tris, n_vertices)
    assert fwd.max() == 1 and back.min() == 1 and back.max() == 1


def components(tris, n_vertices):
    from scipy.sparse import coo_matrix
    from scipy.sparse.csgraph import connected_components
    e = directed_edges(tris)
    g = coo_matrix((np.ones(len(e)), (e[:, 0], e[:, 1])), shape=(n_vertices, n_vertices))
    used = np.unique(np.asarray(tris).reshape(-1))
    _, label = connected_components(g, directed=False)
    return len(np.unique(label[used]))


def euler(tris):
    """V - E + F over the referenced vertices and undirected edges."""
    e = np.sort(directed_edges(tris), axis=1)
    V = len(np.unique(np.asarray(tris).reshape(-1)))
    E = len(np.unique(e[:, 0] * (int(e.max()) + 1) + e[:, 1]))
    return V - E + len(tris)


def normals(verts, tris):
    """(b - a) x (c - a) per triangle (float64)."""
    p = np.asarray(verts, np.float64)[:, :3]
    a, b, c = p[tris[:, 0]], p[tris[:, 1]], p[tris[:, 2]]
    return np.cross(b - a, c - a), (a + b + c) / 3


def area_and_volume(verts, tris):
    n, _ = normals(verts, tris)
    p = np.asarray(verts, np.float64)[:, :3]
    vol = np.einsum("ij,ij->i", p[tris[:, 0]], np.cross(p[tris[:, 1]], p[tris[:, 2]])).sum() / 6
    return np.linalg.norm(n, axis=1).sum() / 2, vol


def surface_point_edges(tsdf, weight):
    """(voxel (i, j, k) [n, 3], axis [n]) of every surface point, in surface_points order (numpy, independent)."""
    nz, ny, nx = tsdf.shape
    near = (weight > 0) & (np.abs(tsdf) < 1)
    k, j, i = np.meshgrid(np.arange(nz), np.arange(ny), np.arange(nx), indexing="ij")
    lin = (k * ny + j) * nx + i
    keys = []
    for axis in range(3):
        a, b = [slice(None)] * 3, [slice(None)] * 3
        a[2 - axis], b[2 - axis] = slice(0, -1), slice(1, None)
        ta, tb = tsdf[tuple(a)], tsdf[tuple(b)]
        sel = near[tuple(a)] & near[tuple(b)] & (((ta > 0) & (tb <= 0)) | ((ta <= 0) & (tb > 0)))
        keys.append(lin[tuple(a)][sel].astype(np.int64) * 3 + axis)
    keys = np.sort(np.concatenate(keys))
    v, axis = keys // 3, keys % 3
    return np.stack([v % nx, (v // nx) % ny, v // (nx * ny)], 1), axis


def on_grid_boundary(tsdf, weight, edges):
    """For each mesh edge (two vertex indices): do both vertices lie on one outer face of the grid?"""
    nz, ny, nx = tsdf.shape
    ijk, axis = surface_point_edges(tsdf, weight)
    hi = np.array([nx - 1, ny - 1, nz - 1])
    ok = np.zeros(len(edges), bool)
    for d in range(3):
        for side in (0, 1):
            # a grid edge lies in the face {coordinate d == side ? hi : 0} when it does not run along d
            inface = (axis != d) & (ijk[:, d] == (hi[d] if side else 0))
            ok |= inface[edges[:, 0]] & inface[edges[:, 1]]
    return ok


def sphere_field(dims, s, origin, centre, radius, tau):
    """tsdf = clamp((|p - c| - R) / tau, -1, 1) (float64, then float32), weight 1."""
    nx, ny, nz = dims
    k, j, i = np.meshgrid(np.arange(nz), np.arange(ny), np.arange(nx), indexing="ij")
    o = np.asarray(origin, np.float32)
    x, y, z = (o[0] + i.astype(np.float32) * np.float32(s), o[1] + j.astype(np.float32) * np.float32(s),
               o[2] + k.astype(np.float32) * np.float32(s))
    d = np.sqrt((x - centre[0]) ** 2.0 + (y - centre[1]) ** 2.0 + (z - centre[2]) ** 2.0) - radius
    return np.clip(d / tau, -1, 1).astype(np.float32), np.ones(d.shape, np.float32)


def assert_sphere_mesh(verts, tris, centre, radius, rel=0.01):
    """Closed, one component, genus 0, outward normals, area and volume within `rel` of the sphere's."""
    assert len(tris) > 100
    assert_closed(tris, len(verts))
    assert components(tris, len(verts)) == 1
    assert euler(tris) == 2
    n, mid = normals(verts, tris)
    big = np.linalg.norm(n, axis=1) > 1e-12 * np.abs(n).max()
    assert np.all(np.einsum("ij,ij->i", n[big], mid[big] - np.asarray(centre)) > 0)
    area, vol = area_and_volume(verts, tris)
    assert abs(area / (4 * np.pi * radius ** 2) - 1) < rel, area
    assert abs(vol / (4 / 3 * np.pi * radius ** 3) - 1) < rel, vol
