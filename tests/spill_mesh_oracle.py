"""ctypes binding of oracle/rmd_oracle_volume_spill_mesh.c -- the CHECKER of the spill mesh of a moving TSDF volume
(DESIGN.md 4.8).

Test infrastructure only, like volume_oracle.py.  The spill mesh filters the outputs of the mesh, volume, intensity and
normals oracles, so the file is compiled together with them and the shift oracle (same flags: IEEE fp32, no
contraction) into oracle/librmd_oracle_volume_spill_mesh.so, or into a temporary directory when the tree is not
writable.  `OracleVolume` is volume_shift_oracle.OracleVolume that also meshes and spills meshes, with the method
names of api.TsdfVolume that api.SceneMesh calls, so that the welder runs on it unchanged.
"""
from __future__ import annotations

import ctypes
import os
import subprocess
import tempfile

import numpy as np

import mesh_oracle
import volume_shift_oracle as vso

_ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
_SRCS = [os.path.join(_ROOT, "oracle", n) for n in
         ("rmd_oracle_volume_spill_mesh.c", "rmd_oracle_volume.c", "rmd_oracle_volume_intensity.c",
          "rmd_oracle_volume_normals.c", "rmd_oracle_mesh.c", "rmd_oracle_volume_shift.c")]
_TABLE = os.path.join(_ROOT, "rpg_open_remode_b200", "csrc", "mc_table.h")
_CFLAGS = ["-O2", "-std=gnu11", "-fPIC", "-ffp-contract=off", "-fno-fast-math", "-Wall", "-Wextra", "-shared"]

_lib = None

POINTS, INTENSITY, NORMALS = vso.POINTS, vso.INTENSITY, vso.NORMALS


def _build() -> str:
    name = "librmd_oracle_volume_spill_mesh.so"
    newest = max(os.path.getmtime(p) for p in _SRCS + [_TABLE])
    for d in (os.path.dirname(_SRCS[0]), os.path.join(tempfile.gettempdir(), "rmd_oracle_%d" % os.getuid())):
        path = os.path.join(d, name)
        if os.path.exists(path) and os.path.getmtime(path) >= newest:
            return path
        try:
            os.makedirs(d, exist_ok=True)
            tmp = "%s.%d.tmp" % (path, os.getpid())
            cc = "/usr/bin/gcc" if os.path.exists("/usr/bin/gcc") else "gcc"
            subprocess.check_call([cc] + _CFLAGS + ["-o", tmp] + _SRCS + ["-lm"])
            os.replace(tmp, path)
            return path
        except (OSError, subprocess.CalledProcessError):
            continue
    raise RuntimeError("spill_mesh_oracle: could not build " + name)


def lib():
    global _lib
    if _lib is None:
        L = ctypes.CDLL(_build())
        vp, ci, cf, cs = ctypes.c_void_p, ctypes.c_int, ctypes.c_float, ctypes.c_size_t
        L.rmd_oracle_volume_spill_mesh.argtypes = [vp, vp, vp, vp, ci, ci, ci, cf, vp, vp, ci, vp, cs, vp, cs, vp,
                                                   ctypes.POINTER(cs)]
        L.rmd_oracle_volume_spill_mesh.restype = cs
        _lib = L
    return _lib


def keys_to_ids(keys, dims, D):
    """int64 [n, 4] ids (i + D0, j + D1, k + D2, axis) of keys 3 * voxel + axis."""
    keys = np.asarray(keys, np.int64)
    nx, ny, _ = dims
    vox = keys // 3
    ids = np.stack([vox % nx, (vox // nx) % ny, vox // (nx * ny), keys - 3 * vox], 1)
    ids[:, :3] += np.asarray(D, np.int64)
    return ids


class OracleVolume(vso.OracleVolume):
    """The moving-volume oracle that also meshes and spills meshes."""

    def spill_mesh(self, d, kind=POINTS, vertex_capacity=None, tri_capacity=None):
        """(vertex values [min(nv, cap)] + per-vertex shape, triangles int32 [min(nt, cap), 3], keys int64, nv, nt)."""
        d = np.ascontiguousarray(np.asarray(d, np.int64).astype(np.int32).reshape(3))
        args = (self.tsdf.ctypes.data, self.weight.ctypes.data, self.cint.ctypes.data, self.cw.ctypes.data,
                *self.dims, self.s, self.origin.ctypes.data, d.ctypes.data, int(kind))
        nv = ctypes.c_size_t()
        if vertex_capacity is None or tri_capacity is None:
            nt = lib().rmd_oracle_volume_spill_mesh(*args, None, 0, None, 0, None, ctypes.byref(nv))
            assert nt != ctypes.c_size_t(-1).value, "spill_mesh_oracle: failed"
            vertex_capacity = nv.value if vertex_capacity is None else vertex_capacity
            tri_capacity = nt if tri_capacity is None else tri_capacity
        per = () if kind == INTENSITY else (4,)
        vals = np.empty((max(int(vertex_capacity), 1),) + per, np.float32)
        keys = np.empty(max(int(vertex_capacity), 1), np.int64)
        tris = np.empty((max(int(tri_capacity), 1), 3), np.int32)
        nt = lib().rmd_oracle_volume_spill_mesh(*args, vals.ctypes.data, int(vertex_capacity), tris.ctypes.data,
                                                int(tri_capacity), keys.ctypes.data, ctypes.byref(nv))
        assert nt != ctypes.c_size_t(-1).value, "spill_mesh_oracle: failed"
        m = min(int(vertex_capacity), nv.value)
        return vals[:m], tris[:min(int(tri_capacity), nt)], keys[:m], nv.value, int(nt)

    # ------------------------------------------------ api.TsdfVolume's names, as api.SceneMesh calls them
    @property
    def offset(self):
        return self.D.copy()

    def spillMesh(self, d):
        verts, tris, keys, _, _ = self.spill_mesh(d, POINTS)
        return verts, tris, keys_to_ids(keys, self.dims, self.D)

    def spillMeshIntensity(self, d):
        return self.spill_mesh(d, INTENSITY)[0]

    def spillMeshNormals(self, d):
        return np.ascontiguousarray(self.spill_mesh(d, NORMALS)[0][:, :3])

    def mesh(self):
        return mesh_oracle.mesh(self)

    def surfaceIds(self):
        """The ids of the surface points: the spill mesh of a shift that drops everything has them all."""
        return keys_to_ids(self.spill_mesh((self.dims[0], 0, 0), POINTS)[2], self.dims, self.D)

    def surfaceIntensity(self):
        return self.surface_intensity()[0]

    def surfaceNormals(self):
        return np.ascontiguousarray(self.surface_normals()[0][:, :3])
