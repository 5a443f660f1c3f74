"""ctypes binding of oracle/rmd_oracle_mesh.c -- the CHECKER of the TSDF volume's triangle mesh (DESIGN.md 4.8).

Test infrastructure only, like volume_oracle.py.  The mesh's vertices are the volume oracle's surface points, so
the file is compiled together with oracle/rmd_oracle_volume.c (same flags: IEEE fp32, no contraction) into
oracle/librmd_oracle_mesh.so, or into a temporary directory when the tree is not writable.  `OracleVolume` is
volume_oracle.OracleVolume with a `mesh()` method; `mesh(o)` meshes any volume_oracle.OracleVolume.
"""
from __future__ import annotations

import ctypes
import os
import subprocess
import tempfile

import numpy as np

import volume_oracle as vo

_ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
_SRCS = [os.path.join(_ROOT, "oracle", "rmd_oracle_mesh.c"), os.path.join(_ROOT, "oracle", "rmd_oracle_volume.c")]
_TABLE = os.path.join(_ROOT, "rpg_open_remode_b200", "csrc", "mc_table.h")   # included by rmd_oracle_mesh.c
_CFLAGS = ["-O2", "-std=gnu11", "-fPIC", "-ffp-contract=off", "-fno-fast-math", "-Wall", "-Wextra", "-shared"]

_lib = None


def _build() -> str:
    name = "librmd_oracle_mesh.so"
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
    raise RuntimeError("mesh_oracle: could not build " + name)


def lib():
    global _lib
    if _lib is None:
        L = ctypes.CDLL(_build())
        vp, ci, cf, cs = ctypes.c_void_p, ctypes.c_int, ctypes.c_float, ctypes.c_size_t
        L.rmd_oracle_volume_mesh.argtypes = [vp, vp, ci, ci, ci, cf, vp, vp, cs, vp, cs, ctypes.POINTER(cs)]
        L.rmd_oracle_volume_mesh.restype = cs
        _lib = L
    return _lib


def mesh(o):
    """(vertices float32 [n, 4] = o.surface_points(), triangles int32 [m, 3]) of a volume_oracle.OracleVolume."""
    args = (o.tsdf.ctypes.data, o.weight.ctypes.data, *o.dims, o.s, o.origin.ctypes.data)
    nv = ctypes.c_size_t()
    m = lib().rmd_oracle_volume_mesh(*args, None, 0, None, 0, ctypes.byref(nv))
    verts = np.empty((max(nv.value, 1), 4), np.float32)
    tris = np.empty((max(m, 1), 3), np.int32)
    m = lib().rmd_oracle_volume_mesh(*args, verts.ctypes.data, nv.value, tris.ctypes.data, m, ctypes.byref(nv))
    return verts[:nv.value], tris[:m]


class OracleVolume(vo.OracleVolume):
    """volume_oracle.OracleVolume that also meshes."""

    def mesh(self):
        return mesh(self)
