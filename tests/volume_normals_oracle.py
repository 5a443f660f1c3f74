"""ctypes binding of oracle/rmd_oracle_volume_normals.c -- the CHECKER of the TSDF volume's normals (DESIGN.md 4.8).

Test infrastructure only, like volume_oracle.py.  The raycast's hits come from the volume oracle, so the file is
compiled together with oracle/rmd_oracle_volume.c (same flags: IEEE fp32, no contraction) into
oracle/librmd_oracle_volume_normals.so, or into a temporary directory when the tree is not writable.
`OracleVolume` is volume_oracle.OracleVolume with the normals.
"""
from __future__ import annotations

import ctypes
import os
import subprocess
import tempfile

import numpy as np

import volume_oracle as vo

_ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
_SRCS = [os.path.join(_ROOT, "oracle", "rmd_oracle_volume_normals.c"),
         os.path.join(_ROOT, "oracle", "rmd_oracle_volume.c")]
_CFLAGS = ["-O2", "-std=gnu11", "-fPIC", "-ffp-contract=off", "-fno-fast-math", "-Wall", "-Wextra", "-shared"]

_lib = None


def _build() -> str:
    name = "librmd_oracle_volume_normals.so"
    newest = max(os.path.getmtime(p) for p in _SRCS)
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
    raise RuntimeError("volume_normals_oracle: could not build " + name)


def lib():
    global _lib
    if _lib is None:
        L = ctypes.CDLL(_build())
        vp, ci, cf, cs = ctypes.c_void_p, ctypes.c_int, ctypes.c_float, ctypes.c_size_t
        L.rmd_oracle_volume_gradients.argtypes = [vp, vp, ci, ci, ci, vp]
        L.rmd_oracle_volume_gradients.restype = None
        L.rmd_oracle_volume_surface_normals.argtypes = [vp, vp, ci, ci, ci, vp, cs]
        L.rmd_oracle_volume_surface_normals.restype = cs
        L.rmd_oracle_volume_raycast_normals.argtypes = [vp, vp, ci, ci, ci, cf, vp, ci, ci, cf, cf, cf, cf, vp, vp,
                                                        vp]
        L.rmd_oracle_volume_raycast_normals.restype = None
        _lib = L
    return _lib


class OracleVolume(vo.OracleVolume):
    """volume_oracle.OracleVolume with the normals of its (tsdf, weight) records."""

    def gradients(self):
        """float32 (nz, ny, nx, 3): every voxel's tsdf gradient."""
        out = np.empty(self.tsdf.shape + (3,), np.float32)
        lib().rmd_oracle_volume_gradients(self.tsdf.ctypes.data, self.weight.ctypes.data, *self.dims,
                                          out.ctypes.data)
        return out

    def surface_normals(self, capacity=None):
        """(normals [min(n, capacity), 4] = (nx, ny, nz, 0), n)."""
        args = (self.tsdf.ctypes.data, self.weight.ctypes.data, *self.dims)
        if capacity is None:
            capacity = lib().rmd_oracle_volume_surface_normals(*args, None, 0)
        out = np.empty((max(int(capacity), 1), 4), np.float32)
        n = lib().rmd_oracle_volume_surface_normals(*args, out.ctypes.data, int(capacity))
        return out[:min(int(capacity), n)], int(n)

    def raycast_normals(self, cam, T_curr_world, width, height):
        """(depth float32 (height, width), normals float32 (height, width, 4))."""
        depth = np.empty((int(height), int(width)), np.float32)
        normals = np.empty((int(height), int(width), 4), np.float32)
        T = vo._pose(T_curr_world)
        lib().rmd_oracle_volume_raycast_normals(
            self.tsdf.ctypes.data, self.weight.ctypes.data, *self.dims, self.s, self.origin.ctypes.data, int(width),
            int(height), *(float(np.float32(v)) for v in cam), T.ctypes.data, depth.ctypes.data,
            normals.ctypes.data)
        return depth, normals
