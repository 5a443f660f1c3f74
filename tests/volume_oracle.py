"""ctypes binding of oracle/rmd_oracle_volume.c -- the CHECKER of the TSDF volume (DESIGN.md 4.8).

Test infrastructure only, like oracle_binding.py.  The file is compiled on its own (same flags as the rest of the
CPU oracle: IEEE fp32, no contraction) into oracle/librmd_oracle_volume.so, or into a temporary directory when the
tree is not writable.
"""
from __future__ import annotations

import ctypes
import os
import subprocess
import tempfile

import numpy as np

_ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
_SRC = os.path.join(_ROOT, "oracle", "rmd_oracle_volume.c")
_CFLAGS = ["-O2", "-std=gnu11", "-fPIC", "-ffp-contract=off", "-fno-fast-math", "-Wall", "-Wextra", "-shared"]

_lib = None


def _build() -> str:
    name = "librmd_oracle_volume.so"
    for d in (os.path.dirname(_SRC), os.path.join(tempfile.gettempdir(), "rmd_oracle_%d" % os.getuid())):
        path = os.path.join(d, name)
        if os.path.exists(path) and os.path.getmtime(path) >= os.path.getmtime(_SRC):
            return path
        try:
            os.makedirs(d, exist_ok=True)
            tmp = "%s.%d.tmp" % (path, os.getpid())
            cc = "/usr/bin/gcc" if os.path.exists("/usr/bin/gcc") else "gcc"
            subprocess.check_call([cc] + _CFLAGS + ["-o", tmp, _SRC, "-lm"])
            os.replace(tmp, path)
            return path
        except (OSError, subprocess.CalledProcessError):
            continue
    raise RuntimeError("volume_oracle: could not build " + name)


def lib():
    global _lib
    if _lib is None:
        L = ctypes.CDLL(_build())
        vp, ci, cf, cs = ctypes.c_void_p, ctypes.c_int, ctypes.c_float, ctypes.c_size_t
        L.rmd_oracle_pose_inverse.argtypes = [vp, vp]
        L.rmd_oracle_pose_inverse.restype = None
        L.rmd_oracle_volume_integrate.argtypes = [vp, vp, ci, ci, ci, cf, vp, ci, ci, cf, cf, cf, cf, vp, vp, vp,
                                                  cf, cf]
        L.rmd_oracle_volume_integrate.restype = cs
        L.rmd_oracle_volume_surface.argtypes = [vp, vp, ci, ci, ci, cf, vp, vp, cs]
        L.rmd_oracle_volume_surface.restype = cs
        L.rmd_oracle_volume_raycast.argtypes = [vp, vp, ci, ci, ci, cf, vp, ci, ci, cf, cf, cf, cf, vp, vp]
        L.rmd_oracle_volume_raycast.restype = None
        _lib = L
    return _lib


def _pose(T):
    return np.ascontiguousarray(np.asarray(T, np.float32).reshape(-1)[:12])


class OracleVolume:
    """The volume's state as two float32 arrays of shape (nz, ny, nx)."""

    def __init__(self, dims, voxel_size, origin, truncation, max_weight):
        nx, ny, nz = (int(n) for n in dims)
        self.dims = (nx, ny, nz)
        self.s = float(np.float32(voxel_size))
        self.origin = np.ascontiguousarray(np.asarray(origin, np.float32).reshape(3))
        self.trunc, self.max_weight = float(np.float32(truncation)), float(np.float32(max_weight))
        self.tsdf = np.zeros((nz, ny, nx), np.float32)
        self.weight = np.zeros((nz, ny, nx), np.float32)

    def integrate(self, depth, cam, T_curr_world, conv=None) -> int:
        """depth: (h, w) float32 distance along the ray; conv: optional int32 states.  Returns updated voxels."""
        d = np.ascontiguousarray(depth, np.float32)
        h, w = d.shape
        c = np.ascontiguousarray(conv, np.int32) if conv is not None else None
        T = _pose(T_curr_world)
        return int(lib().rmd_oracle_volume_integrate(
            self.tsdf.ctypes.data, self.weight.ctypes.data, *self.dims, self.s, self.origin.ctypes.data, w, h,
            *(float(np.float32(v)) for v in cam), T.ctypes.data, d.ctypes.data,
            c.ctypes.data if c is not None else None, self.trunc, self.max_weight))

    def surface_points(self, capacity=None):
        """(points [min(n, capacity), 4], n)."""
        if capacity is None:
            n = lib().rmd_oracle_volume_surface(self.tsdf.ctypes.data, self.weight.ctypes.data, *self.dims, self.s,
                                                self.origin.ctypes.data, None, 0)
            capacity = n
        out = np.empty((max(int(capacity), 1), 4), np.float32)
        n = lib().rmd_oracle_volume_surface(self.tsdf.ctypes.data, self.weight.ctypes.data, *self.dims, self.s,
                                            self.origin.ctypes.data, out.ctypes.data, int(capacity))
        return out[:min(int(capacity), n)], int(n)

    def raycast(self, cam, T_curr_world, width, height):
        out = np.empty((int(height), int(width)), np.float32)
        T = _pose(T_curr_world)
        lib().rmd_oracle_volume_raycast(self.tsdf.ctypes.data, self.weight.ctypes.data, *self.dims, self.s,
                                        self.origin.ctypes.data, int(width), int(height),
                                        *(float(np.float32(v)) for v in cam), T.ctypes.data, out.ctypes.data)
        return out


def pose_inverse(T):
    a, out = _pose(T), np.empty(12, np.float32)
    lib().rmd_oracle_pose_inverse(a.ctypes.data, out.ctypes.data)
    return out.reshape(3, 4)
