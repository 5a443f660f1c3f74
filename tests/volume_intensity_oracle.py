"""ctypes binding of oracle/rmd_oracle_volume_intensity.c -- the CHECKER of the TSDF volume's intensity channel
(DESIGN.md 4.8).

Test infrastructure only, like volume_oracle.py.  The raycast's hits come from the volume oracle, so the file is
compiled together with oracle/rmd_oracle_volume.c (same flags: IEEE fp32, no contraction) into
oracle/librmd_oracle_volume_intensity.so, or into a temporary directory when the tree is not writable.
`OracleVolume` is volume_oracle.OracleVolume with the intensity records (cint, cw) next to (tsdf, weight).
"""
from __future__ import annotations

import ctypes
import os
import subprocess
import tempfile

import numpy as np

import volume_oracle as vo

_ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
_SRCS = [os.path.join(_ROOT, "oracle", "rmd_oracle_volume_intensity.c"),
         os.path.join(_ROOT, "oracle", "rmd_oracle_volume.c")]
_CFLAGS = ["-O2", "-std=gnu11", "-fPIC", "-ffp-contract=off", "-fno-fast-math", "-Wall", "-Wextra", "-shared"]

_lib = None


def _build() -> str:
    name = "librmd_oracle_volume_intensity.so"
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
    raise RuntimeError("volume_intensity_oracle: could not build " + name)


def lib():
    global _lib
    if _lib is None:
        L = ctypes.CDLL(_build())
        vp, ci, cf, cs = ctypes.c_void_p, ctypes.c_int, ctypes.c_float, ctypes.c_size_t
        L.rmd_oracle_volume_integrate_intensity.argtypes = [vp, vp, ci, ci, ci, cf, vp, ci, ci, cf, cf, cf, cf, vp,
                                                            vp, vp, vp, cf, cf]
        L.rmd_oracle_volume_integrate_intensity.restype = cs
        L.rmd_oracle_volume_surface_intensity.argtypes = [vp, vp, vp, vp, ci, ci, ci, vp, cs]
        L.rmd_oracle_volume_surface_intensity.restype = cs
        L.rmd_oracle_volume_raycast_intensity.argtypes = [vp, vp, vp, vp, ci, ci, ci, cf, vp, ci, ci, cf, cf, cf, cf,
                                                          vp, vp, vp]
        L.rmd_oracle_volume_raycast_intensity.restype = None
        _lib = L
    return _lib


class OracleVolume(vo.OracleVolume):
    """volume_oracle.OracleVolume with the intensity channel: cint, cw of shape (nz, ny, nx)."""

    def __init__(self, dims, voxel_size, origin, truncation, max_weight):
        super().__init__(dims, voxel_size, origin, truncation, max_weight)
        self.cint = np.zeros_like(self.tsdf)
        self.cw = np.zeros_like(self.weight)

    def integrate(self, depth, cam, T_curr_world, conv=None, intensity=None) -> int:
        """The tsdf (volume_oracle) and, with an intensity image, the intensity channel.  Returns the number of
        updated (tsdf, weight) records."""
        n = super().integrate(depth, cam, T_curr_world, conv)
        if intensity is not None:
            self.integrate_intensity_only(depth, cam, T_curr_world, conv, intensity)
        return n

    def integrate_intensity_only(self, depth, cam, T_curr_world, conv, intensity) -> int:
        """The intensity half of an integration; returns the number of updated intensity records."""
        d = np.ascontiguousarray(depth, np.float32)
        h, w = d.shape
        c = np.ascontiguousarray(conv, np.int32) if conv is not None else None
        i = np.ascontiguousarray(intensity, np.float32)
        assert i.shape == d.shape
        T = vo._pose(T_curr_world)
        return int(lib().rmd_oracle_volume_integrate_intensity(
            self.cint.ctypes.data, self.cw.ctypes.data, *self.dims, self.s, self.origin.ctypes.data, w, h,
            *(float(np.float32(v)) for v in cam), T.ctypes.data, d.ctypes.data,
            c.ctypes.data if c is not None else None, i.ctypes.data, self.trunc, self.max_weight))

    def surface_intensity(self, capacity=None):
        """(intensity [min(n, capacity)], n)."""
        args = (self.tsdf.ctypes.data, self.weight.ctypes.data, self.cint.ctypes.data, self.cw.ctypes.data,
                *self.dims)
        if capacity is None:
            capacity = lib().rmd_oracle_volume_surface_intensity(*args, None, 0)
        out = np.empty(max(int(capacity), 1), np.float32)
        n = lib().rmd_oracle_volume_surface_intensity(*args, out.ctypes.data, int(capacity))
        return out[:min(int(capacity), n)], int(n)

    def raycast_intensity(self, cam, T_curr_world, width, height):
        """(depth, intensity), float32 (height, width) each."""
        depth = np.empty((int(height), int(width)), np.float32)
        inten = np.empty_like(depth)
        T = vo._pose(T_curr_world)
        lib().rmd_oracle_volume_raycast_intensity(
            self.tsdf.ctypes.data, self.weight.ctypes.data, self.cint.ctypes.data, self.cw.ctypes.data, *self.dims,
            self.s, self.origin.ctypes.data, int(width), int(height), *(float(np.float32(v)) for v in cam),
            T.ctypes.data, depth.ctypes.data, inten.ctypes.data)
        return depth, inten
