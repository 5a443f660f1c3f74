"""ctypes binding of oracle/rmd_oracle_volume_shift.c -- the CHECKER of the moving TSDF volume (DESIGN.md 4.8).

Test infrastructure only, like volume_oracle.py.  The spill filters the surface outputs of the volume, intensity and
normals oracles, so the file is compiled together with them (same flags: IEEE fp32, no contraction) into
oracle/librmd_oracle_volume_shift.so, or into a temporary directory when the tree is not writable.
`OracleVolume` is volume_intensity_oracle.OracleVolume (with the normals) that can shift and spill.
"""
from __future__ import annotations

import ctypes
import os
import subprocess
import tempfile

import numpy as np

import volume_intensity_oracle as vio
import volume_normals_oracle as vno

_ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
_SRCS = [os.path.join(_ROOT, "oracle", n) for n in
         ("rmd_oracle_volume_shift.c", "rmd_oracle_volume.c", "rmd_oracle_volume_intensity.c",
          "rmd_oracle_volume_normals.c")]
_CFLAGS = ["-O2", "-std=gnu11", "-fPIC", "-ffp-contract=off", "-fno-fast-math", "-Wall", "-Wextra", "-shared"]

_lib = None

POINTS, INTENSITY, NORMALS = 0, 1, 2


def _build() -> str:
    name = "librmd_oracle_volume_shift.so"
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
    raise RuntimeError("volume_shift_oracle: could not build " + name)


def lib():
    global _lib
    if _lib is None:
        L = ctypes.CDLL(_build())
        vp, ci, cf, cs = ctypes.c_void_p, ctypes.c_int, ctypes.c_float, ctypes.c_size_t
        L.rmd_oracle_volume_shift.argtypes = [vp, vp, vp, vp, ci, ci, ci, vp]
        L.rmd_oracle_volume_shift.restype = None
        L.rmd_oracle_volume_shift_origin.argtypes = [vp, vp, cf, vp]
        L.rmd_oracle_volume_shift_origin.restype = None
        L.rmd_oracle_volume_spill.argtypes = [vp, vp, vp, vp, ci, ci, ci, cf, vp, vp, ci, vp, cs]
        L.rmd_oracle_volume_spill.restype = cs
        _lib = L
    return _lib


def _d(d):
    return np.ascontiguousarray(np.asarray(d, np.int64).astype(np.int32).reshape(3))


def shift_records(a, b, d):
    """(a, b) of shape (nz, ny, nx) shifted by d: a new pair."""
    a, b = (np.ascontiguousarray(x, np.float32) for x in (a, b))
    nz, ny, nx = a.shape
    ao, bo = np.empty_like(a), np.empty_like(b)
    lib().rmd_oracle_volume_shift(a.ctypes.data, b.ctypes.data, ao.ctypes.data, bo.ctypes.data, nx, ny, nz,
                                  _d(d).ctypes.data)
    return ao, bo


def shift_origin(o0, D, s):
    o0 = np.ascontiguousarray(np.asarray(o0, np.float32).reshape(3))
    D = np.ascontiguousarray(np.asarray(D, np.int64).reshape(3))
    out = np.empty(3, np.float32)
    lib().rmd_oracle_volume_shift_origin(o0.ctypes.data, D.ctypes.data, float(np.float32(s)), out.ctypes.data)
    return out


class OracleVolume(vio.OracleVolume):
    """The volume oracle with the intensity channel and normals, and the creation origin o0 and total offset D of a
    moving volume."""

    def __init__(self, dims, voxel_size, origin, truncation, max_weight):
        super().__init__(dims, voxel_size, origin, truncation, max_weight)
        self.o0 = self.origin.copy()
        self.D = np.zeros(3, np.int64)

    surface_normals = vno.OracleVolume.surface_normals

    def shift(self, d):
        d = np.asarray(d, np.int64).reshape(3)
        if not d.any():
            return
        self.tsdf, self.weight = shift_records(self.tsdf, self.weight, d)
        self.cint, self.cw = shift_records(self.cint, self.cw, d)
        self.D = self.D + d
        self.origin = shift_origin(self.o0, self.D, self.s)

    def spill(self, d, kind=POINTS, capacity=None):
        """(spill [min(n, capacity)] + per-point shape, n) of kind POINTS / INTENSITY / NORMALS."""
        args = (self.tsdf.ctypes.data, self.weight.ctypes.data, self.cint.ctypes.data, self.cw.ctypes.data,
                *self.dims, self.s, self.origin.ctypes.data, _d(d).ctypes.data, int(kind))
        if capacity is None:
            capacity = lib().rmd_oracle_volume_spill(*args, None, 0)
        shape = () if kind == INTENSITY else (4,)
        out = np.empty((max(int(capacity), 1),) + shape, np.float32)
        n = lib().rmd_oracle_volume_spill(*args, out.ctypes.data, int(capacity))
        assert n != ctypes.c_size_t(-1).value, "volume_shift_oracle: out of memory"
        return out[:min(int(capacity), n)], int(n)
