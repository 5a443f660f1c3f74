"""ctypes binding of oracle/rmd_oracle_volume_esdf.c -- the CHECKER of the TSDF volume's Euclidean signed distance
field (DESIGN.md 4.8).

Test infrastructure only, like volume_shift_oracle.py: compiled (IEEE fp32, no contraction) into
oracle/librmd_oracle_volume_esdf.so, or into a temporary directory when the tree is not writable.
"""
from __future__ import annotations

import ctypes
import os
import subprocess
import tempfile

import numpy as np

_ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
_SRCS = [os.path.join(_ROOT, "oracle", "rmd_oracle_volume_esdf.c")]
_CFLAGS = ["-O2", "-std=gnu11", "-fPIC", "-ffp-contract=off", "-fno-fast-math", "-Wall", "-Wextra", "-shared"]

_lib = None


def _build() -> str:
    name = "librmd_oracle_volume_esdf.so"
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
    raise RuntimeError("volume_esdf_oracle: could not build " + name)


def lib():
    global _lib
    if _lib is None:
        L = ctypes.CDLL(_build())
        vp, ci, cf, cs = ctypes.c_void_p, ctypes.c_int, ctypes.c_float, ctypes.c_size_t
        L.rmd_oracle_volume_esdf.argtypes = [vp, vp, ci, ci, ci, cf, vp, vp]
        L.rmd_oracle_volume_esdf.restype = ci
        L.rmd_oracle_volume_esdf_query.argtypes = [vp, vp, ci, ci, ci, cf, vp, vp, cs, vp, vp]
        L.rmd_oracle_volume_esdf_query.restype = None
        _lib = L
    return _lib


def esdf(tsdf, weight, s):
    """(distance, weight) of the snapshot of records (tsdf, weight) of shape (nz, ny, nx) with voxel size s."""
    t, w = (np.ascontiguousarray(x, np.float32) for x in (tsdf, weight))
    nz, ny, nx = t.shape
    dist, wout = np.empty_like(t), np.empty_like(w)
    rc = lib().rmd_oracle_volume_esdf(t.ctypes.data, w.ctypes.data, nx, ny, nz, float(np.float32(s)),
                                      dist.ctypes.data, wout.ctypes.data)
    if rc == -2:
        raise ValueError("volume_esdf_oracle: grid past the size limit")
    assert rc == 0, "volume_esdf_oracle: out of memory"
    return dist, wout


def query(dist, weight, s, origin, points):
    """(dg [N, 4], weight [N]) at points [N, 3] or [N, 4] on a snapshot (distance, weight) computed at origin."""
    d, w = (np.ascontiguousarray(x, np.float32) for x in (dist, weight))
    nz, ny, nx = d.shape
    p = np.asarray(points, np.float32)
    xyzw = np.zeros((len(p), 4), np.float32)
    xyzw[:, :p.shape[1]] = p
    o = np.ascontiguousarray(np.asarray(origin, np.float32).reshape(3))
    dg, wq = np.empty((len(p), 4), np.float32), np.empty(len(p), np.float32)
    lib().rmd_oracle_volume_esdf_query(d.ctypes.data, w.ctypes.data, nx, ny, nz, float(np.float32(s)), o.ctypes.data,
                                       xyzw.ctypes.data, len(p), dg.ctypes.data, wq.ctypes.data)
    return dg, wq


def occupied(tsdf, weight):
    return (weight > 0) & (tsdf <= 0)


def adversarial_grids(rng):
    """Named (tsdf, weight) grids that stress the definition: ragged sizes, nx = 1, a single site, empty O, empty F, all
    unknown, a checkerboard, -0.0 and NaN tsdf."""
    out = []
    for shape in ((7, 5, 9), (13, 1, 6), (5, 11, 1), (1, 1, 17)):
        t = rng.uniform(-1, 1, shape).astype(np.float32)
        w = np.where(rng.random(shape) < 0.7, rng.integers(1, 5, shape), 0).astype(np.float32)
        t[rng.random(shape) < 0.6] = 1.0
        out.append((f"random {shape}", t, w))
    shape = (9, 8, 10)
    t, w = np.ones(shape, np.float32), np.ones(shape, np.float32)
    t[4, 2, 7] = -0.5
    out.append(("single site", t, w.copy()))
    out.append(("empty O", np.ones(shape, np.float32), np.ones(shape, np.float32)))
    out.append(("empty F", -np.ones(shape, np.float32), np.ones(shape, np.float32)))
    out.append(("all unknown", -np.ones(shape, np.float32), np.zeros(shape, np.float32)))
    k, j, i = np.indices(shape)
    out.append(("checkerboard", np.where((i + j + k) % 2 == 0, -1.0, 1.0).astype(np.float32),
                np.ones(shape, np.float32)))
    t = np.ones(shape, np.float32)
    t[1, 1, 1], t[7, 6, 8], t[3, 3, 3] = -0.0, np.nan, 0.0
    out.append(("-0.0 and NaN", t, np.ones(shape, np.float32)))
    return out
