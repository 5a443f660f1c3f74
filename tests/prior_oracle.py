"""ctypes binding of oracle/rmd_oracle_propagate.c -- the CHECKER of the keyframe depth prior (DESIGN.md 4.7).

Test infrastructure only, like oracle_binding.py.  The file is compiled on its own (same flags as the rest of the
CPU oracle: IEEE fp32, no contraction) into oracle/librmd_oracle_propagate.so, or into a temporary directory when
the tree is not writable.
"""
from __future__ import annotations

import ctypes
import os
import subprocess
import tempfile

import numpy as np

_ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
_SRC = os.path.join(_ROOT, "oracle", "rmd_oracle_propagate.c")
_CFLAGS = ["-O2", "-std=gnu11", "-fPIC", "-ffp-contract=off", "-fno-fast-math", "-Wall", "-Wextra", "-shared"]
EMPTY = np.uint32(0xFFFFFFFF)

_lib = None


def _build() -> str:
    name = "librmd_oracle_propagate.so"
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
    raise RuntimeError("prior_oracle: could not build " + name)


def lib():
    global _lib
    if _lib is None:
        L = ctypes.CDLL(_build())
        vp, ci, cf, cs = ctypes.c_void_p, ctypes.c_int, ctypes.c_float, ctypes.c_size_t
        L.rmd_oracle_prior_splat.argtypes = [vp, vp, ci, ci, cf, cf, cf, cf, vp, ci, ci, cf, cf, cf, cf, vp, cf, cf, vp]
        L.rmd_oracle_prior_splat.restype = cs
        L.rmd_oracle_prior_apply.argtypes = [vp, ci, ci, ci, cf, cf, cf, vp, vp, vp, vp, vp]
        L.rmd_oracle_prior_apply.restype = None
        _lib = L
    return _lib


def _pose(T):
    return np.ascontiguousarray(np.asarray(T, np.float32).reshape(-1)[:12])


def prior_splat(src_mu, src_conv, src_cam, T_world_ref_src, dst_size, dst_cam, T_curr_world_dst, min_depth, max_depth):
    """uint32 [dh, dw] z-buffer (bit patterns of the nearest distance, 0xFFFFFFFF = empty), accepted points."""
    mu = np.ascontiguousarray(src_mu, np.float32)
    conv = np.ascontiguousarray(src_conv, np.int32)
    sh, sw = mu.shape
    dw, dh = dst_size
    A, B = _pose(T_world_ref_src), _pose(T_curr_world_dst)
    z = np.empty((dh, dw), np.uint32)
    n = lib().rmd_oracle_prior_splat(mu.ctypes.data, conv.ctypes.data, sw, sh, *src_cam, A.ctypes.data, dw, dh,
                                     *dst_cam, B.ctypes.data, min_depth, max_depth, z.ctypes.data)
    return z, int(n)


def prior_apply(zbuf, patch, min_depth, max_depth, sigma_sq_frac):
    """The new keyframe's (mu, sigma_sq, a, b, convergence) after initialisation and the prior."""
    z = np.ascontiguousarray(zbuf, np.uint32)
    dh, dw = z.shape
    mu, s2, a, b = (np.empty((dh, dw), np.float32) for _ in range(4))
    conv = np.empty((dh, dw), np.int32)
    lib().rmd_oracle_prior_apply(z.ctypes.data, dw, dh, patch, min_depth, max_depth, sigma_sq_frac, mu.ctypes.data,
                                 s2.ctypes.data, a.ctypes.data, b.ctypes.data, conv.ctypes.data)
    return mu, s2, a, b, conv


def propagate_prior(src_mu, src_conv, src_cam, T_world_ref_src, dst_size, dst_cam, T_curr_world_dst, patch,
                    min_depth, max_depth, sigma_sq_frac):
    """Splat + initialise + apply: the destination's (mu, sigma_sq, a, b, convergence)."""
    z, _ = prior_splat(src_mu, src_conv, src_cam, T_world_ref_src, dst_size, dst_cam, T_curr_world_dst, min_depth,
                       max_depth)
    return prior_apply(z, patch, min_depth, max_depth, sigma_sq_frac)
