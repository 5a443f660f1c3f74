"""The records and origin of an ESDF box (DESIGN.md 4.8) -- the CHECKER of rmd_volume_esdf_box, with
volume_esdf_oracle.esdf / .query run on what this returns.

Test infrastructure only.  Box voxel (i, j, k) is voxel u = lo_u + (i, j, k) of the unbounded grid (lo_u = D + lo):
the window's record when u lies in [D, D + n), else the stored brick's when brick floor(u / 8) is stored, else (0, 0).
"""
from __future__ import annotations

import numpy as np

import volume_shift_oracle as vso

B = 8


def box_records(lo_u, dims, D, tsdf, weight, bricks=None):
    """(tsdf, weight) float32 (mz, my, mx) of the box [lo_u, lo_u + dims) of the unbounded grid.  tsdf, weight: the
    window's records (nz, ny, nx) at offset D; bricks: {(bx, by, bz): (tsdf, weight) (8, 8, 8)} or None.  The bricks
    are pasted first and the window over them, so a stale stored copy of a window voxel is never read."""
    lo_u, m, D = (np.asarray(x, np.int64).reshape(3) for x in (lo_u, dims, D))
    n = np.array(tsdf.shape[::-1], np.int64)
    t, w = np.zeros(m[::-1], np.float32), np.zeros(m[::-1], np.float32)

    def paste(src_t, src_w, src_lo, size):
        a = np.maximum(src_lo, lo_u)
        b = np.minimum(src_lo + size, lo_u + m)
        if np.any(a >= b):
            return
        s, d = a - src_lo, a - lo_u
        e = b - a
        t[d[2]:d[2] + e[2], d[1]:d[1] + e[1], d[0]:d[0] + e[0]] = src_t[s[2]:s[2] + e[2], s[1]:s[1] + e[1],
                                                                         s[0]:s[0] + e[0]]
        w[d[2]:d[2] + e[2], d[1]:d[1] + e[1], d[0]:d[0] + e[0]] = src_w[s[2]:s[2] + e[2], s[1]:s[1] + e[1],
                                                                         s[0]:s[0] + e[0]]

    for c, (bt, bw) in (bricks or {}).items():
        paste(bt, bw, np.asarray(c, np.int64) * B, np.full(3, B, np.int64))
    paste(tsdf, weight, D, n)
    return t, w


def model_bricks(model):
    """StoreModel's bricks as box_records wants them (stale copies of window voxels included)."""
    return {c: (r[0], r[1]) for c, r in model.bricks.items()}


def downloaded_bricks(coords, tsdf, weight):
    """api.TsdfVolume.downloadStore()'s bricks as box_records wants them."""
    return {tuple(int(x) for x in c): (a, b) for c, a, b in zip(coords, tsdf, weight)}


def box_records_brute(lo_u, dims, D, tsdf, weight, bricks=None):
    """box_records, one voxel at a time by the definition."""
    lo_u, m, D = (np.asarray(x, np.int64).reshape(3) for x in (lo_u, dims, D))
    n = np.array(tsdf.shape[::-1], np.int64)
    t, w = np.zeros(m[::-1], np.float32), np.zeros(m[::-1], np.float32)
    for k in range(m[2]):
        for j in range(m[1]):
            for i in range(m[0]):
                u = lo_u + (i, j, k)
                x = u - D
                if np.all(x >= 0) and np.all(x < n):
                    t[k, j, i], w[k, j, i] = tsdf[x[2], x[1], x[0]], weight[x[2], x[1], x[0]]
                    continue
                b = tuple(int(c) for c in u // B)
                if bricks and b in bricks:
                    loc = u - np.asarray(b, np.int64) * B
                    t[k, j, i] = bricks[b][0][loc[2], loc[1], loc[0]]
                    w[k, j, i] = bricks[b][1][loc[2], loc[1], loc[0]]
    return t, w


def box_origin(o0, lo_u, s):
    """The box's origin o0 + (float)(lo_u) * s per axis, rmd_volume_shift's rule (the shift oracle's)."""
    return vso.shift_origin(o0, lo_u, s)
