"""A numpy model of a TSDF volume with the brick store (DESIGN.md 4.8) -- the CHECKER of rmd_volume_shift with the
store, rmd_volume_download_store and api.TsdfVolume.mapMesh.

Test infrastructure only.  The map is the window (the moving-volume oracle's records, integrated by the C oracle with
the window's origin) plus a dict of 8 x 8 x 8 bricks for the voxels outside it.  A shift first moves the leaving
voxels into the dict by the eviction rule, then shifts the window with the shift oracle, then takes every entering
voxel from the dict.  `StoreModel` has api.TsdfVolume's method names for what mapMesh calls, so that
api.TsdfVolume.mapMesh runs on it unchanged.
"""
from __future__ import annotations

import numpy as np

import spill_mesh_oracle as smo

B = 8


def kept_box(dims, d):
    """(lo, hi) int64 [3] of the box a shift by d keeps, in pre-shift window indices (x, y, z)."""
    n = np.asarray(dims, np.int64)
    c = np.clip(np.asarray(d, np.int64), -n, n)
    return np.maximum(c, 0), np.where(c < 0, n + c, n)


def moving(dims, lo, hi):
    """bool (nz, ny, nx): the window voxels outside [lo, hi)."""
    nx, ny, nz = dims
    ins = [(np.arange(m) >= lo[a]) & (np.arange(m) < hi[a]) for a, m in enumerate((nx, ny, nz))]
    return ~(ins[2][:, None, None] & ins[1][None, :, None] & ins[0][None, None, :])


def _bricks_of(mask, D):
    """For the voxels of mask: (unique brick coords [m, 3] (x, y, z) in ascending (z, y, x), brick index per voxel,
    local (lz, ly, lx), window (k, j, i))."""
    k, j, i = np.nonzero(mask)
    u = np.stack([i, j, k], 1).astype(np.int64) + np.asarray(D, np.int64)
    b, l = u // B, u % B
    if not len(b):
        return np.empty((0, 3), np.int64), np.empty(0, np.int64), (l[:, 2], l[:, 1], l[:, 0]), (k, j, i)
    lo = b.min(0)
    span = b.max(0) - lo + 1
    key = ((b[:, 2] - lo[2]) * span[1] + (b[:, 1] - lo[1])) * span[0] + (b[:, 0] - lo[0])   # ascending (z, y, x)
    uk, inv = np.unique(key, return_inverse=True)
    coords = np.stack([uk % span[0], (uk // span[0]) % span[1], uk // (span[0] * span[1])], 1) + lo
    return coords, inv.reshape(-1), (l[:, 2], l[:, 1], l[:, 0]), (k, j, i)


class StoreModel(smo.OracleVolume):
    """The moving-volume oracle (with mesh, spill mesh, intensity and normals) plus the brick store."""

    store = True

    def __init__(self, dims, voxel_size, origin, truncation, max_weight):
        super().__init__(dims, voxel_size, origin, truncation, max_weight)
        self.bricks = {}            # (bx, by, bz) -> float32 [4, 8, 8, 8]: tsdf, weight, intensity, intensity weight
        self.restored = 0           # known voxels (weight > 0) the last shift took from the store

    def _channels(self):
        return (self.tsdf, self.weight, self.cint, self.cw)

    def shift(self, d):
        d = np.asarray(d, np.int64).reshape(3)
        if not d.any():
            return
        # eviction: the leaving voxels of every brick that has one
        lo, hi = kept_box(self.dims, d)
        coords, inv, (lz, ly, lx), (k, j, i) = _bricks_of(moving(self.dims, lo, hi), self.D)
        known = np.array([tuple(c) in self.bricks for c in coords.tolist()], bool)
        seen = np.bincount(inv, weights=(self.weight[k, j, i] > 0), minlength=len(coords)) > 0
        rec = np.zeros((len(coords), 4, B, B, B), np.float32)
        for q in np.nonzero(known)[0]:
            rec[q] = self.bricks[tuple(coords[q].tolist())]
        for c, ch in enumerate(self._channels()):
            rec[inv, c, lz, ly, lx] = ch[k, j, i]
        for q in np.nonzero(known | seen)[0]:
            self.bricks[tuple(coords[q].tolist())] = rec[q]
        # the gather, then the entering voxels from the store
        super().shift(d)
        lo, hi = kept_box(self.dims, -d)
        coords, inv, (lz, ly, lx), (k, j, i) = _bricks_of(moving(self.dims, lo, hi), self.D)
        rec = np.zeros((len(coords), 4, B, B, B), np.float32)
        stored = np.zeros(len(coords), bool)
        for q, c in enumerate(coords.tolist()):
            if tuple(c) in self.bricks:
                rec[q], stored[q] = self.bricks[tuple(c)], True
        for c, ch in enumerate(self._channels()):
            ch[k, j, i] = rec[inv, c, lz, ly, lx]
        self.restored = int((stored[inv] & (self.weight[k, j, i] > 0)).sum())

    def download_store(self):
        """(coords int64 [m, 3], records float32 [m, 4, 8, 8, 8]) in ascending (z, y, x), the voxels inside the
        window (0, 0), as rmd_volume_download_store."""
        keys = sorted(self.bricks, key=lambda c: (c[2], c[1], c[0]))
        coords = np.array(keys, np.int64).reshape(-1, 3)
        rec = np.array([self.bricks[c] for c in keys], np.float32).reshape(-1, 4, B, B, B).copy()
        n, D = np.asarray(self.dims, np.int64), self.D
        for q, c in enumerate(keys):
            u = [np.arange(B, dtype=np.int64) + B * c[a] - D[a] for a in range(3)]
            ins = [(x >= 0) & (x < n[a]) for a, x in enumerate(u)]
            rec[q][:, ins[2][:, None, None] & ins[1][None, :, None] & ins[0][None, None, :]] = 0.0
        return coords, rec

    def dense_map(self):
        """(lowest unbounded voxel (x, y, z), tsdf, weight (nz, ny, nx)) of the whole map -- store and window -- as one
        dense grid."""
        D, n = self.D, np.asarray(self.dims, np.int64)
        coords = np.array(list(self.bricks), np.int64).reshape(-1, 3)
        lo = np.minimum(coords.min(0) * B, D) if len(coords) else D
        hi = np.maximum(coords.max(0) * B + B, D + n) if len(coords) else D + n
        size = (hi - lo)[::-1]
        t, w = np.zeros(size, np.float32), np.zeros(size, np.float32)
        for c, r in self.bricks.items():
            o = np.asarray(c, np.int64) * B - lo
            t[o[2]:o[2] + B, o[1]:o[1] + B, o[0]:o[0] + B] = r[0]
            w[o[2]:o[2] + B, o[1]:o[1] + B, o[0]:o[0] + B] = r[1]
        o = D - lo
        t[o[2]:o[2] + n[2], o[1]:o[1] + n[1], o[0]:o[0] + n[0]] = self.tsdf
        w[o[2]:o[2] + n[2], o[1]:o[1] + n[1], o[0]:o[0] + n[0]] = self.weight
        return lo, t, w

    # ------------------------------------------------ api.TsdfVolume's names, as api.TsdfVolume.mapMesh calls them
    def downloadStore(self, records=True):
        assert not records
        return self.download_store()[0]
