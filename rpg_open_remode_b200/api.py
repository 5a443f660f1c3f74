"""Host-side mirror of the reference's C++ interface for the hot path.

Same class and method names, argument meaning and error behaviour as

* ``rmd::SeedMatrix``        include/rmd/seed_matrix.cuh:45-109
* ``rmd::DepthmapDenoiser``  include/rmd/depthmap_denoiser.cuh:27-54
* ``rmd::ImageReducer<T>``   include/rmd/reduction.cuh:27-62
* ``rmd::DeviceImage<T>``    include/rmd/device_image.cuh:34-180
* ``rmd::Depthmap``          include/rmd/depthmap.h:34-129 (OpenCV-free)
* ``rmd::SE3<float>``, ``rmd::PinholeCamera``

so the parity tests read like the reference's gtests.  Every call goes
through the C-ABI (``include/rmd_b200.h``) into the sm_90a kernels; nothing
is computed in Python and there is no CPU fallback.
"""
from __future__ import annotations

import ctypes
import math

import numpy as np

from . import _native
from ._native import RmdError, check

# rmd::ConvergenceStates, include/rmd/seed_matrix.cuh:31-43
class ConvergenceStates:
    UPDATE = 0
    CONVERGED = 1
    BORDER = 2
    DIVERGED = 3
    NO_MATCH = 4
    NOT_VISIBLE = 5


FIELD_MU, FIELD_SIGMA_SQ, FIELD_A, FIELD_B, FIELD_CONVERGENCE = 0, 1, 2, 3, 4
FIELD_SUM_TEMPL, FIELD_CONST_TEMPL_DENOM, FIELD_EPIPOLAR_MATCHES, FIELD_REF_IMG = 5, 6, 7, 8
OPT_RECORD_MATCHES, OPT_KERNEL_VARIANT, OPT_TEX_FRAC_BITS, OPT_DEBUG_TIMELINE, OPT_PINNED_INPUT = 0, 1, 2, 3, 4
OPT_CHAIN_FRAMES, OPT_SEED_MODE_PCT = 5, 6
# tuning knobs of the staged kernel (include/rmd_b200.h RMD_OPT_TUNE_*; results never depend on them)
(OPT_TUNE_SPLIT_MAX, OPT_TUNE_SPLIT_MIN_ITEMS, OPT_TUNE_SPLIT_ITEMS_PER_CTA, OPT_TUNE_SPARSE_MAX_SEEDS,
 OPT_TUNE_HEAVY_MIN_ITEMS, OPT_TUNE_SPLIT_AVG_PCT, OPT_TUNE_PDL) = 10, 11, 12, 13, 14, 15, 16
OPT_TUNE_WARP_TILE_SEEDS = 17
OPT_TUNE_GRID_CTAS = 18
OPT_TUNE_CTAS_PER_SM = 19
OPT_TUNE_WARP_TILE_CANDS = 20
OPT_TUNE_RUN_CHUNKS = 21
FIELD_DEBUG_TIMELINE = 100
VARIANT_STAGED, VARIANT_DIRECT = 0, 1
# sigma^2 of a propagated keyframe prior as a fraction of the uniform prior's range^2 / 36 (DESIGN.md 4.7, 6)
PRIOR_SIGMA_SQ_FRAC = 1.0 / 16.0

_f32 = np.float32


class PinholeCamera:
    """include/rmd/pinhole_camera.cuh:27-63"""

    def __init__(self, fx=0.0, fy=0.0, cx=0.0, cy=0.0):
        self.fx, self.fy, self.cx, self.cy = (float(_f32(v)) for v in (fx, fy, cx, cy))

    def cam2world(self, uv):
        u, v = _f32(uv[0]), _f32(uv[1])
        return np.array([(u - _f32(self.cx)) / _f32(self.fx), (v - _f32(self.cy)) / _f32(self.fy), 1.0], _f32)

    def world2cam(self, xyz):
        x, y, z = (_f32(t) for t in xyz)
        return np.array([_f32(self.fx) * x / z + _f32(self.cx), _f32(self.fy) * y / z + _f32(self.cy)], _f32)

    def getOnePixAngle(self):
        return float(_f32(math.atan2(1.0, 2.0 * self.fx)) * _f32(2.0))


class SE3:
    """include/rmd/se3.cuh:27-168: 3x4 row-major [R|t], float32 arithmetic."""

    def __init__(self, *args):
        if len(args) == 0:
            self.data = np.zeros(12, _f32)
            self.data[[0, 5, 10]] = 1.0
        elif len(args) == 1:
            self.data = np.array(args[0], dtype=_f32).reshape(12).copy()
        elif len(args) == 2:  # (r row-major 3x3, t)
            r, t = np.asarray(args[0], _f32).reshape(3, 3), np.asarray(args[1], _f32).reshape(3)
            self.data = np.concatenate([r, t[:, None]], axis=1).reshape(12).astype(_f32)
        elif len(args) == 7:  # (qw, qx, qy, qz, tx, ty, tz), se3.cuh:37-66
            qw, qx, qy, qz, tx, ty, tz = (_f32(a) for a in args)
            two = _f32(2)
            x, y, z = two * qx, two * qy, two * qz
            wx, wy, wz = x * qw, y * qw, z * qw
            xx, xy, xz = x * qx, y * qx, z * qx
            yy, yz, zz = y * qy, z * qy, z * qz
            one = _f32(1)
            self.data = np.array([one - (yy + zz), xy - wz, xz + wy, tx,
                                  xy + wz, one - (xx + zz), yz - wx, ty,
                                  xz - wy, yz + wx, one - (xx + yy), tz], _f32)
        else:
            raise TypeError("SE3(): expected (), (12 floats), (r, t) or (qw,qx,qy,qz,tx,ty,tz)")

    def __call__(self, r, c):
        return float(self.data[4 * r + c])

    def inv(self):
        d, o = self.data, np.empty(12, _f32)
        o[0], o[1], o[2] = d[0], d[4], d[8]
        o[4], o[5], o[6] = d[1], d[5], d[9]
        o[8], o[9], o[10] = d[2], d[6], d[10]
        o[3] = -d[0] * d[3] - d[4] * d[7] - d[8] * d[11]
        o[7] = -d[1] * d[3] - d[5] * d[7] - d[9] * d[11]
        o[11] = -d[2] * d[3] - d[6] * d[7] - d[10] * d[11]
        return SE3(o)

    def __mul__(self, other):
        if isinstance(other, SE3):
            l, r, o = self.data, other.data, np.empty(12, _f32)
            for row in range(3):
                a = l[4 * row:4 * row + 4]
                for col in range(3):
                    o[4 * row + col] = a[0] * r[col] + a[1] * r[4 + col] + a[2] * r[8 + col]
                o[4 * row + 3] = a[3] + a[0] * r[3] + a[1] * r[7] + a[2] * r[11]
            return SE3(o)
        return self.translate(self.rotate(other))

    def rotate(self, p):
        d, p = self.data, np.asarray(p, _f32)
        return np.array([d[0] * p[0] + d[1] * p[1] + d[2] * p[2],
                         d[4] * p[0] + d[5] * p[1] + d[6] * p[2],
                         d[8] * p[0] + d[9] * p[1] + d[10] * p[2]], _f32)

    def translate(self, p):
        p = np.asarray(p, _f32)
        return np.array([p[0] + self.data[3], p[1] + self.data[7], p[2] + self.data[11]], _f32)

    def getTranslation(self):
        return self.data[[3, 7, 11]].copy()

    def __repr__(self):
        return "SE3(\n%s)" % self.data.reshape(3, 4)


def _box_args(lo, dims, what: str):
    """None when lo and dims are both omitted, else (lo int64 [3], dims int32 [3]) of a box of a volume's map."""
    if lo is None and dims is None:
        return None
    if lo is None or dims is None:
        raise ValueError(what + ": lo and dims come together")
    a, m = list(np.asarray(lo).reshape(-1)), list(np.asarray(dims).reshape(-1))
    if len(a) != 3 or len(m) != 3 or any(int(x) != x for x in a + m):
        raise ValueError(what + ": lo and dims must be three whole numbers each")
    if any(not -2 ** 63 <= int(x) < 2 ** 63 for x in a) or any(not -2 ** 31 <= int(x) < 2 ** 31 for x in m):
        raise ValueError(what + ": lo must fit int64 and dims int32")
    return np.array([int(x) for x in a], np.int64), np.array([int(x) for x in m], np.int32)


def _pose12(T) -> np.ndarray:
    if isinstance(T, SE3):
        return np.ascontiguousarray(T.data, dtype=_f32)
    a = np.ascontiguousarray(np.asarray(T, dtype=_f32).reshape(-1))
    if a.size != 12:
        raise ValueError("pose must be SE3 or 12 floats (3x4 row-major)")
    return a


class DeviceImage:
    """include/rmd/device_image.cuh:34-180.  ``dtype`` in {float32, int32,
    'float2'}.  Public fields as in the reference: width, height, pitch,
    stride (elements), data (device address)."""

    _ELEM = {"float32": (4, np.float32, 1), "int32": (4, np.int32, 1), "float2": (8, np.float32, 2)}

    def __init__(self, width, height, dtype="float32", _view=None):
        key = "float2" if dtype == "float2" else np.dtype(dtype).name
        if key not in self._ELEM:
            raise TypeError(f"DeviceImage: unsupported element type {dtype}")
        self._elem_size, self._np, self._comps = self._ELEM[key]
        self.dtype = key
        self.width, self.height = int(width), int(height)
        self._L = _native.lib()
        if _view is not None:
            self.data, self.pitch = int(_view[0]), int(_view[1])
            self._owned = False
        else:
            ptr, pitch = ctypes.c_void_p(), ctypes.c_size_t()
            check(self._L.rmd_image_alloc(self.width, self.height, self._elem_size,
                                          ctypes.byref(ptr), ctypes.byref(pitch)),
                  "Image: unable to allocate pitched memory.")
            self.data, self.pitch = ptr.value, pitch.value
            self._owned = True
        self.stride = self.pitch // self._elem_size

    def __del__(self):
        if getattr(self, "_owned", False) and getattr(self, "data", None):
            self._L.rmd_image_free(self.data)
            self.data = None

    def _host_shape(self):
        return (self.height, self.width) if self._comps == 1 else (self.height, self.width, self._comps)

    def setDevData(self, aligned_data_row_major):
        a = np.ascontiguousarray(aligned_data_row_major, dtype=self._np)
        if a.shape != self._host_shape():
            raise ValueError(f"setDevData: expected shape {self._host_shape()}, got {a.shape}")
        check(self._L.rmd_image_upload(self.data, self.pitch, a.ctypes.data, self.width, self.height,
                                       self._elem_size), "Image: unable to copy data from host to device.")

    def getDevData(self):
        out = np.empty(self._host_shape(), dtype=self._np)
        check(self._L.rmd_image_download(self.data, self.pitch, out.ctypes.data, self.width, self.height,
                                         self._elem_size), "Image: unable to copy data from device to host.")
        return out

    def zero(self):
        check(self._L.rmd_image_zero(self.data, self.pitch, self.width, self.height, self._elem_size),
              "Image: unable to zero.")

    def assign(self, other: "DeviceImage"):
        """operator= (device to device copy), device_image.cuh:150-171"""
        assert (self.width, self.height, self.dtype) == (other.width, other.height, other.dtype)
        check(self._L.rmd_image_copy(self.data, self.pitch, other.data, other.pitch, self.width,
                                     self.height, self._elem_size),
              "Image, operator '=': unable to copy data from another image.")
        return self


class SeedMatrix:
    """rmd::SeedMatrix -- include/rmd/seed_matrix.cuh:45-109, src/seed_matrix.cu."""

    def __init__(self, width, height, cam: PinholeCamera, patch_side=5, device=-1):
        self.width_, self.height_, self.patch_side = int(width), int(height), int(patch_side)
        self.cam_ = cam
        self._L = _native.lib()
        h = ctypes.c_void_p()
        check(self._L.rmd_seeds_create(self.width_, self.height_, cam.fx, cam.fy, cam.cx, cam.cy,
                                       self.patch_side, int(device), ctypes.byref(h)), "SeedMatrix")
        self._h = h

    def __del__(self):
        h, self._h = getattr(self, "_h", None), None
        if h:
            self._L.rmd_seeds_destroy(h)

    @property
    def handle(self):
        return self._h

    # ---- reference API
    def setReferenceImage(self, host_ref_img_align_row_maj, T_curr_world, min_depth, max_depth) -> bool:
        img = self._frame(host_ref_img_align_row_maj)
        T = _pose12(T_curr_world)
        fn = self._L.rmd_seeds_set_reference_u8 if img.dtype == np.uint8 else self._L.rmd_seeds_set_reference
        check(fn(self._h, img.ctypes.data, T.ctypes.data, float(min_depth), float(max_depth)),
              "SeedMatrix::setReferenceImage")
        return True

    def update(self, host_curr_img_align_row_maj, T_curr_world) -> bool:
        img = self._frame(host_curr_img_align_row_maj)
        T = _pose12(T_curr_world)
        fn = self._L.rmd_seeds_update_u8 if img.dtype == np.uint8 else self._L.rmd_seeds_update
        check(fn(self._h, img.ctypes.data, T.ctypes.data), "SeedMatrix::update")
        return True

    def downloadDepthmap(self):
        return self._download(FIELD_MU)

    def downloadConvergence(self):
        return self._download(FIELD_CONVERGENCE)

    def getMu(self):
        return self._device_image(FIELD_MU)

    def getSigmaSq(self):
        return self._device_image(FIELD_SIGMA_SQ)

    def getA(self):
        return self._device_image(FIELD_A)

    def getB(self):
        return self._device_image(FIELD_B)

    def getConvergence(self):
        return self._device_image(FIELD_CONVERGENCE)

    def getConvergedCount(self) -> int:
        n = ctypes.c_size_t()
        check(self._L.rmd_seeds_converged_count(self._h, ctypes.byref(n)), "SeedMatrix::getConvergedCount")
        return int(n.value)

    def getDistFromRef(self) -> float:
        d = ctypes.c_float()
        check(self._L.rmd_seeds_dist_from_ref(self._h, ctypes.byref(d)), "SeedMatrix::getDistFromRef")
        return float(d.value)

    # RMD_BUILD_TESTS accessors, seed_matrix.cuh:76-83
    def downloadSigmaSq(self):
        return self._download(FIELD_SIGMA_SQ)

    def downloadA(self):
        return self._download(FIELD_A)

    def downloadB(self):
        return self._download(FIELD_B)

    def downloadSumTempl(self):
        return self._download(FIELD_SUM_TEMPL)

    def downloadConstTemplDenom(self):
        return self._download(FIELD_CONST_TEMPL_DENOM)

    def downloadEpipolarMatches(self):
        return self._download(FIELD_EPIPOLAR_MATCHES)

    # ---- additions of this implementation
    def updateDevice(self, dev_ptr: int, pitch_bytes: int, T_curr_world) -> bool:
        """Frame already resident in device memory (16-byte aligned)."""
        T = _pose12(T_curr_world)
        check(self._L.rmd_seeds_update_device(self._h, dev_ptr, pitch_bytes, T.ctypes.data),
              "SeedMatrix::updateDevice")
        return True

    def updateDeviceBatch(self, dev_ptr: int, frame_stride_bytes: int, pitch_bytes: int, poses) -> bool:
        """n consecutive updates from device-resident frames; poses: (n, 12) float32."""
        T = np.ascontiguousarray(np.asarray(poses, dtype=_f32).reshape(-1, 12))
        check(self._L.rmd_seeds_update_device_batch(self._h, dev_ptr, frame_stride_bytes, pitch_bytes,
                                                    T.shape[0], T.ctypes.data),
              "SeedMatrix::updateDeviceBatch")
        return True

    def setReferenceImageDevice(self, dev_ptr: int, pitch_bytes: int, T_curr_world, min_depth, max_depth):
        T = _pose12(T_curr_world)
        check(self._L.rmd_seeds_set_reference_device(self._h, dev_ptr, pitch_bytes, T.ctypes.data,
                                                     float(min_depth), float(max_depth)),
              "SeedMatrix::setReferenceImageDevice")
        return True

    # ---- frame ingest with lens undistortion (rmd::Depthmap::initUndistortionMap / inputImage,
    # src/depthmap.cpp:45-61,95-106); applies to uint8 frames given to setReferenceImage / update
    def initUndistortionMap(self, k1, k2, r1, r2) -> None:
        check(self._L.rmd_seeds_init_undistortion_map(self._h, float(k1), float(k2), float(r1), float(r2)),
              "SeedMatrix::initUndistortionMap")

    def clearUndistortionMap(self) -> None:
        check(self._L.rmd_seeds_clear_undistortion_map(self._h), "SeedMatrix::clearUndistortionMap")

    def getUndistortionMap(self):
        """(map1, map2) as cv::initUndistortRectifyMap(..., CV_16SC2) lays them out."""
        m1 = np.empty((self.height_, self.width_, 2), np.int16)
        m2 = np.empty((self.height_, self.width_), np.uint16)
        check(self._L.rmd_seeds_get_undistortion_map(self._h, m1.ctypes.data, m2.ctypes.data),
              "SeedMatrix::getUndistortionMap")
        return m1, m2

    def undistort(self, img_8uc1):
        """The remapped 8-bit frame (img_undistorted_8uc1_ of rmd::Depthmap)."""
        a = np.ascontiguousarray(img_8uc1, dtype=np.uint8)
        if a.shape != (self.height_, self.width_):
            raise ValueError("undistort: wrong shape")
        out = np.empty_like(a)
        check(self._L.rmd_seeds_undistort_u8(self._h, a.ctypes.data, out.ctypes.data), "SeedMatrix::undistort")
        return out

    @staticmethod
    def updateMany(seeds: "list[SeedMatrix]", host_curr_img_align_row_maj, T_curr_world) -> bool:
        """Several live keyframes against one incoming frame (rmd_seeds_update_many): one upload, one fused kernel
        per keyframe on its own stream.  Same result as update() on each; an 8-bit frame goes through seeds[0]'s
        ingest (undistortion map)."""
        if not seeds:
            raise ValueError("updateMany: no keyframes")
        first = seeds[0]
        img = first._frame(host_curr_img_align_row_maj)
        T = _pose12(T_curr_world)
        arr = (ctypes.c_void_p * len(seeds))(*[s._h.value for s in seeds])
        fn = first._L.rmd_seeds_update_many_u8 if img.dtype == np.uint8 else first._L.rmd_seeds_update_many
        check(fn(arr, len(seeds), img.ctypes.data, T.ctypes.data), "SeedMatrix::updateMany")
        return True

    def pointCloud(self, depth: "DeviceImage | None" = None, capacity: "int | None" = None):
        """rmd::Publisher::publishPointCloud (src/publisher.cpp:54-86): float32 [n, 4] = (x, y, z, intensity) of the
        CONVERGED pixels in row-major order, from the seeds' own depth or from a device depth image (e.g. denoised).
        Returns (points, count); count > len(points) when `capacity` was too small."""
        cap = self.width_ * self.height_ if capacity is None else int(capacity)
        out = np.empty((cap, 4), np.float32)
        n = ctypes.c_size_t()
        ptr, pitch = (depth.data, depth.pitch) if depth is not None else (None, 0)
        check(self._L.rmd_seeds_point_cloud(self._h, ptr, pitch, out.ctypes.data, cap, ctypes.byref(n)),
              "SeedMatrix::pointCloud")
        return out[:min(cap, n.value)], int(n.value)

    def setPriorPropagation(self, sigma_sq_frac: float) -> None:
        """In place: from now on every setReferenceImage* first splats this keyframe's CONVERGED seeds into the new
        reference view and uses them as its depth prior (sigma^2 = sigma_sq_frac * range^2 / 36).  0 = off."""
        check(self._L.rmd_seeds_set_prior_propagation(self._h, float(sigma_sq_frac)), "SeedMatrix::setPriorPropagation")

    def propagatePriorFrom(self, src: "SeedMatrix", sigma_sq_frac: float = PRIOR_SIGMA_SQ_FRAC) -> None:
        """Right after setReferenceImage* (no update since): take this keyframe's depth prior from the CONVERGED
        seeds of another live keyframe `src` (same device; size and camera may differ)."""
        check(self._L.rmd_seeds_propagate_prior(self._h, src.handle, float(sigma_sq_frac)),
              "SeedMatrix::propagatePriorFrom")

    def priorFromVolume(self, volume: "TsdfVolume", sigma_sq_frac: float = PRIOR_SIGMA_SQ_FRAC, lo=None,
                        dims=None) -> None:
        """Right after setReferenceImage* (no update since): every pixel whose ray from the new reference pose hits
        the fused surface of `volume` within [min_depth, max_depth] takes the hit as its depth prior (sigma^2 =
        sigma_sq_frac * range^2 / 36); all other seeds keep the prior they have (uniform, or splatted by the
        propagation above).  Ordered on the device after the volume's queued integrations.  lo, dims: the rays
        march that box of the map instead of the window, brick store included (TsdfVolume.raycast)."""
        what = "SeedMatrix::priorFromVolume"
        box = _box_args(lo, dims, what)
        if box is None:
            check(self._L.rmd_volume_prior_seeds(volume.handle, self._h, float(sigma_sq_frac)), what)
            return
        lo64, m32 = box
        check(self._L.rmd_volume_prior_seeds_box(volume.handle, self._h, float(sigma_sq_frac), lo64.ctypes.data,
                                                 m32.ctypes.data), what)

    def uploadState(self, field: int, values) -> None:
        dt = np.int32 if field == FIELD_CONVERGENCE else np.float32
        a = np.ascontiguousarray(values, dtype=dt)
        if a.shape != (self.height_, self.width_):
            raise ValueError("uploadState: wrong shape")
        check(self._L.rmd_seeds_upload_state(self._h, field, a.ctypes.data), "SeedMatrix::uploadState")

    def copyFieldToDevice(self, field: int, dev_ptr: int, pitch_bytes: int) -> None:
        check(self._L.rmd_seeds_copy_field_to_device(self._h, field, dev_ptr, pitch_bytes),
              "SeedMatrix::copyFieldToDevice")

    def setOption(self, option: int, value: int) -> None:
        check(self._L.rmd_seeds_set_option(self._h, option, value), "SeedMatrix::setOption")

    def setStream(self, cuda_stream: int) -> None:
        check(self._L.rmd_seeds_set_stream(self._h, cuda_stream), "SeedMatrix::setStream")

    def sync(self) -> None:
        check(self._L.rmd_seeds_sync(self._h), "SeedMatrix::sync")

    def launchCount(self):
        a, b = ctypes.c_uint64(), ctypes.c_uint64()
        check(self._L.rmd_seeds_launch_count(self._h, ctypes.byref(a), ctypes.byref(b)))
        return int(a.value), int(b.value)

    def enableKernelTiming(self, on=True):
        check(self._L.rmd_seeds_enable_kernel_timing(self._h, 1 if on else 0))

    def lastKernelMs(self) -> float:
        ms = ctypes.c_float()
        check(self._L.rmd_seeds_last_kernel_ms(self._h, ctypes.byref(ms)), "SeedMatrix::lastKernelMs")
        return float(ms.value)

    # ---- helpers
    def _frame(self, img):
        a = np.asarray(img)
        if a.dtype != np.uint8:
            a = np.ascontiguousarray(a, dtype=np.float32)
        else:
            a = np.ascontiguousarray(a)
        if a.shape != (self.height_, self.width_):
            raise ValueError(f"frame must be ({self.height_}, {self.width_}), got {a.shape}")
        return a

    def downloadTimeline(self):
        """Debug (OPT_DEBUG_TIMELINE): int64[n_tiles, 16] of the last staged launch."""
        n = ((self.width_ + 31) // 32) * ((self.height_ + 7) // 8)
        out = np.empty((n, 16), np.int64)
        check(self._L.rmd_seeds_download(self._h, FIELD_DEBUG_TIMELINE, out.ctypes.data), "SeedMatrix::downloadTimeline")
        return out

    def _download(self, field):
        if field == FIELD_CONVERGENCE:
            out = np.empty((self.height_, self.width_), np.int32)
        elif field == FIELD_EPIPOLAR_MATCHES:
            out = np.empty((self.height_, self.width_, 2), np.float32)
        else:
            out = np.empty((self.height_, self.width_), np.float32)
        check(self._L.rmd_seeds_download(self._h, field, out.ctypes.data), "SeedMatrix::download")
        return out

    def _device_image(self, field):
        ptr, pitch = ctypes.c_void_p(), ctypes.c_size_t()
        check(self._L.rmd_seeds_device_ptr(self._h, field, ctypes.byref(ptr), ctypes.byref(pitch)),
              "SeedMatrix::get*")
        dt = "int32" if field == FIELD_CONVERGENCE else ("float2" if field == FIELD_EPIPOLAR_MATCHES else "float32")
        return DeviceImage(self.width_, self.height_, dt, _view=(ptr.value, pitch.value))


class DepthmapDenoiser:
    """rmd::DepthmapDenoiser -- include/rmd/depthmap_denoiser.cuh:27-54."""

    def __init__(self, width, height, device=-1):
        self.width, self.height = int(width), int(height)
        self._L = _native.lib()
        h = ctypes.c_void_p()
        check(self._L.rmd_denoiser_create(self.width, self.height, int(device), ctypes.byref(h)),
              "DepthmapDenoiser")
        self._h = h

    def __del__(self):
        h, self._h = getattr(self, "_h", None), None
        if h:
            self._L.rmd_denoiser_destroy(h)

    def setLargeSigmaSq(self, depth_range):
        check(self._L.rmd_denoiser_set_large_sigma_sq(self._h, float(depth_range)))

    def denoise(self, mu: DeviceImage, sigma_sq: DeviceImage, a: DeviceImage, b: DeviceImage,
                lam: float, iterations: int):
        """Returns host_denoised (the reference fills a caller buffer)."""
        out = np.empty((self.height, self.width), np.float32)
        check(self._L.rmd_denoiser_run(self._h, mu.data, mu.pitch, sigma_sq.data, sigma_sq.pitch,
                                       a.data, a.pitch, b.data, b.pitch, out.ctypes.data,
                                       float(lam), int(iterations)), "DepthmapDenoiser::denoise")
        return out

    def denoiseSeeds(self, seeds: SeedMatrix, lam: float, iterations: int):
        out = np.empty((self.height, self.width), np.float32)
        check(self._L.rmd_denoiser_run_seeds(self._h, seeds.handle, out.ctypes.data, float(lam),
                                             int(iterations)), "DepthmapDenoiser::denoiseSeeds")
        return out

    def denoiseSeedsToDevice(self, seeds: SeedMatrix, dev_ptr: int, pitch_bytes: int, lam: float,
                             iterations: int):
        check(self._L.rmd_denoiser_run_seeds_to_device(self._h, seeds.handle, dev_ptr, pitch_bytes,
                                                       float(lam), int(iterations)),
              "DepthmapDenoiser::denoiseSeedsToDevice")

    def setStream(self, cuda_stream: int):
        check(self._L.rmd_denoiser_set_stream(self._h, cuda_stream))

    def sync(self):
        check(self._L.rmd_denoiser_sync(self._h))

    def launchCount(self) -> int:
        n = ctypes.c_uint64()
        check(self._L.rmd_denoiser_launch_count(self._h, ctypes.byref(n)))
        return int(n.value)


class TsdfVolume:
    """Dense TSDF voxel grid on one device that fuses finished keyframes (rmd_volume_*, include/rmd_b200.h;
    DESIGN.md 4.8).  dims = (nx, ny, nz), x fastest; origin = world position of the centre of voxel (0, 0, 0);
    truncation in metres; max_weight caps a voxel's weight (one observation = 1).  intensity=True adds the
    intensity channel (8 B per voxel): keyframes then also fuse their reference image, and the surface points, mesh
    vertices and raycast views can be shaded (surfaceIntensity, raycastIntensity).  store=True adds the brick store:
    a shift then keeps the voxels that leave the grid and gives them back when they re-enter, and mapMesh() meshes
    the whole map."""

    def __init__(self, dims, voxel_size: float, origin, truncation: float, max_weight: float = 64.0, device=-1,
                 intensity: bool = False, store: bool = False):
        self.dims = tuple(int(n) for n in dims)
        if len(self.dims) != 3:
            raise ValueError("TsdfVolume: dims must be (nx, ny, nz)")
        self._L = _native.lib()
        o = np.ascontiguousarray(np.asarray(origin, _f32).reshape(3))
        h = ctypes.c_void_p()
        check(self._L.rmd_volume_create(*self.dims, float(voxel_size), o.ctypes.data, float(truncation),
                                        float(max_weight), int(device), ctypes.byref(h)), "TsdfVolume")
        self._h = h
        self.voxel_size, self.origin = float(_f32(voxel_size)), o.copy()
        self.truncation, self.max_weight = float(_f32(truncation)), float(_f32(max_weight))
        self.intensity = False
        if intensity:
            self.enableIntensity()
        self.store = False
        if store:
            self.enableStore()

    def __del__(self):
        h, self._h = getattr(self, "_h", None), None
        if h:
            self._L.rmd_volume_destroy(h)

    @property
    def handle(self):
        return self._h

    def integrate(self, seeds: SeedMatrix, depth: "DeviceImage | None" = None) -> None:
        """A keyframe: the CONVERGED pixels of `seeds`, seen from the pose its reference was set with; depth = the
        seeds' mu or a device image of their size (e.g. denoised).  Ordered on the device against `seeds`."""
        ptr, pitch = (depth.data, depth.pitch) if depth is not None else (None, 0)
        check(self._L.rmd_volume_integrate_seeds(self._h, seeds.handle, ptr, pitch), "TsdfVolume::integrate")

    def enableIntensity(self) -> None:
        """Allocate and zero the intensity channel (no-op when it exists)."""
        check(self._L.rmd_volume_enable_intensity(self._h), "TsdfVolume::enableIntensity")
        self.intensity = True

    def integrateDepth(self, depth, cam: PinholeCamera, T_curr_world, conv=None, intensity=None) -> None:
        """Any depth image (distance along the ray): a float32 DeviceImage or a host array; conv: optional int32
        states (DeviceImage or host array), only CONVERGED pixels count; intensity: optional float32 image of the
        same size (DeviceImage or host array) fused into the intensity channel."""
        keep = []

        def dev(img, dtype):
            if isinstance(img, DeviceImage):
                return img
            a = np.ascontiguousarray(img, dtype)
            d = DeviceImage(a.shape[1], a.shape[0], dtype)
            d.setDevData(a)
            keep.append(d)
            return d

        D = dev(depth, np.float32)
        C = dev(conv, np.int32) if conv is not None else None
        if C is not None and (C.width, C.height) != (D.width, D.height):
            raise ValueError("TsdfVolume::integrateDepth: depth and state maps differ in size")
        I = dev(intensity, np.float32) if intensity is not None else None
        if I is not None and (I.width, I.height) != (D.width, D.height):
            raise ValueError("TsdfVolume::integrateDepth: depth and intensity images differ in size")
        T = _pose12(T_curr_world)
        if I is None:
            check(self._L.rmd_volume_integrate_depth(self._h, D.width, D.height, cam.fx, cam.fy, cam.cx, cam.cy,
                                                     T.ctypes.data, D.data, D.pitch, C.data if C else None,
                                                     C.pitch if C else 0), "TsdfVolume::integrateDepth")
        else:
            check(self._L.rmd_volume_integrate_depth_intensity(
                self._h, D.width, D.height, cam.fx, cam.fy, cam.cx, cam.cy, T.ctypes.data, D.data, D.pitch,
                C.data if C else None, C.pitch if C else 0, I.data, I.pitch), "TsdfVolume::integrateDepth")
        if keep:
            self.sync()   # the staged images must outlive the kernel

    def _surface(self, fn, capacity, shape, what: str) -> np.ndarray:
        """One float32 [shape] per surface point from fn (rmd_volume_surface_points or _intensity): the count first
        when no capacity is given, then at most capacity of them."""
        n = ctypes.c_size_t()
        if capacity is None:
            check(fn(self._h, None, 0, ctypes.byref(n)), what)
            capacity = n.value
        out = np.empty((int(capacity),) + shape, np.float32)
        check(fn(self._h, out.ctypes.data if capacity else None, int(capacity), ctypes.byref(n)), what)
        return out[:min(int(capacity), n.value)]

    def surfacePoints(self, capacity: "int | None" = None) -> np.ndarray:
        """float32 [n, 4] = (x, y, z, weight) of the zero crossings, in voxel order then axis x, y, z.  With a
        capacity, at most that many points."""
        return self._surface(self._L.rmd_volume_surface_points, capacity, (4,), "TsdfVolume::surfacePoints")

    def surfaceIntensity(self, capacity: "int | None" = None) -> np.ndarray:
        """float32 [n]: the intensity of every surface point (and mesh vertex), in surfacePoints() order; -1 where
        neither of the point's voxels has one.  With a capacity, at most that many."""
        return self._surface(self._L.rmd_volume_surface_intensity, capacity, (), "TsdfVolume::surfaceIntensity")

    def surfaceNormals(self, capacity: "int | None" = None) -> np.ndarray:
        """float32 [n, 3]: the unit normal of every surface point (and mesh vertex), in surfacePoints() order,
        towards free space (tsdf > 0); (0, 0, 0) where the tsdf gradient vanishes.  With a capacity, at most that
        many."""
        n = self._surface(self._L.rmd_volume_surface_normals, capacity, (4,), "TsdfVolume::surfaceNormals")
        return np.ascontiguousarray(n[:, :3])

    def mesh(self, vertex_capacity: "int | None" = None, triangle_capacity: "int | None" = None):
        """Marching-cubes mesh of the fused surface: (float32 [n, 4] vertices, int32 [m, 3] triangles).  The vertices
        are surfacePoints(), bit for bit; triangles are ordered by cube and face the tsdf > 0 side, (b - a) x (c - a).
        With capacities, at most that many of each (triangles may then index vertices that were not returned).
        Raises RmdError (RMD_ERR_UNSUPPORTED) for 2^31 or more vertices."""
        nv, nt = ctypes.c_size_t(), ctypes.c_size_t()
        if vertex_capacity is None or triangle_capacity is None:
            check(self._L.rmd_volume_mesh(self._h, None, 0, None, 0, ctypes.byref(nv), ctypes.byref(nt)),
                  "TsdfVolume::mesh")
            vertex_capacity = nv.value if vertex_capacity is None else vertex_capacity
            triangle_capacity = nt.value if triangle_capacity is None else triangle_capacity
        verts = np.empty((int(vertex_capacity), 4), np.float32)
        tris = np.empty((int(triangle_capacity), 3), np.int32)
        check(self._L.rmd_volume_mesh(self._h, verts.ctypes.data if vertex_capacity else None, int(vertex_capacity),
                                      tris.ctypes.data if triangle_capacity else None, int(triangle_capacity),
                                      ctypes.byref(nv), ctypes.byref(nt)), "TsdfVolume::mesh")
        return verts[:min(int(vertex_capacity), nv.value)], tris[:min(int(triangle_capacity), nt.value)]

    def _raycast_box(self, what, box, cam, T, width, height, img, inten=None, nrm=None) -> None:
        lo64, m32 = box
        check(self._L.rmd_volume_raycast_box(self._h, lo64.ctypes.data, m32.ctypes.data, int(width), int(height),
                                             cam.fx, cam.fy, cam.cx, cam.cy, T.ctypes.data, img.data, img.pitch,
                                             inten.data if inten is not None else None,
                                             inten.pitch if inten is not None else 0,
                                             nrm.data if nrm is not None else None,
                                             nrm.pitch if nrm is not None else 0), what)

    def raycast(self, cam: PinholeCamera, T_curr_world, width: int, height: int, lo=None, dims=None) -> np.ndarray:
        """float32 [height, width]: distance along each pixel's ray to the fused surface, 0 where none.

        With lo (int [3], window indices, may be negative or outside the window) and dims (int [3], each > 0): the
        rays march a box of the map instead of the window -- each box voxel takes the window's record, else (with the
        store) its stored brick's, else unknown, as computeEsdf(lo, dims) gathers them.  8 B of scratch per box
        voxel; the box (0, n) gives the window's image bit for bit."""
        what = "TsdfVolume::raycast"
        box = _box_args(lo, dims, what)
        img = DeviceImage(width, height, "float32")
        T = _pose12(T_curr_world)
        if box is not None:
            self._raycast_box(what, box, cam, T, width, height, img)
            self.sync()
            return img.getDevData()
        check(self._L.rmd_volume_raycast(self._h, int(width), int(height), cam.fx, cam.fy, cam.cx, cam.cy,
                                         T.ctypes.data, img.data, img.pitch), "TsdfVolume::raycast")
        self.sync()
        return img.getDevData()

    def raycastIntensity(self, cam: PinholeCamera, T_curr_world, width: int, height: int, lo=None, dims=None):
        """(depth, intensity), float32 [height, width] each: raycast()'s depth, bit for bit, and the fused intensity
        at each hit, -1 where there is no hit or no intensity.  lo, dims: a box of the map, as raycast(); 8 B more
        per box voxel for its intensity records."""
        what = "TsdfVolume::raycastIntensity"
        box = _box_args(lo, dims, what)
        img, inten = DeviceImage(width, height, "float32"), DeviceImage(width, height, "float32")
        T = _pose12(T_curr_world)
        if box is not None:
            self._raycast_box(what, box, cam, T, width, height, img, inten=inten)
            self.sync()
            return img.getDevData(), inten.getDevData()
        check(self._L.rmd_volume_raycast_intensity(self._h, int(width), int(height), cam.fx, cam.fy, cam.cx, cam.cy,
                                                   T.ctypes.data, img.data, img.pitch, inten.data, inten.pitch),
              "TsdfVolume::raycastIntensity")
        self.sync()
        return img.getDevData(), inten.getDevData()

    def raycastNormals(self, cam: PinholeCamera, T_curr_world, width: int, height: int, lo=None, dims=None):
        """(depth float32 [height, width], normals float32 [height, width, 3]): raycast()'s depth, bit for bit, and
        the world-frame unit normal of the fused surface at each hit, (0, 0, 0) where there is no hit or no
        normal.  lo, dims: a box of the map, as raycast()."""
        what = "TsdfVolume::raycastNormals"
        box = _box_args(lo, dims, what)
        img, nrm = DeviceImage(width, height, "float32"), DeviceImage(4 * int(width), height, "float32")
        T = _pose12(T_curr_world)
        if box is not None:
            self._raycast_box(what, box, cam, T, width, height, img, nrm=nrm)
        else:
            check(self._L.rmd_volume_raycast_normals(self._h, int(width), int(height), cam.fx, cam.fy, cam.cx,
                                                     cam.cy, T.ctypes.data, img.data, img.pitch, nrm.data, nrm.pitch),
                  what)
        self.sync()
        return img.getDevData(), np.ascontiguousarray(nrm.getDevData().reshape(int(height), int(width), 4)[..., :3])

    def shift(self, d) -> None:
        """Move the grid by whole voxels d = (dx, dy, dz): voxel (i, j, k) then holds what voxel (i + dx, j + dy,
        k + dz) held, unknown where that lies outside the grid, and the origin moves by d * voxel_size (from the
        creation origin and the total offset, so it never accumulates rounding).  Asynchronous on the volume's
        stream.  Take the surface that leaves the grid with spillPoints(d) etc. first."""
        a = self._offset(d)
        check(self._L.rmd_volume_shift(self._h, a.ctypes.data), "TsdfVolume::shift")
        o = np.empty(3, _f32)
        check(self._L.rmd_volume_size(self._h, None, None, None, None, o.ctypes.data), "TsdfVolume::shift")
        self.origin = o

    @staticmethod
    def _offset(d) -> np.ndarray:
        a = np.asarray(d)
        if a.shape != (3,) or not np.all(a == np.round(a)) or np.any(np.abs(a.astype(np.float64)) > 2**31 - 1):
            raise ValueError("TsdfVolume: d must be three whole voxel counts")
        return np.ascontiguousarray(a.astype(np.int32))

    def _spill(self, fn, d, capacity, shape, what: str) -> np.ndarray:
        a = self._offset(d)
        return self._surface(lambda h, out, cap, n: fn(h, a.ctypes.data, out, cap, n), capacity, shape, what)

    def spillPoints(self, d, capacity: "int | None" = None) -> np.ndarray:
        """The surface points a shift by d would drop (call it before shift(d)): the subsequence of surfacePoints()
        whose voxel or neighbour leaves the grid, in that order and bit for bit.  With a capacity, at most that
        many."""
        return self._spill(self._L.rmd_volume_spill_points, d, capacity, (4,), "TsdfVolume::spillPoints")

    def spillIntensity(self, d, capacity: "int | None" = None) -> np.ndarray:
        """surfaceIntensity() of the points spillPoints(d) returns, in its order."""
        return self._spill(self._L.rmd_volume_spill_intensity, d, capacity, (), "TsdfVolume::spillIntensity")

    def spillNormals(self, d, capacity: "int | None" = None) -> np.ndarray:
        """float32 [n, 3]: surfaceNormals() of the points spillPoints(d) returns, in its order."""
        n = self._spill(self._L.rmd_volume_spill_normals, d, capacity, (4,), "TsdfVolume::spillNormals")
        return np.ascontiguousarray(n[:, :3])

    def spillMesh(self, d, vertex_capacity: "int | None" = None, triangle_capacity: "int | None" = None):
        """The mesh a shift by d would drop (call it before shift(d)): (float32 [n, 4] vertices, int32 [m, 3]
        triangles, int64 [n, 4] ids).  The triangles are mesh()'s of the meshed cubes with a corner leaving the grid,
        in mesh() order; the vertices are the subsequence of surfacePoints() made of the points that spill and the
        seam points those triangles share with the grid that stays.  An id (i + Dx, j + Dy, k + Dz, axis) names the
        vertex's grid edge across shifts (D = offset); SceneMesh welds by it.  With capacities, at most that many of
        each.  Raises RmdError (RMD_ERR_UNSUPPORTED) for 2^31 or more vertices."""
        a = self._offset(d)
        nv, nt = ctypes.c_size_t(), ctypes.c_size_t()
        what = "TsdfVolume::spillMesh"
        if vertex_capacity is None or triangle_capacity is None:
            check(self._L.rmd_volume_spill_mesh(self._h, a.ctypes.data, None, 0, None, 0, None, ctypes.byref(nv),
                                                ctypes.byref(nt)), what)
            vertex_capacity = nv.value if vertex_capacity is None else vertex_capacity
            triangle_capacity = nt.value if triangle_capacity is None else triangle_capacity
        verts = np.empty((int(vertex_capacity), 4), np.float32)
        tris = np.empty((int(triangle_capacity), 3), np.int32)
        ids = np.empty((int(vertex_capacity), 4), np.int64)
        check(self._L.rmd_volume_spill_mesh(self._h, a.ctypes.data, verts.ctypes.data if vertex_capacity else None,
                                            int(vertex_capacity), tris.ctypes.data if triangle_capacity else None,
                                            int(triangle_capacity), ids.ctypes.data if vertex_capacity else None,
                                            ctypes.byref(nv), ctypes.byref(nt)), what)
        m = min(int(vertex_capacity), nv.value)
        return verts[:m], tris[:min(int(triangle_capacity), nt.value)], ids[:m]

    def spillMeshIntensity(self, d, capacity: "int | None" = None) -> np.ndarray:
        """surfaceIntensity() of the vertices spillMesh(d) returns, in its order."""
        return self._spill(self._L.rmd_volume_spill_mesh_intensity, d, capacity, (), "TsdfVolume::spillMeshIntensity")

    def spillMeshNormals(self, d, capacity: "int | None" = None) -> np.ndarray:
        """float32 [n, 3]: surfaceNormals() of the vertices spillMesh(d) returns, in its order."""
        n = self._spill(self._L.rmd_volume_spill_mesh_normals, d, capacity, (4,), "TsdfVolume::spillMeshNormals")
        return np.ascontiguousarray(n[:, :3])

    def surfaceIds(self, capacity: "int | None" = None) -> np.ndarray:
        """int64 [n, 4]: the id (as spillMesh's) of every surface point (and mesh vertex), in surfacePoints()
        order."""
        n = ctypes.c_size_t()
        if capacity is None:
            check(self._L.rmd_volume_surface_ids(self._h, None, 0, ctypes.byref(n)), "TsdfVolume::surfaceIds")
            capacity = n.value
        out = np.empty((int(capacity), 4), np.int64)
        check(self._L.rmd_volume_surface_ids(self._h, out.ctypes.data if capacity else None, int(capacity),
                                             ctypes.byref(n)), "TsdfVolume::surfaceIds")
        return out[:min(int(capacity), n.value)]

    @property
    def offset(self) -> np.ndarray:
        """int64 [3]: the total offset in voxels, the sum of every shift."""
        D = np.empty(3, np.int64)
        check(self._L.rmd_volume_offset(self._h, D.ctypes.data), "TsdfVolume::offset")
        return D

    def enableStore(self) -> None:
        """Turn the brick store on (no-op when it is): from then on shift() keeps the 8x8x8 bricks of the unbounded
        grid that leave the window with a known voxel in device memory, and restores the voxels that re-enter, so
        that shift(d) then shift(-d) gives back the window bit for bit (DESIGN.md 4.8).  Every shift with a new
        candidate brick then synchronises the volume's stream once."""
        check(self._L.rmd_volume_enable_store(self._h), "TsdfVolume::enableStore")
        self.store = True

    def storeInfo(self):
        """(stored bricks, bytes of device memory the store's pool holds)."""
        n, b = ctypes.c_size_t(), ctypes.c_size_t()
        check(self._L.rmd_volume_store_info(self._h, ctypes.byref(n), ctypes.byref(b)), "TsdfVolume::storeInfo")
        return n.value, b.value

    def downloadStore(self, capacity: "int | None" = None, records: bool = True):
        """The stored bricks in ascending (z, y, x): (coords int64 [m, 3] brick coordinates (bx, by, bz), tsdf,
        weight[, intensity, intensity weight] float32 [m, 8, 8, 8] indexed (z, y, x) like download()); voxels inside
        the window are (0, 0).  The intensity pair comes with the channel; records=False returns the coords alone.
        With a capacity, at most that many bricks."""
        what = "TsdfVolume::downloadStore"
        n = ctypes.c_size_t()
        if capacity is None:
            check(self._L.rmd_volume_download_store(self._h, None, None, None, None, None, 0, ctypes.byref(n)), what)
            capacity = n.value
        m = int(capacity)
        coords = np.empty((m, 3), np.int64)
        arrs = [np.empty((m, 8, 8, 8), np.float32) for _ in range((2 + 2 * self.intensity) if records else 0)]
        ptrs = [a.ctypes.data if m else None for a in arrs] + [None] * (4 - len(arrs))
        check(self._L.rmd_volume_download_store(self._h, coords.ctypes.data if m else None, *ptrs, m,
                                                ctypes.byref(n)), what)
        k = min(m, n.value)
        if not records:
            return coords[:k]
        return (coords[:k],) + tuple(a[:k] for a in arrs)

    def uploadStore(self, coords, tsdf, weight, intensity=None, intensity_weight=None) -> None:
        """Replace the store with the bricks given as downloadStore() returns them (intensity pair optional: zeroed
        colour records).  Voxels inside the window are ignored."""
        what = "TsdfVolume::uploadStore"
        c = np.ascontiguousarray(coords, np.int64)
        if c.ndim != 2 or c.shape[1] != 3:
            raise ValueError(what + ": coords must be [m, 3]")
        m = len(c)
        arrs = [np.ascontiguousarray(a, np.float32) for a in (tsdf, weight)]
        if (intensity is None) != (intensity_weight is None):
            raise ValueError(what + ": intensity and its weight come together")
        if intensity is not None:
            arrs += [np.ascontiguousarray(a, np.float32) for a in (intensity, intensity_weight)]
        if any(a.size != m * 512 for a in arrs):
            raise ValueError(what + ": records must be [m, 8, 8, 8]")
        ptrs = [a.ctypes.data if m else None for a in arrs] + [None] * (4 - len(arrs))
        check(self._L.rmd_volume_upload_store(self._h, c.ctypes.data if m else None, *ptrs, m), what)

    def mapMesh(self, intensity: bool = False, normals: bool = False):
        """One mesh of the whole map -- the store and the window -- as SceneMesh.mesh returns it: (float32 [n, 4]
        vertices, int32 [m, 3] triangles, float32 [n] intensity or None, float32 [n, 3] normals or None), ready for
        write_ply (DESIGN.md 4.8).  The window sweeps the map: tiles of its size with stride n - 1 per axis, anchored
        at the lowest corner of the stored bricks once the window's own have been stored, so that every cube lies in
        exactly one tile.  At each tile that meets a stored brick, in ascending (z, y, x), it takes mesh() and
        surfaceIds(); vertices are welded by id, keeping the first tile's values.  The volume then shifts back: its
        window, offset and store are as before, bit for bit.  Requires the store; empty when an axis has n < 2."""
        if not self.store:
            raise RmdError("TsdfVolume::mapMesh: the volume has no brick store", -2)
        n = np.asarray(self.dims, np.int64)
        D0 = self.offset
        empty = (np.empty((0, 4), np.float32), np.empty((0, 3), np.int32),
                 np.empty(0, np.float32) if intensity else None, np.empty((0, 3), np.float32) if normals else None)
        if np.any(n < 2):
            return empty
        self.shift(n)   # every brick of the window with a known voxel goes to the store
        bricks = self.downloadStore(records=False)
        if not len(bricks):
            self.shift(D0 - self.offset)
            return empty
        A, step = bricks.min(0) * 8, n - 1
        # tiles t per axis whose voxels [A + t step, A + t step + n) meet a brick's [8 b, 8 b + 8)
        lo = np.maximum(0, -((A + n - 1 - 8 * bricks) // step))
        hi = (8 * bricks + 7 - A) // step
        tiles = set()
        for a, b in zip(lo, hi):
            for tz in range(a[2], b[2] + 1):
                for ty in range(a[1], b[1] + 1):
                    for tx in range(a[0], b[0] + 1):
                        tiles.add((tz, ty, tx))
        V, T, I, N, ids, base = [], [], [], [], [], 0
        for tz, ty, tx in sorted(tiles):
            self.shift(A + np.array([tx, ty, tz], np.int64) * step - self.offset)
            verts, tris = self.mesh()
            V.append(verts)
            T.append(tris.astype(np.int64) + base)
            ids.append(self.surfaceIds())
            if intensity:
                I.append(self.surfaceIntensity())
            if normals:
                N.append(self.surfaceNormals())
            base += len(verts)
        self.shift(D0 - self.offset)
        ids = np.concatenate(ids)
        _, first, inv = np.unique(ids, axis=0, return_index=True, return_inverse=True)
        order = np.argsort(first)
        rank = np.empty(len(order), np.int64)
        rank[order] = np.arange(len(order))
        keep = first[order]
        if len(keep) >= 2 ** 31:
            raise ValueError("TsdfVolume::mapMesh: 2^31 or more vertices do not fit int32 indices")
        tri = rank[inv.reshape(-1)][np.concatenate(T)].astype(np.int32)
        return (np.concatenate(V)[keep], tri.reshape(-1, 3),
                np.concatenate(I)[keep] if intensity else None, np.concatenate(N)[keep] if normals else None)

    def computeEsdf(self, lo=None, dims=None) -> None:
        """Compute the Euclidean signed distance field of the current window (DESIGN.md 4.8): per voxel the distance
        in metres to the nearest occupied voxel (weight > 0 and tsdf <= 0) for a free or unknown voxel, minus the
        distance to the nearest other voxel for an occupied one; +inf / -inf everywhere when no voxel is occupied /
        free.  Obstacles outside the window are not seen.  Asynchronous on the volume's stream; the snapshot and its
        origin stay as they are until the next computeEsdf(), whatever the volume does meanwhile.  The first call
        allocates 16 B per voxel.  Raises RmdError (RMD_ERR_UNSUPPORTED) unless (nx-1)^2 + (ny-1)^2 + (nz-1)^2 < 2^24.

        With lo (int [3], window indices, may be negative or outside the window) and dims (int [3], each > 0): the
        same over that box of the map.  Each box voxel takes the window's record, else (with the store) its stored
        brick's, else unknown; the snapshot's origin is origin + lo * voxel_size from the creation origin and the
        total offset, so esdfQuery answers around the box and obstacles in the store count.  24 B per box voxel.
        esdfBox() tells which box the snapshot answers for."""
        what = "TsdfVolume::computeEsdf"
        box = _box_args(lo, dims, what)
        if box is None:
            check(self._L.rmd_volume_esdf(self._h), what)
            return
        lo64, m32 = box
        check(self._L.rmd_volume_esdf_box(self._h, lo64.ctypes.data, m32.ctypes.data), what)

    def esdfBox(self):
        """(lo_unbounded int64 [3], dims (mx, my, mz), origin float32 [3]) of the box the snapshot answers for: its
        lowest voxel of the unbounded grid (offset + lo at the compute), its size and the world position of its voxel
        (0, 0, 0).  The window's box after computeEsdf()."""
        lo, m, o = np.empty(3, np.int64), np.empty(3, np.int32), np.empty(3, np.float32)
        check(self._L.rmd_volume_esdf_info(self._h, lo.ctypes.data, m.ctypes.data, o.ctypes.data),
              "TsdfVolume::esdfBox")
        return lo, tuple(int(x) for x in m), o

    def downloadEsdf(self):
        """(distance, weight) of the snapshot, float32 arrays of shape (mz, my, mx), the dims of its box (the
        window's after computeEsdf()); weight = the records' weight at the compute (0 = unknown)."""
        _, (mx, my, mz), _ = self.esdfBox()
        a, b = np.empty((mz, my, mx), np.float32), np.empty((mz, my, mx), np.float32)
        check(self._L.rmd_volume_download_esdf(self._h, a.ctypes.data, b.ctypes.data), "TsdfVolume::downloadEsdf")
        return a, b

    def esdfQuery(self, points):
        """(dg float32 [N, 4] = (distance, d/dx, d/dy, d/dz), weight float32 [N]) at world points [N, 3] or [N, 4]
        (w ignored, so surfacePoints() can be queried as it is): the snapshot trilinear at each point and its
        gradient in metres; weight = the min of the cell's 8 corner weights.  Outside the window: distance NaN,
        gradient 0, weight 0."""
        p = np.asarray(points, np.float32)
        if p.ndim != 2 or p.shape[1] not in (3, 4):
            raise ValueError("TsdfVolume::esdfQuery: points must be [N, 3] or [N, 4]")
        xyzw = np.zeros((len(p), 4), np.float32)
        xyzw[:, :p.shape[1]] = p
        dg, w = np.empty((len(p), 4), np.float32), np.empty(len(p), np.float32)
        n = len(p)
        check(self._L.rmd_volume_esdf_query(self._h, xyzw.ctypes.data if n else None, n,
                                            dg.ctypes.data if n else None, w.ctypes.data if n else None),
              "TsdfVolume::esdfQuery")
        return dg, w

    def esdfQueryDevice(self, dev_xyzw: int, n: int, dev_dg: int, dev_weight: "int | None" = None) -> None:
        """esdfQuery on device memory: n float4 points at dev_xyzw, n float4 (distance, gradient) to dev_dg and,
        when given, n float weights to dev_weight.  Asynchronous on the volume's stream."""
        check(self._L.rmd_volume_esdf_query_device(self._h, dev_xyzw, int(n), dev_dg, dev_weight),
              "TsdfVolume::esdfQueryDevice")

    def _download_records(self, fn, what: str):
        """The two halves of a record array (fn: rmd_volume_download[_intensity]), float32 of shape (nz, ny, nx)."""
        nx, ny, nz = self.dims
        a, b = np.empty((nz, ny, nx), np.float32), np.empty((nz, ny, nx), np.float32)
        check(fn(self._h, a.ctypes.data, b.ctypes.data), what)
        return a, b

    def _upload_records(self, fn, a, b, what: str) -> None:
        nx, ny, nz = self.dims
        a, b = (np.ascontiguousarray(x, np.float32) for x in (a, b))
        if a.size != nx * ny * nz or b.size != nx * ny * nz:
            raise ValueError(what + ": wrong size")
        check(fn(self._h, a.ctypes.data, b.ctypes.data), what)

    def download(self):
        """(tsdf, weight), float32 arrays of shape (nz, ny, nx)."""
        return self._download_records(self._L.rmd_volume_download, "TsdfVolume::download")

    def upload(self, tsdf, weight) -> None:
        self._upload_records(self._L.rmd_volume_upload, tsdf, weight, "TsdfVolume::upload")

    def downloadIntensity(self):
        """(intensity, intensity weight), float32 arrays of shape (nz, ny, nx)."""
        return self._download_records(self._L.rmd_volume_download_intensity, "TsdfVolume::downloadIntensity")

    def uploadIntensity(self, intensity, weight) -> None:
        self._upload_records(self._L.rmd_volume_upload_intensity, intensity, weight, "TsdfVolume::uploadIntensity")

    def reset(self) -> None:
        check(self._L.rmd_volume_reset(self._h), "TsdfVolume::reset")

    def setStream(self, cuda_stream: int) -> None:
        check(self._L.rmd_volume_set_stream(self._h, cuda_stream), "TsdfVolume::setStream")

    def sync(self) -> None:
        check(self._L.rmd_volume_sync(self._h), "TsdfVolume::sync")


def write_ply(path: str, vertices, triangles, intensity=None, normals=None) -> None:
    """Binary little-endian PLY of a mesh such as TsdfVolume.mesh() returns: per vertex float x, y, z and the
    weight as float `weight`; per face a uchar-counted int list `vertex_indices`.  With `normals` (one [3] per
    vertex, e.g. TsdfVolume.surfaceNormals()), each vertex also gets float nx, ny, nz for smooth shading.  With
    `intensity` (one value per vertex in [0, 1], e.g. TsdfVolume.surfaceIntensity()), each vertex then gets uchar
    red, green, blue = clip(rint(255 i), 0, 255); -1 (no intensity) is written as 0."""
    v = np.ascontiguousarray(vertices, "<f4").reshape(-1, 4)
    t = np.ascontiguousarray(triangles, "<i4").reshape(-1, 3)
    faces = np.empty(len(t), np.dtype([("n", "u1"), ("i", "<i4", 3)]))
    faces["n"], faces["i"] = 3, t
    fields, values, extra = [("p", "<f4", 4)], [v], ""
    if normals is not None:
        n = np.asarray(normals, np.float32)
        if n.shape != (len(v), 3):
            raise ValueError("write_ply: one normal (nx, ny, nz) per vertex")
        fields.append(("n", "<f4", 3))
        values.append(n)
        extra += "property float nx\nproperty float ny\nproperty float nz\n"
    if intensity is not None:
        i = np.asarray(intensity, np.float32).reshape(-1)
        if len(i) != len(v):
            raise ValueError("write_ply: one intensity per vertex")
        with np.errstate(invalid="ignore"):
            g = np.clip(np.rint(np.float32(255) * i), 0, 255)
        g = np.where(np.isfinite(g), g, 0).astype(np.uint8)
        fields.append(("c", "u1", 3))
        values.append(np.repeat(g[:, None], 3, 1))
        extra += "property uchar red\nproperty uchar green\nproperty uchar blue\n"
    if len(fields) > 1:
        rec = np.empty(len(v), np.dtype(fields))
        for (name, *_), val in zip(fields, values):
            rec[name] = val
        v = rec
    header = ("ply\nformat binary_little_endian 1.0\n"
              "element vertex %d\nproperty float x\nproperty float y\nproperty float z\nproperty float weight\n"
              "%selement face %d\nproperty list uchar int vertex_indices\nend_header\n" % (len(v), extra, len(t)))
    with open(path, "wb") as f:
        f.write(header.encode("ascii"))
        f.write(v.tobytes())
        f.write(faces.tobytes())


class SceneMesh:
    """One mesh of everything a moving TsdfVolume has seen (DESIGN.md 4.8): the spill mesh of every shift, then the
    current window's mesh(), welded by vertex id.  Call addSpill(volume, d) before each volume.shift(d); mesh(volume)
    returns the scene so far and can be called at any time.

    A vertex whose id is pending -- a seam vertex of an earlier chunk whose two voxels are still in the grid -- reuses
    that vertex; any other vertex is new.  After a chunk, the pending ids with a voxel outside the kept box are dropped
    (that surface has left the grid, and a voxel that re-enters later starts new vertices), and the chunk's seam
    vertices become pending.  With intensity / normals, the vertices' spill-mesh and surface intensities / normals
    are kept as well; a welded vertex keeps those of the chunk that first had it.

    Not for a volume with the brick store: a region it revisits comes back from the store and would spill a second
    time, so its surface would be added twice.  TsdfVolume.mapMesh meshes such a volume's whole map."""

    def __init__(self, intensity: bool = False, normals: bool = False):
        self.intensity, self.normals = bool(intensity), bool(normals)
        self._verts, self._tris, self._inten, self._nrm = [], [], [], []
        self._n = 0                                   # vertices so far
        self._pend_ids = np.empty((0, 4), np.int64)   # pending ids and their vertex indices
        self._pend_idx = np.empty(0, np.int64)

    def _weld(self, ids):
        """(index of each id: the pending vertex's, else a new one from the vertex count on in order; mask of the new
        ones)."""
        ids = np.asarray(ids, np.int64).reshape(-1, 4)
        idx = np.full(len(ids), -1, np.int64)
        if len(self._pend_ids) and len(ids):
            _, inv = np.unique(np.concatenate([self._pend_ids, ids]), axis=0, return_inverse=True)
            inv = inv.reshape(-1)
            pend_of = np.full(int(inv.max()) + 1, -1, np.int64)
            pend_of[inv[:len(self._pend_ids)]] = self._pend_idx
            idx = pend_of[inv[len(self._pend_ids):]]
        new = idx < 0
        idx[new] = self._n + np.arange(int(new.sum()), dtype=np.int64)
        return idx, new

    def _chunk(self, verts, tris, ids, inten, nrm):
        idx, new = self._weld(ids)
        if self._n + int(new.sum()) >= 2 ** 31:
            raise ValueError("SceneMesh: 2^31 or more vertices do not fit int32 indices")
        tri = idx[np.asarray(tris, np.int64).reshape(-1, 3)].astype(np.int32)
        chunk = (np.asarray(verts, np.float32).reshape(-1, 4)[new], tri,
                 None if inten is None else np.asarray(inten, np.float32).reshape(-1)[new],
                 None if nrm is None else np.asarray(nrm, np.float32).reshape(-1, 3)[new])
        return idx, new, chunk

    def addSpill(self, volume, d) -> None:
        """Append the spill mesh of volume's shift by d; call it before volume.shift(d)."""
        d = np.asarray(d, np.int64).reshape(3)
        verts, tris, ids = volume.spillMesh(d)
        inten = volume.spillMeshIntensity(d) if self.intensity else None
        nrm = volume.spillMeshNormals(d) if self.normals else None
        idx, new, chunk = self._chunk(verts, tris, ids, inten, nrm)
        for store, part in zip((self._verts, self._tris, self._inten, self._nrm), chunk):
            store.append(part)
        self._n += int(new.sum())
        # the kept box K in unbounded-grid voxels, as rmd_volume_spill_*: d clamped to [-n, n]
        n = np.asarray(volume.dims, np.int64)
        c = np.clip(d, -n, n)
        D = np.asarray(volume.offset, np.int64)
        lo, hi = D + np.maximum(c, 0), D + np.where(c < 0, n + c, n)
        ids = np.asarray(ids, np.int64).reshape(-1, 4)
        reused = np.isin(self._pend_idx, idx[~new])
        all_ids = np.concatenate([self._pend_ids[~reused], ids])
        all_idx = np.concatenate([self._pend_idx[~reused], idx])
        a = all_ids[:, :3]
        b = a + np.eye(3, dtype=np.int64)[all_ids[:, 3]]
        keep = np.all((a >= lo) & (a < hi) & (b >= lo) & (b < hi), axis=1)
        self._pend_ids, self._pend_idx = all_ids[keep], all_idx[keep]

    def mesh(self, volume):
        """(float32 [n, 4] vertices, int32 [m, 3] triangles, float32 [n] intensity or None, float32 [n, 3] normals or
        None) of the chunks added so far and volume's current mesh(), welded alike: the chunks in the order they were
        added, then the window, each with its new vertices in its own order.  Ready for write_ply.  The accumulated
        state is not changed."""
        verts, tris = volume.mesh()
        inten = volume.surfaceIntensity() if self.intensity else None
        nrm = volume.surfaceNormals() if self.normals else None
        _, _, chunk = self._chunk(verts, tris, volume.surfaceIds(), inten, nrm)
        return (np.concatenate(self._verts + [chunk[0]]), np.concatenate(self._tris + [chunk[1]]),
                np.concatenate(self._inten + [chunk[2]]) if self.intensity else None,
                np.concatenate(self._nrm + [chunk[3]]) if self.normals else None)


class ImageReducer:
    """rmd::ImageReducer<T> -- include/rmd/reduction.cuh:27-62.  The launch
    shape arguments of the reference are accepted and ignored (the kernel
    sizes its own grid)."""

    def __init__(self, dtype="float32", num_threads_per_block=None, num_blocks_per_grid=None):
        self.dtype = np.dtype(dtype).name
        if self.dtype not in ("float32", "int32"):
            raise TypeError("ImageReducer<T>: T must be float32 or int32 (src/reduction.cu:186-187)")
        self._L = _native.lib()

    def sum(self, img: DeviceImage):
        if img.dtype != self.dtype:
            raise TypeError("ImageReducer::sum: element type mismatch")
        if self.dtype == "float32":
            out = ctypes.c_float()
            check(self._L.rmd_reduce_sum_f32(img.data, img.stride, img.width, img.height, ctypes.byref(out)),
                  "sum")
            return float(out.value)
        out = ctypes.c_int32()
        check(self._L.rmd_reduce_sum_i32(img.data, img.stride, img.width, img.height, ctypes.byref(out)), "sum")
        return int(out.value)

    def countEqual(self, img: DeviceImage, value: int) -> int:
        if img.dtype != "int32":
            raise TypeError("countEqual is only instantiated for int (src/reduction.cu:134)")
        out = ctypes.c_size_t()
        check(self._L.rmd_reduce_count_eq_i32(img.data, img.stride, img.width, img.height, int(value),
                                              ctypes.byref(out)), "countEqual")
        return int(out.value)

    def minMax(self, img: DeviceImage):
        lo, hi = ctypes.c_float(), ctypes.c_float()
        check(self._L.rmd_reduce_min_max_f32(img.data, img.stride, img.width, img.height,
                                             ctypes.byref(lo), ctypes.byref(hi)), "minMax")
        return float(lo.value), float(hi.value)


class Depthmap:
    """rmd::Depthmap -- include/rmd/depthmap.h:34-129, src/depthmap.cpp, without
    OpenCV: frames are numpy uint8 (h, w) arrays; the 8U -> 32F * (1/255)
    conversion of inputImage (src/depthmap.cpp:105) runs on the GPU."""

    def __init__(self, width, height, fx, cx, fy, cy, patch_side=5, device=-1):
        self.width_, self.height_ = int(width), int(height)
        self.seeds_ = SeedMatrix(width, height, PinholeCamera(fx, fy, cx, cy), patch_side, device)
        self.denoiser_ = DepthmapDenoiser(width, height, device)
        self.output_depth_32fc1_ = np.zeros((height, width), np.float32)
        self.output_convergence_int_ = np.zeros((height, width), np.int32)
        self.ref_img_undistorted_8uc1_ = np.zeros((height, width), np.uint8)
        self.T_world_ref_ = SE3()
        self.is_distorted_ = False
        self.denoised_dev_ = None   # device copy of the denoised map for fuseDenoisedInto, allocated on first use

    def initUndistortionMap(self, k1, k2, r1, r2):
        """src/depthmap.cpp:45-61; the maps and the per-frame remap live on the GPU."""
        self.seeds_.initUndistortionMap(k1, k2, r1, r2)
        self.is_distorted_ = True

    def setReferenceImage(self, img_curr, T_curr_world, min_depth, max_depth) -> bool:
        self.denoiser_.setLargeSigmaSq(max_depth - min_depth)          # src/depthmap.cpp:69
        img = self._input_image(img_curr)
        ret = self.seeds_.setReferenceImage(img, T_curr_world, min_depth, max_depth)
        # img_undistorted_8uc1_.copyTo(ref_img_undistorted_8uc1_), src/depthmap.cpp:78
        self.ref_img_undistorted_8uc1_ = self.seeds_.undistort(img) if self.is_distorted_ else np.array(img, copy=True)
        self.T_world_ref_ = (T_curr_world if isinstance(T_curr_world, SE3) else SE3(T_curr_world)).inv()
        return ret

    def setPriorPropagation(self, sigma_sq_frac: float = PRIOR_SIGMA_SQ_FRAC) -> None:
        """Each new reference frame takes its depth prior from the converged seeds of the keyframe it replaces
        (SeedMatrix.setPriorPropagation); 0 switches it off (the default of a new Depthmap)."""
        self.seeds_.setPriorPropagation(sigma_sq_frac)

    def priorFromVolume(self, volume: TsdfVolume, sigma_sq_frac: float = PRIOR_SIGMA_SQ_FRAC, lo=None,
                        dims=None) -> None:
        """After setReferenceImage: the new keyframe's depth prior from the model fused so far, or with lo and dims
        from that box of the map (SeedMatrix.priorFromVolume)."""
        self.seeds_.priorFromVolume(volume, sigma_sq_frac, lo, dims)

    def update(self, img_curr, T_curr_world) -> None:
        self.seeds_.update(self._input_image(img_curr), T_curr_world)

    def downloadDepthmap(self) -> None:
        self.output_depth_32fc1_ = self.seeds_.downloadDepthmap()

    def downloadDenoisedDepthmap(self, lam, iterations) -> None:
        self.output_depth_32fc1_ = self.denoiser_.denoiseSeeds(self.seeds_, lam, iterations)

    def fuseDenoisedInto(self, volume: TsdfVolume, lam, iterations) -> None:
        """downloadDenoisedDepthmap (the same host map, bit for bit) and the keyframe's integration into `volume`
        from the denoised device image, masked by the CONVERGED seeds: one denoiser run for both."""
        if self.denoised_dev_ is None:
            self.denoised_dev_ = DeviceImage(self.width_, self.height_, "float32")
        img = self.denoised_dev_
        self.denoiser_.denoiseSeedsToDevice(self.seeds_, img.data, img.pitch, lam, iterations)
        self.denoiser_.sync()
        self.output_depth_32fc1_ = img.getDevData()
        volume.integrate(self.seeds_, img)

    def getDepthmap(self):
        return self.output_depth_32fc1_

    def downloadConvergenceMap(self) -> None:
        self.output_convergence_int_ = self.seeds_.downloadConvergence()

    def getConvergenceMap(self):
        return self.output_convergence_int_

    def getReferenceImage(self):
        return self.ref_img_undistorted_8uc1_

    def getConvergedCount(self) -> int:
        return self.seeds_.getConvergedCount()

    def getConvergedPercentage(self) -> float:
        return float(self.getConvergedCount()) / float(self.width_ * self.height_) * 100.0

    def getDistFromRef(self) -> float:
        return self.seeds_.getDistFromRef()

    def getWidth(self):
        return self.width_

    def getHeight(self):
        return self.height_

    def getT_world_ref(self):
        return self.T_world_ref_

    def _input_image(self, img_8uc1):
        a = np.asarray(img_8uc1)
        if a.dtype != np.uint8:
            raise TypeError("Depthmap expects 8-bit gray frames (CV_8UC1)")
        return np.ascontiguousarray(a)
