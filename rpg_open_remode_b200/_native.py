"""ctypes binding of librmd_b200.so (the C-ABI in include/rmd_b200.h).

There is NO fallback: if the CUDA library is missing or no H100 is present,
every entry point raises.  The CPU oracle under oracle/ is test infrastructure
and is never imported from here.
"""
from __future__ import annotations

import ctypes
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
# RMD_B200_LIB: load another build of the same library (e.g. the debug-counter build of tools/)
LIB_PATH = os.environ.get("RMD_B200_LIB") or os.path.join(_HERE, "librmd_b200.so")

vp, ci, cf, cs = ctypes.c_void_p, ctypes.c_int, ctypes.c_float, ctypes.c_size_t
u64 = ctypes.c_uint64
P = ctypes.POINTER

_SIGNATURES = {
    # name: (restype, argtypes)
    "rmd_abi_version": (ci, []),
    "rmd_last_error_string": (ctypes.c_char_p, []),
    "rmd_device_count": (ci, [P(ci)]),
    "rmd_seeds_create": (ci, [ci, ci, cf, cf, cf, cf, ci, ci, P(vp)]),
    "rmd_seeds_destroy": (ci, [vp]),
    "rmd_seeds_set_stream": (ci, [vp, vp]),
    "rmd_seeds_get_stream": (ci, [vp, P(vp)]),
    "rmd_seeds_set_option": (ci, [vp, ci, ci]),
    "rmd_seeds_set_reference": (ci, [vp, vp, vp, cf, cf]),
    "rmd_seeds_set_reference_device": (ci, [vp, vp, cs, vp, cf, cf]),
    "rmd_seeds_set_reference_u8": (ci, [vp, vp, vp, cf, cf]),
    "rmd_seeds_set_prior_propagation": (ci, [vp, cf]),
    "rmd_seeds_propagate_prior": (ci, [vp, vp, cf]),
    "rmd_seeds_update": (ci, [vp, vp, vp]),
    "rmd_seeds_update_u8": (ci, [vp, vp, vp]),
    "rmd_seeds_update_device": (ci, [vp, vp, cs, vp]),
    "rmd_seeds_update_device_batch": (ci, [vp, vp, cs, cs, ci, vp]),
    "rmd_seeds_sync": (ci, [vp]),
    "rmd_seeds_download": (ci, [vp, ci, vp]),
    "rmd_seeds_upload_state": (ci, [vp, ci, vp]),
    "rmd_seeds_device_ptr": (ci, [vp, ci, P(vp), P(cs)]),
    "rmd_seeds_copy_field_to_device": (ci, [vp, ci, vp, cs]),
    "rmd_seeds_converged_count": (ci, [vp, P(cs)]),
    "rmd_seeds_dist_from_ref": (ci, [vp, P(cf)]),
    "rmd_seeds_size": (ci, [vp, P(ci), P(ci), P(ci)]),
    "rmd_seeds_launch_count": (ci, [vp, P(u64), P(u64)]),
    "rmd_seeds_last_kernel_ms": (ci, [vp, P(cf)]),
    "rmd_seeds_enable_kernel_timing": (ci, [vp, ci]),
    "rmd_debug_host_profile": (ci, [P(ctypes.c_double), ci]),
    "rmd_seeds_init_undistortion_map": (ci, [vp, cf, cf, cf, cf]),
    "rmd_seeds_clear_undistortion_map": (ci, [vp]),
    "rmd_seeds_get_undistortion_map": (ci, [vp, vp, vp]),
    "rmd_seeds_undistort_u8": (ci, [vp, vp, vp]),
    "rmd_seeds_update_many": (ci, [P(vp), ci, vp, vp]),
    "rmd_seeds_update_many_u8": (ci, [P(vp), ci, vp, vp]),
    "rmd_seeds_point_cloud": (ci, [vp, vp, cs, vp, cs, P(cs)]),
    "rmd_seeds_point_cloud_device": (ci, [vp, vp, cs, vp, cs, P(cs)]),
    "rmd_denoiser_create": (ci, [ci, ci, ci, P(vp)]),
    "rmd_denoiser_destroy": (ci, [vp]),
    "rmd_denoiser_set_stream": (ci, [vp, vp]),
    "rmd_denoiser_set_large_sigma_sq": (ci, [vp, cf]),
    "rmd_denoiser_run": (ci, [vp, vp, cs, vp, cs, vp, cs, vp, cs, vp, cf, ci]),
    "rmd_denoiser_run_seeds": (ci, [vp, vp, vp, cf, ci]),
    "rmd_denoiser_run_seeds_to_device": (ci, [vp, vp, vp, cs, cf, ci]),
    "rmd_denoiser_sync": (ci, [vp]),
    "rmd_denoiser_launch_count": (ci, [vp, P(u64)]),
    "rmd_multi_create": (ci, [P(ci), ci, ci, ci, P(vp)]),
    "rmd_multi_unique_id": (ci, [ctypes.c_char_p]),
    "rmd_multi_create_rank": (ci, [ctypes.c_char_p, ci, ci, ci, ci, ci, P(vp)]),
    "rmd_multi_destroy": (ci, [vp]),
    "rmd_multi_size": (ci, [vp, P(ci), P(ci), P(ci)]),
    "rmd_multi_gather_maps": (ci, [vp, P(vp), P(vp), P(cs), ci, vp, vp]),
    "rmd_volume_create": (ci, [ci, ci, ci, cf, vp, cf, cf, ci, P(vp)]),
    "rmd_volume_destroy": (ci, [vp]),
    "rmd_volume_set_stream": (ci, [vp, vp]),
    "rmd_volume_reset": (ci, [vp]),
    "rmd_volume_sync": (ci, [vp]),
    "rmd_volume_size": (ci, [vp, P(ci), P(ci), P(ci), P(cf), vp]),
    "rmd_volume_integrate_seeds": (ci, [vp, vp, vp, cs]),
    "rmd_volume_integrate_depth": (ci, [vp, ci, ci, cf, cf, cf, cf, vp, vp, cs, vp, cs]),
    "rmd_volume_surface_points": (ci, [vp, vp, cs, P(cs)]),
    "rmd_volume_surface_points_device": (ci, [vp, vp, cs, P(cs)]),
    "rmd_volume_mesh": (ci, [vp, vp, cs, vp, cs, P(cs), P(cs)]),
    "rmd_volume_mesh_device": (ci, [vp, vp, cs, vp, cs, P(cs), P(cs)]),
    "rmd_volume_raycast": (ci, [vp, ci, ci, cf, cf, cf, cf, vp, vp, cs]),
    "rmd_volume_prior_seeds": (ci, [vp, vp, cf]),
    "rmd_volume_download": (ci, [vp, vp, vp]),
    "rmd_volume_upload": (ci, [vp, vp, vp]),
    "rmd_volume_enable_intensity": (ci, [vp]),
    "rmd_volume_integrate_depth_intensity": (ci, [vp, ci, ci, cf, cf, cf, cf, vp, vp, cs, vp, cs, vp, cs]),
    "rmd_volume_surface_intensity": (ci, [vp, vp, cs, P(cs)]),
    "rmd_volume_surface_intensity_device": (ci, [vp, vp, cs, P(cs)]),
    "rmd_volume_raycast_intensity": (ci, [vp, ci, ci, cf, cf, cf, cf, vp, vp, cs, vp, cs]),
    "rmd_volume_download_intensity": (ci, [vp, vp, vp]),
    "rmd_volume_upload_intensity": (ci, [vp, vp, vp]),
    "rmd_volume_surface_normals": (ci, [vp, vp, cs, P(cs)]),
    "rmd_volume_surface_normals_device": (ci, [vp, vp, cs, P(cs)]),
    "rmd_volume_raycast_normals": (ci, [vp, ci, ci, cf, cf, cf, cf, vp, vp, cs, vp, cs]),
    "rmd_volume_shift": (ci, [vp, vp]),
    "rmd_volume_spill_points": (ci, [vp, vp, vp, cs, P(cs)]),
    "rmd_volume_spill_intensity": (ci, [vp, vp, vp, cs, P(cs)]),
    "rmd_volume_spill_normals": (ci, [vp, vp, vp, cs, P(cs)]),
    "rmd_volume_spill_mesh": (ci, [vp, vp, vp, cs, vp, cs, vp, P(cs), P(cs)]),
    "rmd_volume_spill_mesh_intensity": (ci, [vp, vp, vp, cs, P(cs)]),
    "rmd_volume_spill_mesh_normals": (ci, [vp, vp, vp, cs, P(cs)]),
    "rmd_volume_surface_ids": (ci, [vp, vp, cs, P(cs)]),
    "rmd_volume_offset": (ci, [vp, vp]),
    "rmd_volume_enable_store": (ci, [vp]),
    "rmd_volume_store_info": (ci, [vp, P(cs), P(cs)]),
    "rmd_volume_download_store": (ci, [vp, vp, vp, vp, vp, vp, cs, P(cs)]),
    "rmd_volume_upload_store": (ci, [vp, vp, vp, vp, vp, vp, cs]),
    "rmd_reduce_sum_f32":(ci, [vp, cs, cs, cs, P(cf)]),
    "rmd_reduce_sum_i32": (ci, [vp, cs, cs, cs, P(ctypes.c_int32)]),
    "rmd_reduce_count_eq_i32": (ci, [vp, cs, cs, cs, ctypes.c_int32, P(cs)]),
    "rmd_reduce_min_max_f32": (ci, [vp, cs, cs, cs, P(cf), P(cf)]),
    "rmd_image_alloc": (ci, [cs, cs, cs, P(vp), P(cs)]),
    "rmd_image_free": (ci, [vp]),
    "rmd_image_upload": (ci, [vp, cs, vp, cs, cs, cs]),
    "rmd_image_download": (ci, [vp, cs, vp, cs, cs, cs]),
    "rmd_image_zero": (ci, [vp, cs, cs, cs, cs]),
    "rmd_image_copy": (ci, [vp, cs, vp, cs, cs, cs, cs]),
}

EXPORTED_SYMBOLS = tuple(_SIGNATURES)

_lib = None


class RmdError(RuntimeError):
    """Mirror of rmd::CudaException (include/rmd/cuda_exception.cuh:27-45):
    message + the cudaError / RMD_ERR_* code."""

    def __init__(self, what: str, code: int):
        super().__init__(f"{what} (code {code})")
        self.code = code


def lib():
    """Load the C-ABI library; raise if it has not been built."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise ImportError(
                f"{LIB_PATH} is missing: build it with `python -c 'import __graft_entry__ as g; g.build()'` "
                "-- there is no CPU fallback")
        L = ctypes.CDLL(LIB_PATH)
        for name, (res, args) in _SIGNATURES.items():
            fn = getattr(L, name)
            fn.restype = res
            fn.argtypes = args
        _lib = L
    return _lib


def check(code: int, what: str = "") -> None:
    if code != 0:
        msg = lib().rmd_last_error_string().decode(errors="replace")
        raise RmdError(f"{what}: {msg}" if what else msg, code)


def device_count() -> int:
    n = ci(0)
    code = lib().rmd_device_count(ctypes.byref(n))
    if code != 0:
        return 0
    return n.value
