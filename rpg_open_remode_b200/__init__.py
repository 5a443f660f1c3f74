"""rpg_open_remode_b200 -- Hopper-native (sm_90a) REMODE depth-filter hot path.

The product is ``librmd_b200.so`` (C-ABI, ``include/rmd_b200.h``) plus
header-compatible C++ classes under ``include/rmd/``.  This package is the
Python host-side mirror of the same interface used by tests and ``bench.py``.
"""
from .api import (ConvergenceStates, DepthmapDenoiser, Depthmap, DeviceImage, ImageReducer,
                  PinholeCamera, SE3, SeedMatrix, RmdError,
                  FIELD_MU, FIELD_SIGMA_SQ, FIELD_A, FIELD_B, FIELD_CONVERGENCE, FIELD_SUM_TEMPL,
                  FIELD_CONST_TEMPL_DENOM, FIELD_EPIPOLAR_MATCHES, FIELD_REF_IMG,
                  OPT_RECORD_MATCHES, OPT_KERNEL_VARIANT, OPT_TEX_FRAC_BITS, OPT_DEBUG_TIMELINE, OPT_PINNED_INPUT, OPT_CHAIN_FRAMES, OPT_SEED_MODE_PCT,
                  OPT_TUNE_SPLIT_MAX, OPT_TUNE_SPLIT_MIN_ITEMS, OPT_TUNE_SPLIT_ITEMS_PER_CTA,
                  OPT_TUNE_SPARSE_MAX_SEEDS, OPT_TUNE_HEAVY_MIN_ITEMS, OPT_TUNE_SPLIT_AVG_PCT, OPT_TUNE_PDL, OPT_TUNE_WARP_TILE_SEEDS, OPT_TUNE_GRID_CTAS, OPT_TUNE_CTAS_PER_SM, OPT_TUNE_WARP_TILE_CANDS, OPT_TUNE_RUN_CHUNKS,
                  VARIANT_STAGED, VARIANT_DIRECT, PRIOR_SIGMA_SQ_FRAC, SceneMesh, TsdfVolume, write_ply)
from ._native import device_count

__all__ = [n for n in dir() if not n.startswith("_")]
