"""In-tree build of the native libraries (nvcc for sm_90a, gcc for host C).

The CUDA library is plain nvcc + cudart (no torch, no pybind): the product is a
C-ABI shared object, ``rpg_open_remode_b200/librmd_b200.so``, that the
reference's C++ callers can link and Python reaches through ctypes.
"""
from __future__ import annotations

import os
import shutil
import subprocess

_HERE = os.path.dirname(os.path.abspath(__file__))
_CSRC = os.path.join(_HERE, "csrc")
LIB_PATH = os.path.join(_HERE, "librmd_b200.so")

CUDA_SOURCES = ["c_api.cu", "depth_filter.cu", "depth_filter_staged.cu", "depth_filter_seeds.cu", "denoiser.cu", "reduction.cu", "ingest.cu", "point_cloud.cu",
                "prior.cu", "volume.cu", "volume_api.cu", "multi_gpu.cu"]

NVCC_FLAGS = [
    "-std=c++17", "-O3",
    "-gencode", "arch=compute_90a,code=sm_90a",
    "-lineinfo",
    # same arithmetic contract as the reference's build (CMakeLists.txt:25)
    "-use_fast_math",
    "-Xcompiler", "-fPIC",
    "-Xptxas", "-v",
]


def nvcc_path() -> str:
    for cand in (os.environ.get("NVCC"), shutil.which("nvcc"), "/usr/local/cuda/bin/nvcc"):
        if cand and os.path.exists(cand):
            return cand
    raise RuntimeError("nvcc not found")


def _newest_source_mtime() -> float:
    newest = 0.0
    for root in (_CSRC, os.path.join(os.path.dirname(_HERE), "include")):
        for dirpath, _, files in os.walk(root):
            for f in files:
                newest = max(newest, os.path.getmtime(os.path.join(dirpath, f)))
    return newest


def build_cuda(force: bool = False, verbose: bool = False) -> str:
    """Compile every CUDA source for sm_90a into librmd_b200.so (in-tree)."""
    if not force and os.path.exists(LIB_PATH) and os.path.getmtime(LIB_PATH) >= _newest_source_mtime():
        return LIB_PATH
    objs = []
    build_dir = os.path.join(_HERE, "build")
    os.makedirs(build_dir, exist_ok=True)
    nvcc = nvcc_path()
    log = []
    for src in CUDA_SOURCES:
        obj = os.path.join(build_dir, src.replace(".cu", ".o"))
        cmd = [nvcc] + NVCC_FLAGS + ["-c", os.path.join(_CSRC, src), "-o", obj]
        res = subprocess.run(cmd, capture_output=True, text=True)
        log.append("$ " + " ".join(cmd) + "\n" + res.stdout + res.stderr)
        if res.returncode != 0:
            raise RuntimeError("nvcc failed:\n" + log[-1])
        objs.append(obj)
    cmd = [nvcc, "-shared", "-o", LIB_PATH] + objs + ["-gencode", "arch=compute_90a,code=sm_90a", "-lpthread", "-ldl",
                                                      ]
    res = subprocess.run(cmd, capture_output=True, text=True)
    log.append("$ " + " ".join(cmd) + "\n" + res.stdout + res.stderr)
    if res.returncode != 0:
        raise RuntimeError("link failed:\n" + log[-1])
    with open(os.path.join(build_dir, "build.log"), "w") as f:
        f.write("\n".join(log))
    if verbose:
        print("\n".join(log))
    return LIB_PATH


def build_all(force: bool = False) -> None:
    from . import synth
    build_cuda(force=force)
    synth.build(force=force)
