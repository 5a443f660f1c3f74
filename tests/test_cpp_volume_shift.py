"""The moving rmd::TsdfVolume (include/rmd/tsdf_volume.cuh) compile with a plain host compiler against the C-ABI
and, on the GPU, behave as tests/cpp/volume_shift_test.cpp checks."""
import os
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EXE = os.path.join(ROOT, "tests", "cpp", "build", "volume_shift_test")
CUDA = os.environ.get("CUDA_HOME", "/usr/local/cuda")


def _build():
    from rpg_open_remode_b200 import _build as b
    b.build_cuda()
    os.makedirs(os.path.dirname(EXE), exist_ok=True)
    pkg = os.path.join(ROOT, "rpg_open_remode_b200")
    cxx = "/usr/bin/g++" if os.path.exists("/usr/bin/g++") else "g++"
    cmd = [cxx, "-std=c++14", "-O1", "-DRMD_BUILD_TESTS=1",
           "-I" + os.path.join(ROOT, "include"), "-I" + os.path.join(CUDA, "include"),
           os.path.join(ROOT, "tests", "cpp", "volume_shift_test.cpp"), "-o", EXE,
           "-L" + pkg, "-lrmd_b200", "-L" + os.path.join(CUDA, "lib64"), "-lcudart",
           "-Wl,-rpath," + pkg + ":" + os.path.join(CUDA, "lib64")]
    subprocess.check_call(cmd)
    return EXE


def test_volume_shift_facade_compiles_with_host_compiler():
    assert os.path.exists(_build())


@pytest.mark.gpu
def test_volume_shift_facade_on_the_gpu():
    exe = _build()
    res = subprocess.run([exe], capture_output=True, text=True, timeout=600)
    print(res.stdout[-2000:], res.stderr[-2000:])
    assert res.returncode == 0, res.stdout[-2000:]
    assert "ALL VOLUME SHIFT TESTS PASSED" in res.stdout
