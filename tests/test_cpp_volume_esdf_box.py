"""The ESDF box from C++.

  * the brick table (csrc/volume_store.h, store_brick_table) is host-only code: built with the system compiler and run
    here, no GPU (tests/cpp/volume_esdf_box_test.cpp), against std::map lookups;
  * rmd::TsdfVolume's computeEsdf(lo, dims) and esdfInfo (include/rmd/tsdf_volume.cuh) compile with a plain host
    compiler against the C-ABI and, on the GPU, give what the same scene gives through the Python API, bit for bit
    (tests/cpp/volume_esdf_box_facade_test.cpp).
"""
import os
import subprocess

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
OUT = os.path.join(ROOT, "tests", "cpp", "build")
CXX = "/usr/bin/g++" if os.path.exists("/usr/bin/g++") else "g++"
CUDA = os.environ.get("CUDA_HOME", "/usr/local/cuda")


def test_brick_table_against_map_lookups():
    os.makedirs(OUT, exist_ok=True)
    exe = os.path.join(OUT, "volume_esdf_box_test")
    subprocess.check_call([CXX, "-std=c++14", "-O2", "-Wall", "-Wextra",
                           os.path.join(ROOT, "tests", "cpp", "volume_esdf_box_test.cpp"), "-o", exe])
    res = subprocess.run([exe], capture_output=True, text=True, timeout=600)
    assert res.returncode == 0 and "ALL VOLUME ESDF BOX HOST TESTS PASSED" in res.stdout, res.stdout[-2000:]


def _build_facade():
    from rpg_open_remode_b200 import _build as b
    b.build_cuda()
    os.makedirs(OUT, exist_ok=True)
    exe = os.path.join(OUT, "volume_esdf_box_facade_test")
    pkg = os.path.join(ROOT, "rpg_open_remode_b200")
    subprocess.check_call([CXX, "-std=c++14", "-O1", "-DRMD_BUILD_TESTS=1",
                           "-I" + os.path.join(ROOT, "include"), "-I" + os.path.join(CUDA, "include"),
                           os.path.join(ROOT, "tests", "cpp", "volume_esdf_box_facade_test.cpp"), "-o", exe,
                           "-L" + pkg, "-lrmd_b200", "-L" + os.path.join(CUDA, "lib64"), "-lcudart",
                           "-Wl,-rpath," + pkg + ":" + os.path.join(CUDA, "lib64")])
    return exe


def test_volume_esdf_box_facade_compiles_with_host_compiler():
    assert os.path.exists(_build_facade())


@pytest.mark.gpu
def test_volume_esdf_box_facade_matches_python(tmp_path):
    import rpg_open_remode_b200 as rmd
    exe = _build_facade()
    out = str(tmp_path / "facade.bin")
    res = subprocess.run([exe, out], capture_output=True, text=True, timeout=600)
    print(res.stdout[-2000:], res.stderr[-2000:])
    assert res.returncode == 0 and "ALL VOLUME ESDF BOX TESTS PASSED" in res.stdout, res.stdout[-2000:]

    # the same scene through the Python API
    N, W, H, s, R = 64, 160, 120, 0.0625, 1.2
    v = rmd.TsdfVolume((N, N, N), s, (-2.0, -2.0, -2.0), 4 * s, 16.0, device=0, store=True)
    cam = rmd.PinholeCamera(100.0, 100.0, (W - 1) / 2.0, (H - 1) / 2.0)
    v.integrateDepth(np.full((H, W), R, np.float32), cam, [1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1, 0])
    v.shift((0, 0, -20))
    v.computeEsdf((-4, -4, -4), (N + 8, N + 8, N + 28))
    lo_u, dims, origin = v.esdfBox()
    d, w = v.downloadEsdf()
    pts = np.array([[0, 0, 1.0], [0, 0, 0.6], [0, 0, 5.0]], np.float32)
    dg, wq = v.esdfQuery(pts)

    raw = open(out, "rb").read()
    nb = int(np.prod(dims))
    got_lo = np.frombuffer(raw, np.int64, 3, 0)
    got_dims = np.frombuffer(raw, np.int32, 3, 24)
    got_o = np.frombuffer(raw, np.float32, 3, 36)
    got_d = np.frombuffer(raw, np.float32, nb, 48)
    got_w = np.frombuffer(raw, np.float32, nb, 48 + 4 * nb)
    got_dg = np.frombuffer(raw, np.float32, 12, 48 + 8 * nb)
    got_wq = np.frombuffer(raw, np.float32, 3, 96 + 8 * nb)
    assert len(raw) == 108 + 8 * nb
    assert list(got_lo) == list(lo_u) == [-4, -4, -24] and tuple(got_dims) == dims
    assert np.array_equal(got_o.view(np.uint32), origin.view(np.uint32))
    assert np.array_equal(got_d.view(np.uint32), d.reshape(-1).view(np.uint32))
    assert np.array_equal(got_w.view(np.uint32), w.reshape(-1).view(np.uint32))
    assert np.array_equal(got_dg.view(np.uint32), dg.reshape(-1).view(np.uint32))
    assert np.array_equal(got_wq.view(np.uint32), wq.view(np.uint32))
