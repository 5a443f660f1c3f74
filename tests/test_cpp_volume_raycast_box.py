"""The box raycasts and the box prior from C++: rmd::TsdfVolume's raycast / raycastIntensity / raycastNormals (..., lo,
dims) and seedPrior(seeds, f, lo, dims) (include/rmd/tsdf_volume.cuh) compile with a plain host compiler against the
C-ABI and, on the GPU, give what the same scene gives through the Python API, bit for bit
(tests/cpp/volume_raycast_box_facade_test.cpp).
"""
import os
import subprocess

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
OUT = os.path.join(ROOT, "tests", "cpp", "build")
CXX = "/usr/bin/g++" if os.path.exists("/usr/bin/g++") else "g++"
CUDA = os.environ.get("CUDA_HOME", "/usr/local/cuda")


def _build_facade():
    from rpg_open_remode_b200 import _build as b
    b.build_cuda()
    os.makedirs(OUT, exist_ok=True)
    exe = os.path.join(OUT, "volume_raycast_box_facade_test")
    pkg = os.path.join(ROOT, "rpg_open_remode_b200")
    subprocess.check_call([CXX, "-std=c++14", "-O1", "-DRMD_BUILD_TESTS=1",
                           "-I" + os.path.join(ROOT, "include"), "-I" + os.path.join(CUDA, "include"),
                           os.path.join(ROOT, "tests", "cpp", "volume_raycast_box_facade_test.cpp"), "-o", exe,
                           "-L" + pkg, "-lrmd_b200", "-L" + os.path.join(CUDA, "lib64"), "-lcudart",
                           "-Wl,-rpath," + pkg + ":" + os.path.join(CUDA, "lib64")])
    return exe


def test_volume_raycast_box_facade_compiles_with_host_compiler():
    assert os.path.exists(_build_facade())


@pytest.mark.gpu
def test_volume_raycast_box_facade_matches_python(tmp_path):
    import rpg_open_remode_b200 as rmd
    exe = _build_facade()
    out = str(tmp_path / "facade.bin")
    res = subprocess.run([exe, out], capture_output=True, text=True, timeout=600)
    print(res.stdout[-2000:], res.stderr[-2000:])
    assert res.returncode == 0 and "ALL VOLUME RAYCAST BOX TESTS PASSED" in res.stdout, res.stdout[-2000:]

    # the same scene through the Python API
    N, W, H, s, R = 64, 160, 120, 0.0625, 1.2
    v = rmd.TsdfVolume((N, N, N), s, (-2.0, -2.0, -2.0), 4 * s, 16.0, device=0, intensity=True, store=True)
    cam = rmd.PinholeCamera(100.0, 100.0, (W - 1) / 2.0, (H - 1) / 2.0)
    T = [1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1, 0]
    v.integrateDepth(np.full((H, W), R, np.float32), cam, T, None, np.full((H, W), 0.5, np.float32))
    v.shift((0, 0, -20))
    lo, m = (-4, -4, -4), (N + 8, N + 8, N + 28)
    d, inten = v.raycastIntensity(cam, T, W, H, lo, m)
    _, nrm = v.raycastNormals(cam, T, W, H, lo, m)
    seeds = rmd.SeedMatrix(W, H, cam, device=0)
    seeds.setReferenceImage(np.full((H, W), 0.5, np.float32), T, 0.5, 2.0)
    seeds.priorFromVolume(v, 1.0 / 16.0, lo, m)
    mu = seeds.downloadDepthmap()

    raw = np.frombuffer(open(out, "rb").read(), np.float32)
    n = W * H
    assert raw.size == 7 * n
    got_d, got_i, got_n, got_mu = raw[:n], raw[n:2 * n], raw[2 * n:6 * n].reshape(H, W, 4), raw[6 * n:]
    u32 = np.uint32
    assert np.array_equal(got_d.view(u32), d.reshape(-1).view(u32))
    assert np.array_equal(got_i.view(u32), inten.reshape(-1).view(u32))
    assert np.array_equal(np.ascontiguousarray(got_n[..., :3]).view(u32), nrm.view(u32))
    assert np.array_equal(got_mu.view(u32), mu.reshape(-1).view(u32))
    assert (d > 0).mean() > 0.5
