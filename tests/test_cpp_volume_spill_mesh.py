"""The spill mesh of rmd::TsdfVolume (include/rmd/tsdf_volume.cuh) compiles with a plain host compiler against the
C-ABI and, on the GPU, behaves as tests/cpp/volume_spill_mesh_test.cpp checks -- and its outputs equal, bit for bit,
the Python path's (api.TsdfVolume) on the same scene."""
import os
import subprocess
import tempfile

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EXE = os.path.join(ROOT, "tests", "cpp", "build", "volume_spill_mesh_test")
CUDA = os.environ.get("CUDA_HOME", "/usr/local/cuda")


def _build():
    from rpg_open_remode_b200 import _build as b
    b.build_cuda()
    os.makedirs(os.path.dirname(EXE), exist_ok=True)
    pkg = os.path.join(ROOT, "rpg_open_remode_b200")
    cxx = "/usr/bin/g++" if os.path.exists("/usr/bin/g++") else "g++"
    cmd = [cxx, "-std=c++14", "-O1", "-DRMD_BUILD_TESTS=1",
           "-I" + os.path.join(ROOT, "include"), "-I" + os.path.join(CUDA, "include"),
           os.path.join(ROOT, "tests", "cpp", "volume_spill_mesh_test.cpp"), "-o", EXE,
           "-L" + pkg, "-lrmd_b200", "-L" + os.path.join(CUDA, "lib64"), "-lcudart",
           "-Wl,-rpath," + pkg + ":" + os.path.join(CUDA, "lib64")]
    subprocess.check_call(cmd)
    return EXE


def _read(path):
    out = []
    with open(path, "rb") as f:
        for dt in (np.float32, np.int32, np.int64, np.float32, np.float32, np.int64):
            n = int(np.frombuffer(f.read(8), np.uint64)[0])
            out.append(np.frombuffer(f.read(n * np.dtype(dt).itemsize), dt))
    return out


def test_volume_spill_mesh_facade_compiles_with_host_compiler():
    assert os.path.exists(_build())


@pytest.mark.gpu
def test_volume_spill_mesh_facade_equals_the_python_path():
    import rpg_open_remode_b200 as rmd
    exe = _build()
    with tempfile.TemporaryDirectory() as tmp:
        path = os.path.join(tmp, "spill_mesh.bin")
        res = subprocess.run([exe, path], capture_output=True, text=True, timeout=600)
        print(res.stdout[-2000:], res.stderr[-2000:])
        assert res.returncode == 0, res.stdout[-2000:]
        assert "ALL VOLUME SPILL MESH TESTS PASSED" in res.stdout
        xyzw, tri, ids, inten, normals, after_ids = _read(path)
    # the same scene through api.TsdfVolume: a sphere of radius 1.2 m seen from its centre
    N, W, H, s = 64, 160, 120, 0.0625
    v = rmd.TsdfVolume((N, N, N), s, (-2.0, -2.0, -2.0), 4 * s, 16.0, device=0, intensity=True)
    cam = rmd.PinholeCamera(100.0, 100.0, (W - 1) / 2.0, (H - 1) / 2.0)
    T = np.hstack([np.eye(3), np.zeros((3, 1))]).astype(np.float32)
    v.integrateDepth(np.full((H, W), 1.2, np.float32), cam, T, None, np.full((H, W), 0.5, np.float32))
    v.shift((2, 0, -1))
    d = (26, -7, -14)
    pv, pt, pids = v.spillMesh(d)
    u32 = np.uint32
    assert np.array_equal(pv.reshape(-1).view(u32), xyzw.view(u32)) and np.array_equal(pt.reshape(-1), tri)
    assert np.array_equal(pids.reshape(-1), ids)
    assert np.array_equal(v.spillMeshIntensity(d).view(u32), inten.view(u32))
    assert np.array_equal(v.spillMeshNormals(d).view(u32), normals.reshape(-1, 4)[:, :3].view(u32))
    v.shift(d)
    assert np.array_equal(v.surfaceIds().reshape(-1), after_ids)
