"""The brick store's host side (csrc/volume_store.h) is host-only code: built with the system compiler and run here,
no GPU (tests/cpp/volume_store_test.cpp): the candidate bricks of a shift against a voxel-by-voxel enumeration for a
negative offset, offsets that are not multiples of 8, ragged grids (97 x 64 x 71, nx = 1), |d| >= n and d = 0, and
the order in which new bricks get their slots."""
import os
import subprocess

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SRC = os.path.join(ROOT, "tests", "cpp", "volume_store_test.cpp")
OUT = os.path.join(ROOT, "tests", "cpp", "build")
CXX = "/usr/bin/g++" if os.path.exists("/usr/bin/g++") else "g++"


def test_candidates_and_slot_order():
    os.makedirs(OUT, exist_ok=True)
    exe = os.path.join(OUT, "volume_store_test")
    subprocess.check_call([CXX, "-std=c++14", "-O2", "-Wall", "-Wextra", SRC, "-o", exe])
    res = subprocess.run([exe], capture_output=True, text=True, timeout=600)
    assert res.returncode == 0 and "ALL VOLUME STORE HOST TESTS PASSED" in res.stdout, res.stdout[-2000:]
