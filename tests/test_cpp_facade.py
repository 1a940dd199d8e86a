"""Builds and runs the C++ facade test (include/m3tsz_b200.hpp over the C ABI).  The binary goes to a temporary
directory: the test writes nothing into the repository tree, which may be read-only."""
import os
import subprocess
import tempfile

import pytest

ROOT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..")
SRC = os.path.join(ROOT, "tests", "cpp", "test_facade.cpp")


@pytest.fixture(scope="module")
def exe():
    path = os.path.join(tempfile.mkdtemp(prefix="m3_cpp_facade_"), "test_facade.bin")
    libdir = os.path.join(ROOT, "m3_b200")
    cmd = ["g++", "-std=c++17", "-O1", "-I", os.path.join(ROOT, "include"), SRC, "-o", path,
           "-L", libdir, "-lm3tsz_b200", "-Wl,-rpath," + libdir, "-L/usr/local/cuda/lib64",
           "-Wl,-rpath,/usr/local/cuda/lib64"]
    subprocess.check_call(cmd)
    return path


def test_cpp_facade_builds_and_refuses_without_gpu(exe):
    import torch
    if torch.cuda.is_available():
        pytest.skip("GPU present: covered by the gpu-marked test")
    r = subprocess.run([exe], capture_output=True, text=True)
    assert r.returncode == 3 and "NO_DEVICE" in r.stdout, (r.returncode, r.stdout, r.stderr)


@pytest.mark.gpu
def test_cpp_facade_goldens_on_gpu(exe):
    r = subprocess.run([exe], capture_output=True, text=True)
    assert r.returncode == 0 and "PASS" in r.stdout, (r.returncode, r.stdout, r.stderr)
