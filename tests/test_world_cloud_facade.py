"""slam::SamplePointsInGrid / slam::WorldCloud of the C++ facade compile with plain g++ against include/cticp.h: without a
GPU they report CTICP_ERR_NO_DEVICE (exit 42); with one they agree with the CPU restatement of the reference
(tests/cpp/world_cloud_facade_test.cpp)."""
import os
import subprocess
import tempfile

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _build(out_dir):
    cxx = "/usr/bin/g++" if os.path.exists("/usr/bin/g++") else "g++"
    exe = os.path.join(out_dir, "world_cloud_facade_test")
    cmd = [cxx, "-std=c++17", "-O1", "-Wall", "-I", os.path.join(ROOT, "include"), "-I",
           os.path.join(ROOT, "ct_icp_b200", "include"), os.path.join(ROOT, "tests", "cpp", "world_cloud_facade_test.cpp"),
           os.path.join(ROOT, "tests", "oracle_grid", "orc_grid.cpp"), "-L", os.path.join(ROOT, "ct_icp_b200"),
           "-lcticp_b200", "-Wl,-rpath," + os.path.join(ROOT, "ct_icp_b200"), "-o", exe]
    r = subprocess.run(cmd, capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    return exe


def test_world_cloud_facade_compiles_and_fails_loudly_without_gpu():
    import torch
    with tempfile.TemporaryDirectory() as d:
        exe = _build(d)
        if torch.cuda.is_available():
            pytest.skip("a CUDA device is present")
        r = subprocess.run([exe], capture_output=True, text=True)
    assert r.returncode == 42, (r.returncode, r.stdout, r.stderr)
    assert "NO_DEVICE" in r.stdout


@pytest.mark.gpu
def test_world_cloud_facade_against_the_oracle():
    with tempfile.TemporaryDirectory() as d:
        exe = _build(d)
        r = subprocess.run([exe], capture_output=True, text=True, timeout=600)
    assert r.returncode == 0 and "WORLD CLOUD FACADE OK" in r.stdout, r.stdout[-3000:] + r.stderr[-2000:]
