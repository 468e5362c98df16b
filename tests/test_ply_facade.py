"""The PLY writers of the C++ facade compile with plain g++ against include/cticp.h: without a GPU they report
CTICP_ERR_NO_DEVICE (exit 42); with one, WritePLY(vector<WPoint3D>) writes the oracle's four-element file, the float and
double mappers the reference's vertex files, and SavePosesAsPLY the oracle's pose file (tests/cpp/ply_facade_test.cpp)."""
import os
import subprocess
import sys
import tempfile

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import oracle_ply_lib as orc  # noqa: E402

from ct_icp_b200 import _abi as abi  # noqa: E402

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _build(out_dir):
    cxx = "/usr/bin/g++" if os.path.exists("/usr/bin/g++") else "g++"
    exe = os.path.join(out_dir, "ply_facade_test")
    cmd = [cxx, "-std=c++17", "-O1", "-Wall", "-I", os.path.join(ROOT, "include"), "-I",
           os.path.join(ROOT, "ct_icp_b200", "include"), os.path.join(ROOT, "tests", "cpp", "ply_facade_test.cpp"),
           "-L", os.path.join(ROOT, "ct_icp_b200"), "-lcticp_b200", "-Wl,-rpath," + os.path.join(ROOT, "ct_icp_b200"),
           "-lm", "-o", exe]
    r = subprocess.run(cmd, capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    return exe


def _points():
    p = np.zeros(5, dtype=abi.wpoint_dtype())
    i = np.arange(5, dtype=np.float64)
    p["raw"] = np.stack([1.5 * i, -1.0 * i, 0.25 * i], 1)
    p["timestamp"] = 0.1 * i
    p["world"] = np.stack([1.5 * i + 10.0, -1.0 * i + 10.0, 0.25 * i + 10.0], 1)
    p["index_frame"] = 7 * np.arange(5)
    return p


def _poses():
    p = np.zeros(3, dtype=abi.pose_dtype())
    for i in range(3):
        p[i]["quat"] = [0.1 * i, 0.2, -0.3, 0.9]
        p[i]["tr"] = [1.0 * i, 2.0, 3.0]
        p[i]["ref_timestamp"], p[i]["dest_timestamp"] = 0.5 * i, 0.5 * i + 0.1
        p[i]["ref_frame_id"], p[i]["dest_frame_id"] = i, 0xFFFFFFFF
    return p


def test_ply_facade_compiles_and_fails_loudly_without_gpu():
    import torch
    with tempfile.TemporaryDirectory() as d:
        exe = _build(d)
        if torch.cuda.is_available():
            pytest.skip("a CUDA device is present")
        r = subprocess.run([exe, d], capture_output=True, text=True)
    assert r.returncode == 42, (r.returncode, r.stdout, r.stderr)
    assert "NO_DEVICE" in r.stdout


@pytest.mark.gpu
def test_ply_facade_on_the_device():
    with tempfile.TemporaryDirectory() as d:
        exe = _build(d)
        r = subprocess.run([exe, d], capture_output=True, text=True, timeout=300)
        assert r.returncode == 0 and "PLY FACADE OK" in r.stdout, r.stdout[-3000:] + r.stderr[-2000:]
        files = {}
        for name in ("default", "float", "double", "poses"):
            with open(os.path.join(d, name + ".ply"), "rb") as f:
                files[name] = f.read()
    pts = _points()
    assert files["default"] == orc.write_wpoints_ply(pts)
    for name, t in (("float", "float"), ("double", "double")):
        cols = [("vertex", "x", t, pts["raw"][:, 0]), ("vertex", "y", t, pts["raw"][:, 1]),
                ("vertex", "z", t, pts["raw"][:, 2]), ("vertex", "timestamp", t, pts["timestamp"])]
        assert files[name] == orc.ply_write(cols), name
    assert files["poses"] == orc.save_poses_ply(_poses())
