"""Loads the CPU restatement of kitti::EvaluatePoses and ComputeTrajectoryMetrics (tests/oracle_eval/liborc_eval.so)
through the generic cticp binding: Binding(lib, "orc_").kitti_evaluate(...) drives it with the engine's calls.
TEST INFRASTRUCTURE."""
import ctypes
import os
import subprocess

from ct_icp_b200._binding import Binding

_ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
_DIR = os.path.join(_ROOT, "tests", "oracle_eval")
LIB = os.path.join(_DIR, "liborc_eval.so")
_SOURCES = [os.path.join(_DIR, "orc_eval.cpp"), os.path.join(_DIR, "orc_eval.h"),
            os.path.join(_ROOT, "oracle", "orc_math.h"), os.path.join(_ROOT, "include", "cticp.h")]
_cached = None


def build(out=LIB):
    """g++ -O2 (no FMA contraction on x86-64 without -march: the arithmetic of the reference's own build)"""
    cxx = "/usr/bin/g++" if os.path.exists("/usr/bin/g++") else "g++"
    subprocess.run([cxx, "-O2", "-std=c++17", "-fPIC", "-shared", "-Wall", "-ffp-contract=off", _SOURCES[0], "-o",
                    out + ".tmp"], check=True, capture_output=True)
    os.replace(out + ".tmp", out)
    return out


def eval_oracle():
    global _cached
    if _cached is None:
        stale = not os.path.exists(LIB) or any(os.path.getmtime(s) > os.path.getmtime(LIB) for s in _SOURCES)
        if stale:
            try:
                build()
            except Exception:
                if not os.path.exists(LIB):
                    raise
        _cached = Binding(ctypes.CDLL(LIB), "orc_")
        f = _cached.fn("svd3")
        f.restype, f.argtypes = None, [ctypes.c_void_p] * 3
    return _cached
