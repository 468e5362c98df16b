"""Loads the CPU restatement of slam::SamplePointsInGrid (tests/oracle_grid/liborc_grid.so) through the generic cticp
binding: Binding(lib, "orc_").sample_points_in_grid(...) drives it with the engine's call. TEST INFRASTRUCTURE."""
import ctypes
import os
import subprocess

from ct_icp_b200._binding import Binding

_ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
_DIR = os.path.join(_ROOT, "tests", "oracle_grid")
LIB = os.path.join(_DIR, "liborc_grid.so")
_SOURCES = [os.path.join(_DIR, "orc_grid.cpp"), os.path.join(_ROOT, "include", "cticp.h")]
_cached = None


def build(out=LIB):
    cxx = "/usr/bin/g++" if os.path.exists("/usr/bin/g++") else "g++"
    subprocess.run([cxx, "-O2", "-std=c++17", "-fPIC", "-shared", "-Wall", _SOURCES[0], "-o", out + ".tmp"], check=True,
                   capture_output=True)
    os.replace(out + ".tmp", out)
    return out


def grid_oracle():
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
    return _cached
