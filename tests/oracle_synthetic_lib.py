"""Loads the CPU restatement of slam::Scene / SyntheticSensorAcquisition (tests/oracle_synthetic/liborc_synthetic.so,
which carries the trajectory oracle too) through the generic cticp binding: Binding(lib, "orc_").synthetic_scene(...)
and .continuous_trajectory(...) drive it with the engine's calls. TEST INFRASTRUCTURE."""
import ctypes
import os
import subprocess

from ct_icp_b200._binding import Binding

_ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
_DIR = os.path.join(_ROOT, "tests", "oracle_synthetic")
LIB = os.path.join(_DIR, "liborc_synthetic.so")
_SOURCES = [os.path.join(_DIR, "orc_synthetic.cpp"), os.path.join(_ROOT, "tests", "oracle_trajectory", "orc_trajectory.cpp"),
            os.path.join(_ROOT, "tests", "oracle_trajectory", "orc_trajectory.h"),
            os.path.join(_ROOT, "oracle", "orc_math.h"), os.path.join(_ROOT, "include", "cticp.h")]
_cached = None


def build(out=LIB):
    """g++ -O2 -ffp-contract=off: host fp64 one operation at a time, as the reference's own build does"""
    cxx = "/usr/bin/g++" if os.path.exists("/usr/bin/g++") else "g++"
    subprocess.run([cxx, "-O2", "-std=c++17", "-fPIC", "-shared", "-Wall", "-ffp-contract=off", _SOURCES[0], "-o",
                    out + ".tmp"], check=True, capture_output=True)
    os.replace(out + ".tmp", out)
    return out


def synthetic_oracle():
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
