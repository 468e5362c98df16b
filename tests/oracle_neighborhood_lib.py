"""Loads the CPU restatement of slam::TNeighborhood (tests/oracle_neighborhood/liborc_neighborhood.so) and wraps it in
NumPy: search(points, queries, k, max_radius) and describe(points, values, ...). TEST INFRASTRUCTURE."""
import ctypes as C
import os
import subprocess

import numpy as np

from ct_icp_b200 import _abi as abi

_ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
_DIR = os.path.join(_ROOT, "tests", "oracle_neighborhood")
LIB = os.path.join(_DIR, "liborc_neighborhood.so")
_SOURCES = [os.path.join(_DIR, "orc_neighborhood.cpp"), os.path.join(_ROOT, "include", "cticp.h"),
            os.path.join(_ROOT, "oracle", "orc_math.h")]
_cached = None
DBL_MAX = np.finfo(np.float64).max


def build(out=LIB):
    cxx = "/usr/bin/g++" if os.path.exists("/usr/bin/g++") else "g++"
    subprocess.run([cxx, "-O2", "-std=c++17", "-fPIC", "-shared", "-Wall", "-ffp-contract=off", _SOURCES[0], "-o",
                    out + ".tmp"], check=True, capture_output=True)
    os.replace(out + ".tmp", out)
    return out


def lib():
    global _cached
    if _cached is None:
        stale = not os.path.exists(LIB) or any(os.path.getmtime(s) > os.path.getmtime(LIB) for s in _SOURCES)
        if stale:
            try:
                build()
            except Exception:
                if not os.path.exists(LIB):
                    raise
        L = C.CDLL(LIB)
        vp, sz = C.c_void_p, C.c_size_t
        L.orn_search.argtypes = [vp, sz, vp, sz, C.c_int, C.c_double, vp, vp, vp]
        L.orn_search.restype = None
        L.orn_describe.argtypes = [vp, sz, vp, C.c_int, C.c_double, C.c_double, C.c_int, vp]
        L.orn_describe.restype = None
        _cached = L
    return _cached


def search(points, queries, k, max_radius=DBL_MAX):
    """(indices (m, k) uint64, d2 (m, k), counts (m,) int32); queries None: the points themselves"""
    p = np.ascontiguousarray(points, dtype=np.float64).reshape(-1, 3)
    q = None if queries is None else np.ascontiguousarray(queries, dtype=np.float64).reshape(-1, 3)
    m = len(p) if q is None else len(q)
    idx = np.zeros((m, k), dtype=np.uint64)
    d2 = np.zeros((m, k))
    cnt = np.zeros(m, dtype=np.int32)
    lib().orn_search(p.ctypes.data, len(p), None if q is None else q.ctypes.data, m, k, float(max_radius),
                     idx.ctypes.data, d2.ctypes.data, cnt.ctypes.data)
    return idx, d2, cnt


def describe(points, values=abi.NB["ALL"], linearity_threshold=0.8, planarity_threshold=0.8, centred=True, centre=None):
    """one abi.neighborhood_description_dtype() record: centred (long double, about `centre` or the first point) or the
    reference's uncentred fp64 formula"""
    p = np.ascontiguousarray(points, dtype=np.float64).reshape(-1, 3)
    out = np.zeros(1, dtype=abi.neighborhood_description_dtype())
    c = None if centre is None else np.ascontiguousarray(centre, dtype=np.float64).reshape(3)
    lib().orn_describe(p.ctypes.data, len(p), None if c is None else c.ctypes.data, int(values), float(linearity_threshold),
                       float(planarity_threshold), 1 if centred else 0, out.ctypes.data)
    return out[0]
