"""Loads the CPU restatement of the reference's dataset readers (tests/oracle_dataset/liborc_dataset.so): NextBatch /
DoNext over velodyne_hits.bin bytes, kitti_frame_filter through Eigen-shaped matrix operations, and LoadPoses with
`istream >> double` and the general 4x4 inverse. TEST INFRASTRUCTURE."""
import ctypes
import os
import subprocess

import numpy as np

_ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
_DIR = os.path.join(_ROOT, "tests", "oracle_dataset")
LIB = os.path.join(_DIR, "liborc_dataset.so")
_SOURCES = [os.path.join(_DIR, "orc_dataset.cpp")]
_cached = None


def build(out=LIB):
    """g++ -O2 -ffp-contract=off: host fp64 one operation at a time, as the reference's own build does"""
    cxx = "/usr/bin/g++" if os.path.exists("/usr/bin/g++") else "g++"
    subprocess.run([cxx, "-O2", "-std=c++17", "-fPIC", "-shared", "-Wall", "-ffp-contract=off", _SOURCES[0], "-o",
                    out + ".tmp"], check=True, capture_output=True)
    os.replace(out + ".tmp", out)
    return out


def _lib():
    global _cached
    if _cached is None:
        if not os.path.exists(LIB) or any(os.path.getmtime(s) > os.path.getmtime(LIB) for s in _SOURCES):
            try:
                build()
            except Exception:
                if not os.path.exists(LIB):
                    raise
        lib = ctypes.CDLL(LIB)
        vp, sz = ctypes.c_void_p, ctypes.c_size_t
        lib.orc_nclt_decode.restype = ctypes.c_int64
        lib.orc_nclt_decode.argtypes = [vp, sz, ctypes.c_uint32, ctypes.c_int, vp, vp, sz, vp, sz, vp]
        lib.orc_kitti_frame_filter.restype = None
        lib.orc_kitti_frame_filter.argtypes = [vp, sz]
        lib.orc_ground_truth.restype = ctypes.c_int64
        lib.orc_ground_truth.argtypes = [ctypes.c_int, ctypes.c_int, vp, sz, vp, sz]
        _cached = lib
    return _cached


def nclt_decode(data, num_aggregated=220, final=True):
    """(xyz (N, 3), t (N,), frame_ends (F,)) of the reference's reader; ValueError where it would stop with an error"""
    lib, buf = _lib(), np.frombuffer(bytes(data), dtype=np.uint8)
    frames = ctypes.c_int64()
    n = lib.orc_nclt_decode(buf.ctypes.data, len(buf), num_aggregated, int(final), None, None, 0, None, 0,
                            ctypes.byref(frames))
    if n < 0:
        raise ValueError("the reference's reader stops with an error on these bytes")
    xyz, t, ends = np.zeros((n, 3)), np.zeros(n), np.zeros(frames.value, dtype=np.uint64)
    lib.orc_nclt_decode(buf.ctypes.data, len(buf), num_aggregated, int(final), xyz.ctypes.data, t.ctypes.data, n,
                        ends.ctypes.data, len(ends), ctypes.byref(frames))
    return xyz, t, ends


def kitti_frame_filter(xyz):
    """kitti_frame_filter of (n, 3) float64 points (a filtered copy)"""
    out = np.ascontiguousarray(xyz, dtype=np.float64).copy()
    _lib().orc_kitti_frame_filter(out.ctypes.data, len(out))
    return out


def ground_truth(dataset, text, sequence_id=0):
    """LoadPoses: an (n, 9) array of qx qy qz qw tx ty tz dest_timestamp dest_frame_id; ValueError where the reference
    CHECK-aborts"""
    from ct_icp_b200 import _abi as abi
    ds = abi.DATASET[dataset] if isinstance(dataset, str) else int(dataset)
    raw = text.encode() if isinstance(text, str) else bytes(text)
    buf = np.frombuffer(raw + b"\0", dtype=np.uint8)
    n = _lib().orc_ground_truth(ds, sequence_id, buf.ctypes.data, len(raw), None, 0)
    if n < 0:
        raise ValueError("the reference's reader aborts on this text")
    out = np.zeros((n, 9))
    _lib().orc_ground_truth(ds, sequence_id, buf.ctypes.data, len(raw), out.ctypes.data, n)
    return out
