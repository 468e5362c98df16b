"""Loads the CPU restatement of the reference's PLY writers and pose reader (tests/oracle_ply/liborc_ply.so):
WriteCollectionToPLY over tinyply 2.x's header and binary writer, SavePosesAsPLY, WritePLY of WPoint3D records with the
default schema mapper, and ReadPosesFromPLY. TEST INFRASTRUCTURE."""
import ctypes
import os
import subprocess

import numpy as np

_ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
_DIR = os.path.join(_ROOT, "tests", "oracle_ply")
LIB = os.path.join(_DIR, "liborc_ply.so")
_SOURCES = [os.path.join(_DIR, "orc_ply.cpp")]
_cached = None


def build(out=LIB):
    cxx = "/usr/bin/g++" if os.path.exists("/usr/bin/g++") else "g++"
    subprocess.run([cxx, "-O2", "-std=c++17", "-fPIC", "-shared", "-Wall", _SOURCES[0], "-o", out + ".tmp"], check=True,
                   capture_output=True)
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
        vp, sz, u64 = ctypes.c_void_p, ctypes.c_size_t, ctypes.c_uint64
        for name, args in (("orc_ply_write", [vp, sz, u64, vp, u64]), ("orc_save_poses_ply", [vp, sz, vp, u64]),
                           ("orc_write_wpoints_ply", [vp, sz, vp, u64]), ("orc_read_poses_ply", [vp, sz, vp, sz])):
            getattr(lib, name).restype = ctypes.c_int64
            getattr(lib, name).argtypes = args
        _cached = lib
    return _cached


def _bytes(fn, *args):
    n = fn(*args, None, 0)
    buf = ctypes.create_string_buffer(max(n, 1))
    assert fn(*args, buf, n) == n
    return buf.raw[:n]


def ply_write(columns, num_items=None):
    """The reference's file of (element, name, ply_dtype, array) columns (NumPy, 1-D or 0-d): bytes"""
    from ct_icp_b200 import _abi as abi
    from ct_icp_b200._binding import _ply_num_items, _ply_props, _ply_src_code
    arrays = [np.asarray(c[3]) for c in columns]
    n = _ply_num_items([a.shape for a in arrays], num_items)
    props, keep = _ply_props(columns, [_ply_src_code(a.dtype.name) for a in arrays],
                             [(a.ctypes.data, a.strides[0] if a.ndim else 0) for a in arrays])
    return _bytes(_lib().orc_ply_write, ctypes.cast(props, ctypes.c_void_p), len(columns), n)


def save_poses_ply(poses):
    """SavePosesAsPLY of an array of abi.pose_dtype()"""
    arr = np.ascontiguousarray(poses)
    return _bytes(_lib().orc_save_poses_ply, arr.ctypes.data, len(arr))


def write_wpoints_ply(points):
    """WritePLY(os, std::vector<WPoint3D>) of an array of 64-byte WPoint3D records (abi.wpoint_dtype())"""
    arr = np.ascontiguousarray(points)
    return _bytes(_lib().orc_write_wpoints_ply, arr.ctypes.data, len(arr))


def read_poses_ply(data):
    """ReadPosesFromPLY: an array of abi.pose_dtype(); ValueError where the reference rejects the file"""
    from ct_icp_b200 import _abi as abi
    buf = np.frombuffer(bytes(data), dtype=np.uint8)
    n = _lib().orc_read_poses_ply(buf.ctypes.data, len(buf), None, 0)
    if n < 0:
        raise ValueError("the reference's reader rejects this file")
    out = np.zeros(n, dtype=abi.pose_dtype())
    _lib().orc_read_poses_ply(buf.ctypes.data, len(buf), out.ctypes.data, n)
    return out
