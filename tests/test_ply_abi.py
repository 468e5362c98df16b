"""PLY files without a GPU: the layout of cticp_ply_property in include/cticp.h and _abi.PlyProperty agree, the engine
exports the entry points, the writers report CTICP_ERR_NO_DEVICE, and the host pose reader reads the oracle's pose
files and refuses what it documents."""
import ctypes as C
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import oracle_ply_lib as orc  # noqa: E402

from ct_icp_b200 import _abi as abi  # noqa: E402
from ct_icp_b200._binding import CticpError  # noqa: E402


def _eng():
    import ct_icp_b200
    return ct_icp_b200.engine()


def test_ply_property_layout():
    assert _eng().fn("abi_sizeof")(b"cticp_ply_property") == C.sizeof(abi.PlyProperty) == 40
    assert abi.PlyProperty.ply_dtype.offset == 16 and abi.PlyProperty.src.offset == 24
    assert abi.PlyProperty.src_stride_bytes.offset == 32
    assert abi.PLY_SRC_DTYPE["int64"] == 9 and abi.PLY_SRC_DTYPE["uint64"] == 10


def test_ply_entry_points_exported():
    for name in ("ply_write", "ply_write_device", "ply_read_poses"):
        assert _eng().has(name), name


def test_ply_writers_without_a_device_report_no_device():
    import torch
    if torch.cuda.is_available():
        pytest.skip("a CUDA device is present")
    with pytest.raises(CticpError) as e:
        _eng().ply_write([("vertex", "x", "float", np.zeros(3))])
    assert e.value.code == abi.ERR_NO_DEVICE
    off = np.zeros(2, dtype=np.uint64)
    props = (abi.PlyProperty * 1)(abi.PlyProperty(b"vertex", b"x", 7, 8, None, 8))
    assert _eng().fn("ply_write_device")(0, props, 1, 0, None, 0, None, 0, off.ctypes.data, None) == abi.ERR_NO_DEVICE


def _poses(n):
    rng = np.random.default_rng(n)
    p = np.zeros(n, dtype=abi.pose_dtype())
    p["quat"] = rng.standard_normal((n, 4))
    p["tr"] = rng.standard_normal((n, 3))
    p["ref_timestamp"], p["dest_timestamp"] = rng.random(n), rng.random(n)
    p["ref_frame_id"] = rng.integers(0, 2 ** 32, n, dtype=np.uint32)
    p["dest_frame_id"] = np.arange(n, dtype=np.uint32)
    return p


@pytest.mark.parametrize("n", [0, 1, 17])
def test_read_poses_of_the_reference_pose_file(n):
    poses = _poses(n)
    assert _eng().read_poses_ply(orc.save_poses_ply(poses)).tobytes() == poses.tobytes()


def test_read_poses_any_order_other_elements_and_uint_fids():
    poses = _poses(4)
    names = ["qx", "qy", "qz", "qw", "x", "y", "z", "ref_t", "dest_t", "ref_fid", "dest_fid"]
    head = "ply\nformat binary_little_endian 1.0\ncomment written elsewhere\nelement other 2\nproperty uchar a\n"
    head += "element pose 4\nproperty short pad\n" + "".join(
        "property %s %s\n" % ("uint" if k.endswith("fid") else "double", k) for k in reversed(names)) + "end_header\n"
    rec = np.zeros(4, dtype=[("pad", "<i2")] + [(k, "<u4" if k.endswith("fid") else "<f8") for k in reversed(names)])
    src = {"qx": poses["quat"][:, 0], "qy": poses["quat"][:, 1], "qz": poses["quat"][:, 2], "qw": poses["quat"][:, 3],
           "x": poses["tr"][:, 0], "y": poses["tr"][:, 1], "z": poses["tr"][:, 2], "ref_t": poses["ref_timestamp"],
           "dest_t": poses["dest_timestamp"], "ref_fid": poses["ref_frame_id"], "dest_fid": poses["dest_frame_id"]}
    for k in names:
        rec[k] = src[k]
    data = head.encode() + b"\x07\x09" + rec.tobytes()
    assert _eng().read_poses_ply(data).tobytes() == poses.tobytes()
    assert orc.read_poses_ply(data).tobytes() == poses.tobytes()


def test_read_poses_refusals():
    good = orc.save_poses_ply(_poses(2))
    cases = {
        abi.ERR_UNSUPPORTED: [good.replace(b"binary_little_endian", b"ascii"),
                              good.replace(b"binary_little_endian", b"binary_big_endian")],
        abi.ERR_INVALID_ARGUMENT: [good.replace(b"double qx", b"float qx"),        # the reference's CHECK
                                   good.replace(b"int ref_fid", b"short ref_fid"),   # stated deviation
                                   good.replace(b"property double qw\n", b""),
                                   good.replace(b"element pose", b"element posed"),
                                   good[:-1], good.replace(b"end_header", b"end_headr"), b"plx\n" + good[4:]],
    }
    for code, datas in cases.items():
        for data in datas:
            with pytest.raises(CticpError) as e:
                _eng().read_poses_ply(data)
            assert e.value.code == code, data[:200]
