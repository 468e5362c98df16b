"""The PLY oracle (tests/oracle_ply, a restatement of WriteCollectionToPLY over tinyply 2.x, SavePosesAsPLY and
ReadPosesFromPLY) against an independent NumPy restatement (tests/ply_ref.py) and literal expected headers."""
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import oracle_ply_lib as orc  # noqa: E402
import ply_ref  # noqa: E402

from ct_icp_b200 import _abi as abi  # noqa: E402

SRC = ["int8", "uint8", "int16", "uint16", "int32", "uint32", "float32", "float64", "int64", "uint64"]


def _values(rng, dtype, n):
    dt = np.dtype(dtype)
    if dt.kind == "f":
        v = rng.standard_normal(n) * 10.0 ** rng.integers(-3, 12, n)
        v[rng.random(n) < 0.05] = np.nan
        v[rng.random(n) < 0.05] = 0.5 + rng.integers(-300, 300, n)[: 1]   # .5 ties
        return v.astype(dt)
    info = np.iinfo(dt)
    return rng.integers(info.min, info.max, n, dtype=dt, endpoint=True)


@pytest.mark.parametrize("src", SRC)
def test_every_dtype_pair_matches_numpy(src):
    rng = np.random.default_rng(abi.PLY_SRC_DTYPE[src])
    for n in (0, 1, 97):
        vals = _values(rng, src, n)
        cols = [("vertex", "p%d" % ply, ply, vals) for ply in range(1, 9)]
        assert orc.ply_write(cols) == ply_ref.ply_file(cols, n)


def test_fp64_to_fp32_ties_round_to_even():
    one = np.float64(1.0)
    ties = np.array([one + 2.0 ** -24, one + 3 * 2.0 ** -24, -(one + 2.0 ** -24)])
    got = orc.ply_write([("v", "x", "float", ties)])
    body = np.frombuffer(got[-12:], dtype="<f4")
    assert body.tolist() == [1.0, np.float32(1.0) + np.float32(2.0 ** -22), -1.0]


def test_float_to_int_saturates_and_nan_is_zero():
    x = np.array([np.nan, 1e30, -1e30, 255.9, -0.9, -1.5, 3e9, np.inf, -np.inf])
    got = orc.ply_write([("v", "u8", "uchar", x), ("v", "i32", "int", x), ("v", "u32", "uint", x)])
    rec = np.frombuffer(got[-len(x) * 9:], dtype=[("u8", "u1"), ("i32", "<i4"), ("u32", "<u4")])
    assert rec["u8"].tolist() == [0, 255, 0, 255, 0, 0, 255, 255, 0]
    assert rec["i32"].tolist() == [0, 2 ** 31 - 1, -2 ** 31, 255, 0, -1, 2 ** 31 - 1, 2 ** 31 - 1, -2 ** 31]
    assert rec["u32"].tolist() == [0, 2 ** 32 - 1, 0, 255, 0, 0, 3000000000, 2 ** 32 - 1, 0]


@pytest.mark.parametrize("seed", range(12))
def test_random_schemas_and_strides(seed):
    rng = np.random.default_rng(100 + seed)
    n = int(rng.choice([0, 1, 2, 13, 1000]))
    cols = []
    for j in range(int(rng.integers(1, 33))):
        src = SRC[rng.integers(len(SRC))]
        if rng.random() < 0.15:
            a = np.asarray(_values(rng, src, 1)[0])               # 0-d: broadcast
        else:
            step = int(rng.integers(1, 4))
            a = _values(rng, src, n * step)[::step]               # strided view
        cols.append(("e%d" % rng.integers(3), "p%d" % j, int(rng.integers(1, 9)), a))
    assert orc.ply_write(cols, num_items=n) == ply_ref.ply_file(cols, n)


def test_float_schema_mapper_header():
    """WPoint3D::FloatSchemaMapper (io.cxx:842-855): vertex x y z timestamp, all float"""
    xyz = np.array([[1.0, 2.0, 3.0], [4.0, 5.0, 6.0]])
    t = np.array([0.25, 0.5])
    cols = [("vertex", "x", "float", xyz[:, 0]), ("vertex", "y", "float", xyz[:, 1]),
            ("vertex", "z", "float", xyz[:, 2]), ("vertex", "timestamp", "float", t)]
    got = orc.ply_write(cols)
    head = (b"ply\nformat binary_little_endian 1.0\nelement vertex 2\nproperty float x\nproperty float y\n"
            b"property float z\nproperty float timestamp\nend_header\n")
    assert got[:len(head)] == head
    assert np.frombuffer(got[len(head):], dtype="<f4").tolist() == [1, 2, 3, 0.25, 4, 5, 6, 0.5]


def _poses(n, rng):
    p = np.zeros(n, dtype=abi.pose_dtype())
    p["quat"] = rng.standard_normal((n, 4))
    p["tr"] = rng.standard_normal((n, 3))
    p["ref_timestamp"] = rng.random(n)
    p["dest_timestamp"] = rng.random(n)
    p["ref_frame_id"] = rng.integers(0, 2 ** 32, n, dtype=np.uint32)
    p["dest_frame_id"] = np.arange(n, dtype=np.uint32)
    return p


def test_pose_file_header_records_and_read_back():
    poses = _poses(3, np.random.default_rng(5))
    got = orc.save_poses_ply(poses)
    head = b"ply\nformat binary_little_endian 1.0\nelement pose 3\n" + b"".join(
        b"property double %s\n" % k for k in (b"qx", b"qy", b"qz", b"qw", b"x", b"y", b"z", b"ref_t", b"dest_t")) + \
        b"property int ref_fid\nproperty int dest_fid\nend_header\n"
    assert got == head + poses.tobytes()          # the records are cticp_pose's 80 bytes
    back = orc.read_poses_ply(got)
    assert back.tobytes() == poses.tobytes()


def test_wpoints_default_schema_header():
    pts = np.zeros(1, dtype=abi.wpoint_dtype())
    got = orc.write_wpoints_ply(pts)
    head = got[:got.index(b"end_header\n")].decode()
    elems = [ln.split()[1] for ln in head.splitlines() if ln.startswith("element")]
    assert elems == ["properties", "raw_point", "world_point", "xyzt"]
    props = [ln.split()[1:] for ln in head.splitlines() if ln.startswith("property")]
    assert props[:8] == [["double", "raw_xyz_0"], ["double", "raw_xyz_1"], ["double", "raw_xyz_2"], ["double", "t"],
                         ["double", "world_xyz_0"], ["double", "world_xyz_1"], ["double", "world_xyz_2"],
                         ["uint", "index_frame"]]
    assert props[-4:] == [["double", "xyz_0"], ["double", "xyz_1"], ["double", "xyz_2"], ["double", "t"]]
    assert len(got) - len(head) - len("end_header\n") == 60 + 24 + 24 + 32
