"""Dataset sequences without a GPU: the layouts of cticp_nclt_frame and cticp_ply_layout, the exports, the PLY header
acceptance and refusal tables, the ground-truth readers (KITTI, KITTI-360, KITTI_CARLA, NCLT, HILTI) on files written
from known poses through the inverse calibration, and the NumPy restatement of kitti_frame_filter the GPU tests use."""
import ctypes as C
import math

import numpy as np
import pytest

from ct_icp_b200 import _abi as abi
from ct_icp_b200._binding import CticpError
import dataset_ref as ref


@pytest.fixture(scope="module")
def lib():
    import ct_icp_b200
    return ct_icp_b200.engine()


def test_dataset_struct_layouts_and_exports(lib):
    assert lib.fn("abi_sizeof")(b"cticp_nclt_frame") == C.sizeof(abi.NcltFrame) == abi.nclt_frame_dtype().itemsize == 24
    assert lib.fn("abi_sizeof")(b"cticp_ply_layout") == C.sizeof(abi.PlyLayout) == 40
    assert abi.PlyLayout.point_step.offset == 16 and abi.PlyLayout.t_dtype.offset == 32
    for name in ("nclt_open", "nclt_open_device", "nclt_destroy", "nclt_num_frames", "nclt_num_packets", "nclt_num_hits",
                 "nclt_bytes_used", "nclt_frame_info", "nclt_read_frames", "nclt_read_frames_device", "ply_layout_parse",
                 "kitti_frame_filter", "kitti_frame_filter_device", "scan_time_ranges", "scan_time_ranges_device",
                 "ground_truth_parse"):
        assert lib.has(name), name


def test_nclt_open_without_a_device_reports_no_device(lib):
    import torch
    if torch.cuda.is_available():
        pytest.skip("a CUDA device is present")
    data = ref.pack_packet(1, [[1, 2, 3]])
    h = C.c_void_p()
    assert lib.fn("nclt_open")(data, len(data), 220, 1, 0, C.byref(h)) == abi.ERR_NO_DEVICE


def _header(*props, fmt="binary_little_endian", extra=()):
    lines = ["ply", "format %s 1.0" % fmt, *extra, "element vertex 2", *["property %s %s" % p for p in props],
             "end_header"]
    return ("\n".join(lines) + "\n").encode()


@pytest.mark.parametrize("props,step,xoff,xdt,toff,tdt", [
    ((("float", "x"), ("float", "y"), ("float", "z")), 12, 0, "float32", 0, 0),
    ((("double", "x"), ("double", "y"), ("double", "z"), ("double", "timestamp")), 32, 0, "float64", 24, "float64"),
    ((("uchar", "intensity"), ("float", "x"), ("float", "y"), ("float", "z"), ("float", "t")), 17, 1, "float32", 13,
     "float32"),
    ((("double", "x"), ("double", "y"), ("double", "z"), ("uint", "timestamps"), ("ushort", "ring")), 30, 0, "float64",
     24, "uint32"),
    ((("float", "x"), ("float", "y"), ("float", "z"), ("double", "t"), ("double", "timestamp")), 28, 0, "float32", 20,
     "float64"),
])
def test_ply_headers_accepted(lib, props, step, xoff, xdt, toff, tdt):
    hdr = _header(*props, extra=("comment a comment", "obj_info x"))
    lay = lib.ply_layout(hdr + bytes(2 * step))
    assert (lay.body_offset, lay.num_points, lay.point_step, lay.xyz_offset) == (len(hdr), 2, step, xoff)
    assert lay.xyz_dtype == abi.DTYPE[xdt] and lay.t_dtype == (abi.DTYPE[tdt] if tdt else 0)
    assert lay.t_offset == toff


XYZ = (("float", "x"), ("float", "y"), ("float", "z"))


@pytest.mark.parametrize("data,code", [
    (_header(*XYZ, fmt="ascii") + b"0 0 0\n0 0 0\n", abi.ERR_UNSUPPORTED),
    (_header(*XYZ, fmt="binary_big_endian") + bytes(24), abi.ERR_UNSUPPORTED),
    (_header(*XYZ, ("list uchar int", "vertex_indices")) + bytes(64), abi.ERR_UNSUPPORTED),
    (b"ply\nformat binary_little_endian 1.0\nelement face 2\nproperty float x\nend_header\n" + bytes(8),
     abi.ERR_UNSUPPORTED),
    (_header(("float", "x"), ("float", "y")) + bytes(16), abi.ERR_INVALID_ARGUMENT),
    (_header(("float", "x"), ("double", "y"), ("float", "z")) + bytes(32), abi.ERR_INVALID_ARGUMENT),
    (_header(("float", "x"), ("float", "z"), ("float", "y")) + bytes(24), abi.ERR_INVALID_ARGUMENT),
    (_header(("int", "x"), ("int", "y"), ("int", "z")) + bytes(24), abi.ERR_INVALID_ARGUMENT),
    (_header(*XYZ) + bytes(23), abi.ERR_INVALID_ARGUMENT),
    (_header(*XYZ)[:-11], abi.ERR_INVALID_ARGUMENT),
    (b"plx\n" + _header(*XYZ)[4:] + bytes(24), abi.ERR_INVALID_ARGUMENT),
    (_header(*XYZ, ("float128", "t")) + bytes(64), abi.ERR_INVALID_ARGUMENT),
], ids=["ascii", "big_endian", "list", "face", "no_z", "mixed", "not_consecutive", "int_xyz", "short_body",
        "no_end_header", "no_magic", "unknown_type"])
def test_ply_headers_refused(lib, data, code):
    with pytest.raises(CticpError) as e:
        lib.ply_layout(data)
    assert e.value.code == code


def _random_poses(rng, n):
    from scipy.spatial.transform import Rotation
    Ms = []
    for _ in range(n):
        M = np.eye(4)
        M[:3, :3] = Rotation.from_rotvec(rng.normal(size=3) * 0.7).as_matrix()
        M[:3, 3] = rng.uniform(-200, 200, 3)
        Ms.append(M)
    return Ms


def _assert_pose_close(p, M, tol=1e-12):
    got = ref.pose_matrix(p)
    assert np.abs(got[:3, :3] - M[:3, :3]).max() < tol
    assert np.abs(got[:3, 3] - M[:3, 3]).max() < tol * max(1.0, np.abs(M[:3, 3]).max())


@pytest.mark.parametrize("dataset,seq", [("KITTI", 0), ("KITTI", 3), ("KITTI", 12), ("KITTI_raw", 2),
                                         ("KITTI_360", 5), ("KITTI_CARLA", 1)])
def test_kitti_family_ground_truth_round_trip(lib, dataset, seq):
    """poses P written as Calib · P · CalibI in KITTI format read back as P, with the family's timestamps"""
    rng = np.random.default_rng(seq + 17)
    Ms = _random_poses(rng, 12)
    C_ = ref.calib_matrix(dataset, seq)
    text = "\n".join(ref.kitti_line(C_ @ M @ np.linalg.inv(C_)) for M in Ms) + "\n\n"
    poses = lib.ground_truth(dataset, text, seq)
    assert len(poses) == len(Ms)
    for i, (p, M) in enumerate(zip(poses, Ms)):
        _assert_pose_close(p, M)
        assert abs(np.linalg.norm(p["quat"]) - 1.0) < 1e-15
        assert p["dest_frame_id"] == i
        assert p["dest_timestamp"] == ((i * 0.1) if dataset == "KITTI_CARLA" else (i + 0.5) * 0.1)


def test_kitti_short_line_keeps_the_identity(lib):
    """a short line leaves its missing entries at the identity's (P starts as Identity on every line)"""
    poses = lib.ground_truth("KITTI_CARLA", "1 0 0 5\n0 1 0 1 0 1 0 2 1 0 0\n", 0)
    _assert_pose_close(poses[0], np.array([[1, 0, 0, 5], [0, 1, 0, 0], [0, 0, 1, 0], [0, 0, 0, 1.0]]))
    # the second line stops after 11 values: P(2, 3) keeps the identity's 0
    assert poses[1]["tr"].tolist() == [1.0, 2.0, 0.0]
    assert len(poses) == 2 and np.all(np.isfinite(poses[1]["quat"]))


def test_nclt_ground_truth_round_trip(lib):
    """rows (t, x, y, z, roll, pitch, yaw) of G_i = G_0 · Calib · P_i · CalibI read back as P_i; NaN rows skipped"""
    from scipy.spatial.transform import Rotation
    rng = np.random.default_rng(3)
    Ms = [np.eye(4)] + _random_poses(rng, 9)
    C_ = ref.nclt_calib()
    G0 = _random_poses(rng, 1)[0]
    rows = []
    for i, M in enumerate(Ms):
        G = G0 @ C_ @ M @ np.linalg.inv(C_)
        yaw, pitch, roll = Rotation.from_matrix(G[:3, :3]).as_euler("ZYX")
        rows.append("%d,%s" % (1_000_000 + 100_000 * i, ",".join(repr(float(v)) for v in (*G[:3, 3], roll, pitch, yaw))))
        if i == 4:
            rows.append("1450000,nan,1,2,0.1,0.2,0.3")
    poses = lib.ground_truth("NCLT", "\n".join(rows) + "\n")
    assert len(poses) == len(Ms)
    for i, (p, M) in enumerate(zip(poses, Ms)):
        _assert_pose_close(p, M, 1e-10)
        assert p["dest_timestamp"] == 1_000_000 + 100_000 * i and p["dest_frame_id"] == 0xFFFFFFFF


@pytest.mark.parametrize("text", ["1,2,3\n", "1,2,3,4,5,6,7,8\n", "1,2,3,x,5,6,7\n", "1,2,3,4,5,6,7\n\n"],
                         ids=["short", "long", "not_a_number", "empty_line"])
def test_nclt_ground_truth_malformed_rows_refused(lib, text):
    with pytest.raises(CticpError) as e:
        lib.ground_truth("NCLT", text)
    assert e.value.code == abi.ERR_INVALID_ARGUMENT


@pytest.mark.parametrize("dataset", ["HILTI_2021", "HILTI_2022"])
def test_hilti_ground_truth_round_trip_and_unnormalised_quaternion(lib, dataset):
    """lines (t, x, y, z, qx, qy, qz, qw) of L2I · P · L2I^-1 read back as P; a quaternion of norm 3 in the file is
    kept as it is (the reference discards its normalized()), which SE3's product then normalises"""
    rng = np.random.default_rng(5)
    Ms = _random_poses(rng, 6)
    L = ref.HILTI_L2I[dataset]
    lines = []
    for i, M in enumerate(Ms):
        G = L @ M @ np.linalg.inv(L)
        q = ref.matrix_to_quat(G[:3, :3]) * (3.0 if i == 2 else 1.0)
        lines.append(" ".join(repr(float(v)) for v in (10.0 + i, *G[:3, 3], *q)))
    poses = lib.ground_truth(dataset, "\n".join(lines) + "\n")
    assert len(poses) == len(Ms)
    for i, (p, M) in enumerate(zip(poses, Ms)):
        _assert_pose_close(p, M, 1e-10)
        assert p["dest_timestamp"] == 10.0 + i
    assert abs(np.linalg.norm(poses[2]["quat"]) - 1.0) < 1e-12


def test_ground_truth_refusals(lib):
    for ds, seq in (("KITTI", 22), ("KITTI", -1), (9, 0)):
        with pytest.raises(CticpError) as e:
            lib.ground_truth(ds, "1 0 0 0 0 1 0 0 0 0 1 0\n", seq)
        assert e.value.code == abi.ERR_INVALID_ARGUMENT


def test_filter_restatement_keeps_norms():
    """the NumPy kitti_frame_filter: norms kept to 1e-12 relative, z-axis points scaled by cos(angle), points with
    !(z > -5) (NaN included) set to 0"""
    rng = np.random.default_rng(0)
    p = rng.uniform(-80, 80, (5000, 3))
    p[:10, :2] = 0.0                      # on the z axis
    p[10:20, 2] = -5.0                    # exactly at the cut
    p[20, 2] = np.nan
    p[21, 0] = np.nan
    out = ref.kitti_frame_filter(p)
    zcut = ~(p[:, 2] > -5.0)
    assert np.all(out[zcut] == 0.0)
    axis = (np.arange(len(p)) < 10) & ~zcut
    c = math.cos(0.205 * math.pi / 180.0)
    assert np.array_equal(out[axis], p[axis] * c)
    rest = ~zcut & ~axis & np.isfinite(p).all(1)
    n0, n1 = np.linalg.norm(p[rest], axis=1), np.linalg.norm(out[rest], axis=1)
    assert np.max(np.abs(n1 - n0) / n0) < 1e-12
    # the rotation is about p x z: the elevation grows by the angle, the azimuth stays
    el0 = np.arctan2(p[rest, 2], np.hypot(p[rest, 0], p[rest, 1]))
    el1 = np.arctan2(out[rest, 2], np.hypot(out[rest, 0], out[rest, 1]))
    assert np.abs(el1 - el0 - 0.205 * math.pi / 180.0).max() < 1e-9


def test_nclt_restatement_on_hand_packets():
    data = ref.pack_packet(7, [[20000, 20000, 20000], [0, 65535, 1]]) + ref.pack_packet(8, []) + \
        ref.pack_packet(9, [[1, 2, 3]])
    d = ref.decode(data, num_aggregated=2, final=True)
    assert d["num_packets"] == 3 and len(d["frames"]) == 2 and d["bytes_used"] == len(data)
    assert d["frames"][0][0][0].tolist() == [0.0, 0.0, 0.0] and d["info"][0] == (2, 7.0, 7.0)
    assert ref.decode(data, num_aggregated=2, final=False)["num_packets"] == 2
    with pytest.raises(ValueError):
        ref.decode(data[:-1])
