"""The dataset readers against the C++ restatement of the reference (tests/oracle_dataset/orc_dataset.cpp), without a
GPU: the ground-truth readers of the engine and of the restatement (which reads with `istream >> double` / std::stod
and inverts the calibration with the general 4x4 inverse) on the same files, and the NumPy kitti_frame_filter the GPU
tests also use against the restatement's Eigen-shaped one, bit for bit; the restatement's NCLT reader on hand packets."""
import math

import numpy as np
import pytest

import dataset_ref as ref
import oracle_dataset_lib as orc


@pytest.fixture(scope="module")
def lib():
    import ct_icp_b200
    return ct_icp_b200.engine()


def _flat(poses):
    return np.concatenate([poses["quat"], poses["tr"], poses["dest_timestamp"][:, None],
                           poses["dest_frame_id"][:, None].astype(np.float64)], 1)


def _rand_kitti(rng, n):
    from scipy.spatial.transform import Rotation
    lines = []
    for _ in range(n):
        M = np.eye(4)[:3]
        M[:, :3] = Rotation.from_rotvec(rng.normal(size=3)).as_matrix()
        M[:, 3] = rng.uniform(-300, 300, 3)
        lines.append(" ".join(repr(float(v)) for v in M.reshape(-1)))
    return lines


@pytest.mark.parametrize("dataset,seq", [("KITTI", 1), ("KITTI", 3), ("KITTI_raw", 20), ("KITTI_360", 0),
                                         ("KITTI_CARLA", 0)])
def test_kitti_family_matches_the_restatement(lib, dataset, seq):
    rng = np.random.default_rng(seq)
    lines = _rand_kitti(rng, 20)
    lines[3] = "1 0 0 5"                                    # a short line
    lines[7] = lines[7].replace(" ", "  ", 3) + "  \t"      # extra blanks
    lines[9] = "0.5 0.1 x 3 0 1 0 4 0 0 1 5"                # a value that is not a number: 0, and the line ends
    lines[11] = "1 0 0 nan 0 1 0 2 0 0 1 3"                 # nan and inf are not numbers to istream
    lines[12] = "1 0 0 0x10 0 1 0 inf 0 0 1 3"              # nor is hex past its leading 0
    lines[13] = "1e0 0 0 -2.5e+1 0 1. 0 .5 0 0 1 +3"
    text = "\n".join(lines[:15]) + "\n\n" + "\n".join(lines[15:])
    got, want = _flat(lib.ground_truth(dataset, text, seq)), orc.ground_truth(dataset, text, seq)
    assert got.shape == want.shape
    assert np.abs(got - want).max() < 1e-12 * max(1.0, np.abs(want).max())
    assert np.array_equal(got[:, 7:], want[:, 7:])


def test_nclt_matches_the_restatement(lib):
    rng = np.random.default_rng(4)
    rows = ["%d,%s" % (1_000_000 + i, ",".join(repr(float(v)) for v in
                                                np.concatenate([rng.uniform(-100, 100, 3), rng.uniform(-3, 3, 3)])))
            for i in range(30)]
    rows[5] = "1000005,nan,1,2,0.1,0.2,0.3"
    rows[9] = " 1000009, 1e1,2,3,inf,0.2,0.3"   # std::stod takes blanks, exponents and inf
    text = "\n".join(rows) + "\n"
    got, want = _flat(lib.ground_truth("NCLT", text)), orc.ground_truth("NCLT", text)
    assert got.shape == want.shape and len(want) == 28
    assert np.abs(got[:, :4] - want[:, :4]).max() < 1e-12 and np.abs(got[:, 4:7] - want[:, 4:7]).max() < 1e-10
    assert np.array_equal(got[:, 7:], want[:, 7:])
    for bad in ("1,2,3\n", "1,2,3,x,5,6,7\n", "1,2,3,4,5,6,7\n\n"):
        with pytest.raises(ValueError):
            orc.ground_truth("NCLT", bad)


@pytest.mark.parametrize("dataset", ["HILTI_2021", "HILTI_2022"])
def test_hilti_matches_the_restatement(lib, dataset):
    rng = np.random.default_rng(8)
    lines = []
    for i in range(12):
        q = rng.normal(size=4) * (3.0 if i == 4 else 1.0 / np.linalg.norm(rng.normal(size=4)))
        lines.append(" ".join(repr(float(v)) for v in (10.0 + i, *rng.uniform(-20, 20, 3), *q)))
    lines[6] = ""                      # an empty line: a default pose, as the reference pushes one
    lines[8] = "11.5 1 2"              # a short line
    text = "\n".join(lines) + "\n"
    got, want = _flat(lib.ground_truth(dataset, text)), orc.ground_truth(dataset, text)
    assert got.shape == want.shape == (12, 9)
    assert np.abs(got - want).max() < 1e-12 * max(1.0, np.abs(want).max())


def test_filter_restatements_agree_bit_for_bit():
    """the NumPy filter (the GPU tests' reference) and the Eigen-shaped C++ one, on random, z-axis, cut and NaN points"""
    rng = np.random.default_rng(1)
    p = rng.uniform(-90, 90, (20000, 3))
    p[:, 2] = rng.uniform(-9, 9, len(p))
    p[:20, :2] = 0.0
    p[20:30, 2] = -5.0
    p[30, 2] = np.nan
    p[31, 1] = np.nan
    p[32] = [0.0, -0.0, 4.0]
    a, b = ref.kitti_frame_filter(p), orc.kitti_frame_filter(p)
    assert np.array_equal(a.view(np.uint64), b.view(np.uint64))
    c = math.cos(0.205 * math.pi / 180.0)
    assert b[0, 2] == (p[0, 2] * c if p[0, 2] > -5 else 0.0)


def test_nclt_restatement_on_hand_packets():
    data = ref.pack_packet(7, [[20000, 20000, 20000], [0, 65535, 1]]) + ref.pack_packet(8, []) + \
        ref.pack_packet(9, [[1, 2, 3]])
    xyz, t, ends = orc.nclt_decode(data, 2, True)
    r = ref.decode(data, 2, True)
    assert np.array_equal(xyz, np.concatenate([f[0] for f in r["frames"]])) and ends.tolist() == [2, 3]
    assert t.tolist() == [7.0, 7.0, 9.0]
    assert len(orc.nclt_decode(data[:-2], 2, False)[2]) == 1
    with pytest.raises(ValueError):
        orc.nclt_decode(data[:-2], 2, True)
    bad = bytearray(data)
    bad[len(data) - 32] ^= 1
    with pytest.raises(ValueError):
        orc.nclt_decode(bytes(bad), 2, True)
