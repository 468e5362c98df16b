"""The CPU restatement of slam::Scene / SyntheticSensorAcquisition (tests/oracle_synthetic) on hand-computed cases and
invariants: each primitive's Distance (the line's projection quirk, rank-2 and rank-3 triangles, points on vertices),
the draw contract, GeneratePoses on the courtyard, and the geometry of generated frames over random scenes. No GPU."""
import json
import math
import os

import numpy as np
import pytest

from ct_icp_b200 import _abi as abi
from oracle_synthetic_lib import synthetic_oracle

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
COURTYARD = os.path.join(ROOT, "tests", "golden", "synthetic_courtyard.json")
RAND_MAX = 2147483647


def _splitmix64(x):
    m = (1 << 64) - 1
    x = (x + 0x9E3779B97F4A7C15) & m
    x = ((x ^ (x >> 30)) * 0xBF58476D1CE4E5B9) & m
    x = ((x ^ (x >> 27)) * 0x94D049BB133111EB) & m
    return x ^ (x >> 31)


def _u(seed, frame_key, prim, point, j):
    """the draw contract of include/cticp.h, restated"""
    key = _splitmix64(_splitmix64(_splitmix64(seed) ^ frame_key) ^ prim)
    return _splitmix64(key ^ ((point << 3) | j)) >> 33


def _rnd(u):
    return -1.0 + (2.0 * u) / RAND_MAX


def test_draw_mapping_endpoints():
    assert _rnd(0) == -1.0 and _rnd(RAND_MAX) == 1.0
    assert 0 / RAND_MAX == 0.0 and RAND_MAX / RAND_MAX == 1.0
    us = [_u(7, 3, p, i, j) for p in range(3) for i in range(50) for j in range(5)]
    assert all(0 <= u <= RAND_MAX for u in us) and len(set(us)) == len(us)


def test_line_points_follow_the_draw_contract():
    o = synthetic_oracle()
    sc = o.synthetic_scene(lines=[[[1, 2, 3], [4, -5, 6]]])
    xyz, src = sc.generate_points(20, seed=11)
    points_key = (1 << 32) | 1
    for i in range(20):
        c0, c1 = abs(_rnd(_u(11, points_key, 0, i, 0))), abs(_rnd(_u(11, points_key, 0, i, 1)))
        s = c0 + c1
        c0, c1 = c0 / s, c1 / s
        want = [1 * c0 + 4 * c1, 2 * c0 + -5 * c1, 3 * c0 + 6 * c1]
        assert list(xyz[i]) == want
    assert (src[:, 0] == 0).all() and (src[:, 1] == np.arange(20)).all()


def test_distance_spheres_and_balls():
    o = synthetic_oracle()
    sc = o.synthetic_scene(spheres=[[0, 0, 0, 2]], balls=[[0, 0, 0, 2]])
    d = sc.distance([[3, 0, 0], [1, 0, 0], [0, 0, 0]])
    assert d.tolist() == [[1.0, 1.0], [1.0, 0.0], [2.0, 0.0]]


def test_distance_line_projects_with_abs():
    """p0 + |(x - p0).d| d with d = normalized(p0 - p1): a point beside the segment projects beyond p0, so the distance is
    that of the nearest of p0 / p1 / barycentre, not the distance to the segment"""
    o = synthetic_oracle()
    sc = o.synthetic_scene(lines=[[[0, 0, 0], [1, 0, 0]]])
    d = sc.distance([[0.25, 0.1, 0.0], [0.0, 0.0, 0.0], [1.0, 0.0, 0.0], [-2.0, 0.0, 0.0]])
    assert d[0, 0] == pytest.approx(math.sqrt(0.25 * 0.25 + 0.1 * 0.1), rel=1e-15)   # the segment is 0.1 away
    assert d[1, 0] == 0.0 and d[2, 0] == 0.0
    assert d[3, 0] == 2.0


def test_distance_rank2_triangle_of_the_floor():
    """courtyard's floor: A = [p0 p1 p2] has rank 2 (every corner at z = 0), the free coefficient is 0"""
    o = synthetic_oracle()
    sc = o.synthetic_scene(triangles=[[[0, 0, 0], [0, 10, 0], [5, 10, 0]]])
    d = sc.distance([[1, 5, 2], [4, 2, 0], [0, 0, 0], [5, 10, 0], [1, 5, 0]])[:, 0]
    assert d[0] == 2.0                     # inside: |point to plane|
    assert d[1] == math.sqrt(20.0)         # outside: the nearest corner (0, 0, 0)
    assert d[2] == 0.0 and d[3] == 0.0     # on vertices
    assert d[4] == 0.0


def test_distance_rank3_triangle():
    o = synthetic_oracle()
    sc = o.synthetic_scene(triangles=[[[1, 0, 0], [0, 1, 0], [0, 0, 1]]])
    d = sc.distance([[1, 1, 1], [1, 0, 0], [-1, -1, -1]])[:, 0]
    assert d[0] == pytest.approx(2 / math.sqrt(3), rel=1e-15)
    assert d[1] == 0.0
    assert d[2] == pytest.approx(4 / math.sqrt(3), rel=1e-15)   # projects onto the barycentre: inside


def _courtyard():
    with open(COURTYARD) as f:
        return json.load(f)


def test_courtyard_fixture_shape():
    spec = _courtyard()
    acq = spec["acquisition"]
    assert len(acq["poses"]) == 11 and len(acq["triangles"]) == 40 and len(acq["lines"]) == 9
    assert len(acq["spheres"]) == 4 and acq["balls"] == []
    assert spec["sample_frequency"] == 40.0 and spec["max_lidar_distance"] == 15.0
    assert spec["num_points_per_primitives"] == 300


def test_courtyard_generate_poses_count():
    """t += 1/40 summed in fp64 passes 10 after 400 steps (10.000000000000075), so the pose at t = 10 is not sampled"""
    o = synthetic_oracle()
    seq = o.synthetic_sequence(_courtyard(), num_frames=2)
    gt = seq["ground_truth"]
    assert len(gt) == 400 and len(seq["frames"]) == 2
    assert (gt["dest_frame_id"] == np.arange(400)).all()
    assert gt[0]["quat"].tolist() == [0, 0, 0, 1] or np.allclose(gt[0]["quat"], [0, 0, 0, 1], atol=1e-15)
    assert np.abs(gt[0]["tr"]).max() < 1e-15


def _random_scene(rng, nt=20, nl=10, ns=8, nb=8, spread=20.0):
    tri = rng.uniform(-spread, spread, (nt, 3, 3))
    tri[: nt // 4, :, 2] = 0.0   # floor triangles: rank-2 factors
    lines = rng.uniform(-spread, spread, (nl, 2, 3))
    sph = np.concatenate([rng.uniform(-spread, spread, (ns, 3)), rng.uniform(0.1, 3.0, (ns, 1))], axis=1)
    ball = np.concatenate([rng.uniform(-spread, spread, (nb, 3)), rng.uniform(0.1, 3.0, (nb, 1))], axis=1)
    return tri, lines, sph, ball


def _random_poses(rng, n=6, spin=2.0):
    poses = []
    for k in range(n):
        axis = rng.normal(size=3)
        axis /= np.linalg.norm(axis)
        ang = rng.uniform(-spin, spin)
        q = list(axis * math.sin(ang / 2)) + [math.cos(ang / 2)]
        poses.append(abi.Pose.make(q, rng.uniform(-5, 5, 3).tolist(), float(k), k))
    return poses


def _qrot(q, v):
    x, y, z, w = q
    qv = np.array([x, y, z])
    uv = 2 * np.cross(qv, v)
    return v + w * uv + np.cross(qv, uv)


def _slerp(a, b, t):
    d = float(np.dot(a, b))
    if abs(d) >= 1 - 2.220446049250313e-16:
        s0, s1 = 1 - t, t
    else:
        th = math.acos(abs(d))
        s0, s1 = math.sin((1 - t) * th) / math.sin(th), math.sin(t * th) / math.sin(th)
    if d < 0:
        s1 = -s1
    return s0 * a + s1 * b


@pytest.mark.parametrize("seed", [1, 2, 3])
def test_generated_frames_geometry(seed):
    rng = np.random.default_rng(seed)
    tri, lines, sph, ball = _random_scene(rng)
    o = synthetic_oracle()
    sc = o.synthetic_scene(tri, lines, sph, ball)
    traj = o.continuous_trajectory(_random_poses(rng))
    frames = [(0.0, 0.7, 0), (1.2, 2.0, 1), (2.5, 2.5, 2), (3.0, 4.6, 3)]
    d = 18.0
    raw = sc.generate_frames(traj, frames, 40, d, seed=seed, with_source_index=True)
    world = sc.generate_frames(traj, frames, 40, d, seed=seed, world=True)
    n = len(raw["t"])
    assert n > 100 and (raw["frame_ends"] == world["frame_ends"]).all() and raw["frame_ends"][-1] == n
    src = raw["src_index"]
    starts = np.concatenate([[0], raw["frame_ends"][:-1]]).astype(np.int64)
    nt, nl, ns = len(tri), len(lines), len(sph)
    for k, (b, e, _) in enumerate(frames):
        sl = slice(starts[k], int(raw["frame_ends"][k]))
        pb, pe = traj.interpolate([b, e])
        t0, t1 = pb["dest_timestamp"], pe["dest_timestamp"]   # the interpolated poses' own timestamps
        t = raw["t"][sl]
        # begin.ts (1 - alpha) + alpha end.ts rounds: within an ulp of [t0, t1]
        ulp = np.spacing(max(abs(t0), abs(t1), 1.0))
        assert ((t >= t0 - ulp) & (t <= t1 + ulp)).all()
        assert (np.linalg.norm(raw["xyz"][sl], axis=1) < d).all()
        # (primitive, point) ascending: the order of GenerateSensorPoints
        key = src[sl, 0].astype(np.int64) * 100 + src[sl, 1]
        assert (np.diff(key) > 0).all()
        for i in range(sl.start, sl.stop, 7):
            alpha = 0.0 if t1 == t0 else (raw["t"][i] - t0) / (t1 - t0)
            q = _slerp(np.array(pb["quat"]), np.array(pe["quat"]), alpha)
            q = q / np.linalg.norm(q)
            tr = (1 - alpha) * np.array(pb["tr"]) + alpha * np.array(pe["tr"])
            w = _qrot(q, raw["xyz"][i]) + tr
            assert np.abs(w - world["xyz"][i]).max() < 1e-12 * max(1.0, np.abs(w).max())
    # each primitive's points lie on it
    for i in range(n):
        p, w = int(src[i, 0]), world["xyz"][i]
        if p < nt:
            A = np.vstack([tri[p].T, np.ones(3)])   # a convex combination of the corners
            c = np.linalg.lstsq(A, np.append(w, 1.0), rcond=None)[0]
            assert (c > -1e-9).all() and np.abs(A @ c - np.append(w, 1.0)).max() < 1e-9
        elif p < nt + nl:
            a, bb = lines[p - nt]
            assert np.linalg.norm(np.cross(w - a, bb - a)) <= 1e-9 * np.linalg.norm(bb - a) * max(1, np.abs(w).max())
        elif p < nt + nl + ns:
            c, r = sph[p - nt - nl, :3], sph[p - nt - nl, 3]
            assert abs(np.linalg.norm(w - c) - r) <= 1e-15 * 8 * max(r, np.abs(c).max())
        else:
            c, r = ball[p - nt - nl - ns, :3], ball[p - nt - nl - ns, 3]
            assert np.linalg.norm(w - c) <= r * (1 + 1e-15) + 1e-14


def test_refusals():
    o = synthetic_oracle()
    sc = o.synthetic_scene(spheres=[[0, 0, 0, 1]])
    traj = o.continuous_trajectory(_random_poses(np.random.default_rng(0), 3))
    from ct_icp_b200._binding import CticpError
    for args in [((0.0, 1.0, 0),), ]:
        with pytest.raises(CticpError):
            sc.generate_frames(traj, list(args), 1, 5.0)          # fewer than two points per primitive
        with pytest.raises(CticpError):
            sc.generate_frames(traj, list(args), 10, 0.0)         # d <= 0
        with pytest.raises(CticpError):
            sc.generate_frames(traj, [(1.0, 0.5, 0)], 10, 5.0)    # begin_ts > end_ts
    with pytest.raises(CticpError):
        o.synthetic_scene(spheres=[[0, 0, 0, -1]])
    with pytest.raises(CticpError):
        o.synthetic_scene(triangles=[[[0, 0, float("nan")], [0, 1, 0], [1, 0, 0]]])
