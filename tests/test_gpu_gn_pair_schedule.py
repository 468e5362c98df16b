"""Paired tile schedule of k_gn_persistent (icp_gn.cu, gn_pair_schedule): from the second Gauss-Newton iteration on, a
gather CTA with 17..32 keypoints gives each warp one tile, the heaviest keypoints alone and the others in pairs. Which warp
computes which keypoint's row must not change a bit of the result: every output is compared byte for byte with the
one-keypoint-per-grab schedule (CTICP_DEBUG_FLAGS=8, read at every registration call), with a repeat of the same call and
with the CPU oracle.

Keypoint counts are chosen for the per-CTA ranges: a solo call of K >= 1032 keypoints gathers on all 131 gather CTAs of an
H100 SXM (132 co-resident CTAs of the kernel), so K = 131 s gives every gather CTA a range of s keypoints."""

import numpy as np
import pytest

from conftest import frame_diff
from test_gpu_icp_batch import _gn_options, _map_options, _perturbed, _with_world, case, emap  # noqa: F401

pytestmark = pytest.mark.gpu

GATHER_CTAS = 131


def _keypoints(kp, n):
    """n keypoints: the frame's, every 9th first (spread over the scan), repeated where the frame has fewer"""
    order = np.concatenate([np.arange(j, len(kp), 9) for j in range(9)])
    idx = np.resize(order, n)
    return kp[idx].copy()


def _register(m, io, kp, frame, prev, mm, monkeypatch, flags):
    monkeypatch.setenv("CTICP_DEBUG_FLAGS", str(flags))
    k, f = kp.copy(), frame.copy()
    s = m.icp_register(io, k, f, prev, mm)
    monkeypatch.delenv("CTICP_DEBUG_FLAGS")
    return k, f, s


def _same(a, b):
    ka, fa, sa = a
    kb, fb, sb = b
    assert bytes(fa) == bytes(fb)
    assert (sa.success, sa.num_residuals_used, sa.num_iters) == (sb.success, sb.num_residuals_used, sb.num_iters)
    assert ka["world"].tobytes() == kb["world"].tobytes()


@pytest.mark.parametrize("span", [16, 17, 24, 32, 33])
def test_solo_register_same_bits_as_grab_schedule(orc, eng, case, emap, span, monkeypatch):  # noqa: F811
    map_xyz, kp, frame, prev = case
    io = _gn_options(eng)
    mm = eng.default_odometry_options().default_motion_model
    f0 = _perturbed(frame, span)
    k = _with_world(orc, _keypoints(kp, GATHER_CTAS * span), f0)
    new = _register(emap, io, k, f0, prev, mm, monkeypatch, 0)
    assert new[2].success and new[2].num_iters > 1
    _same(new, _register(emap, io, k, f0, prev, mm, monkeypatch, 0))
    _same(new, _register(emap, io, k, f0, prev, mm, monkeypatch, 8))
    # the CPU oracle, with the tolerances of the batch parity test
    mo = orc.voxel_map(_map_options(orc))
    mo.insert(map_xyz)
    ko, fo = k.copy(), f0.copy()
    so = mo.icp_register(_gn_options(orc), ko, fo, prev, orc.default_odometry_options().default_motion_model)
    assert so.success and so.num_residuals_used == new[2].num_residuals_used
    dt, dr = frame_diff(fo, new[1])
    assert dt < 1e-6 and dr < 1e-6, (dt, dr)
    assert np.abs(ko["world"] - new[0]["world"]).max() < 1e-5


@pytest.mark.parametrize("n", [600, 1000])
def test_batch_same_bits_as_grab_schedule(eng, case, emap, n, monkeypatch):  # noqa: F811
    """4 problems on the 128 gather CTAs left: 32 each, ranges of 18..19 (n = 600) and 31..32 (n = 1000) keypoints"""
    _, kp, frame, prev = case
    io = _gn_options(eng)
    mm = eng.default_odometry_options().default_motion_model
    kps = [_keypoints(kp[b::4], n) for b in range(4)]
    frames = [_perturbed(frame, b) for b in range(4)]

    def batch(flags):
        monkeypatch.setenv("CTICP_DEBUG_FLAGS", str(flags))
        ks, fs = [k.copy() for k in kps], [f.copy() for f in frames]
        ss = emap.icp_register_batch(io, ks, fs, [prev] * 4, mm)
        monkeypatch.delenv("CTICP_DEBUG_FLAGS")
        return list(zip(ks, fs, ss))

    got, again, grab = batch(0), batch(0), batch(8)
    for b in range(4):
        assert got[b][2].success
        _same(got[b], again[b])
        _same(got[b], grab[b])
    # one problem runs the solo launch: the solo call's result
    k24 = _keypoints(kp, GATHER_CTAS * 24)
    ks, fs = [k24.copy()], [frame.copy()]
    s1 = emap.icp_register_batch(io, ks, fs, [prev], mm)
    _same((ks[0], fs[0], s1[0]), _register(emap, io, k24, frame, prev, mm, monkeypatch, 0))


def test_odometry_same_bits_as_grab_schedule(eng, monkeypatch):
    """the bench workload (2.4k-2.6k keypoints a frame: ranges of 18..20 on 131 gather CTAs)"""
    import bench
    seq = bench.make_scans(8, bench.WORKLOADS["kitti64_gn"][0])

    def run(flags):
        monkeypatch.setenv("CTICP_DEBUG_FLAGS", str(flags))
        od = eng.odometry(bench.make_options(eng))
        out = [od.RegisterFrame(s["xyz"], s["t"], s["frame_idx"]) for s in seq]
        monkeypatch.delenv("CTICP_DEBUG_FLAGS")
        return out

    new, grab = run(0), run(8)
    assert any(GATHER_CTAS * 16 < s.num_keypoints <= GATHER_CTAS * 32 for s in new)
    for a, b in zip(new, grab):
        assert a.success and b.success
        assert a.num_keypoints == b.num_keypoints
        assert bytes(a.frame) == bytes(b.frame)
