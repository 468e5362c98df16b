"""Paired tiles of k_gn_persistent from the first Gauss-Newton iteration on (icp_gn.cu, gn_pair_schedule): a gather CTA
with 17..32 keypoints gives each warp one tile in every iteration, the first one pairing in keypoint order (no costs
yet). Neither the schedule nor where the kernel reads its parameters from may change a bit of the result: every output
is compared byte for byte with the one-keypoint-per-grab schedule (CTICP_DEBUG_FLAGS=8, read at every registration
call), with a repeat of the same call and with the CPU oracle — for solo calls (with and without the rigid first
iteration), for pairs whose candidates overflow the staging area (sel_compact inside a pair) and for grouped launches.

A solo call of K >= 1032 keypoints gathers on all 131 gather CTAs of an H100 SXM (132 co-resident CTAs of the kernel),
so K = 131 s gives every gather CTA a range of s keypoints."""

import numpy as np
import pytest

from ct_icp_b200 import _abi as abi
from ct_icp_b200 import synthetic as syn
from conftest import frame_diff
from test_gpu_gn_pair_schedule import GATHER_CTAS, _keypoints, _register, _same
from test_gpu_icp_batch import _gn_options, _map_options, _perturbed, _with_world, case, emap  # noqa: F401
from test_gpu_odometry_batch import _summary_bytes
from test_gpu_parity import POSE_TOL_M, POSE_TOL_RAD

pytestmark = pytest.mark.gpu

CORESIDENT = GATHER_CTAS + 1


def _check_solo(orc, eng, m, map_options, map_xyz, io_of, k, f0, prev, monkeypatch):
    """k registered on map m with options io_of(backend): default schedule == repeat == grab schedule, and the oracle"""
    mm = eng.default_odometry_options().default_motion_model
    io = io_of(eng)
    new = _register(m, io, k, f0, prev, mm, monkeypatch, 0)
    assert new[2].success and new[2].num_iters > 1
    _same(new, _register(m, io, k, f0, prev, mm, monkeypatch, 0))
    _same(new, _register(m, io, k, f0, prev, mm, monkeypatch, 8))
    mo = orc.voxel_map(map_options(orc))
    mo.insert(map_xyz)
    ko, fo = k.copy(), f0.copy()
    so = mo.icp_register(io_of(orc), ko, fo, prev, orc.default_odometry_options().default_motion_model)
    assert so.success and so.num_residuals_used == new[2].num_residuals_used
    dt, dr = frame_diff(fo, new[1])
    assert dt < 1e-6 and dr < 1e-6, (dt, dr)
    assert np.abs(ko["world"] - new[0]["world"]).max() < 1e-5


def _rigid_options(b):
    """parametrization SIMPLE without distortion: the first iteration transforms the keypoints rigidly (rigid_first)"""
    io = _gn_options(b)
    io.parametrization = abi.PARAMETRIZATION["SIMPLE"]
    io.point_to_plane_with_distortion = 0
    return io


@pytest.mark.parametrize("rigid", [False, True])
@pytest.mark.parametrize("span", [16, 17, 24, 32, 33])
def test_solo_spans(orc, eng, case, emap, span, rigid, monkeypatch):  # noqa: F811
    map_xyz, kp, frame, prev = case
    f0 = _perturbed(frame, span + 7 * rigid)
    k = _with_world(orc, _keypoints(kp, GATHER_CTAS * span), f0)
    _check_solo(orc, eng, emap, _map_options, map_xyz, _rigid_options if rigid else _gn_options, k, f0, prev, monkeypatch)


def _dense_map_options(b):
    """60 points per 1 m voxel, 2 cm apart: several hundred in-radius candidates per stencil, more than a batch leaves
    room for in the staging area (sel_compact runs inside the pairs)"""
    o = b.legacy_map_options(1.0, 60, 0.02)
    o.capacity_voxels = 1 << 18
    return o


@pytest.mark.parametrize("kmax", [20, 32])
def test_pairs_that_compact(orc, eng, case, kmax, monkeypatch):  # noqa: F811
    map_xyz, kp, frame, prev = case
    m = eng.voxel_map(_dense_map_options(eng))
    m.insert(map_xyz)

    def io_of(b):
        io = _gn_options(b)
        io.max_number_neighbors = kmax
        return io

    f0 = _perturbed(frame, kmax)
    k = _with_world(orc, _keypoints(kp, GATHER_CTAS * 20), f0)
    _check_solo(orc, eng, m, _dense_map_options, map_xyz, io_of, k, f0, prev, monkeypatch)


def _gather_ctas(n, kp_per_cta):
    """icp_batch.cu BatchGatherCtas for these counts on CORESIDENT CTAs"""
    solo = [max(1, min(-(-(x + 16) // kp_per_cta), CORESIDENT - 1)) for x in n]
    if sum(1 + s for s in solo) <= CORESIDENT:
        return solo
    g = [1] * len(n)
    for _ in range(CORESIDENT - 2 * len(n)):
        best = -1
        for b in range(len(n)):
            if g[b] < solo[b] and (best < 0 or n[b] * g[best] > n[best] * g[b]):
                best = b
        if best < 0:
            break
        g[best] += 1
    return g


def _odometry_options(b, i):
    o = b.default_odometry_options()
    o.ct_icp_options.solver = abi.SOLVER["GN"]
    o.ct_icp_options.num_iters_icp = 5
    o.ct_icp_options.min_number_neighbors = 10
    o.ct_icp_options.max_number_neighbors = (20, 16, 28, 24)[i % 4]
    o.map_options = b.legacy_map_options(1.0, 20, 0.1)
    o.voxel_size, o.sample_voxel_size, o.max_distance = 0.5, 2.0, 100.0
    o.init_num_frames = 3
    o.debug_print = 0
    o.ct_icp_options.debug_print = 0
    return o


@pytest.mark.parametrize("B", [2, 4])
def test_grouped_odometry_batch(orc, eng, B, monkeypatch):
    """cticp_odometry_register_batch: the grouped launch (k_gn_persistent<false, true>), 24 keypoints per gather CTA"""
    monkeypatch.setenv("CTICP_GN_KP_PER_CTA", "24")
    seqs = [syn.make_sequence(6, syn.SMALL16, seed=700 + i) for i in range(B)]

    def run(flags):
        monkeypatch.setenv("CTICP_DEBUG_FLAGS", str(flags))
        ods = [eng.odometry(_odometry_options(eng, i)) for i in range(B)]
        sums = [eng.register_batch(ods, [(s[k]["xyz"], s[k]["t"]) for s in seqs], [s[k]["frame_idx"] for s in seqs])
                for k in range(len(seqs[0]))]
        monkeypatch.delenv("CTICP_DEBUG_FLAGS")
        return sums

    got, again, grab = run(0), run(0), run(8)
    paired = False
    for k in range(len(got)):
        n = [got[k][b].num_keypoints for b in range(B)]
        paired |= any(16 * g < x <= 32 * g for x, g in zip(n, _gather_ctas(n, 24)))
        for b in range(B):
            assert got[k][b].success
            assert _summary_bytes(got[k][b]) == _summary_bytes(again[k][b])
            assert bytes(got[k][b].frame) == bytes(grab[k][b].frame)
    assert paired, "no group had ranges of 17..32 keypoints"
    for b, seq in enumerate(seqs):
        od = orc.odometry(_odometry_options(orc, b))
        for k, s in enumerate(seq):
            so = od.RegisterFrame(s["xyz"], s["t"], s["frame_idx"])
            assert so.success, (b, k)
            dt, dr = frame_diff(so.frame, got[k][b].frame)
            assert dt < POSE_TOL_M and dr < POSE_TOL_RAD, (b, k, dt, dr)
