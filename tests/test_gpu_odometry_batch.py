"""cticp_odometry_register_batch (Binding.register_batch): one frame on each of many handles in one call, the eligible
Gauss-Newton loops in one grouped launch across their maps. Every handle is compared with a twin driven by the
single-frame entries: summaries (wall-clock and device-time fields aside), trajectory, the three point vectors and the
map, byte for byte — or, when the problems do not fit on the device together, against the CPU oracle and against a
second identical run."""
import ctypes as C

import numpy as np
import pytest

from ct_icp_b200 import _abi as abi
from ct_icp_b200 import synthetic as syn
from ct_icp_b200._binding import CticpError
from conftest import frame_diff
from test_gpu_device_io import _assert_same, _options, _state, _summary_bytes
from test_gpu_parity import POSE_TOL_M, POSE_TOL_RAD, _sequence_options

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

N_FRAMES = 8


@pytest.fixture
def solo_grids_fit(monkeypatch):
    """512 keypoints per gather CTA (CTICP_GN_KP_PER_CTA, read when a handle is created): the solo grids of a few
    small-scan problems fit on the device together — the condition for bit-identity with the single-frame calls. With
    the default of 8, two small16 problems (~1.2k keypoints each, and ~10k points in the first registration's estimate)
    already share the device's CTAs."""
    monkeypatch.setenv("CTICP_GN_KP_PER_CTA", "512")


def _small_seq(seed, n=N_FRAMES, f32=False):
    seq = syn.make_sequence(n, syn.SMALL16, seed=seed)
    if f32:   # float32-representable coordinates: no residual plane
        for s in seq:
            s["xyz"] = s["xyz"].astype(np.float32).astype(np.float64)
    return seq


def _gn_variant(eng, i):
    """bench GN options, varied per handle: neighbor count, map kind, start-up length"""
    o = _options(eng, "gn")
    o.ct_icp_options.max_number_neighbors = (20, 12, 28, 16)[i % 4]
    o.init_num_frames = (3, 5, 2, 6)[i % 4]
    if i % 2 == 1:   # a two-resolution map instead of the legacy one
        m = eng.default_map_options()
        m.num_resolutions = 2
        o.map_options = m
    return o


def _run_twins(eng, options, seqs):
    """the single-frame twins: every handle registers its sequence alone"""
    out = []
    for o, seq in zip(options, seqs):
        od = eng.odometry(o)
        out.append((od, [od.RegisterFrame(s["xyz"], s["t"], s["frame_idx"]) for s in seq]))
    return out


@pytest.mark.parametrize("B", [2, 3, 4])
def test_fitting_batch_is_bit_identical(eng, solo_grids_fit, B):
    options = [_gn_variant(eng, i) for i in range(B)]
    seqs = [_small_seq(100 + i, f32=(i != B - 1)) for i in range(B)]   # the last handle's scans need the residual plane
    twins = _run_twins(eng, options, seqs)
    ods = [eng.odometry(o) for o in options]
    sums = [[] for _ in range(B)]
    for k in range(N_FRAMES):
        out = eng.register_batch(ods, [(seqs[b][k]["xyz"], seqs[b][k]["t"]) for b in range(B)],
                                 [seqs[b][k]["frame_idx"] for b in range(B)])
        for b in range(B):
            sums[b].append(out[b])
            assert ods[b].last_timing().icp_batch_groups == (B if k > 0 else 0), (k, b)
    for b in range(B):
        _assert_same(twins[b][0], ods[b], twins[b][1], sums[b])


def test_mixed_eligibility(eng, solo_grids_fit):
    """one batch mixing joining frames with every kind of frame that takes its single-frame path"""
    profiles = ["gn", "gn", "default_driving_ceres", "robust_driving", "constant_velocity", "gn", "gn", "gn", "gn"]
    seqs = [_small_seq(200 + i, n=5, f32=True) for i in range(len(profiles))]
    options = [_options(eng, p) for p in profiles]
    options[6].quit_on_error = 1   # handles 6 and 7: too few keypoints from frame 2 on
    options[7].quit_on_error = 0
    twins = [eng.odometry(o) for o in options]
    ods = [eng.odometry(o) for o in options]
    events = {"twin": [], "batch": []}
    twins[5].RegisterCallback(lambda e: events["twin"].append(e) or True)
    ods[5].RegisterCallback(lambda e: events["batch"].append(e) or True)
    few = 60
    for k in range(4):
        # handle 8 starts late: its frame 0 rides along with the others' frame 2
        members = [i for i in range(9) if i < 8 or k >= 2]
        scans, fids = [], []
        for i in members:
            s = seqs[i][k - 2 if i == 8 else k]
            xyz, t = s["xyz"], s["t"]
            if i in (6, 7) and k >= 2:
                xyz, t = xyz[::len(xyz) // few][:few], t[::len(t) // few][:few]
            scans.append((xyz, t))
            fids.append(s["frame_idx"])
        want = [twins[i].RegisterFrame(xyz, t, f) for i, (xyz, t), f in zip(members, scans, fids)]
        got = eng.register_batch([ods[i] for i in members], scans, fids)
        joiners = ([0, 1, 6, 7] if k >= 1 else []) + ([8] if k == 3 else [])
        for i, a, b in zip(members, want, got):
            assert _summary_bytes(a) == _summary_bytes(b), (k, i)
            first_frame = k == 0 or (i == 8 and k == 2)
            expect = len(joiners) if i in joiners else 0 if first_frame else 1
            assert ods[i].last_timing().icp_batch_groups == expect, (k, i)
        if k >= 2:
            assert not got[members.index(6)].success and not got[members.index(7)].success
    for i in range(9):
        _assert_same(twins[i], ods[i], [], [])
    assert events["twin"] == events["batch"] and len(events["batch"]) > 0


def test_input_kinds(eng, solo_grids_fit):
    seqs = [_small_seq(300 + i) for i in range(3)]
    options = [_options(eng, "gn") for _ in range(3)]
    twins = [eng.odometry(o) for o in options]
    ods = [eng.odometry(o) for o in options]
    side = torch.cuda.Stream()
    sums_t, sums_b = [[] for _ in range(3)], [[] for _ in range(3)]
    for k in range(6):
        s0, s1, s2 = seqs[0][k], seqs[1][k], seqs[2][k]
        sums_t[0].append(twins[0].RegisterFrame(s0["xyz"], s0["t"], s0["frame_idx"]))
        sums_t[1].append(twins[1].RegisterFrame(torch.from_numpy(s1["xyz"]).cuda(), torch.from_numpy(s1["t"]).cuda(),
                                                s1["frame_idx"]))
        slot_t = twins[2].stage_frame(s2["xyz"], s2["t"])
        sums_t[2].append(twins[2].RegisterStaged(slot_t, s2["frame_idx"]))
        with torch.cuda.stream(side):   # written on a side stream: the batch reads it behind that stream's work
            xyz = torch.from_numpy(s1["xyz"]).to("cuda", non_blocking=True) * 1.0
            t = torch.from_numpy(s1["t"]).to("cuda", non_blocking=True) + 0.0
            slot = ods[2].stage_frame(s2["xyz"], s2["t"])
            out = eng.register_batch(ods, [(s0["xyz"], s0["t"]), (xyz, t), slot],
                                     [s0["frame_idx"], s1["frame_idx"], s2["frame_idx"]])
        for b in range(3):
            sums_b[b].append(out[b])
            if k > 0:
                assert ods[b].last_timing().icp_batch_groups == 3
    for b in range(3):
        _assert_same(twins[b], ods[b], sums_t[b], sums_b[b])


def _hdl64_batch(eng, seqs):
    ods = [eng.odometry(_sequence_options(eng, "GN")) for _ in seqs]
    sums = []
    for k in range(len(seqs[0])):
        sums.append(eng.register_batch(ods, [(s[k]["xyz"], s[k]["t"]) for s in seqs], [s[k]["frame_idx"] for s in seqs]))
    return ods, sums


def test_oversubscribed_hdl64_matches_oracle_and_itself(orc, eng):
    """four bench-size problems do not fit with their solo grids: the CTAs are shared, results differ from the solo
    call by summation order only — within the parity tolerance of the oracle, and reproducible run to run"""
    seqs = [syn.make_sequence(6, syn.HDL64, seed=400 + i) for i in range(4)]
    ods, sums = _hdl64_batch(eng, seqs)
    assert ods[0].last_timing().icp_batch_groups == 4
    for b, seq in enumerate(seqs):
        od = orc.odometry(_sequence_options(orc, "GN"))
        for k, s in enumerate(seq):
            so = od.RegisterFrame(s["xyz"], s["t"], s["frame_idx"])
            assert so.success and sums[k][b].success, (b, k)
            dt, dr = frame_diff(so.frame, sums[k][b].frame)
            assert dt < POSE_TOL_M and dr < POSE_TOL_RAD, (b, k, dt, dr)
    ods2, sums2 = _hdl64_batch(eng, seqs)
    for b in range(4):
        assert _state(ods[b]) == _state(ods2[b])
        for k in range(len(sums)):
            assert _summary_bytes(sums[k][b]) == _summary_bytes(sums2[k][b])


def test_argument_errors_touch_nothing(eng, solo_grids_fit):
    seqs = [_small_seq(500 + i, n=3) for i in range(2)]
    ods = [eng.odometry(_options(eng, "gn")) for _ in range(2)]
    for k in range(2):
        eng.register_batch(ods, [(s[k]["xyz"], s[k]["t"]) for s in seqs], [s[k]["frame_idx"] for s in seqs])
    before = [_state(od) for od in ods]
    s = [x[2] for x in seqs]
    bad = [([ods[0], ods[0]], [(s[0]["xyz"], s[0]["t"])] * 2, [9, 9]),   # the same handle twice
           ([ods[0], ods[1]], [(s[0]["xyz"], s[0]["t"]), (s[1]["xyz"], s[1]["t"]), 3], [9, 9, 9])]
    with pytest.raises(CticpError) as e:
        eng.register_batch(*bad[0])
    assert e.value.code == abi.ERR_INVALID_ARGUMENT
    with pytest.raises(ValueError):
        eng.register_batch(*bad[1])
    # raw calls: a batch of 0 and of 65 items, a null handle, a staged item with an initial estimate
    items = (abi.BatchFrame * 2)()
    fn = eng.fn("odometry_register_batch")
    assert fn(items, 0) == abi.ERR_INVALID_ARGUMENT
    assert fn(items, 65) == abi.ERR_INVALID_ARGUMENT
    out = abi.Summary()
    items[0].kind, items[0].out = abi.BATCH_STAGED, C.addressof(out)
    assert fn(items, 1) == abi.ERR_INVALID_ARGUMENT   # null handle
    items[0].handle = ods[0].h.value
    est = abi.Frame()
    items[0].initial_estimate = C.addressof(est)
    assert fn(items, 1) == abi.ERR_INVALID_ARGUMENT
    for od, b in zip(ods, before):
        assert _state(od) == b


def test_timestamp_error_ends_its_item_alone(eng, solo_grids_fit):
    seqs = [_small_seq(600 + i, n=5) for i in range(3)]
    options = [_options(eng, "gn") for _ in range(3)]
    twins = [eng.odometry(o) for o in options]
    ods = [eng.odometry(o) for o in options]
    sums_t, sums_b = [[] for _ in range(3)], [[] for _ in range(3)]
    for k in range(5):
        ests = [None, None, None]
        if k == 3:   # handle 1's estimate ends before its scan does
            s = seqs[1][k]
            est = abi.Frame()
            for p, ts in ((est.begin_pose, s["t"].min() - 2.0), (est.end_pose, s["t"].min() - 1.0)):
                p.quat[:] = (0, 0, 0, 1)
                p.dest_timestamp = ts
            ests[1] = est
        for b in range(3):
            s = seqs[b][k]
            if ests[b] is None:
                sums_t[b].append(twins[b].RegisterFrame(s["xyz"], s["t"], s["frame_idx"]))
            else:
                with pytest.raises(CticpError) as e:
                    twins[b].RegisterFrameWithEstimate(s["xyz"], s["t"], ests[b], s["frame_idx"])
                assert e.value.code == abi.ERR_TIMESTAMP
        scans = [(seqs[b][k]["xyz"], seqs[b][k]["t"]) for b in range(3)]
        fids = [seqs[b][k]["frame_idx"] for b in range(3)]
        if k == 3:
            with pytest.raises(CticpError) as e:
                eng.register_batch(ods, scans, fids, initial_estimates=ests)
            assert e.value.code == abi.ERR_TIMESTAMP
            assert e.value.statuses == [0, abi.ERR_TIMESTAMP, 0]
            for b in (0, 2):
                assert ods[b].last_timing().icp_batch_groups == 2
                sums_t[b].pop()   # (the raising call returns no summaries: trajectory, points and map still compared)
            continue
        out = eng.register_batch(ods, scans, fids)
        for b in range(3):
            sums_b[b].append(out[b])
    for b in (0, 2):
        _assert_same(twins[b], ods[b], sums_t[b], sums_b[b])
    assert _state(twins[1]) == _state(ods[1])
