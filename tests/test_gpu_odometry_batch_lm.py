"""cticp_odometry_register_batch (Binding.register_batch) with solver CERES and ROBUST frames: their Levenberg-Marquardt
loops run in one grouped launch of k_lm_persistent per mode (CERES nearest neighbour, CERES distance-based, ROBUST),
each group against its own handle's map, options and buffers. Every handle is compared with a twin driven by the
single-frame entries: summaries (wall-clock and device-time fields aside), trajectory, the three point vectors and the
map, byte for byte — or, when the problems do not fit on the device together, against the CPU oracle and against a
second identical run."""
import numpy as np
import pytest

from ct_icp_b200 import _abi as abi
from ct_icp_b200 import synthetic as syn
from ct_icp_b200._binding import CticpError
from conftest import frame_diff
from test_gpu_device_io import _assert_same, _options, _state, _summary_bytes
from test_gpu_parity import POSE_TOL_M, POSE_TOL_RAD, _sequence_options

pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

N_FRAMES = 6
LOSSES = ("CAUCHY", "HUBER", "TOLERANT", "TRUNCATED")


@pytest.fixture
def solo_grids_fit(monkeypatch):
    """512 keypoints per gather / worker CTA (CTICP_GN_KP_PER_CTA, read when a handle is created; it sizes the LM solo
    grid too): the solo grids of a few small-scan problems fit on the device together, the condition for bit-identity
    with the single-frame calls."""
    monkeypatch.setenv("CTICP_GN_KP_PER_CTA", "512")


def _small_seq(seed, n=N_FRAMES, f32=True):
    seq = syn.make_sequence(n, syn.SMALL16, seed=seed)
    if f32:   # float32-representable coordinates: no residual plane
        for s in seq:
            s["xyz"] = s["xyz"].astype(np.float32).astype(np.float64)
    return seq


def _lm_variant(eng, i, solver="CERES", strategy="NEAREST_NEIGHBOR_STRATEGY"):
    """the driving profile with solver CERES, varied per handle: loss and inner iterations, closest neighbours and
    residual cap, map kind, start-up length (so that groups run different iteration counts side by side)"""
    o = _options(eng, "default_driving_ceres")
    c = o.ct_icp_options
    c.solver = abi.SOLVER[solver]
    c.loss_function = abi.LOSS[LOSSES[i % 4]]
    c.ls_max_num_iters = (5, 3, 7, 4)[i % 4]
    c.num_closest_neighbors = (1, 2)[i % 2] if solver == "CERES" else 1
    c.max_num_residuals = (600, -1, 900, 1200)[i % 4]
    o.init_num_frames = (3, 5, 2, 4)[i % 4]
    o.neighborhood_strategy.type = abi.STRATEGY[strategy]
    if i % 2 == 0:
        o.map_options = eng.legacy_map_options(1.0, 20, 0.1)
    else:   # a two-resolution map instead of the legacy one
        m = eng.default_map_options()
        m.num_resolutions = 2
        o.map_options = m
    if strategy == "DISTANCE_BASED_STRATEGY":   # the sensor-side normal filter: the map keeps normals
        o.map_options.select_valid_normals_direction = 1
    return o


def _run_twins(eng, options, seqs):
    out = []
    for o, seq in zip(options, seqs):
        od = eng.odometry(o)
        out.append((od, [od.RegisterFrame(s["xyz"], s["t"], s["frame_idx"]) for s in seq]))
    return out


def _batch_matches_twins(eng, options, seqs, groups, require_success=True):
    """B handles through register_batch frame by frame, against their single-frame twins; `groups[b]`: handle b's
    icp_batch_groups from frame 1 on"""
    B = len(options)
    twins = _run_twins(eng, options, seqs)
    ods = [eng.odometry(o) for o in options]
    sums = [[] for _ in range(B)]
    for k in range(len(seqs[0])):
        out = eng.register_batch(ods, [(seqs[b][k]["xyz"], seqs[b][k]["t"]) for b in range(B)],
                                 [seqs[b][k]["frame_idx"] for b in range(B)])
        for b in range(B):
            sums[b].append(out[b])
            assert ods[b].last_timing().icp_batch_groups == (groups[b] if k > 0 else 0), (k, b)
    for b in range(B):
        assert not require_success or all(s.success for s in sums[b]), b
        _assert_same(twins[b][0], ods[b], twins[b][1], sums[b])


@pytest.mark.parametrize("B", [2, 3, 4])
def test_fitting_ceres_batch_is_bit_identical(eng, solo_grids_fit, B):
    options = [_lm_variant(eng, i) for i in range(B)]
    seqs = [_small_seq(700 + i, f32=(i != B - 1)) for i in range(B)]   # the last handle's scans need the residual plane
    _batch_matches_twins(eng, options, seqs, [B] * B)


def test_fitting_robust_batch_is_bit_identical(eng, solo_grids_fit):
    options = [_lm_variant(eng, i, solver="ROBUST") for i in range(3)]
    for o in options:
        o.robust_registration = 0
    seqs = [_small_seq(720 + i, f32=(i != 2)) for i in range(3)]
    _batch_matches_twins(eng, options, seqs, [3] * 3, require_success=False)


def test_fitting_distance_based_batch_is_bit_identical(eng, solo_grids_fit):
    options = [_lm_variant(eng, i, strategy="DISTANCE_BASED_STRATEGY") for i in range(3)]
    seqs = [_small_seq(740 + i, f32=(i != 2)) for i in range(3)]
    _batch_matches_twins(eng, options, seqs, [3] * 3)


def test_mixed_batch_one_launch_per_mode(eng, solo_grids_fit):
    """two frames each of GN, CERES nearest neighbour, CERES distance-based and ROBUST (four grouped launches), and a
    CERES frame with a callback, which takes its single-frame path"""
    kinds = ["gn", "gn", "nn", "nn", "db", "db", "robust", "robust", "callback"]
    options = []
    for i, kind in enumerate(kinds):
        if kind == "gn":
            options.append(_options(eng, "gn"))
        elif kind == "db":
            options.append(_lm_variant(eng, i, strategy="DISTANCE_BASED_STRATEGY"))
        elif kind == "robust":
            o = _lm_variant(eng, i, solver="ROBUST")
            o.robust_registration = 0
            options.append(o)
        else:
            options.append(_lm_variant(eng, i))
    seqs = [_small_seq(760 + i, n=5) for i in range(len(kinds))]
    twins = [eng.odometry(o) for o in options]
    ods = [eng.odometry(o) for o in options]
    events = {"twin": [], "batch": []}
    twins[8].RegisterCallback(lambda e: events["twin"].append(e) or True)
    ods[8].RegisterCallback(lambda e: events["batch"].append(e) or True)
    size = {"gn": 2, "nn": 2, "db": 2, "robust": 2, "callback": 1}
    for k in range(5):
        scans = [(s[k]["xyz"], s[k]["t"]) for s in seqs]
        fids = [s[k]["frame_idx"] for s in seqs]
        want = [tw.RegisterFrame(xyz, t, f) for tw, (xyz, t), f in zip(twins, scans, fids)]
        got = eng.register_batch(ods, scans, fids)
        for i, (a, b) in enumerate(zip(want, got)):
            assert _summary_bytes(a) == _summary_bytes(b), (k, i)
            assert ods[i].last_timing().icp_batch_groups == (size[kinds[i]] if k > 0 else 0), (k, i)
    for i in range(len(kinds)):
        _assert_same(twins[i], ods[i], [], [])
    assert events["twin"] == events["batch"] and len(events["batch"]) > 0


def _hdl64_batch(eng, seqs):
    ods = [eng.odometry(_sequence_options(eng, "CERES")) for _ in seqs]
    sums = []
    for k in range(len(seqs[0])):
        sums.append(eng.register_batch(ods, [(s[k]["xyz"], s[k]["t"]) for s in seqs], [s[k]["frame_idx"] for s in seqs]))
    return ods, sums


def test_oversubscribed_hdl64_ceres_matches_oracle_and_itself(orc, eng):
    """four bench-size CERES problems at the default CTA policy ask for ~131-CTA solo grids each: the groups share the
    device's CTAs, and results differ from the solo call by summation order only — within the parity tolerance of the
    oracle, and reproducible run to run"""
    seqs = [syn.make_sequence(5, syn.HDL64, seed=800 + i) for i in range(4)]
    ods, sums = _hdl64_batch(eng, seqs)
    assert ods[0].last_timing().icp_batch_groups == 4
    for b, seq in enumerate(seqs):
        od = orc.odometry(_sequence_options(orc, "CERES"))
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


def test_per_item_failures_end_alone(eng, solo_grids_fit):
    """handle 1: five closest neighbours (UNSUPPORTED on the LM path, which builds at most four); handle 3: the distance-based strategy with radius_max 0
    (INVALID_ARGUMENT); handle 4: an estimate that ends before its scan at frame 3 (TIMESTAMP). The frames the LM path
    rejects do not join; every failing item gets its twin's status and state, the others join and match their twins."""
    options = [_lm_variant(eng, i) for i in range(6)]
    options[1].ct_icp_options.num_closest_neighbors = 5
    options[3].neighborhood_strategy.type = abi.STRATEGY["DISTANCE_BASED_STRATEGY"]
    options[3].neighborhood_strategy.radius_max = 0.0
    seqs = [_small_seq(820 + i, n=5) for i in range(6)]
    twins = [eng.odometry(o) for o in options]
    ods = [eng.odometry(o) for o in options]
    ok = [0, 2, 4, 5]
    sums_t, sums_b = [[] for _ in range(6)], [[] for _ in range(6)]
    for k in range(5):
        ests = [None] * 6
        if k == 3:
            s = seqs[4][k]
            est = abi.Frame()
            for p, ts in ((est.begin_pose, s["t"].min() - 2.0), (est.end_pose, s["t"].min() - 1.0)):
                p.quat[:] = (0, 0, 0, 1)
                p.dest_timestamp = ts
            ests[4] = est
        want = [0] * 6
        for b in range(6):
            s = seqs[b][k]
            try:
                if ests[b] is None:
                    sums_t[b].append(twins[b].RegisterFrame(s["xyz"], s["t"], s["frame_idx"]))
                else:
                    twins[b].RegisterFrameWithEstimate(s["xyz"], s["t"], ests[b], s["frame_idx"])
            except CticpError as e:
                want[b] = e.code
        if k >= 1:
            assert want[1] == abi.ERR_UNSUPPORTED and want[3] == abi.ERR_INVALID_ARGUMENT, (k, want)
        assert want[4] == (abi.ERR_TIMESTAMP if k == 3 else 0), (k, want)
        scans = [(seqs[b][k]["xyz"], seqs[b][k]["t"]) for b in range(6)]
        fids = [seqs[b][k]["frame_idx"] for b in range(6)]
        kw = {"initial_estimates": ests} if k == 3 else {}
        if any(want):
            with pytest.raises(CticpError) as e:
                eng.register_batch(ods, scans, fids, **kw)
            assert e.value.statuses == want, (k, e.value.statuses, want)
            for b in range(6):
                if not want[b]:
                    sums_t[b].pop()   # (the raising call returns no summaries: trajectory, points and map still compared)
        else:
            out = eng.register_batch(ods, scans, fids, **kw)
            for b in range(6):
                sums_b[b].append(out[b])
        if k >= 1:
            joiners = [b for b in ok if want[b] == 0]
            for b in joiners:
                assert ods[b].last_timing().icp_batch_groups == len(joiners), (k, b)
    for b in ok:
        _assert_same(twins[b], ods[b], sums_t[b], sums_b[b])
    for b in (1, 3):
        assert _state(twins[b]) == _state(ods[b])
