"""Snapshots of odometry handles and voxel maps (cticp_odometry_save / _load / _clone, cticp_map_save / _load): a handle
loaded from a snapshot, or cloned, registers every later frame exactly as the handle it came from. Compared byte for byte
(the wall-clock fields of the summaries aside): summaries, trajectories, the three point vectors after the next frame,
the map's points, every level's export, map_size; and the snapshot bytes themselves (save twice, load -> save, the map
section of an odometry snapshot against cticp_map_save of its map). Malformed snapshots are refused before the device is
touched, and neither refusals nor save / load / clone cycles keep device memory."""
import ctypes as C
import struct

import numpy as np
import pytest

from ct_icp_b200 import _abi as abi
from ct_icp_b200 import synthetic as syn
from ct_icp_b200._binding import CticpError
from test_gpu_device_io import _options, _summary_bytes

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

N_FRAMES = 8
HEADER = 72            # snapshot_format.h kHeaderBytes
SECTIONS = 5           # options, host state, trajectory, map, origins
MIB = 1 << 20


@pytest.fixture(scope="module")
def seq():
    return syn.make_sequence(N_FRAMES, syn.SMALL16, seed=4321)


def _profile(eng, name):
    """the GN bench options and the shipped profiles, every one with a three-frame start-up phase"""
    if name in ("gn", "adaptive", "mc_none", "mc_iterative", "small_tables"):
        o = _options(eng, "adaptive" if name == "adaptive" else "gn")
        if name == "mc_none":
            o.motion_compensation = abi.MOTION_COMPENSATION["NONE"]
        elif name == "mc_iterative":
            o.motion_compensation = abi.MOTION_COMPENSATION["ITERATIVE"]
        elif name == "small_tables":   # tables that grow, and evictions that leave tombstones, before the save
            o.map_options.capacity_voxels = 1024
            o.max_distance = 12.0
    elif name in ("robust_driving", "robust_outdoor_low_inertia"):
        o = eng.profile(name)
    elif name == "distance":   # CERES with the distance-based strategy: the map keeps voxel normals
        o = _options(eng, "default_driving_ceres")
        o.neighborhood_strategy.type = abi.STRATEGY["DISTANCE_BASED_STRATEGY"]
        o.map_options.select_valid_normals_direction = 1
    else:
        o = _options(eng, name)
    o.init_num_frames = 3
    o.debug_print = 0
    o.ct_icp_options.debug_print = 0
    return o


def _register(od, s):
    return od.RegisterFrame(s["xyz"], s["t"], s["frame_idx"])


def _levels(od):
    m = od.GetMapPointer()
    n = od.options.map_options.num_resolutions
    return [b"".join(a.tobytes() for a in m.export(i)) for i in range(n)]


def _state(od):
    """trajectory, the three point vectors of the last frame, the map points, every level's export, map_size"""
    tr = od.Trajectory()
    return (b"".join(bytes(memoryview(f)) for f in tr),
            [od.points(w).tobytes() for w in (abi.POINTS_CORRECTED, abi.POINTS_ALL_CORRECTED, abi.POINTS_KEYPOINTS)],
            od.GetMapPointCloud().tobytes(), _levels(od), od.MapSize())


def _assert_same_run(a, b, sums_a, sums_b):
    assert len(sums_a) == len(sums_b)
    for i, (x, y) in enumerate(zip(sums_a, sums_b)):
        assert _summary_bytes(x) == _summary_bytes(y), i
    sa, sb = _state(a), _state(b)
    assert sa[0] == sb[0]
    for w in range(3):
        assert sa[1][w] == sb[1][w], w
    assert sa[2] == sb[2]
    assert sa[3] == sb[3]
    assert sa[4] == sb[4]


def _sections(blob):
    sizes = struct.unpack_from("<%dQ" % SECTIONS, blob, 16)
    offs, at = [], HEADER
    for s in sizes:
        offs.append(at)
        at += s
    return offs, sizes


def _map_section(blob):
    offs, sizes = _sections(blob)
    return blob[offs[3]:offs[3] + sizes[3]]


def _level_header(blob, level):
    """the map section's level header: capacity and counters (snapshot_format.h WriteMapHeader)"""
    at = _sections(blob)[0][3] + C.sizeof(abi.MapOptions) + 16 + 48 * level
    cap, B, _, points, voxels, tombs = struct.unpack_from("<QIIQII", blob, at)
    return dict(cap=cap, B=B, points=points, voxels=voxels, tombs=tombs)


def _host_state(blob):
    """the host-state section's leading fields (snapshot_format.h WriteHostState)"""
    v = struct.unpack_from("<iiiiddiiQii", blob, _sections(blob)[0][1])
    keys = ("registered_frames", "robust_num_consecutive_failures", "next_robust_level", "suspect_registration_error",
            "cum_distance", "cum_orientation", "skipped_frames", "total_insertions", "last_num_keypoints",
            "default_model_present", "prev_frame_points")
    return dict(zip(keys, v))


PROFILES = ["gn", "default_driving_ceres", "robust_driving", "robust_outdoor_low_inertia", "distance", "adaptive",
            "mc_none", "mc_iterative", "small_tables"]


@pytest.mark.parametrize("j", [0, 2, 5], ids=["fresh", "startup", "after_startup"])
@pytest.mark.parametrize("profile", PROFILES)
def test_resume_is_bit_exact(eng, seq, profile, j):
    o = _profile(eng, profile)
    a = eng.odometry(o)
    for s in seq[:j]:
        _register(a, s)
    blob = a.save()
    assert a.save() == blob                                    # save twice: the same bytes
    b = eng.load_odometry(blob)
    assert b.save() == blob                                    # load -> save: the same bytes
    assert a.GetMapPointer().save()[HEADER:HEADER + len(_map_section(blob))] == _map_section(blob)
    assert _levels(a) == _levels(b) and a.MapSize() == b.MapSize()
    sums_a = [_register(a, s) for s in seq[j:]]
    sums_b = [_register(b, s) for s in seq[j:]]
    _assert_same_run(a, b, sums_a, sums_b)
    if profile == "small_tables" and j == 5:   # the 1024-slot level-0 table had grown when the handle was saved
        assert _level_header(blob, 0)["cap"] > 1024


@pytest.mark.parametrize("profile", ["gn", "default_driving_ceres", "robust_driving", "distance"])
def test_clone_is_bit_exact_and_leaves_the_original_alone(eng, seq, profile):
    o = _profile(eng, profile)
    a, twin = eng.odometry(o), eng.odometry(o)
    for s in seq[:4]:
        _register(a, s)
        _register(twin, s)
    c = a.clone()
    assert c.save() == a.save()
    sums_c = [_register(c, s) for s in seq[4:]]
    sums_a = [_register(a, s) for s in seq[4:]]
    sums_t = [_register(twin, s) for s in seq[4:]]
    _assert_same_run(twin, c, sums_t, sums_c)
    _assert_same_run(twin, a, sums_t, sums_a)


@pytest.mark.parametrize("profile", ["gn", "default_driving_ceres"])
def test_loaded_and_cloned_handles_join_a_batch(eng, seq, profile, monkeypatch):
    monkeypatch.setenv("CTICP_GN_KP_PER_CTA", "512")   # the solo grids of the batch fit on the device together
    o = _profile(eng, profile)
    a = eng.odometry(o)
    for s in seq[:4]:
        _register(a, s)
    loaded, cloned = eng.load_odometry(a.save()), a.clone()
    sums_a, sums_l, sums_c = [], [], []
    for s in seq[4:]:
        sl, sc = eng.register_batch([loaded, cloned], [(s["xyz"], s["t"])] * 2, [s["frame_idx"]] * 2)
        sums_l.append(sl)
        sums_c.append(sc)
        sums_a.append(_register(a, s))
    _assert_same_run(a, loaded, sums_a, sums_l)
    _assert_same_run(a, cloned, sums_a, sums_c)


def test_load_for_localisation_keeps_the_map(eng, seq):
    """do_no_insert = 1 and a max_distance that covers the whole map: the map export stays the snapshot's"""
    o = _profile(eng, "gn")
    a = eng.odometry(o)
    for s in seq[:5]:
        _register(a, s)
    blob, levels = a.save(), _levels(a)
    loc = _profile(eng, "gn")
    loc.do_no_insert = 1
    loc.max_distance = 1e6
    b = eng.load_odometry(blob, options=loc)
    for s in seq[5:]:
        sm = _register(b, s)
        assert sm.success
        assert _levels(b) == levels
    other = _profile(eng, "gn")
    other.map_options.resolutions[0].max_num_points = 19
    with pytest.raises(CticpError) as e:
        eng.load_odometry(blob, options=other)
    assert e.value.code == abi.ERR_INVALID_ARGUMENT
    normals = _profile(eng, "gn")   # a strategy that needs voxel normals this snapshot does not keep
    normals.neighborhood_strategy.type = abi.STRATEGY["DISTANCE_BASED_STRATEGY"]
    normals.map_options.select_valid_normals_direction = 1
    with pytest.raises(CticpError) as e:
        eng.load_odometry(blob, options=normals)
    assert e.value.code == abi.ERR_INVALID_ARGUMENT


def test_voxel_map_round_trip(eng):
    rng = np.random.default_rng(11)
    opts = eng.legacy_map_options(1.0, 20, 0.1)
    opts.select_valid_normals_direction = 1
    m = eng.voxel_map(opts)
    for k in range(4):
        m.insert(rng.uniform(-15, 15, size=(4000, 3)), origin=(k, 0.5 * k, 0.0))
    m.remove_far((0.0, 0.0, 0.0), 12.0)
    blob = m.save()
    n = eng.load_voxel_map(blob)
    assert n.save() == blob
    assert [a.tobytes() for a in m.export(0)] == [a.tobytes() for a in n.export(0)]
    q = rng.uniform(-10, 10, size=(256, 3))
    ra, rb = m.radius_search(q, 1.0, 20, (0.0, 0.0, 0.0)), n.radius_search(q, 1.0, 20, (0.0, 0.0, 0.0))
    assert ra[0].tobytes() == rb[0].tobytes() and ra[1].tobytes() == rb[1].tobytes()


def _checksum(payload):
    """snapshot_format.h Checksum"""
    M = (1 << 64) - 1
    P = ((0x100000001b3 * 0x9E3779B97F4A7C15) | 1) & M
    h = 0xcbf29ce484222325
    pad = payload + b"\0" * (-len(payload) % 8)
    for w in np.frombuffer(pad, dtype="<u8").tolist():
        h = ((h ^ w) * P) & M
    h = ((h ^ len(payload)) * P) & M
    return h ^ (h >> 29)


def _reseal(blob):
    b = bytearray(blob)
    struct.pack_into("<Q", b, HEADER - 8, _checksum(bytes(b[HEADER:])))
    return bytes(b)


def _refusals(eng):
    """truncated, bit-flipped and structurally corrupted map and odometry snapshots (re-checksummed)"""
    m = eng.voxel_map(eng.legacy_map_options(1.0, 20, 0.1))
    m.insert(np.random.default_rng(3).uniform(-10, 10, size=(3000, 3)))
    mblob = m.save()
    fixed = C.sizeof(abi.MapOptions) + 16
    lvl = HEADER + fixed                      # level 0 header: u64 cap | u32 B | u32 0 | u64 points | u32 voxels ...
    rec = lvl + 48                            # first record: u32 slot | u32 count | u64 key
    cap = struct.unpack_from("<Q", mblob, lvl)[0]
    bad = []
    for n in (0, HEADER - 1, HEADER, len(mblob) // 2, len(mblob) - 1):
        bad.append(("map", mblob[:n]))
    flip = bytearray(mblob)
    flip[len(mblob) // 3] ^= 0x10
    bad.append(("map", bytes(flip)))
    for at, v in ((rec, cap), (rec + 16, struct.unpack_from("<I", mblob, rec)[0])):   # slot >= cap; repeated slot
        b = bytearray(mblob)
        struct.pack_into("<I", b, at, v)
        bad.append(("map", _reseal(bytes(b))))
    b = bytearray(mblob)
    struct.pack_into("<I", b, rec + 4, 21)    # count > B
    bad.append(("map", _reseal(bytes(b))))
    b = bytearray(mblob)
    struct.pack_into("<Q", b, lvl + 16, struct.unpack_from("<Q", mblob, lvl + 16)[0] + 1)   # totals != counters
    bad.append(("map", _reseal(bytes(b))))
    od = eng.odometry(_profile(eng, "gn"))
    oblob = od.save()
    bad.append(("odometry", oblob[:-1]))
    bad.append(("odometry", mblob))           # a map snapshot is not an odometry snapshot
    b = bytearray(oblob)
    b[0] ^= 1
    bad.append(("odometry", _reseal(bytes(b))))
    return bad, m, od


def test_malformed_snapshots_are_refused(eng):
    bad, _, _ = _refusals(eng)
    for kind, blob in bad:
        with pytest.raises(CticpError) as e:
            (eng.load_voxel_map if kind == "map" else eng.load_odometry)(blob)
        assert e.value.code == abi.ERR_INVALID_ARGUMENT, (kind, len(blob))
    od = eng.odometry(_profile(eng, "gn"))
    n = eng.fn("odometry_save")(od.h, None, 0)
    buf = C.create_string_buffer(n)
    assert eng.fn("odometry_save")(od.h, buf, n - 1) == abi.ERR_INVALID_ARGUMENT   # below the size: nothing written
    assert buf.raw == b"\0" * n


def _free_bytes():
    torch.cuda.synchronize()
    return torch.cuda.mem_get_info(0)[0]


def test_refusals_and_cycles_release_memory(eng, seq):
    bad, m, od = _refusals(eng)
    a = eng.odometry(_profile(eng, "gn"))
    for s in seq[:3]:
        _register(a, s)
    a.clone().close()   # warm-up
    eng.load_odometry(a.save()).close()
    before = _free_bytes()
    for i in range(20):
        kind, blob = bad[i % len(bad)]
        with pytest.raises(CticpError):
            (eng.load_voxel_map if kind == "map" else eng.load_odometry)(blob)
    for _ in range(20):
        eng.load_odometry(a.save()).close()
        a.clone().close()
    lost = before - _free_bytes()
    assert lost < 256 * MIB, "refusals and cycles kept %.1f MiB of device memory" % (lost / MIB)


def test_clone_to_another_gpu(eng, seq):
    if torch.cuda.device_count() < 2:
        pytest.skip("only one GPU")
    o = _profile(eng, "gn")
    a, twin = eng.odometry(o), eng.odometry(o)
    for s in seq[:4]:
        _register(a, s)
        _register(twin, s)
    c = a.clone(device=1)
    sums_c = [_register(c, s) for s in seq[4:]]
    sums_t = [_register(twin, s) for s in seq[4:]]
    _assert_same_run(twin, c, sums_t, sums_c)


# robust_driving with options that force the ladder to retry (tests/test_gpu_robust_ladder.py): rotations above 1e-4
# degrees fail every attempt, so every frame runs to robust_num_attempts; a tight translation threshold retries some
RETRY_CASES = {
    "rotation": dict(robust_threshold_ego_orientation=1e-4, robust_threshold_relative_orientation=1e-4, robust_num_attempts=3),
    "translation": dict(robust_relative_trans_threshold=1e-3, robust_num_attempts=3),
}


@pytest.mark.parametrize("case", sorted(RETRY_CASES))
@pytest.mark.parametrize("profile", ["robust_driving", "robust_outdoor_low_inertia"])
def test_resume_right_after_a_retried_frame(eng, seq, profile, case):
    o = _profile(eng, profile)
    for k, v in RETRY_CASES[case].items():
        setattr(o, k, v)
    a = eng.odometry(o)
    sums = []
    for k, s in enumerate(seq):
        sums.append(_register(a, s))
        if k >= 2 and sums[-1].number_of_attempts > 1:
            break
    assert sums[-1].number_of_attempts > 1, [sm.number_of_attempts for sm in sums]   # the frame just saved was retried
    j = len(sums)
    assert j < len(seq)
    blob = a.save()
    st = _host_state(blob)
    if case == "rotation":   # the ladder ran out: the robust state the retries leave is not the fresh one
        assert st["suspect_registration_error"] == 1 and st["next_robust_level"] > 0, st
    b = eng.load_odometry(blob)
    assert b.save() == blob
    sums_a = [_register(a, s) for s in seq[j:]]
    sums_b = [_register(b, s) for s in seq[j:]]
    _assert_same_run(a, b, sums_a, sums_b)


def test_resume_with_frames_larger_than_the_tail_head_room(eng):
    """HDL-64 scans: F is far above the 4096 points of head-room a handle without a previous frame gives the device tail.
    The snapshot carries the saved handle's F, so the first resumed frame takes the same tail as on the saved handle."""
    hdl = syn.make_sequence(6, syn.HDL64, seed=99)
    a = eng.odometry(_profile(eng, "gn"))
    for s in hdl[:3]:
        _register(a, s)
    blob = a.save()
    assert _host_state(blob)["prev_frame_points"] > 4096
    b = eng.load_odometry(blob)
    c = a.clone()
    sums_a = [_register(a, s) for s in hdl[3:]]
    sums_b = [_register(b, s) for s in hdl[3:]]
    sums_c = [_register(c, s) for s in hdl[3:]]
    _assert_same_run(a, b, sums_a, sums_b)
    _assert_same_run(a, c, sums_a, sums_c)
    assert a.last_timing().kernel_launches == b.last_timing().kernel_launches == c.last_timing().kernel_launches


@pytest.mark.parametrize("how", ["load", "clone"])
def test_last_timing_before_the_first_resumed_frame(eng, seq, how):
    """last_timing() on a loaded or cloned handle before its first frame: no event of it has been recorded yet, so it
    answers as a fresh handle does and leaves no CUDA error behind for the frames that follow"""
    a = eng.odometry(_profile(eng, "gn"))
    for s in seq[:4]:
        _register(a, s)
    b = eng.load_odometry(a.save()) if how == "load" else a.clone()
    t = b.last_timing()
    assert t.total_ms == 0.0 and t.kernel_launches == 0
    sums_a = [_register(a, s) for s in seq[4:]]
    sums_b = [_register(b, s) for s in seq[4:]]
    _assert_same_run(a, b, sums_a, sums_b)
    assert b.last_timing().total_ms > 0.0
