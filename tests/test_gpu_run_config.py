"""The odometry runner (ct_icp_b200/runner.py, tools/run_odometry.py) end to end on the device, from reference-shaped
configurations over a SYNTHETIC dataset: a temporary root holding config/synthetic/courtyard.yaml and shorter variants
of it. Checks the runner's <sequence>.PLY against a hand loop of register_device, its mid-frame poses against the
trajectory oracle, metrics.yaml against a direct trajectory_kitti_evaluate call, the periodic saves, exit_early, and a
concurrent run against the serial one."""
import os
import shutil
import struct

import numpy as np
import pytest

from ct_icp_b200 import config, datasets, runner

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
COURTYARD = os.path.join(ROOT, "tests", "golden", "configs", "synthetic", "courtyard.yaml")

SOLVERS = {
    "GN": "    solver: GN\n",
    "CERES": "    solver: CERES\n    loss_function: CAUCHY\n    ls_max_num_iters: 5\n",
    "ROBUST": "    solver: ROBUST\n",
}


def odometry_node(solver, extra=""):
    return ("odometry_options:\n" + extra + "  voxel_size: 0.2\n  sample_voxel_size: 0.4\n  max_distance: 100.0\n"
            "  distance_error_threshold: 100.0\n  init_num_frames: 3\n  motion_compensation: CONTINUOUS\n"
            "  initialization: INIT_CONSTANT_VELOCITY\n  map_options:\n    map_type: MULTI_RESOLUTION_VOXEL_HASHMAP\n"
            "    resolutions:\n      - {resolution: 0.5, max_num_points: 20, min_distance_between_points: 0.05}\n"
            "  ct_icp_options:\n    num_iters_icp: 10\n    min_number_neighbors: 10\n    max_number_neighbors: 20\n"
            + SOLVERS[solver])


def variant(text, num_poses, frequency, scene=None):
    """courtyard.yaml with its first num_poses poses, sampled at `frequency`, optionally with another scene"""
    lines = text.splitlines()
    out, pose_count, in_poses = [], 0, False
    for ln in lines:
        s = ln.strip()
        if s.startswith("sample_frequency:"):
            ln = "sample_frequency: %s" % frequency
        if s == "poses:":
            in_poses = True
        elif in_poses and s.startswith("- quaternion"):
            pose_count += 1
        elif in_poses and ln.startswith("  ") and not ln.startswith("    ") and s:
            in_poses = False
            if scene is not None:
                out.append(scene)
                break
        if in_poses and pose_count > num_poses:
            continue
        out.append(ln)
    return "\n".join(out) + "\n"


@pytest.fixture(scope="module")
def scenes(tmp_path_factory):
    root = tmp_path_factory.mktemp("synthetic")
    text = open(COURTYARD).read()
    shutil.copy(COURTYARD, root / "courtyard.yaml")
    for n in (3, 4, 5, 6):   # the first n poses: 40 (n - 1) frames
        (root / ("c%d.yaml" % n)).write_text(variant(text, n, 40.0))
    # a scene of one ball around the first pose, seen within 2 m: it leaves the sensor's range within a second, and
    # the first frame without a point is refused
    (root / "c4fail.yaml").write_text(variant(text, 3, 40.0, scene="  balls:\n    - center: [2.5, 5, 2]\n"
                                              "      radius: 1.0").replace("max_lidar_distance: 15.0",
                                                                         "max_lidar_distance: 2.0"))
    return root


def config_text(root, out, solver="GN", names=None, extra="", odometry_extra=""):
    seqs = "" if names is None else "    use_all_datasets: false\n    sequence_options:\n" + "".join(
        "      - sequence_name: %s\n" % n for n in names)
    return ("generate_directory_prefix: false\noutput_dir: %s\n%s\ndataset_options:\n  - dataset: SYNTHETIC\n"
            "    root_path: %s\n%s%s" % (out, extra, root, seqs, odometry_node(solver, odometry_extra)))


def run(eng, text, concurrent=None, saves=None):
    root = config.compose(text)
    opts = config.load_runner_options(root, eng)
    if concurrent is not None:
        opts.concurrent_sequences = concurrent
    seqs = datasets.load_dataset_from_options(eng, config.dataset_options_from_config(root))
    r = runner.OdometryRunner(eng, seqs, opts)
    if saves is not None:
        orig = r._save

        def spy(run_, is_driving=True):
            saves.append((run_.name, len(run_.od.Trajectory()), is_driving))
            orig(run_, is_driving)
        r._save = spy
    return r.Run(), r


def hand_loop(eng, spec, options):
    """register_device over every frame of Binding.synthetic_sequence(spec), stopping after the first failure: the
    summaries' frames, the ground truth, and the handle's trajectory (what SaveTrajectoryAndMetrics writes)"""
    import torch
    o = options.copy()
    o.debug_print = 0
    o.ct_icp_options.debug_print = 0
    od = eng.odometry(o)
    d = eng.synthetic_sequence(spec, device=True)
    ends = [0] + d["frame_ends"].tolist()
    stream = torch.cuda.current_stream().cuda_stream
    frames = []
    for k in range(len(ends) - 1):
        xyz, t = d["xyz"][ends[k]:ends[k + 1]], d["t"][ends[k]:ends[k + 1]]
        sm = od.register_device(datasets.device_scan({"xyz": xyz, "t": t}), k, stream=stream)
        frames.append(sm.frame.copy())
        if not sm.success:
            break
    trajectory = od.Trajectory()
    od.close()
    return frames, d["ground_truth"], trajectory


def bits(x):
    """a double's bits; every NaN is one value (metrics.yaml writes any NaN as .nan)"""
    return b"nan" if np.isnan(x) else struct.pack("<d", float(x))


@pytest.mark.parametrize("solver", ["GN", "CERES", "ROBUST"])
def test_courtyard_matches_a_hand_loop(eng, scenes, tmp_path, solver):
    from oracle_trajectory_lib import trajectory_oracle
    text = config_text(scenes, tmp_path, solver, ["courtyard"], extra="exit_early: false\n")
    ok, r = run(eng, text)
    assert ok
    spec = config.yaml_to_synthetic_scene(config.load_config(COURTYARD))
    frames, gt, _ = hand_loop(eng, spec, config.load_runner_options(config.compose(text), eng).odometry_options)
    assert len(frames) > 300
    mids = [runner.mid_frame_pose(f.begin_pose, f.end_pose) for f in frames]
    data = open(tmp_path / "SYNTHETIC_courtyard.PLY", "rb").read()
    assert data == eng.save_poses_ply(mids)
    # InterpolatePoseAlpha at exactly 0.5: the oracle's DoInterpolatePose between the frame's poses re-stamped 0 and 1
    orc = trajectory_oracle()
    got = eng.read_poses_ply(data)
    for k in range(0, len(frames), 7):
        b, e = frames[k].begin_pose.copy(), frames[k].end_pose.copy()
        b.dest_timestamp, e.dest_timestamp, b.dest_frame_id, e.dest_frame_id = 0.0, 1.0, 0, 0
        tr = orc.continuous_trajectory([b, e])
        want = tr.interpolate(np.array([0.5]))[0]
        assert got[k]["quat"].tobytes() == want["quat"].tobytes() and got[k]["tr"].tobytes() == want["tr"].tobytes()
        assert got[k]["dest_frame_id"] == frames[k].begin_pose.dest_frame_id
    # metrics.yaml: EvaluatePoses(runner's poses, LinearContinuousTrajectory(gt), driving)
    m = runner.read_metrics_yaml(str(tmp_path / "metrics.yaml"))["SYNTHETIC_courtyard"]
    e = eng.continuous_trajectory(datasets.pose_list(gt)).kitti_evaluate(mids, lengths="driving")
    for key, field in (("MAX_APE", "max_ape"), ("MEAN_APE", "mean_ape"), ("MEAN_RPE", "mean_rpe"),
                       ("MEAN_LOCAL_ERROR", "mean_local_err"), ("MAX_LOCAL_ERROR", "max_local_err")):
        assert bits(m[key]) == bits(e[field]), key
    assert m["INDEX_MAX_LOCAL_ERROR"] == e["index_max_local_err"]
    assert (m["success"], m["finished"], m["AVG_NUM_ATTEMPTS"]) == (False, False, -1.0)
    assert m["Average(ms)"] > 0 and bits(m["Average(ms)"]) == bits(r.summaries["SYNTHETIC_courtyard"]["avg_time_ms"])


def test_begin_and_end_poses_without_mid_frames(eng, scenes, tmp_path):
    text = config_text(scenes, tmp_path, "GN", ["c4"], extra="save_mid_frame: 0\n")
    ok, _ = run(eng, text)
    assert ok
    spec = config.yaml_to_synthetic_scene(config.load_config(str(scenes / "c4.yaml")))
    frames, _, _ = hand_loop(eng, spec, config.load_runner_options(config.compose(text), eng).odometry_options)
    want = eng.save_poses_ply([frames[0].begin_pose] + [f.end_pose for f in frames])
    assert len(frames) == 120 and open(tmp_path / "SYNTHETIC_c4.PLY", "rb").read() == want


def test_periodic_saves(eng, scenes, tmp_path):
    saves = []
    ok, r = run(eng, config_text(scenes, tmp_path, "GN", ["c5", "c6"],
                                 extra="compute_metrics_period: 50\nuse_outdoor_evaluation: 0\n"), saves=saves)
    assert ok
    n5, n6 = r.summaries["SYNTHETIC_c5"]["num_frames"], r.summaries["SYNTHETIC_c6"]["num_frames"]
    assert (n5, n6) == (160, 199)   # 40 Hz over 5 s samples 200 poses (the last instant falls past the end)
    # after frame_id k > 0 with k % period == 0, the trajectory holds k + 1 frames; indoor lengths unless
    # use_outdoor_evaluation; the final save always with the driving lengths
    want = [("SYNTHETIC_c5", k + 1, False) for k in (50, 100, 150)] + [("SYNTHETIC_c5", n5, True)] + \
        [("SYNTHETIC_c6", k + 1, False) for k in (50, 100, 150)] + [("SYNTHETIC_c6", n6, True)]
    assert saves == want
    assert sorted(runner.read_metrics_yaml(str(tmp_path / "metrics.yaml"))) == ["SYNTHETIC_c5", "SYNTHETIC_c6"]


@pytest.mark.parametrize("exit_early", [True, False])
@pytest.mark.parametrize("concurrent", [1, 3])
def test_exit_early(eng, scenes, tmp_path, exit_early, concurrent):
    text = config_text(scenes, tmp_path, "GN", ["c3", "c4fail", "c5"],
                       extra="exit_early: %s\n" % ("true" if exit_early else "false"))
    ok, r = run(eng, text, concurrent=concurrent)   # sequences run in name order: c3, c4fail, c5
    assert r.summaries["SYNTHETIC_c4fail"]["success"] is False
    assert 0 < r.summaries["SYNTHETIC_c4fail"]["num_frames"] < 80
    files = sorted(os.listdir(tmp_path))
    if exit_early:   # the run stops at the failed frame: no final save, and the later sequence never runs
        assert not ok and files == ["SYNTHETIC_c3.PLY", "metrics.yaml"]
        assert "SYNTHETIC_c5" not in r.summaries
        assert list(runner.read_metrics_yaml(str(tmp_path / "metrics.yaml"))) == ["SYNTHETIC_c3"]
    else:            # the failed sequence is saved as far as it went, and the next one runs
        assert ok and files == ["SYNTHETIC_c3.PLY", "SYNTHETIC_c4fail.PLY", "SYNTHETIC_c5.PLY", "metrics.yaml"]
        assert r.summaries["SYNTHETIC_c5"]["success"]
    assert r.summaries["SYNTHETIC_c3"]["success"]


@pytest.fixture
def solo_grids_fit(monkeypatch):
    """512 keypoints per gather CTA (CTICP_GN_KP_PER_CTA, read when a handle is created, so by both runs): the solo
    grids of four synthetic problems then fit on the device together, the condition under which the batched call gives
    the single-frame call's results byte for byte (cticp.h, "one frame on each of many handles")"""
    monkeypatch.setenv("CTICP_GN_KP_PER_CTA", "512")


@pytest.mark.parametrize("solver", ["GN", "CERES"])
def test_concurrent_sequences_give_the_serial_files(eng, scenes, tmp_path, solo_grids_fit, solver):
    names = ["c3", "c4", "c5", "c6", "courtyard"]
    serial, conc = tmp_path / "serial", tmp_path / "conc"
    ok1, r1 = run(eng, config_text(scenes, serial, solver, names, extra="exit_early: false\n"))
    joins = []
    text = config_text(scenes, conc, solver, names, extra="exit_early: false\nconcurrent_sequences: 4\n")
    root = config.compose(text)
    opts = config.load_runner_options(root, eng)
    assert opts.concurrent_sequences == 4
    seqs = datasets.load_dataset_from_options(eng, config.dataset_options_from_config(root))
    r2 = runner.OdometryRunner(eng, seqs, opts)
    orig_start = r2._start

    def spy(run_):   # how many frames the other active sequences had registered when each one joined
        joins.append((run_.name, {n: s["num_frames"] for n, s in r2.summaries.items()}))
        orig_start(run_)
    r2._start = spy
    assert ok1 and r2.Run()
    assert sorted(os.listdir(serial)) == sorted(os.listdir(conc))
    for f in sorted(os.listdir(serial)):
        if f.endswith(".PLY"):
            assert open(serial / f, "rb").read() == open(conc / f, "rb").read(), f
    m1, m2 = runner.read_metrics_yaml(str(serial / "metrics.yaml")), runner.read_metrics_yaml(str(conc / "metrics.yaml"))
    assert sorted(m1) == sorted(m2) == ["SYNTHETIC_" + n for n in names]
    for name in m1:   # every field but the timing
        for k in runner.METRIC_KEYS:
            if k != "Average(ms)":
                assert bits(m1[name][k]) == bits(m2[name][k]) if isinstance(m1[name][k], float) else \
                    m1[name][k] == m2[name][k], (name, k)
    # the fifth sequence joins mid-run: one of the first four has left the batch, the others are part way
    name, seen = joins[4]
    final = {n: r1.summaries[n]["num_frames"] for n in seen}
    assert name == "SYNTHETIC_courtyard" and sorted(seen) == ["SYNTHETIC_c%d" % n for n in (3, 4, 5, 6)]
    assert sum(seen[n] == final[n] for n in seen) == 1 and sum(0 < seen[n] < final[n] for n in seen) == 3
    assert [r2.summaries[n]["num_frames"] for n in sorted(r2.summaries)] == \
        [r1.summaries[n]["num_frames"] for n in sorted(r1.summaries)]


@pytest.mark.parametrize("exit_early", [True, False])
@pytest.mark.parametrize("concurrent", [1, 2])
def test_registration_failure(eng, scenes, tmp_path, solo_grids_fit, exit_early, concurrent):
    """a frame the registration rejects (summary.success == 0: it moved more than distance_error_threshold): the
    sequence stops there, and <seq>.PLY holds the handle's trajectory, as the reference's odom.Trajectory()"""
    text = config_text(scenes, tmp_path, "GN", ["c3", "c4"],
                       extra="exit_early: %s\n" % ("true" if exit_early else "false")).replace(
        "distance_error_threshold: 100.0", "distance_error_threshold: 0.01")
    ok, r = run(eng, text, concurrent=concurrent)
    frames, _, trajectory = hand_loop(eng, config.yaml_to_synthetic_scene(config.load_config(str(scenes / "c3.yaml"))),
                                      config.load_runner_options(config.compose(text), eng).odometry_options)
    s3 = r.summaries["SYNTHETIC_c3"]
    assert s3["success"] is False and s3["num_frames"] == len(frames) < 80
    assert [bytes(p) for p in s3["trajectory"]] == [bytes(f.end_pose) for f in frames]
    files = sorted(os.listdir(tmp_path))
    if exit_early:   # serial: c4 never starts; side by side: c4 comes after c3, so its files are removed
        assert not ok and files == [] and "SYNTHETIC_c4" not in r.summaries
    else:
        assert ok and files == ["SYNTHETIC_c3.PLY", "SYNTHETIC_c4.PLY", "metrics.yaml"]
        mids = [runner.mid_frame_pose(f.begin_pose, f.end_pose) for f in trajectory]
        assert open(tmp_path / "SYNTHETIC_c3.PLY", "rb").read() == eng.save_poses_ply(mids)


def test_run_odometry_tool(eng, scenes, tmp_path):
    import subprocess
    import sys
    cfg = tmp_path / "config.yaml"
    cfg.write_text(config_text(scenes, tmp_path / "out", "GN", ["c3", "c4"]))
    p = subprocess.run([sys.executable, os.path.join(ROOT, "tools", "run_odometry.py"), "-c", str(cfg),
                        "--concurrent", "2"], capture_output=True, text=True)
    assert p.returncode == 0, p.stderr[-2000:]
    assert sorted(os.listdir(tmp_path / "out")) == ["SYNTHETIC_c3.PLY", "SYNTHETIC_c4.PLY", "metrics.yaml"]
