"""The YAML configuration readers (ct_icp_b200/config.py) against the reference's clauses: every configuration the
reference ships parses (or is refused where the reference refuses it), driving_config and nclt_config give the values
tests/golden/reference_defaults.json holds, and each quirk of the readers has its own case. CPU only."""
import glob
import json
import math
import os
import struct

import numpy as np
import pytest

import ct_icp_b200
from ct_icp_b200 import _abi as abi
from ct_icp_b200 import config, datasets, runner

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CONFIGS = os.path.join(ROOT, "tests", "golden", "configs")
REF = json.load(open(os.path.join(ROOT, "tests", "golden", "reference_defaults.json")))
ENUMS = {"solver": abi.SOLVER, "loss_function": abi.LOSS, "weighting_scheme": abi.WEIGHTING,
         "parametrization": abi.PARAMETRIZATION, "distance": abi.DISTANCE,
         "motion_compensation": abi.MOTION_COMPENSATION, "initialization": abi.INITIALIZATION,
         "sampling": abi.SAMPLING}


def fixture_files():
    return sorted(os.path.relpath(p, CONFIGS) for p in glob.glob(os.path.join(CONFIGS, "**", "*.yaml"), recursive=True))


def odometry_nodes(rel):
    """(label, odometry node) of every odometry configuration a fixture holds: the runner's and the ROS node's
    top-level odometry_options, or each regression run's"""
    root = config.load_config(os.path.join(CONFIGS, rel))
    if "runs" in root:
        return [(rel + ":" + k, v["odometry_options"]) for k, v in root["runs"].items()]
    if "odometry_options" in root:
        return [(rel, root["odometry_options"])]
    return []


# the fixtures the reference itself refuses, with the message it gives
REFUSED = {"synthetic_ct_icp_config.yaml": "Distance CT_POINT_TO_PLANE not recognized as a valid distance",
           "regression/regression_config_short_nclt.yaml:run_nclt_robust_short_ceres":
               "Distance CT_POINT_TO_PLANE not recognized as a valid distance"}


@pytest.mark.parametrize("rel", fixture_files())
def test_every_fixture_parses(rel):
    nodes = odometry_nodes(rel)
    if rel.startswith("synthetic/"):
        assert config.yaml_to_synthetic_scene(config.load_config(os.path.join(CONFIGS, rel)))["acquisition"]["poses"]
        return
    assert nodes, rel
    for label, node in nodes:
        if label in REFUSED:
            with pytest.raises(config.ConfigError, match="^" + REFUSED[label] + "$"):
                config.yaml_to_odometry_options(node)
        else:
            o = config.yaml_to_odometry_options(node)
            assert o.map_options.num_resolutions >= 1, label


def check_fields(expect, got, skip=()):
    for k, v in expect.items():
        if k in skip or isinstance(v, (dict, list)):
            continue
        want = ENUMS[k][v] if k in ENUMS else int(v) if isinstance(v, bool) else v
        assert got[k] == want, (k, got[k], v)


@pytest.mark.parametrize("name", ["driving_config", "nclt_config"])
def test_shipped_configs_field_by_field(name):
    root = config.load_config(os.path.join(CONFIGS, "odometry", name + ".yaml"))
    opts = config.load_runner_options(root)
    got = opts.odometry_options.to_dict()
    y = REF["yaml"][name]
    carried_top = {k: v for k, v in y.items() if k not in ("size_voxel_map", "max_num_points_in_voxel",
                                                           "min_distance_points", "voxel_neighborhood")}
    check_fields(carried_top, got)
    icp = y["ct_icp_options"]
    check_fields(icp, got["ct_icp_options"], skip={k for k in icp if k.startswith("beta_")} | {"output_weights"})
    # the betas under ct_icp_options name no clause of yaml_to_ct_icp_options: the motion model keeps its defaults
    assert got["default_motion_model"] == ct_icp_b200.default_odometry_options().to_dict()["default_motion_model"]
    m = got["map_options"]
    res = sorted(y["map_options"]["resolutions"], key=lambda r: r["resolution"])
    assert m["num_resolutions"] == len(res)
    for g, r in zip(m["resolutions"], res):
        assert {k: g[k] for k in r} == r
    assert m["default_radius"] == y["map_options"].get("default_radius", REF["MapOptions"]["default_radius"])
    ns, ys = got["neighborhood_strategy"], y["neighborhood_strategy"]
    assert (ns["type"], ns["max_num_neighbors"], ns["min_num_neighbors"]) == \
        (abi.STRATEGY[ys["type"]], ys["max_num_neighbors"], ys["min_num_neighbors"])
    assert opts.dropped["ct_icp_options.output_weights"] is False and opts.dropped["with_viz3d"] is True
    if name == "nclt_config":   # the old map keys are read, and dropped: the node has map_options
        assert opts.dropped["size_voxel_map"] == 1.0 and opts.dropped["max_num_points_in_voxel"] == 20
    assert opts.exit_early and opts.output_results and opts.output_dir == ".outputs"


def test_sequence_name_00_stays_a_string():
    d = config.dataset_options_from_config(config.load_config(os.path.join(CONFIGS, "odometry", "driving_config.yaml")))
    assert d.dataset == "KITTI_raw" and not d.use_all_datasets
    assert [s.sequence_name for s in d.sequence_options] == ["00"]


def test_scalar_rules():
    assert config.as_double("1e-3", "k") == 1e-3 and config.as_double("5", "k") == 5.0
    assert math.isnan(config.as_double(".NaN", "k")) and config.as_double("-.inf", "k") == -math.inf
    assert [config.as_int(v, "k") for v in ("0x1F", "010", "-7", "+3")] == [31, 8, -7, 3]
    for v in ("true", "1.5", "08", "2147483648", "", None):
        with pytest.raises(config.ConfigError):
            config.as_int(v, "k")
    for v in ("1e999", "0x10", "abc", "1.0.0"):
        with pytest.raises(config.ConfigError):
            config.as_double(v, "k")
    trues = ("y", "Y", "yes", "Yes", "YES", "true", "True", "TRUE", "on", "On", "ON")
    falses = ("n", "N", "no", "No", "NO", "false", "False", "FALSE", "off", "Off", "OFF")
    assert all(config.as_bool(v, "k") for v in trues) and not any(config.as_bool(v, "k") for v in falses)
    for v in ("tRue", "1", "0", "yess", None):
        with pytest.raises(config.ConfigError):
            config.as_bool(v, "k")
    assert config.as_float("0.1", "k") == float(np.float32(0.1))
    assert config.as_string(None, "k") == "null"


def odo(text):
    return config.yaml_to_odometry_options(config.compose(text))


def test_beta_keys_under_ct_icp_options_are_ignored():
    o = odo("ct_icp_options:\n  beta_location_consistency: 7.0\n  beta_constant_velocity: 3.0\n")
    assert o.default_motion_model.beta_location_consistency == REF["MotionModelOptions"]["beta_location_consistency"]
    assert o.default_motion_model.beta_constant_velocity == REF["MotionModelOptions"]["beta_constant_velocity"]
    o = odo("default_motion_model:\n  beta_location_consistency: 7.0\n  model: SMALL_VELOCITY\n")
    assert o.default_motion_model.beta_location_consistency == 7.0
    assert o.default_motion_model.model == abi.MOTION_MODEL["SMALL_VELOCITY"]


def test_keys_no_clause_names_are_ignored():
    d = {}
    o = config.yaml_to_odometry_options(config.compose(
        "ct_icp_options:\n  size_voxel_map: 9.0\n  voxel_neighborhood: 3\n  max_dist_to_plane_icp: 0.5\n"
        "  ls_sigma: 1e-3\nnot_a_key: 4\n"), dropped=d)
    assert o.ct_icp_options.ls_sigma == 1e-3
    assert o.ct_icp_options.max_dist_to_plane_ct_icp == REF["CTICPOptions"]["max_dist_to_plane_ct_icp"]
    assert d == {}


@pytest.mark.parametrize("key", ["save_mid_frame", "use_outdoor_evaluation"])
def test_int_typed_runner_keys_refuse_true(key):
    with pytest.raises(config.ConfigError, match=key):
        config.load_runner_options(config.compose("%s: true\n" % key))
    assert getattr(config.load_runner_options(config.compose("%s: 0\n" % key)), key) == 0


def test_enum_errors_are_the_references():
    with pytest.raises(config.ConfigError, match="^Distance CT_POINT_TO_PLANE not recognized as a valid distance$"):
        odo("ct_icp_options:\n  distance: CT_POINT_TO_PLANE\n")
    with pytest.raises(config.ConfigError, match=r"^Invalid Solver Options found: LM Not in \[GN, CERES, ROBUST\]$"):
        odo("ct_icp_options:\n  solver: LM\n")
    with pytest.raises(config.ConfigError, match="^Unrecognised loss function L1$"):
        odo("ct_icp_options:\n  loss_function: L1\n")
    with pytest.raises(config.ConfigError, match="^Parametrization is not supported !$"):
        odo("ct_icp_options:\n  parametrization: SPLINE\n")
    with pytest.raises(config.ConfigError, match="^Not implemented error$"):
        odo("map_options:\n  map_type: OCTREE\n")


def test_unsorted_resolutions_are_sorted_stably():
    o = odo("map_options:\n  map_type: MULTI_RESOLUTION_VOXEL_HASHMAP\n  max_frames_to_keep: 7\n  resolutions:\n"
            "    - {resolution: 2.0, max_num_points: 12.9}\n"
            "    - {resolution: 0.5, min_distance_between_points: 0.05}\n"
            "    - {resolution: 2.0, max_num_points: 3}\n")
    m = o.map_options
    assert m.num_resolutions == 3 and m.max_frames_to_keep == 7 and m.default_radius == REF["MapOptions"]["default_radius"]
    got = [(r.resolution, r.min_distance_between_points, r.max_num_points) for r in m.resolutions[:3]]
    assert got == [(0.5, 0.05, 40), (2.0, 0.1, 12), (2.0, 0.1, 3)]
    assert all(r.resolution == 0 and r.max_num_points == 0 for r in m.resolutions[3:])
    with pytest.raises(config.ConfigError, match="Invalid Resolution Param"):
        odo("map_options:\n  map_type: MULTI_RESOLUTION_VOXEL_HASHMAP\n  resolutions:\n    - {max_num_points: 3}\n")


def test_old_map_path():
    b = ct_icp_b200.engine()
    o = odo("map_options:\n  size_voxel_map: 0.7\n  max_num_points_in_voxel: 25.8\n")
    first = b.default_map_options().resolutions[0]
    want = b.legacy_map_options(0.7, 25, first.min_distance_between_points)
    assert bytes(o.map_options) == bytes(want)
    assert o.map_options.max_frames_to_keep == 1


def test_no_map_options_reads_the_odometry_node():
    b = ct_icp_b200.engine()
    warnings = []
    o = config.yaml_to_odometry_options(config.compose(
        "size_voxel_map: 1.5\nmax_num_points_in_voxel: 20\nmin_distance_points: 0.2\n"), warnings=warnings)
    assert bytes(o.map_options) == bytes(b.legacy_map_options(1.5, 20, 0.2))
    assert "does not have any node `map_options`" in warnings[0]
    with pytest.raises(config.ConfigError):   # the int clause of the old keys still runs after the double read
        odo("map_options: {}\nmax_num_points_in_voxel: 20.5\n")


def test_unknown_strategy_type_warns_and_reads_its_keys():
    warnings = []
    o = config.yaml_to_odometry_options(config.compose(
        "neighborhood_strategy:\n  type: KDTREE\n  max_num_neighbors: 12\n  min_num_neighbors: 4\n  radius_max: 9\n"),
        warnings=warnings)
    s = o.neighborhood_strategy
    assert s.type == abi.STRATEGY["NEAREST_NEIGHBOR_STRATEGY"] and (s.max_num_neighbors, s.min_num_neighbors) == (12, 4)
    assert s.radius_max == REF["NeighborStrategyOptions"]["DISTANCE_BASED_STRATEGY"]["radius_max"]
    assert warnings[-1] == "The neighborhood strategy type :KDTREE is not recognised"
    o = odo("neighborhood_strategy:\n  type: DISTANCE_BASED_STRATEGY\n  radius_max: 9\n  exponent: 2\n")
    s = o.neighborhood_strategy
    assert (s.type, s.radius_max, s.exponent, s.max_num_neighbors, s.min_num_neighbors) == (1, 9.0, 2.0, 20, 8)


def test_dataset_options_sequence_uses_its_first_entry():
    root = config.compose("dataset_options:\n  - dataset: nclt\n    root_path: /a\n    nclt_num_aggregated_pc: 110\n"
                          "  - dataset: KITTI\n    root_path: /b\n")
    d = config.dataset_options_from_config(root)
    assert (d.dataset, d.root_path, d.nclt_num_aggregated_pc, d.use_all_datasets) == ("NCLT", "/a", 110, True)
    with pytest.raises(config.ConfigError, match="The `dataset` name: MARS is invalid."):   # every entry is read
        config.dataset_options_from_config(config.compose(
            "dataset_options:\n  - dataset: nclt\n  - dataset: MARS\n"))
    d = config.dataset_options_from_config(config.compose("dataset_options:\n  dataset: hilti\n  root_path: x\n"))
    assert d.dataset == "HILTI_2021"


def test_missing_named_sequence_is_an_error(tmp_path):
    os.makedirs(tmp_path / "00" / "frames")
    node = config.compose("dataset: KITTI_raw\nroot_path: %s\nuse_all_datasets: false\nsequence_options:\n"
                          "  - sequence_name: 00\n    start_frame_id: 3\n    max_num_frames: 5\n" % tmp_path)
    found = datasets.load_dataset_from_options(ct_icp_b200.engine(), config.yaml_to_dataset_options(node))
    assert [label for label, _ in found] == ["KITTI_raw_00"]
    seq = found[0][1]
    assert (seq.init, seq.current, seq.max_frames) == (3, 3, 5)
    node["sequence_options"].append({"sequence_name": "01"})
    with pytest.raises(config.ConfigError, match="Could not find all the sequences"):
        datasets.load_dataset_from_options(ct_icp_b200.engine(), config.yaml_to_dataset_options(node))


def test_courtyard_scene_parses_to_the_golden_dict():
    spec = config.yaml_to_synthetic_scene(config.load_config(os.path.join(CONFIGS, "synthetic", "courtyard.yaml")))
    assert spec == json.load(open(os.path.join(ROOT, "tests", "golden", "synthetic_courtyard.json")))


def test_metrics_yaml_round_trips_every_bit(tmp_path):
    rng = np.random.default_rng(5)
    vals = [math.nan, math.inf, -math.inf, 0.0, -0.0, 5e-324, 1.7976931348623157e308, 0.1, 1e20, 1 / 3.0] + \
        list(rng.standard_normal(20) * 10.0 ** rng.integers(-30, 30, 20))
    metrics = {}
    for i in range(0, len(vals), 5):
        v = vals[i:i + 5]
        metrics["SEQ_%d#" % i] = {"MAX_APE": v[0], "MEAN_APE": v[1], "MEAN_RPE": v[2], "success": False,
                                  "finished": False, "MEAN_LOCAL_ERROR": v[3], "MAX_LOCAL_ERROR": v[4],
                                  "INDEX_MAX_LOCAL_ERROR": i - 3, "Average(ms)": v[0], "AVG_NUM_ATTEMPTS": -1.0}
    path = tmp_path / "metrics.yaml"
    path.write_text(runner.metrics_yaml(metrics))
    back = runner.read_metrics_yaml(str(path))
    assert list(back) == sorted(metrics)
    for name, m in metrics.items():
        assert list(back[name]) == list(runner.METRIC_KEYS)
        for k, v in m.items():
            if isinstance(v, float):
                assert struct.pack("<d", back[name][k]) == struct.pack("<d", v), (name, k, v)
            else:
                assert back[name][k] == v and type(back[name][k]) is type(v)
    import yaml   # any YAML reader sees the same keys and numbers
    plain = yaml.safe_load(path.read_text())
    assert list(plain[sorted(metrics)[0]]) == list(runner.METRIC_KEYS)
