"""The facade's YAML readers (ct_icp::yaml_to_odometry_options / yaml_to_dataset_options, templates over a node type
with yaml-cpp's interface in ct_icp_b200/include/ct_icp_b200/odometry.hpp) over the stub node of
tests/cpp/yaml_node_stub.h give the Python readers' results: the same OdometryOptions bytes for every odometry node of
every configuration in tests/golden/configs, the same DatasetOptions, and the same refusals. CPU only: plain g++ against
include/cticp.h (the option defaults come from the engine library, which needs no device)."""
import os
import subprocess
import tempfile

import pytest

from ct_icp_b200 import config

from test_config_yaml import CONFIGS, fixture_files, odometry_nodes

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

# the quirks of the readers, each through both
CASES = [
    "ct_icp_options:\n  beta_location_consistency: 7.0\n  ls_sigma: 1e-3\n  size_voxel_map: 9\n",
    "map_options:\n  map_type: MULTI_RESOLUTION_VOXEL_HASHMAP\n  max_frames_to_keep: 7\n  resolutions:\n"
    "    - {resolution: 2.0, max_num_points: 12.9}\n    - {resolution: 0.5, min_distance_between_points: 0.05}\n"
    "    - {resolution: 2.0, max_num_points: 3}\n",
    "map_options:\n  size_voxel_map: 0.7\n  max_num_points_in_voxel: 25.8\n",
    "size_voxel_map: 1.5\nmax_num_points_in_voxel: 20\nmin_distance_points: 0.2\n",
    "neighborhood_strategy:\n  type: KDTREE\n  max_num_neighbors: 12\n  min_num_neighbors: 4\n  radius_max: 9\n",
    "neighborhood_strategy:\n  type: DISTANCE_BASED_STRATEGY\n  radius_max: 9\n  exponent: 2\n",
    "default_motion_model:\n  beta_location_consistency: 7.0\n  model: SMALL_VELOCITY\n  log_if_invalid: off\n",
    "ct_icp_options:\n  distance: CT_POINT_TO_PLANE\n",
    "ct_icp_options:\n  solver: LM\n",
    "ct_icp_options:\n  loss_function: L1\n",
    "map_options:\n  map_type: OCTREE\n",
    "sampling: RANDOM\n",
    "max_num_keypoints: 0x40\ninit_num_frames: 010\nrobust_registration: Yes\ndebug_print: OFF\n",
    "max_num_keypoints: true\n",
    "voxel_size: 1e999\n",
]


def serialise(node):
    """the length-prefixed text yaml_node_stub.h reads"""
    if node is None:
        return "N\n"
    if isinstance(node, str):
        b = node.encode("utf-8")
        return "V %d %s\n" % (len(b), node)
    if isinstance(node, list):
        return "S %d\n" % len(node) + "".join(serialise(x) for x in node)
    return "M %d\n" % len(node) + "".join("K %d %s\n" % (len(k.encode("utf-8")), k) + serialise(v)
                                         for k, v in node.items())


@pytest.fixture(scope="module")
def facade():
    cxx = "/usr/bin/g++" if os.path.exists("/usr/bin/g++") else "g++"
    d = tempfile.mkdtemp()
    exe = os.path.join(d, "config_facade_test")
    cmd = [cxx, "-std=c++17", "-O1", "-Wall", "-I", os.path.join(ROOT, "include"), "-I",
           os.path.join(ROOT, "ct_icp_b200", "include"), "-I", os.path.join(ROOT, "tests", "cpp"),
           os.path.join(ROOT, "tests", "cpp", "config_facade_test.cpp"), "-L", os.path.join(ROOT, "ct_icp_b200"),
           "-lcticp_b200", "-Wl,-rpath," + os.path.join(ROOT, "ct_icp_b200"), "-lm", "-o", exe]
    r = subprocess.run(cmd, capture_output=True, text=True)
    assert r.returncode == 0, r.stderr

    def run(kind, node):
        path = os.path.join(d, "tree.txt")
        with open(path, "w", encoding="utf-8") as f:
            f.write(serialise(node))
        p = subprocess.run([exe, kind, path], capture_output=True, text=True)
        assert p.returncode == 0, p.stderr
        return p.stdout.strip()
    return run


def python_odometry(node):
    try:
        return "OK " + bytes(config.yaml_to_odometry_options(node)).hex()
    except config.ConfigError as e:
        return "ERR " + str(e)


def test_facade_matches_python_on_every_fixture(facade):
    compared = 0
    for rel in fixture_files():
        for label, node in odometry_nodes(rel):
            py = python_odometry(node)
            got = facade("odometry", node)
            if py.startswith("ERR"):   # the same refusal: the enum messages are the reference's in both
                assert got == py, label
            else:
                assert got == py, label
            compared += 1
    assert compared >= 12


@pytest.mark.parametrize("text", CASES)
def test_facade_matches_python_on_each_quirk(facade, text):
    node = config.compose(text)
    py, got = python_odometry(node), facade("odometry", node)
    if py.startswith("ERR bad conversion") or py.startswith("ERR `"):   # conversion errors: only both refuse
        assert got.startswith("ERR"), got
    else:
        assert got == py


def dataset_line(d):
    return "OK " + "|".join([d.dataset or "", d.root_path, str(int(d.fail_if_incomplete)),
                             "%.17g" % d.min_dist_lidar_center, "%.17g" % d.max_dist_lidar_center,
                             str(d.nclt_num_aggregated_pc), str(int(d.use_all_datasets))] +
                            ["%s,%d,%d" % (s.sequence_name, s.start_frame_id, s.max_num_frames)
                             for s in d.sequence_options])


@pytest.mark.parametrize("rel", ["odometry/driving_config.yaml", "odometry/nclt_config.yaml",
                                 "synthetic_ct_icp_config.yaml"])
def test_facade_dataset_options(facade, rel):
    root = config.load_config(os.path.join(CONFIGS, rel))
    node = root["dataset_options"]
    assert facade("dataset", node if isinstance(node, list) else [node]) == \
        dataset_line(config.dataset_options_from_config(root))


def test_facade_dataset_quirks(facade):
    node = config.compose("- dataset: hilti\n  root_path: /a\n  min_dist_lidar_center: 0.1\n  use_all_datasets: no\n"
                          "  sequence_options:\n    - {sequence_name: 00, start_frame_id: 3}\n- dataset: KITTI\n")
    assert facade("dataset", node) == dataset_line(config.yaml_to_dataset_options_vector(node)[0])
    bad = config.compose("- dataset: MARS\n")
    assert facade("dataset", bad) == "ERR The `dataset` name: MARS is invalid."
