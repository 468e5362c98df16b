"""The reference's YAML configuration readers (src/ct_icp/config.cpp, src/ct_icp/map.cpp:10-77,
include/ct_icp/neighborhood_strategy.h:51-114, command/odometry_runner.cpp OdometryRunner::Options::LoadYAML), clause by
clause, returning the engine's option structs (the abi types Binding.default_odometry_options() returns).

A configuration is composed with PyYAML's BaseLoader, so every scalar keeps its text, and each clause converts that
text with yaml-cpp's `as<T>` rules for the clause's type (DESIGN §5.13): `sequence_name: 00` stays "00", `1e-3` is a
double, `as<bool>` takes the y / yes / true / on and n / no / false / off families, and `as<int>` refuses `true`.
Exactly the keys the reference's clauses name are read; every other key is ignored. Keys the reference reads into
fields the engine's structs do not carry (the ones tests/test_reference_defaults.py lists) are converted all the same,
so a bad value fails as it would in the reference, and land in the `dropped` dict a reader is given.

A node is what `compose` makes of a YAML node: a dict (a map, first occurrence of a key wins), a list (a sequence),
a str (a scalar) or None (a null: an empty value, or a plain ~ / null / Null / NULL).
"""
import math
import re

from . import _abi as abi


class ConfigError(ValueError):
    """A configuration the reference refuses (a failed conversion, a CHECK or a throw), with the reference's message
    where it has one"""


_NULLS = ("", "~", "null", "Null", "NULL")


def _tree(node):
    import yaml
    if isinstance(node, yaml.ScalarNode):
        return None if node.style is None and node.value in _NULLS else node.value
    if isinstance(node, yaml.SequenceNode):
        return [_tree(n) for n in node.value]
    out = {}
    for k, v in node.value:
        key = _tree(k)
        if not isinstance(key, str):
            key = "null" if key is None else repr(key)
        out.setdefault(key, _tree(v))
    return out


def compose(text):
    """the node tree of a YAML document (an empty document is an empty map)"""
    import yaml   # only here and in the tools: nothing else in the package needs PyYAML
    node = yaml.compose(text, Loader=yaml.BaseLoader)
    return {} if node is None else _tree(node)


def load_config(path):
    """YAML::LoadFile(path) as a node tree"""
    with open(path, "r", encoding="utf-8") as f:
        return compose(f.read())


# ---- yaml-cpp's as<T> on a scalar's text ------------------------------------------------------------------------------
_INT = re.compile(r"[+-]?(0[xX][0-9a-fA-F]+|0[0-7]*|[1-9][0-9]*)\Z")
_FLOAT = re.compile(r"[+-]?([0-9]+\.?[0-9]*|\.[0-9]+)([eE][+-]?[0-9]+)?\Z")
_INF = (".inf", ".Inf", ".INF", "+.inf", "+.Inf", "+.INF")
_NINF = ("-.inf", "-.Inf", "-.INF")
_NAN = (".nan", ".NaN", ".NAN")
_BOOLS = (("y", "n"), ("yes", "no"), ("true", "false"), ("on", "off"))


def _bad(key, v, what):
    return ConfigError("bad conversion: `%s` is %s, not %s" % (key, "a null" if v is None else
                                                                 ("%r" % v if isinstance(v, str) else "not a scalar"),
                                                                 what))


def as_string(v, key):
    """as<std::string>: a scalar's text; a null reads "null"; a map or a sequence is an error"""
    if v is None:
        return "null"
    if not isinstance(v, str):
        raise _bad(key, v, "a string")
    return v


def _as_integer(v, key, lo, hi, what):
    # std::stringstream with the base left to the prefix (0x → hex, 0 → octal), whole text consumed, no overflow
    if not isinstance(v, str) or not _INT.match(v):
        raise _bad(key, v, what)
    s = v.lstrip("+-")
    x = int(s, 16) if s[:2] in ("0x", "0X") else int(s, 8) if len(s) > 1 and s[0] == "0" else int(s)
    x = -x if v.startswith("-") else x
    if not lo <= x <= hi:
        raise _bad(key, v, what)
    return x


def as_int(v, key):
    return _as_integer(v, key, -2 ** 31, 2 ** 31 - 1, "an int")


def as_size_t(v, key):
    if isinstance(v, str) and v.startswith("-"):
        raise _bad(key, v, "a size_t")
    return _as_integer(v, key, 0, 2 ** 64 - 1, "a size_t")


def as_double(v, key):
    """as<double>: a decimal number with an optional exponent (no hex), or one of YAML's .inf / -.inf / .nan
    spellings; a finite text that overflows is an error"""
    if isinstance(v, str):
        if _FLOAT.match(v):
            x = float(v)
            if not math.isinf(x):
                return x
        elif v in _INF:
            return math.inf
        elif v in _NINF:
            return -math.inf
        elif v in _NAN:
            return math.nan
    raise _bad(key, v, "a double")


def as_float(v, key):
    """as<float>: as<double>'s grammar, rounded to binary32 (overflow is an error)"""
    import numpy as np
    x = as_double(v, key)
    with np.errstate(over="ignore"):
        f = np.float32(x)
    if np.isinf(f) and not math.isinf(x):
        raise _bad(key, v, "a float")
    return float(f)


def as_bool(v, key):
    """as<bool>: y / yes / true / on or n / no / false / off, all lower case, all upper case or capitalised"""
    if isinstance(v, str) and (v in (v.lower(), v.upper()) or v == v[:1].upper() + v[1:].lower()):
        low = v.lower()
        for t, f in _BOOLS:
            if low == t:
                return True
            if low == f:
                return False
    raise _bad(key, v, "a bool")


_CONVERT = {"int": as_int, "double": as_double, "bool": as_bool, "string": as_string, "float": as_float,
            "size_t": as_size_t}
_MISSING = object()


def _get(node, key):
    """node[key]: the child, or _MISSING when the node has no such key (yaml-cpp's undefined node)"""
    if isinstance(node, dict):
        return node.get(key, _MISSING)
    if node is None:
        return _MISSING
    raise ConfigError("operator[] call on a scalar or a sequence (key: \"%s\")" % key)


def _clauses(node, target, clauses, dropped=None, prefix=""):
    """OPTION_CLAUSE / FIND_OPTION over (name, type) clauses in source order: a present key is converted; a field the
    target struct carries is set (bools as 0 / 1), any other lands in dropped[prefix + name]"""
    for name, typ in clauses:
        v = _get(node, name)
        if v is _MISSING:
            continue
        x = _CONVERT[typ](v, prefix + name)
        if target is not None and hasattr(target, name):
            setattr(target, name, int(x) if typ == "bool" else x)
        elif dropped is not None:
            dropped[prefix + name] = x


def _binding(binding):
    if binding is None:
        from ._lib import engine
        binding = engine()
    return binding


# ---- ct_icp::CTICPOptions (config.cpp:26-122) ------------------------------------------------------------------------
_ICP_CLAUSES = [
    ("threshold_voxel_occupancy", "int"), ("num_iters_icp", "int"), ("min_number_neighbors", "int"),
    ("max_number_neighbors", "int"), ("max_dist_to_plane_ct_icp", "double"), ("threshold_orientation_norm", "double"),
    ("threshold_translation_norm", "double"), ("debug_print", "bool"), ("point_to_plane_with_distortion", "bool"),
    ("num_closest_neighbors", "int"), ("ls_max_num_iters", "int"), ("ls_num_threads", "int"), ("ls_sigma", "double"),
    ("min_num_residuals", "int"), ("max_num_residuals", "int"), ("weight_alpha", "double"),
    ("weight_neighborhood", "double"), ("ls_tolerant_min_threshold", "double"), ("power_planarity", "double"),
    ("point_to_plane_with_distortion", "bool"),
    ("output_normals", "bool"), ("output_lines", "bool"), ("output_weights", "bool"), ("output_residuals", "bool"),
    ("output_neighborhood_info", "bool"),
    ("threshold_linearity", "double"), ("threshold_planarity", "double"), ("weight_point_to_point", "double"),
    ("outlier_distance", "double"), ("use_barycenter", "bool"),
]


def yaml_to_ct_icp_options(icp_node, binding=None, dropped=None, prefix="ct_icp_options."):
    """ct_icp::yaml_to_ct_icp_options: CTICPOptions() defaults, then every clause of the node"""
    o = _binding(binding).default_icp_options()
    _clauses(icp_node, o, _ICP_CLAUSES, dropped, prefix)
    v = _get(icp_node, "distance")
    if v is not _MISSING:
        d = as_string(v, prefix + "distance")
        if d not in ("POINT_TO_PLANE", "POINT_TO_LINE", "POINT_TO_POINT", "POINT_TO_DISTRIBUTION"):
            raise ConfigError("Distance " + d + " not recognized as a valid distance")
        o.distance = abi.DISTANCE[d]
    v = _get(icp_node, "parametrization")
    if v is not _MISSING:
        p = as_string(v, prefix + "parametrization")
        if p not in abi.PARAMETRIZATION:
            raise ConfigError("Parametrization is not supported !")
        o.parametrization = abi.PARAMETRIZATION[p]
    v = _get(icp_node, "solver")
    if v is not _MISSING:
        s = as_string(v, prefix + "solver")
        if s not in abi.SOLVER:
            raise ConfigError("Invalid Solver Options found: " + s + " Not in [GN, CERES, ROBUST]")
        o.solver = abi.SOLVER[s]
    v = _get(icp_node, "loss_function")
    if v is not _MISSING:
        f = as_string(v, prefix + "loss_function")
        if f not in abi.LOSS:
            raise ConfigError("Unrecognised loss function " + f)
        o.loss_function = abi.LOSS[f]
    return o


# ---- ct_icp::PreviousFrameMotionModel::Options (config.cpp:304-318) --------------------------------------------------
_MOTION_CLAUSES = [("beta_location_consistency", "double"), ("beta_small_velocity", "double"),
                   ("beta_orientation_consistency", "double"), ("beta_constant_velocity", "double"),
                   ("threshold_orientation_deg", "double"), ("threshold_translation_diff", "double"),
                   ("log_if_invalid", "bool")]


def yaml_to_motion_model_options(node, binding=None, dropped=None, prefix="default_motion_model."):
    o = _binding(binding).default_odometry_options().default_motion_model
    _clauses(node, o, _MOTION_CLAUSES, dropped, prefix)
    v = _get(node, "model")
    if v is not _MISSING:
        m = as_string(v, prefix + "model")
        if m not in abi.MOTION_MODEL:
            raise ConfigError("[ERROR] The option " + m + " is not a valid option. Valid options are: {" +
                              ", ".join(sorted(abi.MOTION_MODEL)) + "}")
        o.model = abi.MOTION_MODEL[m]
    return o


# ---- map options (map.cpp:10-77) -------------------------------------------------------------------------------------
def _old_map_options(node, b):
    """old_map_options_from_yaml: one resolution (the default options' first, keys overriding it), max_frames_to_keep
    1: Binding.legacy_map_options. max_num_points_in_voxel is read as a double and truncated."""
    first = b.default_map_options().resolutions[0]
    size, npts, dmin = first.resolution, first.max_num_points, first.min_distance_between_points
    v = _get(node, "size_voxel_map")
    if v is not _MISSING:
        size = as_double(v, "size_voxel_map")
    v = _get(node, "max_num_points_in_voxel")
    if v is not _MISSING:
        npts = _trunc_int(as_double(v, "max_num_points_in_voxel"), "max_num_points_in_voxel")
    v = _get(node, "min_distance_points")
    if v is not _MISSING:
        dmin = as_double(v, "min_distance_points")
    return b.legacy_map_options(size, npts, dmin)


def _trunc_int(x, key):
    # the double → int assignment of the reference; a value outside int's range is undefined there and refused here
    if not (-2.0 ** 31 < x < 2.0 ** 31):
        raise ConfigError("`%s` = %r does not fit an int" % (key, x))
    return int(x)


def yaml_to_map_options(node, binding=None):
    """ct_icp::yaml_to_map_options: MULTI_RESOLUTION_VOXEL_HASHMAP, any other map_type an error, no map_type the old
    options. The resolutions are sorted by resolution, stably (std::sort leaves equal resolutions in an unspecified
    order); more than CTICP_MAX_RESOLUTIONS is refused."""
    b = _binding(binding)
    v = _get(node, "map_type")
    if v is _MISSING:
        return _old_map_options(node, b)
    if as_string(v, "map_type") != "MULTI_RESOLUTION_VOXEL_HASHMAP":
        raise ConfigError("Not implemented error")
    o = b.default_map_options()
    res_node = _get(node, "resolutions")
    if res_node is not _MISSING:
        if not isinstance(res_node, list):
            raise ConfigError("The node 'resolutions' in the yaml is not a sequence")
        params = []
        for child in res_node:
            if not isinstance(child, dict):
                raise ConfigError("The following child node is not a Map: %r" % (child,))
            p = abi.ResolutionParam()
            p.resolution, p.min_distance_between_points, p.max_num_points = 0.5, 0.1, 40   # ResolutionParam() (map.h)
            v = _get(child, "min_distance_between_points")
            if v is not _MISSING:
                p.min_distance_between_points = as_double(v, "min_distance_between_points")
            v = _get(child, "max_num_points")
            if v is not _MISSING:
                p.max_num_points = _trunc_int(as_double(v, "max_num_points"), "max_num_points")
            v = _get(child, "resolution")
            if v is _MISSING:
                raise ConfigError("Invalid Resolution Param in the yaml: %r" % (child,))
            p.resolution = as_double(v, "resolution")
            params.append(p)
        if not params:
            raise ConfigError("The yaml does not define a valid set of resolutions for the map")
        if len(params) > abi.CTICP_MAX_RESOLUTIONS:
            raise ConfigError("%d resolutions: the engine's map holds at most %d" %
                              (len(params), abi.CTICP_MAX_RESOLUTIONS))
        params.sort(key=lambda p: p.resolution)
        o.num_resolutions = len(params)
        for i in range(abi.CTICP_MAX_RESOLUTIONS):   # the slots past the last resolution are zero
            o.resolutions[i] = params[i] if i < len(params) else abi.ResolutionParam()
    _clauses(node, o, [("max_frames_to_keep", "int"), ("default_radius", "double")])
    return o


# ---- neighbourhood strategy (odometry config.cpp:155-168, neighborhood_strategy.h:51-114) ----------------------------
def strategy_from_yaml(strategy_node, current=None):
    """the strategy clause of yaml_to_odometry_options: the node's type (or the current one's) chooses the options
    object (DISTANCE_BASED_STRATEGY a fresh one; any other type than NEAREST_NEIGHBOR_STRATEGY warns and keeps the
    current), whose FromYAML then reads its keys. Returns (options, warning or None)."""
    o = abi.StrategyOptions() if current is None else current.copy()
    names = {v: k for k, v in abi.STRATEGY.items()}
    v = _get(strategy_node, "type")
    typ = as_string(v, "neighborhood_strategy.type") if v is not _MISSING else names[o.type]
    warning = None
    if typ == "DISTANCE_BASED_STRATEGY":
        o = abi.StrategyOptions(type=abi.STRATEGY["DISTANCE_BASED_STRATEGY"])
    elif typ != "NEAREST_NEIGHBOR_STRATEGY":
        warning = "The neighborhood strategy type :" + typ + " is not recognised"
    clauses = [("max_num_neighbors", "int"), ("min_num_neighbors", "int")]
    if o.type == abi.STRATEGY["DISTANCE_BASED_STRATEGY"]:
        clauses += [("distance_max", "double"), ("radius_min", "double"), ("radius_max", "double"),
                    ("exponent", "double")]
    _clauses(strategy_node, o, clauses, prefix="neighborhood_strategy.")
    return o, warning


# ---- ct_icp::OdometryOptions (config.cpp:132-255) --------------------------------------------------------------------
_ODOMETRY_HEAD = [("voxel_size", "double"), ("max_distance", "double"), ("distance_error_threshold", "double"),
                  ("orientation_error_threshold", "double"), ("max_num_keypoints", "int"),
                  ("sample_voxel_size", "double")]
_ODOMETRY_TAIL = [
    ("min_distance_points", "double"), ("max_num_points_in_voxel", "int"), ("size_voxel_map", "double"),
    ("voxel_neighborhood", "int"), ("max_radius_neighborhood", "double"),
    ("init_num_frames", "int"), ("init_voxel_size", "double"), ("init_sample_voxel_size", "double"),
    ("log_to_file", "bool"), ("log_file_destination", "string"), ("debug_print", "bool"), ("debug_viz", "bool"),
    ("do_no_insert", "bool"), ("always_insert", "bool"),
    ("robust_minimal_level", "int"), ("robust_registration", "bool"), ("robust_full_voxel_threshold", "double"),
    ("robust_fail_early", "bool"), ("robust_num_attempts", "int"), ("robust_max_voxel_neighborhood", "int"),
    ("robust_threshold_relative_orientation", "double"), ("robust_threshold_ego_orientation", "double"),
]


def _check_enum(node, key, names, table):
    v = _get(node, key)
    if v is _MISSING:
        return None
    s = as_string(v, key)
    if s not in names:
        raise ConfigError("Check failed: " + " || ".join('%s == "%s"' % (key, n) for n in names) + " (got " + s + ")")
    return table[s]


def yaml_to_odometry_options(odometry_node, binding=None, dropped=None, warnings=None):
    """ct_icp::yaml_to_odometry_options: OdometryOptions() defaults, then the clauses in the reference's order.
    Keys the structs do not carry go to `dropped` (by their dotted path), warnings the reference logs to `warnings`."""
    b = _binding(binding)
    dropped = {} if dropped is None else dropped
    o = b.default_odometry_options()
    _clauses(odometry_node, o, _ODOMETRY_HEAD, dropped)
    map_node = _get(odometry_node, "map_options")
    if map_node is not _MISSING:
        o.map_options = yaml_to_map_options(map_node, b)
    else:
        if warnings is not None:
            warnings.append("The config does not have any node `map_options`, using the default (deprecated) set of "
                            "parameters to define the map")
        o.map_options = yaml_to_map_options(odometry_node, b)
    strategy_node = _get(odometry_node, "neighborhood_strategy")
    if strategy_node is not _MISSING:
        o.neighborhood_strategy, w = strategy_from_yaml(strategy_node, o.neighborhood_strategy)
        if w and warnings is not None:
            warnings.append(w)
    _clauses(odometry_node, o, _ODOMETRY_TAIL, dropped)
    mm = _get(odometry_node, "default_motion_model")
    if mm is not _MISSING:
        o.default_motion_model = yaml_to_motion_model_options(mm, b, dropped)
    x = _check_enum(odometry_node, "motion_compensation", ["NONE", "CONSTANT_VELOCITY", "ITERATIVE", "CONTINUOUS"],
                    abi.MOTION_COMPENSATION)
    if x is not None:
        o.motion_compensation = x
    x = _check_enum(odometry_node, "sampling", ["GRID", "ADAPTIVE", "NONE"], abi.SAMPLING)
    if x is not None:
        o.sampling = x
    x = _check_enum(odometry_node, "initialization", ["INIT_NONE", "INIT_CONSTANT_VELOCITY"], abi.INITIALIZATION)
    if x is not None:
        o.initialization = x
    icp_node = _get(odometry_node, "ct_icp_options")
    if icp_node is not _MISSING:
        o.ct_icp_options = yaml_to_ct_icp_options(icp_node, b, dropped)
    return o


# ---- ct_icp::DatasetOptions (config.cpp:264-301, include/ct_icp/dataset.h:270-293) -----------------------------------
# DATASETFromString: case-insensitive; hilti is HILTI_2021
_DATASET_NAMES = {"kitti_carla": "KITTI_CARLA", "kitti_360": "KITTI_360", "kitti": "KITTI", "hilti": "HILTI_2021",
                  "hilti_2021": "HILTI_2021", "hilti_2022": "HILTI_2022", "kitti_raw": "KITTI_raw", "nclt": "NCLT",
                  "synthetic": "SYNTHETIC", "ply_directory": "PLY_DIRECTORY"}


class SequenceOptions:
    def __init__(self, sequence_name="", start_frame_id=0, max_num_frames=-1):
        self.sequence_name, self.start_frame_id, self.max_num_frames = sequence_name, start_frame_id, max_num_frames

    def __repr__(self):
        return "SequenceOptions(%r, %d, %d)" % (self.sequence_name, self.start_frame_id, self.max_num_frames)


class DatasetOptions:
    """ct_icp::DatasetOptions: dataset is the DATASETEnumToString name ("KITTI_raw", "NCLT", "SYNTHETIC", ...) or
    None when the node names none"""

    def __init__(self):
        self.dataset = None
        self.root_path = ""
        self.fail_if_incomplete = False
        self.min_dist_lidar_center = 3.0
        self.max_dist_lidar_center = 100.0
        self.nclt_num_aggregated_pc = 220
        self.use_all_datasets = True
        self.sequence_options = []


def yaml_to_dataset_options(dataset_node):
    o = DatasetOptions()
    v = _get(dataset_node, "dataset")
    if v is not _MISSING:
        name = as_string(v, "dataset")
        if name.lower() not in _DATASET_NAMES:
            raise ConfigError("The `dataset` name: " + name + " is invalid.")
        o.dataset = _DATASET_NAMES[name.lower()]
    _clauses(dataset_node, o, [("root_path", "string"), ("fail_if_incomplete", "bool"),
                               ("min_dist_lidar_center", "float"), ("nclt_num_aggregated_pc", "int"),
                               ("max_dist_lidar_center", "float"), ("use_all_datasets", "bool")])
    for k in ("fail_if_incomplete", "use_all_datasets"):
        setattr(o, k, bool(getattr(o, k)))
    seqs = _get(dataset_node, "sequence_options")
    if seqs is not _MISSING:
        o.sequence_options = []
        for seq_node in _children(seqs):
            s = SequenceOptions()
            _clauses(seq_node, s, [("sequence_name", "string"), ("start_frame_id", "int"), ("max_num_frames", "int")],
                     prefix="sequence_options.")
            o.sequence_options.append(s)
    return o


def _children(node):
    """range-for over a node: a sequence's items, a map's values (yaml-cpp iterates a map's pairs; a pair is not a map,
    so any key read from it is absent), nothing for a scalar or a null"""
    if isinstance(node, list):
        return node
    if isinstance(node, dict):
        return [None] * len(node)
    return []


def yaml_to_dataset_options_vector(node):
    return [yaml_to_dataset_options(child) for child in _children(node)]


# ---- OdometryRunner::Options (command/odometry_runner.h, odometry_runner.cpp:347-363) --------------------------------
class RunnerOptions:
    """OdometryRunner::Options with the reference's defaults, plus concurrent_sequences (not a reference key): how many
    sequences register side by side, 1 being the reference's serial order"""

    def __init__(self, binding=None):
        self.odometry_options = _binding(binding).default_odometry_options()
        self.generate_directory_prefix = True
        self.progress_bar = True
        self.debug_information = False
        self.output_results = True
        self.exit_early = True
        self.compute_metrics_period = 500
        self.save_mid_frame = True
        self.use_outdoor_evaluation = True
        self.output_dir = ""
        self.concurrent_sequences = 1
        self.dropped = {}
        self.warnings = []


def load_runner_options(config, binding=None):
    """OdometryRunner::Options::LoadYAML of a configuration's root node (use_outdoor_evaluation and save_mid_frame are
    read as int, as the reference reads them, so `true` is an error); with_viz3d is read and dropped"""
    o = RunnerOptions(binding)
    node = _get(config, "odometry_options")
    if node is not _MISSING:
        o.odometry_options = yaml_to_odometry_options(node, binding, o.dropped, o.warnings)
    _clauses(config, o, [("with_viz3d", "bool"), ("generate_directory_prefix", "bool"), ("progress_bar", "bool"),
                         ("debug_information", "bool"), ("output_results", "bool"), ("exit_early", "bool"),
                         ("compute_metrics_period", "int"), ("use_outdoor_evaluation", "int"),
                         ("save_mid_frame", "int"), ("output_dir", "string"), ("concurrent_sequences", "int")],
             o.dropped)
    for k in ("generate_directory_prefix", "progress_bar", "debug_information", "output_results", "exit_early"):
        setattr(o, k, bool(getattr(o, k)))
    if not 1 <= o.concurrent_sequences <= 64:   # a cticp_odometry_register_batch call takes 1 to 64 items
        raise ConfigError("concurrent_sequences must be in [1, 64]")
    return o


def dataset_options_from_config(config):
    """the dataset of a run (cmd_run_odometry.cpp DatasetFromConfig): the top-level dataset_options node as a map, or
    the first entry of it as a sequence (the reference returns inside its loop over the entries)"""
    node = _get(config, "dataset_options")
    if node is _MISSING:
        raise ConfigError("The config does not contain a node `dataset_options`")
    if isinstance(node, list):
        if not node:
            raise ConfigError("The node `dataset_options` is an empty sequence")
        return yaml_to_dataset_options_vector(node)[0]   # every entry is read, the first is used
    return yaml_to_dataset_options(node)


# ---- the scene of a SYNTHETIC sequence (dataset.cpp SyntheticSequence::PtrFromNode, synthetic.cxx ReadYAML) ----------
def _vector(node, n, key):
    if not isinstance(node, list) or len(node) != n:
        raise ConfigError("Check failed: `%s` is not a sequence of %d scalars" % (key, n))
    return [as_double(v, key) for v in node]


def _points(node, n, key):
    if not isinstance(node, list) or len(node) != n:
        raise ConfigError("The node is not a sequence of size %d (`%s`)" % (n, key))
    return [_vector(p, 3, key) for p in node]


def _round(node, key):
    if _get(node, "radius") is _MISSING or _get(node, "center") is _MISSING:
        raise ConfigError("A Ball cannot be read from Node: %r" % (node,))
    return {"center": _vector(node["center"], 3, key + ".center"), "radius": as_double(node["radius"], key + ".radius")}


def yaml_to_synthetic_scene(root):
    """the dict Binding.synthetic_sequence takes, read from a scene YAML's root node: sample_frequency,
    max_lidar_distance and num_points_per_primitives when present (sequence_name too), the acquisition's poses with the
    keys each one has, and its triangles, lines, balls and spheres (an absent kind is an empty list)"""
    acq = _get(root, "acquisition")
    if acq is _MISSING:
        raise ConfigError("The root node does not contain a node `acquisition` at its root.")
    poses = _get(acq, "poses")
    if poses is _MISSING:
        raise ConfigError("The node does not contain a `poses` node")
    if not isinstance(poses, list):
        raise ConfigError("The `poses` node is not a sequence")
    out_poses = []
    for child in poses:
        p = {}
        for key, n in (("quaternion", 4), ("translation", 3)):
            v = _get(child, key)
            if v is not _MISSING:
                p[key] = _vector(v, n, "poses." + key)
        v = _get(child, "dest_frame_id")
        if v is not _MISSING:
            p["dest_frame_id"] = as_int(v, "poses.dest_frame_id")
        v = _get(child, "dest_timestamp")
        if v is not _MISSING:
            p["dest_timestamp"] = as_double(v, "poses.dest_timestamp")
        out_poses.append(p)
    spec = {"acquisition": {"poses": out_poses}}
    for key, read in (("triangles", lambda n: _points(n, 3, "triangles")), ("lines", lambda n: _points(n, 2, "lines")),
                      ("balls", lambda n: _round(n, "balls")), ("spheres", lambda n: _round(n, "spheres"))):
        v = _get(acq, key)
        if v is not _MISSING and not isinstance(v, list):
            raise ConfigError("The node with key `" + key + "` is not a sequence")
        spec["acquisition"][key] = [] if v is _MISSING else [read(x) for x in v]
    for key, conv in (("sample_frequency", as_double), ("max_lidar_distance", as_double),
                      ("num_points_per_primitives", as_size_t), ("sequence_name", as_string)):
        v = _get(root, key)
        if v is not _MISSING:
            spec[key] = conv(v, key)
    return spec
