"""ctypes mirror of include/cticp.h (the C ABI of the engine).

Field order and types must match the header exactly; tests/test_abi.py checks sizeof() of every struct against
the values compiled into the shared library (cticp_abi_sizeof).
"""
import ctypes as C

CTICP_MAX_RESOLUTIONS = 8

# status codes
OK = 0
ERR_INVALID_ARGUMENT = -1
ERR_NO_DEVICE = -2
ERR_CUDA = -3
ERR_CAPACITY = -4
ERR_TIMESTAMP = -5
ERR_UNSUPPORTED = -6
ERR_NCCL = -7
ERR_INTERNAL = -8

# enums (same numeric order as the reference, see cticp.h)
SOLVER = {"GN": 0, "CERES": 1, "ROBUST": 2}
LOSS = {"STANDARD": 0, "CAUCHY": 1, "HUBER": 2, "TOLERANT": 3, "TRUNCATED": 4}
WEIGHTING = {"PLANARITY": 0, "NEIGHBORHOOD": 1, "ALL": 2}
PARAMETRIZATION = {"SIMPLE": 0, "CONTINUOUS_TIME": 1}
DISTANCE = {"POINT_TO_PLANE": 0, "POINT_TO_POINT": 1, "POINT_TO_LINE": 2, "POINT_TO_DISTRIBUTION": 3}
MOTION_COMPENSATION = {"NONE": 0, "CONSTANT_VELOCITY": 1, "ITERATIVE": 2, "CONTINUOUS": 3}
INITIALIZATION = {"INIT_NONE": 0, "INIT_CONSTANT_VELOCITY": 1}
SAMPLING = {"NONE": 0, "GRID": 1, "ADAPTIVE": 2}
MOTION_MODEL = {"CONSTANT_VELOCITY": 0, "SMALL_VELOCITY": 1}

POINTS_CORRECTED, POINTS_ALL_CORRECTED, POINTS_KEYPOINTS = 0, 1, 2
EVENT_BEFORE_ITERATION, EVENT_ITERATION_COMPLETED, EVENT_FINISHED_REGISTRATION = 0, 1, 2
EVENT_FN = C.CFUNCTYPE(C.c_int, C.c_int, C.c_void_p)   # cticp_event_fn
ERR_CALLBACK = -9


class _Struct(C.Structure):
    def to_dict(self):
        out = {}
        for name, _ in self._fields_:
            if name.startswith("_pad"):
                continue
            v = getattr(self, name)
            if isinstance(v, _Struct):
                v = v.to_dict()
            elif isinstance(v, C.Array):
                v = [x.to_dict() if isinstance(x, _Struct) else x for x in v]
            out[name] = v
        return out

    def copy(self):
        other = type(self)()
        C.memmove(C.byref(other), C.byref(self), C.sizeof(self))
        return other


class IcpOptions(_Struct):
    _fields_ = [
        ("num_iters_icp", C.c_int32), ("parametrization", C.c_int32), ("distance", C.c_int32),
        ("solver", C.c_int32), ("max_num_residuals", C.c_int32), ("min_num_residuals", C.c_int32),
        ("weighting_scheme", C.c_int32), ("max_number_neighbors", C.c_int32), ("min_number_neighbors", C.c_int32),
        ("threshold_voxel_occupancy", C.c_int32), ("num_closest_neighbors", C.c_int32),
        ("point_to_plane_with_distortion", C.c_int32), ("loss_function", C.c_int32),
        ("ls_max_num_iters", C.c_int32), ("ls_num_threads", C.c_int32), ("debug_print", C.c_int32),
        ("weight_alpha", C.c_double), ("weight_neighborhood", C.c_double), ("power_planarity", C.c_double),
        ("threshold_orientation_norm", C.c_double), ("threshold_translation_norm", C.c_double),
        ("ls_sigma", C.c_double), ("ls_tolerant_min_threshold", C.c_double),
        ("max_dist_to_plane_ct_icp", C.c_double),
        ("threshold_linearity", C.c_double), ("threshold_planarity", C.c_double),
        ("weight_point_to_point", C.c_double), ("outlier_distance", C.c_double),
        ("use_barycenter", C.c_int32), ("use_lines", C.c_int32),
    ]


class ResolutionParam(_Struct):
    _fields_ = [("resolution", C.c_double), ("min_distance_between_points", C.c_double),
                ("max_num_points", C.c_int32), ("_pad0", C.c_int32)]


class MapOptions(_Struct):
    _fields_ = [
        ("num_resolutions", C.c_int32), ("select_valid_normals_direction", C.c_int32),
        ("max_frames_to_keep", C.c_int32), ("_pad0", C.c_int32),
        ("default_radius", C.c_double),
        ("resolutions", ResolutionParam * CTICP_MAX_RESOLUTIONS),
        ("capacity_voxels", C.c_uint64),
    ]


STRATEGY = {"NEAREST_NEIGHBOR_STRATEGY": 0, "DISTANCE_BASED_STRATEGY": 1}


class StrategyOptions(_Struct):
    _fields_ = [("type", C.c_int32), ("max_num_neighbors", C.c_int32), ("min_num_neighbors", C.c_int32),
                ("_pad0", C.c_int32), ("distance_max", C.c_double), ("radius_min", C.c_double),
                ("radius_max", C.c_double), ("exponent", C.c_double)]

    def __init__(self, type=0, max_num_neighbors=20, min_num_neighbors=8, _pad0=0, distance_max=60.0, radius_min=0.1,
                 radius_max=2.0, exponent=1.0):
        super().__init__(type, max_num_neighbors, min_num_neighbors, _pad0, distance_max, radius_min, radius_max, exponent)


class MotionModelOptions(_Struct):
    _fields_ = [
        ("model", C.c_int32), ("log_if_invalid", C.c_int32),
        ("beta_location_consistency", C.c_double), ("beta_constant_velocity", C.c_double),
        ("beta_small_velocity", C.c_double), ("beta_orientation_consistency", C.c_double),
        ("threshold_orientation_deg", C.c_double), ("threshold_translation_diff", C.c_double),
    ]


class AdaptiveOptions(_Struct):
    _fields_ = [("num_points_per_voxel", C.c_int32), ("max_num_points", C.c_int32), ("num_bands", C.c_int32),
                ("_pad0", C.c_int32), ("distance", C.c_double * 8), ("voxel_size", C.c_double * 8)]


# sensor_msgs/PointField datatype codes (cticp.h CTICP_DTYPE_*)
DTYPE = {"int8": 1, "uint8": 2, "int16": 3, "uint16": 4, "int32": 5, "uint32": 6, "float32": 7, "float64": 8}


class CloudView(_Struct):
    _fields_ = [("data", C.c_void_p), ("num_points", C.c_uint64), ("point_step", C.c_uint32),
                ("xyz_offset", C.c_uint32), ("xyz_dtype", C.c_int32), ("t_offset", C.c_uint32),
                ("t_dtype", C.c_int32), ("_pad0", C.c_int32)]


class CloudSink(_Struct):
    _fields_ = [("data", C.c_void_p), ("capacity_points", C.c_uint64), ("point_step", C.c_uint32),
                ("xyz_offset", C.c_uint32), ("xyz_dtype", C.c_int32), ("t_offset", C.c_uint32),
                ("t_dtype", C.c_int32), ("world", C.c_int32)]


class DeviceScan(_Struct):   # cticp_device_scan: a scan in device memory (cticp_odometry_register_device)
    _fields_ = [("xyz", C.c_void_p), ("xyz_stride_bytes", C.c_uint64), ("t", C.c_void_p), ("t_stride_bytes", C.c_uint64),
                ("num_points", C.c_uint64), ("xyz_dtype", C.c_int32), ("t_dtype", C.c_int32)]


class SyntheticFrame(_Struct):   # cticp_synthetic_frame: one SyntheticSensorAcquisition::GenerateFrame call
    _fields_ = [("begin_ts", C.c_double), ("end_ts", C.c_double), ("frame_id", C.c_uint32), ("_pad0", C.c_uint32)]


def synthetic_frame_dtype():
    import numpy as np
    return np.dtype({"names": ["begin_ts", "end_ts", "frame_id"], "formats": [np.float64, np.float64, np.uint32],
                     "offsets": [0, 8, 16], "itemsize": C.sizeof(SyntheticFrame)})


class LidarSensor(_Struct):   # cticp_lidar_sensor: a spinning LiDAR (ring elevations in host memory)
    _fields_ = [("elevations_deg", C.c_void_p), ("n_rings", C.c_uint32), ("n_azimuth", C.c_uint32),
                ("period", C.c_double), ("min_range", C.c_double), ("max_range", C.c_double),
                ("noise_sigma", C.c_double)]


class LidarFrame(_Struct):   # cticp_lidar_frame: one sweep
    _fields_ = [("t0", C.c_double), ("frame_id", C.c_uint32), ("_pad0", C.c_uint32)]


class NcltFrame(_Struct):   # cticp_nclt_frame: one frame of an NCLT velodyne_hits.bin stream
    _fields_ = [("num_points", C.c_uint64), ("t_first", C.c_double), ("t_max", C.c_double)]


def nclt_frame_dtype():
    import numpy as np
    return np.dtype([("num_points", "<u8"), ("t_first", "<f8"), ("t_max", "<f8")])


class PlyLayout(_Struct):   # cticp_ply_layout: the vertex records of a binary_little_endian PLY file
    _fields_ = [("body_offset", C.c_uint64), ("num_points", C.c_uint64), ("point_step", C.c_uint32),
                ("xyz_offset", C.c_uint32), ("xyz_dtype", C.c_int32), ("t_offset", C.c_uint32), ("t_dtype", C.c_int32),
                ("_pad0", C.c_int32)]


# source types of a PLY column (cticp.h CTICP_DTYPE_INT64 / _UINT64 are valid there only)
PLY_SRC_DTYPE = dict(DTYPE, int64=9, uint64=10)
# PLY property type names (tinyply's), by CTICP_DTYPE_*
PLY_TYPE_NAME = {1: "char", 2: "uchar", 3: "short", 4: "ushort", 5: "int", 6: "uint", 7: "float", 8: "double"}


class PlyProperty(_Struct):   # cticp_ply_property: one PLY property as a strided column of scalars
    _fields_ = [("element", C.c_char_p), ("name", C.c_char_p), ("ply_dtype", C.c_int32), ("src_dtype", C.c_int32),
                ("src", C.c_void_p), ("src_stride_bytes", C.c_uint64)]


# CTICP_DATASET_*:the reference's ct_icp::DATASET values (include/ct_icp/dataset.h)
DATASET = {"KITTI_raw": 0, "KITTI_CARLA": 1, "KITTI": 2, "KITTI_360": 3, "NCLT": 4, "HILTI_2021": 5, "HILTI_2022": 6}


def lidar_frame_dtype():
    import numpy as np
    return np.dtype({"names": ["t0", "frame_id"], "formats": [np.float64, np.uint32], "offsets": [0, 8],
                     "itemsize": C.sizeof(LidarFrame)})


SYN = {"TRIANGLE": 0, "LINE": 1, "SPHERE": 2, "BALL": 3}   # CTICP_SYN_*: primitive kinds, in generation order


class OdometryOptions(_Struct):
    _fields_ = [
        ("ct_icp_options", IcpOptions), ("map_options", MapOptions),
        ("neighborhood_strategy", StrategyOptions), ("default_motion_model", MotionModelOptions),
        ("motion_compensation", C.c_int32), ("initialization", C.c_int32), ("init_num_frames", C.c_int32),
        ("max_num_keypoints", C.c_int32), ("sampling", C.c_int32), ("quit_on_error", C.c_int32),
        ("robust_minimal_level", C.c_int32), ("robust_registration", C.c_int32), ("robust_fail_early", C.c_int32),
        ("robust_num_attempts", C.c_int32), ("robust_num_attempts_when_rotation", C.c_int32),
        ("robust_max_voxel_neighborhood", C.c_int32), ("always_insert", C.c_int32), ("do_no_insert", C.c_int32),
        ("debug_print", C.c_int32), ("with_default_motion_model", C.c_int32),
        ("init_voxel_size", C.c_double), ("init_sample_voxel_size", C.c_double), ("sample_voxel_size", C.c_double),
        ("voxel_size", C.c_double), ("max_distance", C.c_double), ("distance_error_threshold", C.c_double),
        ("orientation_error_threshold", C.c_double), ("robust_full_voxel_threshold", C.c_double),
        ("robust_empty_voxel_threshold", C.c_double), ("robust_neighborhood_min_dist", C.c_double),
        ("robust_neighborhood_min_orientation", C.c_double), ("robust_relative_trans_threshold", C.c_double),
        ("robust_threshold_ego_orientation", C.c_double), ("robust_threshold_relative_orientation", C.c_double),
        ("insertion_ego_rotation_threshold", C.c_double), ("insertion_threshold_frames_skipped", C.c_double),
        ("insertion_cum_distance_threshold", C.c_double), ("insertion_cum_orientation_threshold", C.c_double),
        ("shuffle_seed", C.c_uint64), ("max_points_per_frame", C.c_uint64),
        ("adaptive_options", AdaptiveOptions),
    ]


class Pose(_Struct):
    _fields_ = [("quat", C.c_double * 4), ("tr", C.c_double * 3), ("ref_timestamp", C.c_double),
                ("dest_timestamp", C.c_double), ("ref_frame_id", C.c_uint32), ("dest_frame_id", C.c_uint32)]

    @staticmethod
    def make(quat=(0, 0, 0, 1), tr=(0, 0, 0), dest_timestamp=-1.0, dest_frame_id=0xFFFFFFFF):
        p = Pose()
        p.quat[:] = quat
        p.tr[:] = tr
        p.ref_timestamp = 0.0
        p.dest_timestamp = dest_timestamp
        p.ref_frame_id = 0
        p.dest_frame_id = dest_frame_id
        return p


class Frame(_Struct):
    _fields_ = [("begin_pose", Pose), ("end_pose", Pose)]


class MotionPrior(_Struct):   # cticp_motion_prior: the AMotionModel* argument of RegisterFrame (a PreviousFrameMotionModel)
    _fields_ = [("options", MotionModelOptions), ("previous_frame", Frame)]


class WPoint(_Struct):
    _fields_ = [("raw", C.c_double * 3), ("timestamp", C.c_double), ("world", C.c_double * 3),
                ("index_frame", C.c_uint32), ("_pad0", C.c_uint32)]


class IcpSummary(_Struct):
    _fields_ = [("success", C.c_int32), ("num_residuals_used", C.c_int32), ("num_iters", C.c_int32),
                ("_pad0", C.c_int32), ("duration_total", C.c_double), ("duration_init", C.c_double),
                ("avg_duration_iter", C.c_double), ("avg_duration_neighborhood", C.c_double),
                ("avg_duration_solve", C.c_double)]


class Summary(_Struct):
    _fields_ = [
        ("frame", Frame), ("initial_frame", Frame), ("icp_summary", IcpSummary),
        ("sample_size", C.c_int32), ("number_of_residuals", C.c_int32), ("robust_level", C.c_int32),
        ("success", C.c_int32), ("points_added", C.c_int32), ("number_of_attempts", C.c_int32),
        ("distance_correction", C.c_double), ("relative_distance", C.c_double),
        ("relative_orientation", C.c_double), ("ego_orientation", C.c_double),
        ("num_corrected_points", C.c_uint64), ("num_all_corrected_points", C.c_uint64),
        ("num_keypoints", C.c_uint64),
        ("odometry_total", C.c_double), ("odometry_initialization", C.c_double),
        ("odometry_try_register", C.c_double), ("odometry_duration_sampling", C.c_double),
        ("odometry_map_update", C.c_double), ("odometry_transform", C.c_double),
        ("error_message", C.c_char * 256),
    ]


class DeviceTiming(_Struct):
    _fields_ = [
        ("total_ms", C.c_double), ("ingest_ms", C.c_double), ("icp_ms", C.c_double), ("gather_ms", C.c_double),
        ("map_update_ms", C.c_double), ("icp_iterations", C.c_int32), ("kernel_launches", C.c_int32),
        ("gather_keypoint_iterations", C.c_uint64), ("gather_stencil_points", C.c_uint64),
        ("gather_stencil_voxels", C.c_uint64), ("h2d_bytes", C.c_uint64), ("d2h_bytes", C.c_uint64),
        ("gather_launches", C.c_int32), ("icp_batch_groups", C.c_int32),
    ]


class KittiErrors(_Struct):   # cticp_kitti_errors: kitti::seq_errors without tab_errors and the runner-filled fields
    _fields_ = [("mean_rpe", C.c_double), ("mean_ape", C.c_double), ("max_ape", C.c_double),
                ("mean_local_err", C.c_double), ("max_local_err", C.c_double), ("index_max_local_err", C.c_int64)]


class TrajSegment(_Struct):   # cticp_traj_segment: slam::segment_t of a counted segment and its loc error
    _fields_ = [("segment_length", C.c_double), ("start_idx", C.c_int64), ("end_idx", C.c_int64),
                ("loc_error", C.c_double), ("quat", C.c_double * 4), ("tr", C.c_double * 3)]


class TrajMetrics(_Struct):   # cticp_traj_metrics: slam::metrics_t without the vectors
    _fields_ = [("total_distance", C.c_double), ("mean_ate", C.c_double), ("max_ate", C.c_double),
                ("max_ate_idx", C.c_int64), ("segment_mean_ate", C.c_double), ("segment_mean_ate_ratio", C.c_double),
                ("num_segments", C.c_int64), ("quat", C.c_double * 4), ("tr", C.c_double * 3)]


class GridSamplingOptions(_Struct):   # cticp_grid_sampling_options: slam::GridSamplingOptions
    _fields_ = [("grid_size", C.c_double), ("num_points_per_voxel", C.c_int32), ("_pad0", C.c_int32),
                ("max_num_points", C.c_int64)]


class WorldCloudStats(_Struct):   # cticp_world_cloud_stats: what one add of a world cloud did
    _fields_ = [("submitted", C.c_uint64), ("kept", C.c_uint64), ("rejected", C.c_uint64), ("new_voxels", C.c_uint64)]


class NeighborhoodDescription(_Struct):   # cticp_neighborhood_description: slam::NeighborhoodDescription<double>
    _fields_ = [("planarity", C.c_double), ("linearity", C.c_double), ("a2D", C.c_double), ("cov_det", C.c_double),
                ("line", C.c_double * 3), ("normal", C.c_double * 3), ("barycenter", C.c_double * 3),
                ("covariance", C.c_double * 6), ("is_valid", C.c_int32), ("type", C.c_int32)]


def neighborhood_description_dtype():
    """NumPy view of cticp_neighborhood_description (160 bytes)"""
    import numpy as np
    return np.dtype([("planarity", "f8"), ("linearity", "f8"), ("a2D", "f8"), ("cov_det", "f8"), ("line", "f8", 3),
                     ("normal", "f8", 3), ("barycenter", "f8", 3), ("covariance", "f8", 6), ("is_valid", "i4"),
                     ("type", "i4")])


# slam::NEIGHBORHOOD_PROPERTIES and slam::NEIGHBORHOOD_TYPE (neighborhood.h), the reference's values
NB = {"NO_VALUES": 0, "LINE": 1, "NORMAL": 2, "PLANARITY": 4, "LINEARITY": 8, "COV_DET": 16, "KDTREE": 32, "A2D": 64,
      "ALL": 127, "ALL_BUT_KDTREE": 95}
NB_TYPE = {"NONE": 0, "LINEAR": 1, "PLANAR": 2, "VOLUMIC": 3}


KITTI_LENGTHS = {"driving": (100., 200., 300., 400., 500., 600., 700., 800.),   # eval.h kitti_segment_lengths
                 "indoor": (10., 20., 30., 40., 50., 60., 70., 80.)}            # eval.h indoor_segment_lengths


# cticp_batch_frame kinds
BATCH_HOST, BATCH_DEVICE, BATCH_STAGED = 0, 1, 2


class BatchFrame(_Struct):   # cticp_batch_frame: one item of cticp_odometry_register_batch
    _fields_ = [("handle", C.c_void_p), ("kind", C.c_int32), ("frame_id", C.c_uint32),
                ("xyz", C.c_void_p), ("xyz_stride_bytes", C.c_size_t), ("t", C.c_void_p), ("t_stride_bytes", C.c_size_t),
                ("n", C.c_size_t), ("device_scan", C.c_void_p), ("stream", C.c_void_p), ("staged_slot", C.c_int64),
                ("initial_estimate", C.c_void_p), ("motion_model", C.c_void_p), ("out", C.c_void_p),
                ("status", C.c_int32), ("_pad0", C.c_int32)]


# numpy dtype of cticp_wpoint (64 bytes, same as slam::WPoint3D)
def wpoint_dtype():
    import numpy as np
    return np.dtype([("raw", "<f8", 3), ("timestamp", "<f8"), ("world", "<f8", 3), ("index_frame", "<u4"),
                     ("_pad0", "<u4")])


# numpy dtype of cticp_pose (72 bytes): the output of ContinuousTrajectory.interpolate
def pose_dtype():
    import numpy as np
    return np.dtype([("quat", "<f8", 4), ("tr", "<f8", 3), ("ref_timestamp", "<f8"), ("dest_timestamp", "<f8"),
                     ("ref_frame_id", "<u4"), ("dest_frame_id", "<u4")])


# numpy dtype of cticp_traj_segment (88 bytes): the segments of Binding.trajectory_metrics
def traj_segment_dtype():
    import numpy as np
    return np.dtype([("segment_length", "<f8"), ("start_idx", "<i8"), ("end_idx", "<i8"), ("loc_error", "<f8"),
                     ("quat", "<f8", 4), ("tr", "<f8", 3)])


def frame_to_arrays(frame):
    """cticp_frame → (begin_quat, begin_tr, end_quat, end_tr) as python lists."""
    return (list(frame.begin_pose.quat), list(frame.begin_pose.tr), list(frame.end_pose.quat),
            list(frame.end_pose.tr))
