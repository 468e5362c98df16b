"""Thin ctypes binding over a shared library that implements the include/cticp.h entry points.

`Binding(lib, prefix)` works for any library exporting `<prefix>odometry_create`, ... — the engine uses
prefix "cticp_"; the test-suite binds the CPU oracle (prefix "orc_") through the same class so both are
driven by identical calls. Nothing in this module computes anything: it marshals numpy arrays and PODs.
"""
import ctypes as C
import math

import numpy as np

from . import _abi as abi


class CticpError(RuntimeError):
    def __init__(self, code, message, statuses=None):
        super().__init__(f"[{code}] {message}")
        self.code = code
        self.statuses = statuses   # register_batch: every item's status (0 = registered)


def _is_cuda_tensor(a):
    """A torch CUDA tensor, recognised without importing torch."""
    return type(a).__module__.split(".")[0] == "torch" and bool(getattr(a, "is_cuda", False))


def _torch_dtype_codes(torch):
    codes = {torch.int8: 1, torch.uint8: 2, torch.int16: 3, torch.int32: 5, torch.float32: 7, torch.float64: 8}
    for name, code in (("uint16", 4), ("uint32", 6)):
        if hasattr(torch, name):
            codes[getattr(torch, name)] = code
    return codes


def _as_f64_rows(a, cols):
    a = np.ascontiguousarray(a, dtype=np.float64)
    if a.ndim != 2 or a.shape[1] != cols:
        raise ValueError(f"expected an (n, {cols}) array, got {a.shape}")
    return a


def _pose_array(poses):
    """a contiguous array of abi.pose_dtype() from abi.Pose items or such an array"""
    if isinstance(poses, np.ndarray):
        if poses.dtype != abi.pose_dtype():
            raise TypeError("expected an array of abi.pose_dtype()")
        return np.ascontiguousarray(poses.reshape(-1))
    out = np.zeros(len(poses), dtype=abi.pose_dtype())
    for i, p in enumerate(poses):
        if not isinstance(p, abi.Pose):
            raise TypeError("expected abi.Pose items, got %r" % type(p))
        C.memmove(out.ctypes.data + i * out.itemsize, C.addressof(p), C.sizeof(abi.Pose))
    return out


def _estimates_array(estimates, n):
    """(B × n poses, B, single): one estimate (a pose list or array) or a list of them; each must have n poses"""
    single = isinstance(estimates, np.ndarray) or (len(estimates) > 0 and isinstance(estimates[0], abi.Pose))
    ests = [_pose_array(estimates)] if single else [_pose_array(e) for e in estimates]
    if not ests:
        raise CticpError(abi.ERR_INVALID_ARGUMENT, "no estimates")
    for e in ests:
        if len(e) != n:
            raise CticpError(abi.ERR_INVALID_ARGUMENT, "an estimate has %d poses, the ground truth %d" % (len(e), n))
    return np.concatenate(ests), len(ests), single


def _lengths(lengths):
    if isinstance(lengths, str):
        lengths = abi.KITTI_LENGTHS[lengths]
    return np.ascontiguousarray(lengths, dtype=np.float64).reshape(-1)


def _kitti_dict(e, tab):
    d = {name: getattr(e, name) for name, _ in abi.KittiErrors._fields_}
    d["tab_errors"] = np.array(tab)
    return d


def _metrics_dict(m, segs):
    d = {name: getattr(m, name) for name, _ in abi.TrajMetrics._fields_ if name not in ("quat", "tr")}
    d["quat"], d["tr"] = np.array(m.quat[:]), np.array(m.tr[:])
    d["segments"] = np.array(segs)
    return d


_SNAPSHOT_HEADER_BYTES = 72   # snapshot_format.h kHeaderBytes


def _pose_of_spec(p):
    """slam::ReadPosesFromYAML of one pose: the quaternion (x, y, z, w) normalised as Eigen does, dest_frame_id also
    setting dest_timestamp, dest_timestamp overriding it"""
    q = [float(v) for v in p.get("quaternion", (0.0, 0.0, 0.0, 1.0))]
    if "quaternion" in p:
        nrm = math.sqrt(((q[0] * q[0] + q[1] * q[1]) + q[2] * q[2]) + q[3] * q[3])
        q = [v / nrm for v in q]
    pose = abi.Pose.make(q, [float(v) for v in p.get("translation", (0.0, 0.0, 0.0))])
    if "dest_frame_id" in p:
        pose.dest_frame_id = int(p["dest_frame_id"])
        pose.dest_timestamp = float(pose.dest_frame_id)
    if "dest_timestamp" in p:
        pose.dest_timestamp = float(p["dest_timestamp"])
    return pose


def _qrot(q, v):   # Eigen _transformVector: uv = 2 (q.vec x v); v + w uv + q.vec x uv
    x, y, z, w = q
    uv = (y * v[2] - z * v[1], z * v[0] - x * v[2], x * v[1] - y * v[0])
    uv = (uv[0] + uv[0], uv[1] + uv[1], uv[2] + uv[2])
    c = (y * uv[2] - z * uv[1], z * uv[0] - x * uv[2], x * uv[1] - y * uv[0])
    return [v[i] + w * uv[i] + c[i] for i in range(3)]


def _qnormalized(q):
    nrm = math.sqrt(((q[0] * q[0] + q[1] * q[1]) + q[2] * q[2]) + q[3] * q[3])
    return [v / nrm for v in q]


def _se3_inverse(q, t):   # slam::TSE3::Inverse: quat.inverse(), tr = -(quat.inverse() * tr)
    q = [float(v) for v in q]
    n2 = ((q[0] * q[0] + q[1] * q[1]) + q[2] * q[2]) + q[3] * q[3]
    qi = [-q[0] / n2, -q[1] / n2, -q[2] / n2, q[3] / n2]
    return qi, [-v for v in _qrot(qi, [float(v) for v in t])]


def _se3_mul(a, b):   # slam::TSE3::operator*: normalised product, quat.normalized() * rhs.tr + tr
    (ax, ay, az, aw), at = a
    (bx, by, bz, bw), bt = [float(v) for v in b[0]], [float(v) for v in b[1]]
    q = [aw * bx + ax * bw + ay * bz - az * by, aw * by + ay * bw + az * bx - ax * bz,
         aw * bz + az * bw + ax * by - ay * bx, aw * bw - ax * bx - ay * by - az * bz]
    r = _qrot(_qnormalized(a[0]), bt)
    return _qnormalized(q), [r[i] + at[i] for i in range(3)]


def _snapshot_bytes(binding, fn, handle):
    n = binding.check(binding.fn(fn)(handle, None, 0))
    buf = C.create_string_buffer(n)
    m = binding.check(binding.fn(fn)(handle, buf, n))
    assert m == n, (m, n)
    return buf.raw


def _ply_code(t):
    """a PLY property type: a CTICP_DTYPE_* code, a tinyply name or a NumPy dtype name"""
    if isinstance(t, (int, np.integer)):
        return int(t)
    names = {v: k for k, v in abi.PLY_TYPE_NAME.items()}
    return names[t] if t in names else abi.DTYPE[np.dtype(t).name]


def _ply_src_code(name):
    if name not in abi.PLY_SRC_DTYPE:
        raise ValueError("no PLY source type for %s" % name)
    return abi.PLY_SRC_DTYPE[name]


def _ply_num_items(shapes, num_items):
    lengths = {s[0] for s in shapes if len(s) == 1}
    if num_items is None:
        if len(lengths) > 1:
            raise ValueError("the columns have different lengths %s" % sorted(lengths))
        return lengths.pop() if lengths else 1
    if any(length < num_items for length in lengths):
        raise ValueError("a column is shorter than num_items")
    return int(num_items)


def _ply_props(cols, src_codes, sources):
    """a cticp_ply_property array (and the encoded names it points to) from (element, name, ply_dtype, _) columns and
    (pointer, stride) sources"""
    props = (abi.PlyProperty * len(cols))()
    keep = []
    for i, ((elem, name, ply, _), code, (ptr, stride)) in enumerate(zip(cols, src_codes, sources)):
        e, nm = elem.encode(), name.encode()
        keep += [e, nm]
        props[i] = abi.PlyProperty(e, nm, _ply_code(ply), code, ptr, stride)
    return props, keep


def _pose_columns(arr):
    """SavePosesAsPLY's eleven columns: strided views of a cticp_pose array, whose records are the file's records"""
    cols = [("pose", nm, "double", arr["quat"][:, i]) for i, nm in enumerate(["qx", "qy", "qz", "qw"])]
    cols += [("pose", nm, "double", arr["tr"][:, i]) for i, nm in enumerate(["x", "y", "z"])]
    cols += [("pose", "ref_t", "double", arr["ref_timestamp"]), ("pose", "dest_t", "double", arr["dest_timestamp"]),
             ("pose", "ref_fid", "int", arr["ref_frame_id"]), ("pose", "dest_fid", "int", arr["dest_frame_id"])]
    return cols


class Binding:
    def __init__(self, lib, prefix):
        self.lib = lib
        self.prefix = prefix
        self._declare()

    # ------------------------------------------------------------------------------------------------------
    def fn(self, name):
        return getattr(self.lib, self.prefix + name)

    def has(self, name):
        return hasattr(self.lib, self.prefix + name)

    def _declare(self):
        P = C.POINTER
        vp, i32, i64, u32, u64, dbl, sz = C.c_void_p, C.c_int32, C.c_int64, C.c_uint32, C.c_uint64, C.c_double, C.c_size_t
        sigs = {
            "last_error": (C.c_char_p, []),
            "default_icp_options": (None, [P(abi.IcpOptions)]),
            "default_map_options": (None, [P(abi.MapOptions)]),
            "default_odometry_options": (None, [P(abi.OdometryOptions)]),
            "legacy_map_options": (None, [P(abi.MapOptions), dbl, C.c_int, dbl]),
            "profile_default_driving": (None, [P(abi.OdometryOptions)]),
            "profile_robust_driving": (None, [P(abi.OdometryOptions)]),
            "profile_robust_outdoor_low_inertia": (None, [P(abi.OdometryOptions)]),
            "odometry_create": (C.c_int, [P(abi.OdometryOptions), C.c_int, P(vp)]),
            "odometry_destroy": (None, [vp]),
            "odometry_register_frame": (C.c_int, [vp, vp, sz, vp, sz, sz, u32, P(abi.Frame), P(abi.Summary)]),
            "odometry_get_points": (i64, [vp, C.c_int, vp, sz]),
            "odometry_trajectory": (i64, [vp, P(abi.Frame), sz]),
            "odometry_map_size": (i64, [vp]),
            "odometry_reset": (C.c_int, [vp]),
            "odometry_map": (vp, [vp]),
            "map_create": (C.c_int, [P(abi.MapOptions), C.c_int, P(vp)]),
            "map_destroy": (None, [vp]),
            "map_insert": (C.c_int, [vp, vp, sz, sz]),
            "map_insert_from": (C.c_int, [vp, vp, sz, sz, vp]),
            "map_radius_search": (C.c_int, [vp, vp, vp, sz, C.c_int, vp, vp, vp]),
            "map_remove_far": (C.c_int, [vp, P(dbl), dbl]),
            "map_num_points": (i64, [vp, C.c_int]),
            "map_num_voxels": (i64, [vp, C.c_int]),
            "map_export": (i64, [vp, C.c_int, vp, vp, sz]),
            "map_compute_neighborhoods": (C.c_int, [vp, vp, sz, C.c_int, vp, vp]),
            "map_clear": (C.c_int, [vp]),
            "icp_register": (C.c_int, [vp, P(abi.IcpOptions), P(abi.StrategyOptions), vp, sz, P(abi.Frame),
                                       P(abi.Frame), P(abi.MotionModelOptions), P(abi.IcpSummary)]),
            "icp_register_batch": (C.c_int, [vp, P(abi.IcpOptions), sz, P(vp), P(sz), P(abi.Frame), P(vp),
                                             P(abi.MotionModelOptions), P(abi.IcpSummary)]),
            "icp_register_batch_ex": (C.c_int, [vp, P(abi.IcpOptions), P(abi.StrategyOptions), sz, P(vp), P(sz),
                                                P(abi.Frame), P(vp), P(abi.MotionModelOptions), P(abi.IcpSummary)]),
            "icp_gn_normal_equations": (C.c_int, [vp, P(abi.IcpOptions), vp, sz, P(abi.Frame), P(abi.Frame),
                                                  P(abi.MotionModelOptions), vp, vp, P(i32)]),
            "grid_sample_indices": (i64, [C.c_int, vp, sz, sz, dbl, vp, sz]),
            "permutation": (C.c_int, [u64, u64, u32, vp]),
            "adaptive_sample_indices": (i64, [C.c_int, P(abi.AdaptiveOptions), vp, sz, sz, vp, sz]),
            "default_adaptive_options": (None, [P(abi.AdaptiveOptions)]),
            # engine only
            "abi_version": (u32, []),
            "abi_sizeof": (sz, [C.c_char_p]),
            "odometry_map_points": (i64, [vp, vp, sz]),
            "odometry_last_timing": (C.c_int, [vp, P(abi.DeviceTiming)]),
            "nccl_unique_id": (C.c_int, [vp]),
            "odometry_stage_frame": (i64, [vp, vp, sz, vp, sz, sz]),
            "odometry_register_cloud": (C.c_int, [vp, P(abi.CloudView), u32, P(abi.Frame), P(abi.Summary)]),
            "odometry_stage_cloud": (i64, [vp, P(abi.CloudView)]),
            "odometry_write_points": (i64, [vp, C.c_int, P(abi.CloudSink)]),
            "odometry_register_device": (C.c_int, [vp, P(abi.DeviceScan), vp, u32, P(abi.Frame), P(abi.MotionPrior),
                                                   P(abi.Summary)]),
            "odometry_write_points_device": (i64, [vp, C.c_int, P(abi.CloudSink), vp]),
            "odometry_register_staged": (C.c_int, [vp, i64, u32, P(abi.Summary)]),
            "odometry_clear_staged": (C.c_int, [vp]),
            "odometry_register_batch": (C.c_int, [P(abi.BatchFrame), sz]),
            "odometry_timer_start": (C.c_int, [vp]),
            "odometry_timer_stop": (C.c_int, [vp, P(dbl)]),
            "odometry_flush_l2": (C.c_int, [vp, sz]),
            "odometry_set_gather_timing": (C.c_int, [vp, C.c_int]),
            "odometry_set_summary_points": (C.c_int, [vp, C.c_int]),
            "odometry_register_frame_ex": (C.c_int, [vp, vp, sz, vp, sz, sz, u32, P(abi.Frame), P(abi.MotionPrior), P(abi.Summary)]),
            "odometry_set_callback": (C.c_int, [vp, abi.EVENT_FN, vp]),
            "odometry_reset_options": (C.c_int, [vp, P(abi.OdometryOptions)]),
            "odometry_enable_sharding": (C.c_int, [vp, vp, C.c_int, C.c_int]),
            "odometry_sharding_mode": (C.c_int, [vp]),
            "odometry_save": (i64, [vp, vp, sz]),
            "odometry_load": (C.c_int, [vp, sz, P(abi.OdometryOptions), C.c_int, P(vp)]),
            "odometry_clone": (C.c_int, [vp, C.c_int, P(vp)]),
            "map_save": (i64, [vp, vp, sz]),
            "map_load": (C.c_int, [vp, sz, C.c_int, P(vp)]),
            "trajectory_create": (C.c_int, [vp, sz, C.c_int, P(vp)]),
            "trajectory_destroy": (None, [vp]),
            "trajectory_poses": (i64, [vp, vp, sz]),
            "trajectory_interpolate": (C.c_int, [vp, vp, vp, sz, vp]),
            "trajectory_transform": (i64, [vp, P(abi.CloudView), vp, vp, sz, P(abi.CloudSink)]),
            "trajectory_transform_device": (i64, [vp, P(abi.DeviceScan), vp, vp, sz, P(abi.CloudSink), vp]),
            "kitti_evaluate": (i64, [C.c_int, vp, sz, vp, sz, vp, sz, vp, vp, sz]),
            "trajectory_kitti_evaluate": (i64, [vp, vp, sz, vp, sz, vp, vp, sz]),
            "trajectory_metrics": (i64, [C.c_int, vp, sz, vp, sz, dbl, vp, vp, sz]),
            "trajectory_distances": (C.c_int, [C.c_int, vp, sz, C.c_int, vp]),
            "default_grid_sampling_options": (None, [P(abi.GridSamplingOptions)]),
            "sample_points_in_grid": (i64, [C.c_int, P(abi.GridSamplingOptions), vp, sz, sz, vp, sz]),
            "world_cloud_create": (C.c_int, [P(abi.GridSamplingOptions), u64, u64, C.c_int, P(vp)]),
            "world_cloud_destroy": (None, [vp]),
            "world_cloud_add": (C.c_int, [vp, vp, P(abi.CloudView), vp, vp, sz, P(abi.WorldCloudStats)]),
            "world_cloud_add_device": (C.c_int, [vp, vp, P(abi.DeviceScan), vp, vp, sz, P(abi.WorldCloudStats), vp]),
            "world_cloud_add_odometry": (C.c_int, [vp, vp, P(abi.WorldCloudStats)]),
            "world_cloud_num_points": (i64, [vp]),
            "world_cloud_num_voxels": (i64, [vp]),
            "world_cloud_export": (i64, [vp, P(abi.CloudSink), vp]),
            "world_cloud_export_device": (i64, [vp, P(abi.CloudSink), vp, vp]),
            "world_cloud_clear": (C.c_int, [vp]),
            # oracle only (KAT taps)
            "odometry_last_counters": (None, [vp, P(u64), P(u64)]),
            "neighborhood_describe": (C.c_int, [vp, sz, vp, P(dbl), P(dbl), P(dbl), vp]),
            "pose_transform": (C.c_int, [P(abi.Frame), P(dbl), dbl, P(dbl)]),
            "se3_inverse": (None, [vp, vp, vp, vp]),
            "se3_mul": (None, [vp, vp, vp, vp, vp, vp]),
            "angular_distance": (dbl, [vp, vp]),
            "se3_interpolate": (None, [vp, vp, vp, vp, dbl, vp, vp]),
            "se3_apply": (None, [vp, vp, vp, vp]),
            "ct_point_to_plane_residual": (dbl, [dbl, vp, vp, vp, dbl, vp, vp, vp, vp, vp]),
            "ct_residual": (dbl, [C.c_int, dbl, vp, vp, vp, vp, dbl, vp, vp, vp, vp, vp]),
            "loss_evaluate": (None, [P(abi.IcpOptions), dbl, vp]),
            "corrector": (None, [dbl, vp, P(dbl), P(dbl)]),
            "quat_plus": (None, [vp, vp, vp]),
            "lm_solve_plane_blocks": (None, [P(abi.IcpOptions), C.c_int, vp, vp, vp, vp, vp, vp, vp]),
            "quat_from_matrix": (None, [vp, vp]),
            "quat_to_matrix": (None, [vp, vp]),
            "symmetric_svd3": (None, [vp, vp, vp]),
            "ldlt_solve12": (None, [vp, vp, vp]),
        }
        if self.prefix == "cticp_":
            # the engine's cticp_neighborhood_describe is the index's; the oracle's orc_neighborhood_describe (above) is
            # the KAT tap of the GN gather
            sigs["neighborhood_describe"] = (C.c_int, [vp, vp, sz, C.c_int, dbl, C.c_int, dbl, dbl, vp])
        sigs.update({
            "neighborhood_describe_sets": (C.c_int, [C.c_int, vp, sz, sz, vp, sz, C.c_int, dbl, dbl, vp]),
            "neighborhood_create": (C.c_int, [vp, sz, sz, C.c_int, P(vp)]),
            "neighborhood_create_device": (C.c_int, [P(abi.DeviceScan), vp, C.c_int, P(vp)]),
            "neighborhood_create_world_cloud": (C.c_int, [vp, P(vp)]),
            "neighborhood_destroy": (None, [vp]),
            "neighborhood_num_points": (i64, [vp]),
            "neighborhood_num_rejected": (i64, [vp]),
            "neighborhood_search": (C.c_int, [vp, vp, sz, C.c_int, dbl, vp, vp, vp]),
            "neighborhood_search_device": (C.c_int, [vp, vp, sz, C.c_int, dbl, vp, vp, vp, vp]),
            "neighborhood_describe_device": (C.c_int, [vp, vp, sz, C.c_int, dbl, C.c_int, dbl, dbl, vp, vp]),
            "synthetic_scene_create": (C.c_int, [vp, sz, vp, sz, vp, sz, vp, sz, C.c_int, P(vp)]),
            "synthetic_scene_destroy": (None, [vp]),
            "synthetic_scene_num_primitives": (i64, [vp]),
            "synthetic_scene_distance": (C.c_int, [vp, vp, sz, vp]),
            "synthetic_generate_points": (i64, [vp, sz, vp, dbl, u64, vp, sz, vp]),
            "synthetic_generate_frames": (i64, [vp, vp, vp, sz, sz, dbl, u64, P(abi.CloudSink), vp, vp]),
            "synthetic_generate_frames_device": (C.c_int, [vp, vp, vp, sz, sz, dbl, u64, P(abi.CloudSink), vp, vp, vp]),
            "synthetic_generate_poses": (i64, [vp, dbl, vp, sz]),
            "apply_uniform_noise": (C.c_int, [vp, sz, dbl, dbl, u64]),
            "lidar_scene_create": (C.c_int, [vp, sz, vp, sz, C.c_int, C.c_int, P(vp)]),
            "lidar_scene_destroy": (None, [vp]),
            "lidar_scene_raycast": (C.c_int, [vp, vp, vp, sz, dbl, u64, vp]),
            "lidar_scene_raycast_device": (C.c_int, [vp, vp, vp, sz, dbl, u64, vp, vp]),
            "lidar_generate_sweeps": (i64, [vp, vp, P(abi.LidarSensor), vp, sz, u64, P(abi.CloudSink), vp, vp]),
            "lidar_generate_sweeps_device": (C.c_int, [vp, vp, P(abi.LidarSensor), vp, sz, u64, P(abi.CloudSink), vp, vp,
                                                        vp]),
            "nclt_open": (C.c_int, [vp, sz, u32, C.c_int, C.c_int, P(vp)]),
            "nclt_open_device": (C.c_int, [vp, sz, u32, C.c_int, C.c_int, vp, P(vp)]),
            "nclt_destroy": (None, [vp]),
            "nclt_num_frames": (i64, [vp]),
            "nclt_num_packets": (i64, [vp]),
            "nclt_num_hits": (i64, [vp]),
            "nclt_bytes_used": (i64, [vp]),
            "nclt_index_walked": (C.c_int, [vp]),
            "nclt_frame_info": (C.c_int, [vp, sz, sz, vp]),
            "nclt_read_frames": (i64, [vp, sz, sz, P(abi.CloudSink), vp]),
            "nclt_read_frames_device": (C.c_int, [vp, sz, sz, P(abi.CloudSink), vp, vp]),
            "ply_layout_parse": (C.c_int, [vp, sz, P(abi.PlyLayout)]),
            "kitti_frame_filter": (C.c_int, [C.c_int, P(abi.CloudView), P(abi.CloudSink)]),
            "kitti_frame_filter_device": (C.c_int, [C.c_int, P(abi.DeviceScan), P(abi.CloudSink), vp]),
            "scan_time_ranges": (C.c_int, [C.c_int, P(abi.CloudView), vp, sz, vp]),
            "scan_time_ranges_device": (C.c_int, [C.c_int, P(abi.DeviceScan), vp, sz, vp, vp]),
            "ground_truth_parse": (i64, [C.c_int, C.c_int, vp, sz, vp, sz]),
            "ply_write": (i64, [C.c_int, P(abi.PlyProperty), sz, u64, vp, u64]),
            "ply_write_device": (C.c_int, [C.c_int, P(abi.PlyProperty), sz, u64, vp, sz, vp, u64, vp, vp]),
            "ply_read_poses": (i64, [vp, sz, vp, sz]),
        })
        for name, (res, args) in sigs.items():
            if self.has(name):
                f = self.fn(name)
                f.restype = res
                f.argtypes = args

    def check(self, code):
        if code < 0:
            msg = self.fn("last_error")()
            raise CticpError(code, msg.decode("utf-8", "replace") if msg else "")
        return code

    # ---- options -------------------------------------------------------------------------------------------
    def default_odometry_options(self):
        o = abi.OdometryOptions()
        self.fn("default_odometry_options")(C.byref(o))
        return o

    def default_icp_options(self):
        o = abi.IcpOptions()
        self.fn("default_icp_options")(C.byref(o))
        return o

    def default_map_options(self):
        o = abi.MapOptions()
        self.fn("default_map_options")(C.byref(o))
        return o

    def legacy_map_options(self, size_voxel_map=1.0, max_num_points_in_voxel=20, min_distance_points=0.1):
        o = abi.MapOptions()
        self.fn("legacy_map_options")(C.byref(o), size_voxel_map, max_num_points_in_voxel, min_distance_points)
        return o

    def profile(self, name):
        o = abi.OdometryOptions()
        self.fn("profile_" + name)(C.byref(o))
        return o

    # ---- factories -----------------------------------------------------------------------------------------
    def odometry(self, options, device=0):
        return Odometry(self, options, device)

    def voxel_map(self, options, device=0):
        return VoxelMap(self, options=options, device=device)

    # ---- snapshots -----------------------------------------------------------------------------------------
    def load_odometry(self, blob, options=None, device=0):
        """A new Odometry on `device` from the bytes of Odometry.save() (cticp_odometry_load). options None: the saved
        options, and every later frame registers exactly as on the saved handle; otherwise options may differ from the
        saved ones only outside map_options (e.g. do_no_insert = 1 to localise against the saved map)."""
        blob = bytes(blob)
        h = C.c_void_p()
        self.check(self.fn("odometry_load")(blob, len(blob), C.byref(options) if options is not None else None, device,
                                            C.byref(h)))
        if options is None:   # the options section follows the fixed header (snapshot_format.h)
            options = abi.OdometryOptions.from_buffer_copy(blob, _SNAPSHOT_HEADER_BYTES)
        return Odometry._adopt(self, h, options, device)

    def load_voxel_map(self, blob, device=0):
        """A new standalone VoxelMap on `device` from the bytes of VoxelMap.save() (cticp_map_load)."""
        blob = bytes(blob)
        m = VoxelMap.__new__(VoxelMap)
        m.b, m._owner, m._borrowed, m._free_wrapper = self, None, False, False
        m.h = C.c_void_p()
        self.check(self.fn("map_load")(blob, len(blob), device, C.byref(m.h)))
        return m

    def continuous_trajectory(self, poses_or_frames, device=0):
        """slam::LinearContinuousTrajectory::Create (cticp_trajectory_create) of abi.Pose items, or of abi.Frame items
        (each contributes its begin and end pose, e.g. Odometry.Trajectory())."""
        return ContinuousTrajectory(self, poses_or_frames, device)

    # ---- scoring against ground truth ----------------------------------------------------------------------
    def kitti_evaluate(self, gt, estimates, lengths="driving", device=0):
        """kitti::EvaluatePoses (cticp_kitti_evaluate) of one estimate or of a list of estimates against the ground truth
        `gt`. Poses: lists of abi.Pose or arrays of abi.pose_dtype(). lengths: "driving", "indoor" or a sequence.
        Returns a dict (a list of dicts for a list of estimates): the seq_errors fields and tab_errors, a (count, 2)
        array of (t_err / len, r_err / len)."""
        g = _pose_array(gt)
        est, B, single = _estimates_array(estimates, len(g))
        lens = _lengths(lengths)
        cap = -(-len(g) // 10) * len(lens)   # every (first frame, length) pair kept
        out = (abi.KittiErrors * B)()
        tab = np.zeros((B, max(cap, 1), 2))
        count = self.check(self.fn("kitti_evaluate")(device, g.ctypes.data, len(g), est.ctypes.data, B, lens.ctypes.data,
                                                     len(lens), out, tab.ctypes.data, cap))
        res = [_kitti_dict(out[b], tab[b, :count]) for b in range(B)]
        return res[0] if single else res

    def trajectory_metrics(self, gt, estimates, segment_length=10.0, device=0):
        """ComputeTrajectoryMetrics (cticp_trajectory_metrics) of one estimate or of a list of estimates against the
        ground truth `gt`. Returns a dict (a list of dicts for a list of estimates): the metrics_t scalars, the global
        rigid transform (quat, tr) and `segments`, an array of abi.traj_segment_dtype() holding the counted segments."""
        g = _pose_array(gt)
        est, B, single = _estimates_array(estimates, len(g))
        cap = max((len(g) - 1) // 5, 1)   # a counted segment spans at least 5 steps
        out = (abi.TrajMetrics * B)()
        segs = np.zeros((B, cap), dtype=abi.traj_segment_dtype())
        count = self.check(self.fn("trajectory_metrics")(device, g.ctypes.data, len(g), est.ctypes.data, B,
                                                         float(segment_length), out, segs.ctypes.data, cap))
        res = [_metrics_dict(out[b], segs[b, :count]) for b in range(B)]
        return res[0] if single else res

    def trajectory_distances(self, gt, kind="kitti", device=0):
        """The distances along the ground truth that kitti_evaluate ("kitti") or trajectory_metrics ("metrics") selects
        pairs and segments with (cticp_trajectory_distances)."""
        g = _pose_array(gt)
        out = np.zeros(len(g))
        self.check(self.fn("trajectory_distances")(device, g.ctypes.data, len(g), {"kitti": 0, "metrics": 1}[kind],
                                                   out.ctypes.data))
        return out

    # ---- many handles, one frame each ------------------------------------------------------------------------
    def register_batch(self, odometries, scans, frame_ids, initial_estimates=None, motion_models=None, statuses=None):
        """One frame on each Odometry of `odometries` in one call (cticp_odometry_register_batch): the eligible
        Gauss-Newton loops run in one grouped launch, the eligible CERES / ROBUST loops in one grouped launch per LM mode
        (CERES nearest neighbour, CERES distance-based, ROBUST); the attempts of robust_registration frames run in rounds
        of such launches, apart from the plain frames; every result is that of the single-frame call.
        scans[i]: (xyz, timestamps) NumPy arrays (RegisterFrame's host path), (xyz, timestamps) torch CUDA tensors (read
        after the work queued on torch's current stream, as RegisterFrame), or an int staged slot (RegisterStaged).
        initial_estimates / motion_models: None or one entry (abi.Frame / abi.MotionPrior or None) per item.
        Returns the summaries; raises CticpError after the call when an item fails (.statuses: every item's status).
        statuses: a list that receives every item's status instead of the raise, so the items that registered keep their
        summaries (a failed item's summary is left zero; cticp_last_error() holds the first failing item's message). A
        call refused before any item ran still raises."""
        B = len(odometries)
        for name, lst in (("scans", scans), ("frame_ids", frame_ids), ("initial_estimates", initial_estimates),
                          ("motion_models", motion_models)):
            if lst is not None and len(lst) != B:
                raise ValueError(f"{name} has {len(lst)} entries for {B} odometries")
        items = (abi.BatchFrame * max(B, 1))()
        outs = [abi.Summary() for _ in range(B)]
        keep = []   # every buffer the items point to, alive until the call returns
        for i, (od, scan) in enumerate(zip(odometries, scans)):
            it = items[i]
            it.handle = od.h.value if od.h else None
            it.frame_id = int(frame_ids[i])
            it.staged_slot = -1
            if isinstance(scan, (int, np.integer)):
                it.kind = abi.BATCH_STAGED
                it.staged_slot = int(scan)
            else:
                xyz, ts = scan
                if _is_cuda_tensor(xyz) or _is_cuda_tensor(ts):
                    dscan, stream = od._device_scan(xyz, ts)
                    keep.append(dscan)
                    it.kind = abi.BATCH_DEVICE
                    it.device_scan = C.addressof(dscan)
                    it.stream = stream or None
                else:
                    xyz = np.asarray(xyz)
                    if xyz.dtype != np.float64 or xyz.ndim != 2 or xyz.shape[1] < 3 or xyz.strides[1] != 8:
                        xyz = np.ascontiguousarray(xyz[:, :3], dtype=np.float64)
                    ts = np.ascontiguousarray(ts, dtype=np.float64).reshape(-1)
                    if len(xyz) != len(ts):
                        raise ValueError("xyz and timestamps must have the same length")
                    keep += [xyz, ts]
                    it.kind = abi.BATCH_HOST
                    it.xyz, it.xyz_stride_bytes = xyz.ctypes.data, xyz.strides[0]
                    it.t, it.t_stride_bytes, it.n = ts.ctypes.data, ts.strides[0], len(xyz)
            if initial_estimates is not None and initial_estimates[i] is not None:
                it.initial_estimate = C.addressof(initial_estimates[i])
            if motion_models is not None and motion_models[i] is not None:
                it.motion_model = C.addressof(motion_models[i])
            it.out = C.addressof(outs[i])
        rc = self.fn("odometry_register_batch")(items, B)
        item_status = [items[i].status for i in range(B)]
        if rc < 0 and (statuses is None or not any(item_status)):
            msg = self.fn("last_error")()
            raise CticpError(rc, msg.decode("utf-8", "replace") if msg else "", item_status)
        if statuses is not None:
            statuses[:] = item_status
        return outs

    # ---- sampling ------------------------------------------------------------------------------------------
    def grid_sample_indices(self, xyz, voxel_size, device=0):
        xyz = _as_f64_rows(xyz, 3)
        out = np.empty(len(xyz), dtype=np.uint32)
        n = self.check(self.fn("grid_sample_indices")(device, xyz.ctypes.data, 24, len(xyz), voxel_size,
                                                       out.ctypes.data, len(out)))
        return out[:n].copy()

    def adaptive_sample_indices(self, xyz, options=None, device=0):
        xyz = _as_f64_rows(xyz, 3)
        if options is None:
            options = abi.AdaptiveOptions()
            self.fn("default_adaptive_options")(C.byref(options))
        out = np.empty(len(xyz) + 1, dtype=np.uint32)
        n = self.check(self.fn("adaptive_sample_indices")(device, C.byref(options), xyz.ctypes.data, 24, len(xyz),
                                                           out.ctypes.data, len(out)))
        return out[:n].copy()

    def grid_sampling_options(self, grid_size=1.0, num_points_per_voxel=1, max_num_points=-1):
        o = abi.GridSamplingOptions()
        self.fn("default_grid_sampling_options")(C.byref(o))
        o.grid_size, o.num_points_per_voxel, o.max_num_points = float(grid_size), int(num_points_per_voxel), int(max_num_points)
        return o

    def sample_points_in_grid(self, xyz, grid_size, num_points_per_voxel=1, max_num_points=-1, device=0):
        """slam::SamplePointsInGrid (cticp_sample_points_in_grid) of (n, 3) points: the indices kept (uint64), voxel by
        voxel in order of first appearance, each voxel's points in input order."""
        xyz = _as_f64_rows(xyz, 3)
        o = self.grid_sampling_options(grid_size, num_points_per_voxel, max_num_points)
        out = np.empty(max(len(xyz), 1), dtype=np.uint64)
        n = self.check(self.fn("sample_points_in_grid")(device, C.byref(o), xyz.ctypes.data, 24, len(xyz), out.ctypes.data,
                                                        len(out)))
        return out[:n].copy()

    def world_cloud(self, grid_size=1.0, num_points_per_voxel=1, max_num_points=-1, capacity_voxels=0,
                    capacity_points=0, device=0):
        """A WorldCloud (cticp_world_cloud_create): SamplePointsInGrid grown add by add on `device`."""
        return WorldCloud(self, self.grid_sampling_options(grid_size, num_points_per_voxel, max_num_points),
                          capacity_voxels, capacity_points, device)

    def neighborhood(self, points, device=0):
        """A Neighborhood (cticp_neighborhood_create / _create_device): the k-nearest index of slam::TNeighborhood over
        (n, 3) points, a NumPy array (fp64) or a torch CUDA tensor (float32 / float64, unit column stride) on `device`,
        read after the work of torch's current stream. Index i is row i."""
        return Neighborhood(self, points, device)

    def describe_point_sets(self, points, segment_ends=None, values=abi.NB["ALL"], linearity_threshold=0.8,
                            planarity_threshold=0.8, device=0):
        """TNeighborhood(points).ComputeNeighborhood(values) + ClassifyNeighborhood(linearity, planarity) of each set
        (cticp_neighborhood_describe_sets): set s is rows [segment_ends[s - 1], segment_ends[s]); None: one set of every
        row. Returns an array of abi.neighborhood_description_dtype()."""
        xyz = _as_f64_rows(points, 3)
        ends = np.ascontiguousarray([len(xyz)] if segment_ends is None else segment_ends, dtype=np.uint64).reshape(-1)
        out = np.zeros(len(ends), dtype=abi.neighborhood_description_dtype())
        self.check(self.fn("neighborhood_describe_sets")(device, xyz.ctypes.data if len(xyz) else None, 24, len(xyz),
                                                         ends.ctypes.data if len(ends) else None, len(ends), int(values),
                                                         float(linearity_threshold), float(planarity_threshold),
                                                         out.ctypes.data if len(out) else None))
        return out

    def synthetic_scene(self, triangles=(), lines=(), spheres=(), balls=(), device=0):
        """slam::Scene on `device`: triangles (n, 3, 3), lines (n, 2, 3), spheres and balls (n, 4) as (centre, radius);
        primitive i runs over triangles, lines, spheres, balls in that order."""
        return SyntheticScene(self, triangles, lines, spheres, balls, device)

    def lidar_scene(self, boxes=(), cylinders=(), ground=True, device=0):
        """A ray-cast scene on `device`: boxes (n, 7) x0 y0 z0 x1 y1 z1 mean_free_path, cylinders (n, 4) cx cy r h and
        the ground plane z = 0 (synthetic.UrbanScene's .boxes and .cyl load as they are)."""
        return LidarScene(self, boxes, cylinders, ground, device)

    # ---- dataset sequences ------------------------------------------------------------------------------------
    def nclt_hits(self, data, num_aggregated=220, final=True, device=0):
        """An NCLT velodyne_hits.bin stream (bytes, a uint8 NumPy array, or a uint8 CUDA tensor on `device`, read after
        torch's current stream), indexed on `device` into frames of num_aggregated packets (include/cticp.h, "Dataset
        sequences"). With final=False only whole frames are kept and .bytes_used says where the next chunk starts."""
        return NcltHits(self, data, num_aggregated, final, device)

    def ply_layout(self, data):
        """The vertex record layout of a binary_little_endian PLY file's bytes: an abi.PlyLayout"""
        buf = np.frombuffer(bytes(data) if not isinstance(data, np.ndarray) else data.tobytes(), dtype=np.uint8)
        out = abi.PlyLayout()
        self.check(self.fn("ply_layout_parse")(buf.ctypes.data, len(buf), C.byref(out)))
        return out

    def ply_records(self, data):
        """(layout, records): the vertex records of a PLY file as a NumPy structured array with fields x, y, z and t
        (when the file has a timestamp), a view of a copy of the body"""
        lay = self.ply_layout(data)
        raw = np.frombuffer(bytes(data), dtype=np.uint8)
        names = {v: k for k, v in abi.DTYPE.items()}
        xs = np.dtype(names[lay.xyz_dtype]).itemsize
        fields = {"names": ["x", "y", "z"], "formats": [names[lay.xyz_dtype]] * 3,
                  "offsets": [lay.xyz_offset, lay.xyz_offset + xs, lay.xyz_offset + 2 * xs], "itemsize": lay.point_step}
        if lay.t_dtype:
            fields["names"].append("t")
            fields["formats"].append(names[lay.t_dtype])
            fields["offsets"].append(lay.t_offset)
        body = raw[lay.body_offset:lay.body_offset + lay.num_points * lay.point_step].copy()
        return lay, body.view(np.dtype(fields))

    def kitti_frame_filter(self, scan, device=0, in_place=False):
        """kitti_frame_filter of a scan: a NumPy structured array with fields x, y, z (host; returns a filtered copy) or
        an (N, >=3) float32 / float64 CUDA tensor with unit column stride (on torch's current stream; a new tensor, or
        the same one with in_place=True)"""
        if _is_cuda_tensor(scan):
            import torch
            if scan.dim() != 2 or scan.shape[1] < 3 or scan.stride(1) != 1 or scan.dtype not in (torch.float32,
                                                                                                  torch.float64):
                raise ValueError("scan must be an (N, >=3) float32 / float64 tensor with unit column stride")
            out = scan if in_place else torch.empty_like(scan)
            code = abi.DTYPE["float32" if scan.dtype == torch.float32 else "float64"]
            es = scan.element_size()
            ds = abi.DeviceScan(scan.data_ptr(), scan.stride(0) * es, None, 0, scan.shape[0], code, 0)
            sink = abi.CloudSink(out.data_ptr(), out.shape[0], out.stride(0) * es, 0, code, 0, 0, 0)
            if not in_place and scan.shape[1] > 3:
                out[:, 3:] = scan[:, 3:]
            if scan.shape[0]:
                self.check(self.fn("kitti_frame_filter_device")(device, C.byref(ds), C.byref(sink),
                                                                C.c_void_p(torch.cuda.current_stream(device).cuda_stream)))
            return out
        rec = np.ascontiguousarray(scan)
        f = rec.dtype.fields
        xdt, xoff = f["x"][0], f["x"][1]
        view = abi.CloudView(rec.ctypes.data, len(rec), rec.dtype.itemsize, xoff, abi.DTYPE[xdt.name], 0, 0, 0)
        out = rec.view(np.uint8).copy().view(rec.dtype).reshape(-1)   # every byte of a record, named or not
        sink = abi.CloudSink(out.ctypes.data, len(out), out.dtype.itemsize, xoff, abi.DTYPE[xdt.name], 0, 0, 0)
        if len(rec):
            self.check(self.fn("kitti_frame_filter")(device, C.byref(view), C.byref(sink)))
        return out

    def scan_time_ranges(self, t, frame_ends, device=0):
        """(m, 2) per-frame (min, max) of timestamps t split at frame_ends: NumPy arrays on the host (a NaN timestamp
        raises), or CUDA tensors (t 1-D, frame_ends int64 / uint64) on torch's current stream (NaN rows for NaN frames)"""
        if _is_cuda_tensor(t):
            import torch
            codes = _torch_dtype_codes(torch)
            ends = frame_ends.to(device=t.device, dtype=torch.int64).contiguous()
            out = torch.empty((ends.shape[0], 2), dtype=torch.float64, device=t.device)
            ds = abi.DeviceScan(None, 0, t.data_ptr() if t.shape[0] else None, t.stride(0) * t.element_size(), t.shape[0],
                                abi.DTYPE["float64"], codes[t.dtype])
            if ends.shape[0]:
                self.check(self.fn("scan_time_ranges_device")(device, C.byref(ds), ends.data_ptr(), ends.shape[0],
                                                              out.data_ptr(),
                                                              C.c_void_p(torch.cuda.current_stream(device).cuda_stream)))
            return out
        tt = np.ascontiguousarray(t)
        ends = np.ascontiguousarray(frame_ends, dtype=np.uint64)
        out = np.zeros((len(ends), 2))
        rec = np.zeros(len(tt), dtype=np.dtype({"names": ["x", "y", "z", "t"], "formats": ["<f8"] * 3 + [tt.dtype],
                                                "offsets": [0, 8, 16, 24], "itemsize": 24 + tt.dtype.itemsize}))
        rec["t"] = tt
        view = abi.CloudView(rec.ctypes.data if len(rec) else None, len(rec), rec.dtype.itemsize, 0,
                             abi.DTYPE["float64"], 24, abi.DTYPE[tt.dtype.name], 0)
        if len(ends):
            if len(rec) == 0:
                rec = np.zeros(1, dtype=rec.dtype)
                view.data = rec.ctypes.data
            self.check(self.fn("scan_time_ranges")(device, C.byref(view), ends.ctypes.data, len(ends), out.ctypes.data))
        return out

    def ground_truth(self, dataset, text, sequence_id=0):
        """LoadPoses of a ground-truth file's text (str or bytes) for `dataset` (a name of abi.DATASET or its value):
        an array of abi.pose_dtype() in the LiDAR frame"""
        ds = abi.DATASET[dataset] if isinstance(dataset, str) else int(dataset)
        raw = text.encode() if isinstance(text, str) else bytes(text)
        buf = np.frombuffer(raw, dtype=np.uint8)
        n = self.check(self.fn("ground_truth_parse")(ds, int(sequence_id), buf.ctypes.data if len(buf) else None,
                                                     len(buf), None, 0))
        out = np.zeros(n, dtype=abi.pose_dtype())
        if n:
            self.check(self.fn("ground_truth_parse")(ds, int(sequence_id), buf.ctypes.data, len(buf), out.ctypes.data, n))
        return out

    # ---- PLY files -------------------------------------------------------------------------------------------
    def ply_write(self, columns, file_ends=None, device=0, num_items=None):
        """PLY files of columns (include/cticp.h, "PLY files"): `columns` is an ordered list of (element, name,
        ply_dtype, array), ply_dtype a CTICP_DTYPE_* code, a tinyply name ("float") or a NumPy dtype name ("float32");
        each array is 1-D (any stride) or 0-d (one value for every item), NumPy arrays or torch CUDA tensors on `device`.
        num_items defaults to the 1-D columns' common length. Host arrays: the bytes of one file, or with file_ends
        (non-decreasing, at most num_items) (bytes of every file back to back, int64 offsets of m + 1). CUDA tensors: a
        uint8 tensor of every file and an int64 tensor of the m + 1 offsets, written in order with torch's current
        stream (one host synchronisation reads the total size)."""
        cols = list(columns)
        if not cols:
            raise CticpError(abi.ERR_INVALID_ARGUMENT, "no columns")
        if any(_is_cuda_tensor(c[3]) for c in cols):
            return self._ply_write_device(cols, file_ends, device, num_items)
        arrays = []
        for c in cols:
            a = np.asarray(c[3])
            if a.ndim > 1:
                raise ValueError("column %s: expected a 1-D or 0-d array" % c[1])
            if a.ndim == 1 and a.strides[0] < 0:
                a = np.ascontiguousarray(a)
            arrays.append(a)
        n = _ply_num_items([a.shape for a in arrays], num_items)
        codes = [_ply_src_code(a.dtype.name) for a in arrays]

        def encode(first, count):
            props, keep = _ply_props(cols, codes, [(a.ctypes.data + (first * a.strides[0] if a.ndim else 0)
                                                    if a.size else None, a.strides[0] if a.ndim else 0)
                                                   for a in arrays])
            size = self.check(self.fn("ply_write")(device, props, len(cols), count, None, 0))
            buf = C.create_string_buffer(size)
            self.check(self.fn("ply_write")(device, props, len(cols), count, buf, size))
            return buf.raw

        if file_ends is None:
            return encode(0, n)
        ends = np.asarray(file_ends, dtype=np.int64).reshape(-1)
        if (np.diff(ends) < 0).any() or (len(ends) and (ends[0] < 0 or ends[-1] > n)):
            raise CticpError(abi.ERR_INVALID_ARGUMENT, "file_ends must be non-decreasing and at most num_items")
        files = [encode(int(b), int(e - b)) for b, e in zip(np.concatenate([[0], ends[:-1]]), ends)]
        return b"".join(files), np.concatenate([[0], np.cumsum([len(f) for f in files])]).astype(np.int64)

    def _ply_write_device(self, cols, file_ends, device, num_items):
        import torch
        dev = torch.device("cuda", device)
        codes = {torch.int8: 1, torch.uint8: 2, torch.int16: 3, torch.int32: 5, torch.float32: 7, torch.float64: 8,
                 torch.int64: 9}
        for name, code in (("uint16", 4), ("uint32", 6), ("uint64", 10)):
            if hasattr(torch, name):
                codes[getattr(torch, name)] = code
        tensors = []
        for c in cols:
            t = c[3]
            if not _is_cuda_tensor(t) or t.device != dev:
                raise ValueError("column %s: every column must be a CUDA tensor on cuda:%d" % (c[1], device))
            if t.dim() > 1 or t.dtype not in codes:
                raise ValueError("column %s: expected a 1-D or 0-d tensor of a scalar type" % c[1])
            tensors.append(t)
        n = _ply_num_items([tuple(t.shape) for t in tensors], num_items)
        props, keep = _ply_props(cols, [codes[t.dtype] for t in tensors],
                                 [(t.data_ptr() if t.numel() else None, t.stride(0) * t.element_size() if t.dim() else 0)
                                  for t in tensors])
        ends = torch.tensor([n], dtype=torch.int64, device=dev) if file_ends is None else \
            torch.as_tensor(file_ends).to(device=dev, dtype=torch.int64).reshape(-1).contiguous()
        m = ends.shape[0]
        offsets = torch.empty(m + 1, dtype=torch.int64, device=dev)
        stream = C.c_void_p(torch.cuda.current_stream(device).cuda_stream)
        fn = self.fn("ply_write_device")
        self.check(fn(device, props, len(cols), n, ends.data_ptr() if m else None, m, None, 0, offsets.data_ptr(),
                      stream))
        out = torch.empty(int(offsets[-1].item()), dtype=torch.uint8, device=dev)
        if out.numel():
            self.check(fn(device, props, len(cols), n, ends.data_ptr() if m else None, m, out.data_ptr(), out.numel(),
                          offsets.data_ptr(), stream))
        return out, offsets

    def save_poses_ply(self, poses, device=0):
        """slam::SavePosesAsPLY: element pose with qx qy qz qw x y z ref_t dest_t (double) and ref_fid dest_fid (int),
        eleven columns over the cticp_pose records; returns the file's bytes"""
        arr = _pose_array(poses)
        return self.ply_write(_pose_columns(arr), device=device, num_items=len(arr))

    def read_poses_ply(self, data):
        """slam::ReadPosesFromPLY of a file's bytes: an array of abi.pose_dtype()"""
        buf = np.frombuffer(bytes(data), dtype=np.uint8)
        n = self.check(self.fn("ply_read_poses")(buf.ctypes.data, len(buf), None, 0))
        out = np.zeros(n, dtype=abi.pose_dtype())
        if n:
            self.check(self.fn("ply_read_poses")(buf.ctypes.data, len(buf), out.ctypes.data, n))
        return out

    def apply_uniform_noise(self, poses, scale_rot_deg, scale_trans_m, seed=0):
        """slam::ApplyUniformNoise of every pose (a copy, as an array of abi.pose_dtype()); pose i draws under key
        (seed, noise, i)"""
        out = _pose_array(poses).copy()
        self.check(self.fn("apply_uniform_noise")(out.ctypes.data, len(out), float(scale_rot_deg), float(scale_trans_m),
                                                  int(seed)))
        return out

    def synthetic_sequence(self, spec, seed=0, num_frames=None, device=False, device_index=0):
        """ct_icp::SyntheticSequence of `spec`, the dict the reference's YAML parses to (acquisition: {poses, triangles,
        lines, balls, spheres}, sample_frequency 10, max_lidar_distance 100, num_points_per_primitives 300). Returns a dict:
        ground_truth (init^-1 pose_k with dest_frame_id k, abi.pose_dtype()), frames (synthetic_frame_dtype(): frame k
        spans [pose_k.ts, pose_k+1.ts]), and the raw points of the first num_frames frames (all by default) as xyz (N, 3)
        float64, t (N,), frame_ends (m,) and src_index (N, 2): NumPy arrays, or torch CUDA tensors on device_index with
        device=True (generated into device memory, without a host copy of the points)."""
        acq = spec["acquisition"]
        freq = float(spec.get("sample_frequency", 10.0))
        d = float(spec.get("max_lidar_distance", 100.0))
        n = int(spec.get("num_points_per_primitives", 300))
        poses = [_pose_of_spec(p) for p in acq["poses"]]
        def rounds(key):   # {center, radius} items → (centre, radius) rows
            return [list(r["center"]) + [r["radius"]] for r in (acq.get(key) or ())]
        scene = self.synthetic_scene(acq.get("triangles") or (), acq.get("lines") or (), rounds("spheres"),
                                     rounds("balls"), device=device_index)
        traj = self.continuous_trajectory(poses, device=device_index)
        sampled = traj.generate_poses(freq)
        init_inv = _se3_inverse(sampled[0]["quat"], sampled[0]["tr"])
        gt = sampled.copy()
        for k in range(len(gt)):
            gt[k]["quat"], gt[k]["tr"] = _se3_mul(init_inv, (sampled[k]["quat"], sampled[k]["tr"]))
            gt[k]["dest_frame_id"] = k
        frames = np.zeros(max(len(sampled) - 1, 0), dtype=abi.synthetic_frame_dtype())
        frames["begin_ts"] = sampled["dest_timestamp"][:-1]
        frames["end_ts"] = sampled["dest_timestamp"][1:]
        frames["frame_id"] = np.arange(len(frames))
        if num_frames is not None:
            frames = frames[:num_frames]
        out = scene.generate_frames(traj, frames, n, d, seed=seed, with_source_index=True, device=device)
        out.update(ground_truth=gt, frames=frames, scene=scene, trajectory=traj)
        return out

    def permutation(self, seed, counter, n):
        out = np.empty(n, dtype=np.uint32)
        self.check(self.fn("permutation")(seed, counter, n, out.ctypes.data))
        return out


class VoxelMap:
    """ct_icp::MultipleResolutionVoxelMap (include/ct_icp/map.h:99-606) behind the C ABI."""

    def __init__(self, binding, options=None, device=0, borrowed_handle=None, owner=None):
        self.b = binding
        self._owner = owner
        self._borrowed = borrowed_handle is not None
        # the oracle hands out a heap wrapper even for borrowed maps; the engine returns an interior pointer
        self._free_wrapper = self._borrowed and binding.prefix == "orc_"
        if borrowed_handle is not None:
            self.h = C.c_void_p(borrowed_handle)
        else:
            self.h = C.c_void_p()
            binding.check(binding.fn("map_create")(C.byref(options), device, C.byref(self.h)))

    def close(self):
        if self.h and (not self._borrowed or self._free_wrapper):
            self.b.fn("map_destroy")(self.h)
        self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def insert(self, xyz, origin=None):          # InsertPointCloud, map.h:153-254 (origin = frame_poses.front().tr)
        xyz = _as_f64_rows(xyz, 3)
        if origin is None:
            self.b.check(self.b.fn("map_insert")(self.h, xyz.ctypes.data, 24, len(xyz)))
        else:
            o = (C.c_double * 3)(*[float(v) for v in origin])
            self.b.check(self.b.fn("map_insert_from")(self.h, xyz.ctypes.data, 24, len(xyz), o))

    def remove_far(self, location, distance):    # RemoveElementsFarFromLocation, map.h:305-322
        loc = (C.c_double * 3)(*location)
        self.b.check(self.b.fn("map_remove_far")(self.h, loc, distance))

    def num_points(self, map_idx=0):
        return self.b.check(self.b.fn("map_num_points")(self.h, map_idx))

    def num_voxels(self, map_idx=0):
        return self.b.check(self.b.fn("map_num_voxels")(self.h, map_idx))

    def export(self, map_idx=0):
        """Returns (xyz (P,3) f64, voxel (P,3) i32), sorted by (voxel, insertion order)."""
        n = self.num_points(map_idx)
        xyz = np.empty((n, 3), dtype=np.float64)
        vox = np.empty((n, 3), dtype=np.int32)
        m = self.b.check(self.b.fn("map_export")(self.h, map_idx, xyz.ctypes.data, vox.ctypes.data, n))
        assert m == n, (m, n)
        return xyz, vox

    def compute_neighborhoods(self, queries, max_num_neighbors=20):
        q = _as_f64_rows(queries, 3)
        pts = np.zeros((len(q), max_num_neighbors, 3), dtype=np.float64)
        cnt = np.zeros(len(q), dtype=np.int32)
        self.b.check(self.b.fn("map_compute_neighborhoods")(self.h, q.ctypes.data, len(q), max_num_neighbors,
                                                            pts.ctypes.data, cnt.ctypes.data))
        return pts, cnt

    def radius_search(self, queries, radiuses, max_num_neighbors=20, sensor_location=None):
        """ComputeNeighborhoods(queries, radiuses, max_num_neighbors, true, sensor_location), map.h:434-447."""
        q = _as_f64_rows(queries, 3)
        r = np.ascontiguousarray(np.broadcast_to(np.asarray(radiuses, dtype=np.float64), (len(q),)))
        pts = np.zeros((len(q), max_num_neighbors, 3), dtype=np.float64)
        cnt = np.zeros(len(q), dtype=np.int32)
        loc = (C.c_double * 3)(*[float(v) for v in sensor_location]) if sensor_location is not None else None
        self.b.check(self.b.fn("map_radius_search")(self.h, q.ctypes.data, r.ctypes.data, len(q), max_num_neighbors, loc,
                                                    pts.ctypes.data, cnt.ctypes.data))
        return pts, cnt

    def clear(self):
        self.b.check(self.b.fn("map_clear")(self.h))

    def save(self):
        """The map's snapshot (cticp_map_save): every table slot, point and normal, loadable bit for bit with
        Binding.load_voxel_map. For an odometry's map it is the map section of the odometry's snapshot."""
        return _snapshot_bytes(self.b, "map_save", self.h)

    # CT_ICP_Registration::Register(map, keypoints, frame, motion_model), ct_icp.cpp:1026-1037
    def icp_register(self, icp_options, keypoints, frame, previous_frame=None, motion_options=None,
                     strategy=None):
        """keypoints: structured array of abi.wpoint_dtype() (world rewritten in place); frame: abi.Frame (in/out).
        Returns abi.IcpSummary."""
        assert keypoints.dtype == abi.wpoint_dtype() and keypoints.flags.c_contiguous
        summary = abi.IcpSummary()
        st = strategy if strategy is not None else abi.StrategyOptions(0, 20, 8, 0)
        self.b.check(self.b.fn("icp_register")(
            self.h, C.byref(icp_options), C.byref(st), keypoints.ctypes.data, len(keypoints), C.byref(frame),
            C.byref(previous_frame) if previous_frame is not None else None,
            C.byref(motion_options) if motion_options is not None else None, C.byref(summary)))
        return summary

    def icp_register_batch(self, icp_options, keypoints_list, frames, previous_frames=None, motion_options=None):
        """B independent registrations (solver GN) in one launch (cticp_icp_register_batch). keypoints_list: B arrays of
        abi.wpoint_dtype() (world rewritten in place); frames: B abi.Frame (updated in place); previous_frames: None or
        B entries, each an abi.Frame or None (no motion prior for that problem). Returns the B abi.IcpSummary."""
        return self._register_batch(None, icp_options, keypoints_list, frames, previous_frames, motion_options)

    def icp_register_batch_ex(self, icp_options, keypoints_list, frames, previous_frames=None, motion_options=None,
                              strategy=None):
        """icp_register_batch for every solver (cticp_icp_register_batch_ex): GN, CERES or ROBUST, with the neighborhood
        strategy CERES consults (None: icp_register's default). Returns the B abi.IcpSummary."""
        st = strategy if strategy is not None else abi.StrategyOptions(0, 20, 8, 0)
        return self._register_batch(st, icp_options, keypoints_list, frames, previous_frames, motion_options)

    def _register_batch(self, strategy, icp_options, keypoints_list, frames, previous_frames, motion_options):
        B = len(keypoints_list)
        if len(frames) != B or (previous_frames is not None and len(previous_frames) != B):
            raise ValueError("keypoints_list, frames and previous_frames must have one entry per problem")
        for kp in keypoints_list:
            assert kp.dtype == abi.wpoint_dtype() and kp.flags.c_contiguous
        m = max(B, 1)
        kps = (C.c_void_p * m)(*[kp.ctypes.data if len(kp) else None for kp in keypoints_list])
        ns = (C.c_size_t * m)(*[len(kp) for kp in keypoints_list])
        fr = (abi.Frame * m)()
        for b, f in enumerate(frames):
            C.memmove(C.addressof(fr[b]), C.addressof(f), C.sizeof(abi.Frame))
        prev = None
        if previous_frames is not None:
            prev = (C.c_void_p * m)(*[C.addressof(p) if p is not None else None for p in previous_frames])
        out = (abi.IcpSummary * m)()
        mo = C.byref(motion_options) if motion_options is not None else None
        if strategy is None:
            rc = self.b.fn("icp_register_batch")(self.h, C.byref(icp_options), B, kps, ns, fr, prev, mo, out)
        else:
            rc = self.b.fn("icp_register_batch_ex")(self.h, C.byref(icp_options), C.byref(strategy), B, kps, ns, fr, prev,
                                                    mo, out)
        if rc >= 0 or rc == abi.ERR_INTERNAL:   # ERR_INTERNAL: a timed-out problem; every output is written all the same
            for b, f in enumerate(frames):
                C.memmove(C.addressof(f), C.addressof(fr[b]), C.sizeof(abi.Frame))
        self.b.check(rc)
        return [out[b].copy() for b in range(B)]

    def gn_normal_equations(self, icp_options, keypoints, frame, previous_frame=None, motion_options=None):
        assert keypoints.dtype == abi.wpoint_dtype() and keypoints.flags.c_contiguous
        A = np.zeros((12, 12))
        b = np.zeros(12)
        n = C.c_int32(0)
        self.b.check(self.b.fn("icp_gn_normal_equations")(
            self.h, C.byref(icp_options), keypoints.ctypes.data, len(keypoints), C.byref(frame),
            C.byref(previous_frame) if previous_frame is not None else None,
            C.byref(motion_options) if motion_options is not None else None, A.ctypes.data, b.ctypes.data,
            C.byref(n)))
        return A, b, n.value


class Odometry:
    """ct_icp::Odometry (include/ct_icp/odometry.h:159-402) behind the C ABI.

    Method names follow the reference: RegisterFrame, RegisterFrameWithEstimate, Trajectory, MapSize,
    GetMapPointCloud, Reset, GetMapPointer."""

    def __init__(self, binding, options, device=0):
        self.b = binding
        self.options = options.copy()
        self.device = device
        self.h = C.c_void_p()
        binding.check(binding.fn("odometry_create")(C.byref(self.options), device, C.byref(self.h)))

    @classmethod
    def _adopt(cls, binding, handle, options, device):
        od = cls.__new__(cls)
        od.b, od.options, od.device, od.h = binding, options.copy(), device, handle
        return od

    def save(self):
        """The handle's snapshot (cticp_odometry_save): voxel map, trajectory, motion model and counters as bytes;
        Binding.load_odometry resumes from it bit for bit."""
        return _snapshot_bytes(self.b, "odometry_save", self.h)

    def clone(self, device=None):
        """A new Odometry holding the same state, on `device` (None: this handle's), copied device to device."""
        device = self.device if device is None else device
        h = C.c_void_p()
        self.b.check(self.b.fn("odometry_clone")(self.h, device, C.byref(h)))
        return Odometry._adopt(self.b, h, self.options, device)

    def close(self):
        if self.h:
            self.b.fn("odometry_destroy")(self.h)
        self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def _register(self, xyz, timestamps, frame_id, initial_estimate):
        xyz = np.asarray(xyz)
        timestamps = np.asarray(timestamps)
        if xyz.dtype != np.float64 or xyz.ndim != 2 or xyz.shape[1] < 3 or xyz.strides[1] != 8:
            xyz = np.ascontiguousarray(xyz[:, :3], dtype=np.float64)
        if timestamps.dtype != np.float64 or timestamps.ndim != 1:
            timestamps = np.ascontiguousarray(timestamps, dtype=np.float64).reshape(-1)
        if len(xyz) != len(timestamps):
            raise ValueError("xyz and timestamps must have the same length")
        summary = abi.Summary()
        self.b.check(self.b.fn("odometry_register_frame")(
            self.h, xyz.ctypes.data, xyz.strides[0], timestamps.ctypes.data, timestamps.strides[0], len(xyz),
            frame_id, C.byref(initial_estimate) if initial_estimate is not None else None, C.byref(summary)))
        return summary

    def RegisterFrame(self, xyz, timestamps, frame_id, motion_model=None):
        """motion_model: an abi.MotionPrior — the AMotionModel* of the reference's overloads (odometry.h:231-248).
        xyz / timestamps: numpy arrays, or torch CUDA tensors on the handle's device (read in place, see _register_tensors)"""
        if _is_cuda_tensor(xyz) or _is_cuda_tensor(timestamps):
            return self._register_tensors(xyz, timestamps, frame_id, None, motion_model)
        if motion_model is not None:
            return self._register_ex(xyz, timestamps, frame_id, None, motion_model)
        return self._register(xyz, timestamps, frame_id, None)

    def _register_ex(self, xyz, timestamps, frame_id, initial_estimate, motion_model):
        xyz = np.ascontiguousarray(np.asarray(xyz)[:, :3], dtype=np.float64)
        timestamps = np.ascontiguousarray(timestamps, dtype=np.float64).reshape(-1)
        summary = abi.Summary()
        self.b.check(self.b.fn("odometry_register_frame_ex")(
            self.h, xyz.ctypes.data, xyz.strides[0], timestamps.ctypes.data, timestamps.strides[0], len(xyz), frame_id,
            C.byref(initial_estimate) if initial_estimate is not None else None,
            C.byref(motion_model) if motion_model is not None else None, C.byref(summary)))
        return summary

    def RegisterCallback(self, fn):
        """fn(event) -> bool, called at BEFORE_ITERATION / ITERATION_COMPLETED / FINISHED_REGISTRATION
        (Odometry::RegisterCallback, odometry.h:260); None removes it."""
        self._callback = abi.EVENT_FN(lambda event, user: 1 if fn(event) else 0) if fn else abi.EVENT_FN()
        self.b.check(self.b.fn("odometry_set_callback")(self.h, self._callback, None))

    def ResetWithOptions(self, options):        # Odometry::Reset(const OdometryOptions&), odometry.h:269
        self.options = options.copy()
        self.b.check(self.b.fn("odometry_reset_options")(self.h, C.byref(self.options)))

    def RegisterFrameWithEstimate(self, xyz, timestamps, initial_estimate, frame_id, motion_model=None):
        if _is_cuda_tensor(xyz) or _is_cuda_tensor(timestamps):
            return self._register_tensors(xyz, timestamps, frame_id, initial_estimate, motion_model)
        if motion_model is not None:
            return self._register_ex(xyz, timestamps, frame_id, initial_estimate, motion_model)
        return self._register(xyz, timestamps, frame_id, initial_estimate)

    # ---- device memory in and out (engine only) ----------------------------------------------------------------
    def _register_tensors(self, xyz, timestamps, frame_id, initial_estimate, motion_model):
        scan, stream = self._device_scan(xyz, timestamps)
        return self.register_device(scan, frame_id, initial_estimate, motion_model, stream=stream)

    def _device_scan(self, xyz, timestamps):
        """(abi.DeviceScan, producer stream) of a tensor scan. xyz: (N, >=3) float32 / float64 CUDA tensor with unit
        column stride (an (N, 4) xyzi tensor is read in place); timestamps: 1-D CUDA tensor of any supported dtype and stride. Both on the handle's device; the scan is read after
        the work already queued on torch's current stream of that device."""
        import torch
        if not (_is_cuda_tensor(xyz) and _is_cuda_tensor(timestamps)):
            raise ValueError("xyz and timestamps must both be CUDA tensors (or both host arrays)")
        if xyz.device.index != self.device or timestamps.device.index != self.device:
            raise ValueError("xyz and timestamps must be on cuda:%d, the handle's device" % self.device)
        if xyz.dim() != 2 or xyz.shape[1] < 3 or xyz.stride(1) != 1 or xyz.dtype not in (torch.float32, torch.float64):
            raise ValueError("xyz must be an (N, >=3) float32 / float64 tensor with unit column stride")
        codes = _torch_dtype_codes(torch)
        if timestamps.dim() != 1 or timestamps.dtype not in codes:
            raise ValueError("timestamps must be a 1-D tensor of a supported dtype")
        if xyz.shape[0] != timestamps.shape[0]:
            raise ValueError("xyz and timestamps must have the same length")
        scan = abi.DeviceScan(xyz.data_ptr(), xyz.stride(0) * xyz.element_size(), timestamps.data_ptr(),
                              timestamps.stride(0) * timestamps.element_size(), xyz.shape[0], codes[xyz.dtype],
                              codes[timestamps.dtype])
        return scan, torch.cuda.current_stream(self.device).cuda_stream

    def register_device(self, scan, frame_id, initial_estimate=None, motion_model=None, stream=0):
        """cticp_odometry_register_device on an abi.DeviceScan (any record layout); stream: the producer's cudaStream_t."""
        summary = abi.Summary()
        self.b.check(self.b.fn("odometry_register_device")(
            self.h, C.byref(scan), C.c_void_p(stream or None), frame_id,
            C.byref(initial_estimate) if initial_estimate is not None else None,
            C.byref(motion_model) if motion_model is not None else None, C.byref(summary)))
        return summary

    def write_points_device(self, which, sink, stream=0):
        """cticp_odometry_write_points_device on an abi.CloudSink in device memory; returns the count."""
        return self.b.check(self.b.fn("odometry_write_points_device")(self.h, which, C.byref(sink),
                                                                      C.c_void_p(stream or None)))

    def points_device(self, which, world=True, dtype=None, with_timestamps=False):
        """One of the summary's point vectors as an (n, 3) — (n, 4) with the timestamps — CUDA tensor of `dtype`
        (float64 by default, or float32) on the handle's device, written in order with torch's current stream."""
        import torch
        dtype = torch.float64 if dtype is None else dtype
        if dtype not in (torch.float32, torch.float64):
            raise ValueError("dtype must be torch.float32 or torch.float64")
        stream = torch.cuda.current_stream(self.device).cuda_stream
        n = self.write_points_device(which, abi.CloudSink(None, 0, 0, 0, 0, 0, 0, 0), stream)
        cols = 4 if with_timestamps else 3
        out = torch.empty((n, cols), dtype=dtype, device=torch.device("cuda", self.device))
        if n:
            code = abi.DTYPE["float32" if dtype == torch.float32 else "float64"]
            size = out.element_size()
            sink = abi.CloudSink(out.data_ptr(), n, cols * size, 0, code, 3 * size, code if with_timestamps else 0,
                                 1 if world else 0)
            self.write_points_device(which, sink, stream)
        return out

    # ---- record buffers (sensor_msgs/PointCloud2-like), zero-copy in and out (engine only) -------------------
    @staticmethod
    def _cloud_view(records, xyz_field="x", t_field="t"):
        """records: 1-D numpy structured array with fields x, y, z (contiguous, same float type) and a timestamp."""
        assert records.ndim == 1 and records.flags.c_contiguous and records.dtype.fields is not None
        f = records.dtype.fields
        xdt, xoff = f[xyz_field][0], f[xyz_field][1]
        assert f["y"] == (xdt, xoff + xdt.itemsize) and f["z"] == (xdt, xoff + 2 * xdt.itemsize), "x, y, z must be contiguous"
        tdt, toff = f[t_field][0], f[t_field][1]
        return abi.CloudView(records.ctypes.data, len(records), records.dtype.itemsize, xoff, abi.DTYPE[xdt.name], toff,
                             abi.DTYPE[tdt.name], 0)

    def RegisterCloud(self, records, frame_id, initial_estimate=None, t_field="t"):
        """RegisterFrame(const slam::PointCloud&, frame_id) on an interleaved record buffer, read in place."""
        view = self._cloud_view(records, t_field=t_field)
        summary = abi.Summary()
        self.b.check(self.b.fn("odometry_register_cloud")(
            self.h, C.byref(view), frame_id, C.byref(initial_estimate) if initial_estimate is not None else None,
            C.byref(summary)))
        return summary

    def stage_cloud(self, records, t_field="t"):
        view = self._cloud_view(records, t_field=t_field)
        return self.b.check(self.b.fn("odometry_stage_cloud")(self.h, C.byref(view)))

    def write_points(self, which, records, world=True, t_field="t"):
        """Fills `records` (structured array with x, y, z [+ timestamp field]) with one of the summary's point vectors;
        returns the number of points the vector holds."""
        f = records.dtype.fields
        xdt, xoff = f["x"][0], f["x"][1]
        has_t = t_field in f
        sink = abi.CloudSink(records.ctypes.data, len(records), records.dtype.itemsize, xoff, abi.DTYPE[xdt.name],
                             f[t_field][1] if has_t else 0, abi.DTYPE[f[t_field][0].name] if has_t else 0,
                             1 if world else 0)
        return self.b.check(self.b.fn("odometry_write_points")(self.h, which, C.byref(sink)))

    # ---- device-resident input / measurement helpers (engine only) ---------------------------------------
    def stage_frame(self, xyz, timestamps):
        xyz = np.ascontiguousarray(np.asarray(xyz)[:, :3], dtype=np.float64)
        timestamps = np.ascontiguousarray(timestamps, dtype=np.float64).reshape(-1)
        return self.b.check(self.b.fn("odometry_stage_frame")(self.h, xyz.ctypes.data, xyz.strides[0],
                                                              timestamps.ctypes.data, 8, len(xyz)))

    def RegisterStaged(self, slot, frame_id):
        summary = abi.Summary()
        self.b.check(self.b.fn("odometry_register_staged")(self.h, slot, frame_id, C.byref(summary)))
        return summary

    def clear_staged(self):
        self.b.check(self.b.fn("odometry_clear_staged")(self.h))

    def timer_start(self):
        self.b.check(self.b.fn("odometry_timer_start")(self.h))

    def timer_stop(self):
        ms = C.c_double(0.0)
        self.b.check(self.b.fn("odometry_timer_stop")(self.h, C.byref(ms)))
        return ms.value

    def flush_l2(self, nbytes=256 << 20):
        self.b.check(self.b.fn("odometry_flush_l2")(self.h, nbytes))

    def set_gather_timing(self, on):
        self.b.check(self.b.fn("odometry_set_gather_timing")(self.h, 1 if on else 0))

    def set_summary_points(self, mask):
        """bit POINTS_* set: every RegisterFrame produces that vector of the RegistrationSummary eagerly."""
        self.b.check(self.b.fn("odometry_set_summary_points")(self.h, int(mask)))

    def points_into(self, which, buf):
        """one of the summary's point vectors into a caller-owned record array (abi.wpoint_dtype()); returns the count"""
        return self.b.check(self.b.fn("odometry_get_points")(self.h, which, buf.ctypes.data, len(buf)))

    def points(self, which):
        cap = 1 << 16
        while True:
            buf = np.zeros(cap, dtype=abi.wpoint_dtype())
            n = self.b.check(self.b.fn("odometry_get_points")(self.h, which, buf.ctypes.data, cap))
            if n <= cap:
                return buf[:n].copy()
            cap = int(n)

    def corrected_points(self):
        return self.points(abi.POINTS_CORRECTED)

    def all_corrected_points(self):
        return self.points(abi.POINTS_ALL_CORRECTED)

    def keypoints(self):
        return self.points(abi.POINTS_KEYPOINTS)

    def Trajectory(self):
        n = self.b.check(self.b.fn("odometry_trajectory")(self.h, None, 0))
        arr = (abi.Frame * max(n, 1))()
        self.b.check(self.b.fn("odometry_trajectory")(self.h, arr, n))
        return [arr[i].copy() for i in range(n)]

    def MapSize(self):
        return self.b.check(self.b.fn("odometry_map_size")(self.h))

    def GetMapPointer(self):
        return VoxelMap(self.b, borrowed_handle=self.b.fn("odometry_map")(self.h), owner=self)

    def GetMapPointCloud(self):
        xyz, _ = self.GetMapPointer().export(0)
        return xyz

    def Reset(self):
        self.b.check(self.b.fn("odometry_reset")(self.h))

    def last_timing(self):
        t = abi.DeviceTiming()
        self.b.check(self.b.fn("odometry_last_timing")(self.h, C.byref(t)))
        return t

    def enable_sharding(self, unique_id_bytes, rank, world):
        buf = (C.c_char * 128).from_buffer_copy(unique_id_bytes)
        self.b.check(self.b.fn("odometry_enable_sharding")(self.h, buf, rank, world))

    def sharding_mode(self):
        """0 = single GPU, 1 = NCCL all-reduce per exchange, 2 = in-kernel exchange over NVLink peer mailboxes."""
        return self.b.fn("odometry_sharding_mode")(self.h)


class ContinuousTrajectory:
    """slam::LinearContinuousTrajectory (include/SlamCore/trajectory.h:28-130) behind the C ABI: the sorted poses, the
    pose at any timestamp, and RawPointsToWorldPoints (src/SlamCore/pointcloud.cxx:313-326) of host or device points."""

    def __init__(self, binding, poses_or_frames, device=0):
        self.b = binding
        self.device = device
        poses = []
        for item in poses_or_frames:
            if isinstance(item, abi.Frame):
                poses += [item.begin_pose, item.end_pose]
            elif isinstance(item, abi.Pose):
                poses.append(item)
            else:
                raise TypeError("expected abi.Pose or abi.Frame items, got %r" % type(item))
        arr = (abi.Pose * max(len(poses), 1))()
        for i, p in enumerate(poses):
            C.memmove(C.addressof(arr[i]), C.addressof(p), C.sizeof(abi.Pose))
        self.h = C.c_void_p()
        binding.check(binding.fn("trajectory_create")(arr, len(poses), device, C.byref(self.h)))

    def close(self):
        if self.h:
            self.b.fn("trajectory_destroy")(self.h)
        self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def poses(self):
        """Poses(): sorted by (dest_frame_id, dest_timestamp), as a structured array of abi.pose_dtype()"""
        n = self.b.check(self.b.fn("trajectory_poses")(self.h, None, 0))
        out = np.zeros(n, dtype=abi.pose_dtype())
        self.b.check(self.b.fn("trajectory_poses")(self.h, out.ctypes.data, n))
        return out

    def interpolate(self, timestamps, frame_ids=None):
        """InterpolatePose(t) of every timestamp, or InterpolatePoseWithFrameId(t, frame_id) when frame_ids is given
        (one per timestamp); a structured array of abi.pose_dtype()."""
        ts = np.ascontiguousarray(timestamps, dtype=np.float64).reshape(-1)
        fid = None
        if frame_ids is not None:
            fid = np.ascontiguousarray(frame_ids, dtype=np.uint32).reshape(-1)
            if len(fid) != len(ts):
                raise ValueError("frame_ids must have one entry per timestamp")
        out = np.zeros(len(ts), dtype=abi.pose_dtype())
        self.b.check(self.b.fn("trajectory_interpolate")(self.h, ts.ctypes.data, fid.ctypes.data if fid is not None else None,
                                                         len(ts), out.ctypes.data))
        return out

    def generate_poses(self, frequency):
        """SyntheticSensorAcquisition::GeneratePoses(frequency): InterpolatePose at MinTimestamp + k / frequency (summed
        in fp64) up to MaxTimestamp, as an array of abi.pose_dtype()"""
        n = self.b.check(self.b.fn("synthetic_generate_poses")(self.h, float(frequency), None, 0))
        out = np.zeros(n, dtype=abi.pose_dtype())
        self.b.check(self.b.fn("synthetic_generate_poses")(self.h, float(frequency), out.ctypes.data, n))
        return out

    def kitti_evaluate(self, gt, lengths="driving"):
        """kitti::EvaluatePoses(gt, trajectory) (cticp_trajectory_kitti_evaluate): the estimate is the pose of this
        trajectory at every ground-truth dest_timestamp, interpolated on the trajectory's device. A dict as
        Binding.kitti_evaluate returns."""
        g = _pose_array(gt)
        lens = _lengths(lengths)
        cap = -(-len(g) // 10) * len(lens)
        out = abi.KittiErrors()
        tab = np.zeros((max(cap, 1), 2))
        count = self.b.check(self.b.fn("trajectory_kitti_evaluate")(self.h, g.ctypes.data, len(g), lens.ctypes.data,
                                                                    len(lens), C.byref(out), tab.ctypes.data, cap))
        return _kitti_dict(out, tab[:count])

    @staticmethod
    def _segments(segments, n):
        """segments: None, or (ends, frame_ids): segment s holds points [ends[s-1], ends[s]) of frame frame_ids[s]"""
        if segments is None:
            return None, None, 0
        ends, fids = segments
        ends = np.ascontiguousarray(ends, dtype=np.uint64).reshape(-1)
        fids = np.ascontiguousarray(fids, dtype=np.uint32).reshape(-1)
        if len(ends) != len(fids):
            raise ValueError("segment ends and frame ids must have the same length")
        return ends, fids, len(ends)

    def transform_records(self, records, sink, segments=None):
        """cticp_trajectory_transform of a 1-D structured host array (fields x, y, z contiguous of one float type and t)
        into `sink`, a 1-D structured host array with x, y, z and optionally t; returns the number of points."""
        view = Odometry._cloud_view(records)
        f = sink.dtype.fields
        has_t = "t" in f
        cs = abi.CloudSink(sink.ctypes.data, len(sink), sink.dtype.itemsize, f["x"][1], abi.DTYPE[f["x"][0].name],
                           f["t"][1] if has_t else 0, abi.DTYPE[f["t"][0].name] if has_t else 0, 1)
        ends, fids, ns = self._segments(segments, len(records))
        return self.b.check(self.b.fn("trajectory_transform")(
            self.h, C.byref(view), ends.ctypes.data if ns else None, fids.ctypes.data if ns else None, ns, C.byref(cs)))

    def transform_device(self, scan, sink, segments=None, stream=0):
        """cticp_trajectory_transform_device of an abi.DeviceScan into an abi.CloudSink in device memory"""
        ends, fids, ns = self._segments(segments, scan.num_points)
        return self.b.check(self.b.fn("trajectory_transform_device")(
            self.h, C.byref(scan), ends.ctypes.data if ns else None, fids.ctypes.data if ns else None, ns, C.byref(sink),
            C.c_void_p(stream or None)))

    def transform(self, xyz, t, segments=None, dtype=np.float64, with_timestamps=False):
        """World coordinates of raw points xyz (N, 3) with timestamps t (N,): TransformPoint(raw, t) of every point, or
        TransformPoint(raw, t, frame_id) with segments = (ends, frame_ids) for N scans concatenated.
        NumPy arrays: the host path, returns an (N, 3) array of `dtype` ((N, 4) with the timestamps).
        torch CUDA tensors on the trajectory's device (xyz (N, >=3) float32 / float64 with unit column stride, t 1-D of any
        supported dtype): the device path, read after and written before the work of torch's current stream; returns a
        CUDA tensor."""
        if _is_cuda_tensor(xyz) or _is_cuda_tensor(t):
            return self._transform_tensors(xyz, t, segments, dtype, with_timestamps)
        xyz = np.asarray(xyz)
        t = np.asarray(t).reshape(-1)
        if xyz.ndim != 2 or xyz.shape[1] < 3 or xyz.dtype not in (np.float32, np.float64):
            raise ValueError("xyz must be an (N, >=3) float32 / float64 array")
        if len(xyz) != len(t):
            raise ValueError("xyz and t must have the same length")
        rec = np.zeros(len(xyz), dtype=np.dtype([("x", xyz.dtype), ("y", xyz.dtype), ("z", xyz.dtype), ("t", t.dtype)]))
        rec["x"], rec["y"], rec["z"], rec["t"] = xyz[:, 0], xyz[:, 1], xyz[:, 2], t
        dtype = np.dtype(dtype)
        fields = [("x", dtype), ("y", dtype), ("z", dtype)] + ([("t", dtype)] if with_timestamps else [])
        out = np.zeros(len(xyz), dtype=np.dtype(fields))
        self.transform_records(rec, out, segments)
        return out.view(dtype).reshape(len(xyz), len(fields))

    def _transform_tensors(self, xyz, t, segments, dtype, with_timestamps):
        import torch
        if not (_is_cuda_tensor(xyz) and _is_cuda_tensor(t)):
            raise ValueError("xyz and t must both be CUDA tensors (or both host arrays)")
        if xyz.device.index != self.device or t.device.index != self.device:
            raise ValueError("xyz and t must be on cuda:%d, the trajectory's device" % self.device)
        if xyz.dim() != 2 or xyz.shape[1] < 3 or xyz.stride(1) != 1 or xyz.dtype not in (torch.float32, torch.float64):
            raise ValueError("xyz must be an (N, >=3) float32 / float64 tensor with unit column stride")
        codes = _torch_dtype_codes(torch)
        if t.dim() != 1 or t.dtype not in codes:
            raise ValueError("t must be a 1-D tensor of a supported dtype")
        if xyz.shape[0] != t.shape[0]:
            raise ValueError("xyz and t must have the same length")
        tdtype = {np.dtype(np.float32): torch.float32, np.dtype(np.float64): torch.float64}.get(np.dtype(dtype), dtype)
        if tdtype not in (torch.float32, torch.float64):
            raise ValueError("dtype must be float32 or float64")
        n = xyz.shape[0]
        scan = abi.DeviceScan(xyz.data_ptr(), xyz.stride(0) * xyz.element_size(), t.data_ptr(),
                              t.stride(0) * t.element_size(), n, codes[xyz.dtype], codes[t.dtype])
        cols = 4 if with_timestamps else 3
        stream = torch.cuda.current_stream(self.device).cuda_stream
        out = torch.empty((n, cols), dtype=tdtype, device=torch.device("cuda", self.device))
        code = abi.DTYPE["float32" if tdtype == torch.float32 else "float64"]
        size = out.element_size()
        sink = abi.CloudSink(out.data_ptr() if n else None, n, cols * size, 0, code, 3 * size,
                             code if with_timestamps else 0, 1)
        self.transform_device(scan, sink, segments, stream)
        return out


class WorldCloud:
    """slam::SamplePointsInGrid grown call by call on the device (cticp_world_cloud_*): after any sequence of adds, export
    returns SamplePointsInGrid over every point submitted, in call order, with each point's source index (its position in
    that concatenation) and timestamp."""

    def __init__(self, binding, options, capacity_voxels=0, capacity_points=0, device=0):
        self.b = binding
        self.device = device
        self.options = options.copy()
        self.h = C.c_void_p()
        binding.check(binding.fn("world_cloud_create")(C.byref(self.options), int(capacity_voxels), int(capacity_points),
                                                       device, C.byref(self.h)))

    def close(self):
        if self.h:
            self.b.fn("world_cloud_destroy")(self.h)
        self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    @staticmethod
    def _traj(trajectory):
        return trajectory.h if trajectory is not None else None

    def add_records(self, records, trajectory=None, segments=None, t_field="t"):
        """cticp_world_cloud_add of a 1-D structured host array (x, y, z contiguous of one float type, and a timestamp
        field, which may be absent without a trajectory). Returns abi.WorldCloudStats."""
        assert records.ndim == 1 and records.flags.c_contiguous and records.dtype.fields is not None
        f = records.dtype.fields
        xdt, xoff = f["x"][0], f["x"][1]
        assert f["y"] == (xdt, xoff + xdt.itemsize) and f["z"] == (xdt, xoff + 2 * xdt.itemsize), "x, y, z must be contiguous"
        has_t = t_field in f
        view = abi.CloudView(records.ctypes.data if len(records) else None, len(records), records.dtype.itemsize, xoff,
                             abi.DTYPE[xdt.name], f[t_field][1] if has_t else 0, abi.DTYPE[f[t_field][0].name] if has_t else 0,
                             0)
        ends, fids, ns = ContinuousTrajectory._segments(segments, len(records))
        st = abi.WorldCloudStats()
        self.b.check(self.b.fn("world_cloud_add")(self.h, self._traj(trajectory), C.byref(view),
                                                  ends.ctypes.data if ns else None, fids.ctypes.data if ns else None, ns,
                                                  C.byref(st)))
        return st

    def add_device(self, scan, trajectory=None, segments=None, stream=0):
        """cticp_world_cloud_add_device of an abi.DeviceScan; stream: the producer's cudaStream_t"""
        ends, fids, ns = ContinuousTrajectory._segments(segments, scan.num_points)
        st = abi.WorldCloudStats()
        self.b.check(self.b.fn("world_cloud_add_device")(self.h, self._traj(trajectory), C.byref(scan),
                                                         ends.ctypes.data if ns else None,
                                                         fids.ctypes.data if ns else None, ns, C.byref(st),
                                                         C.c_void_p(stream or None)))
        return st

    def add(self, xyz, t=None, trajectory=None, segments=None):
        """Adds points: world coordinates without a trajectory, else raw coordinates placed by
        trajectory.transform(xyz, t, segments). NumPy arrays: the host path; torch CUDA tensors on the cloud's device
        (xyz (N, >=3) float32 / float64 with unit column stride, t 1-D of any supported dtype or None): read in place
        after the work of torch's current stream. Returns abi.WorldCloudStats."""
        if _is_cuda_tensor(xyz) or _is_cuda_tensor(t):
            return self._add_tensors(xyz, t, trajectory, segments)
        xyz = np.asarray(xyz)
        if xyz.ndim != 2 or xyz.shape[1] < 3 or xyz.dtype not in (np.float32, np.float64):
            raise ValueError("xyz must be an (N, >=3) float32 / float64 array")
        fields = [("x", xyz.dtype), ("y", xyz.dtype), ("z", xyz.dtype)]
        if t is not None:
            t = np.asarray(t).reshape(-1)
            if len(t) != len(xyz):
                raise ValueError("xyz and t must have the same length")
            fields.append(("t", t.dtype))
        rec = np.zeros(len(xyz), dtype=np.dtype(fields))
        rec["x"], rec["y"], rec["z"] = xyz[:, 0], xyz[:, 1], xyz[:, 2]
        if t is not None:
            rec["t"] = t
        return self.add_records(rec, trajectory, segments)

    def _add_tensors(self, xyz, t, trajectory, segments):
        import torch
        if not _is_cuda_tensor(xyz) or (t is not None and not _is_cuda_tensor(t)):
            raise ValueError("xyz and t must both be CUDA tensors (or both host arrays)")
        if xyz.device.index != self.device or (t is not None and t.device.index != self.device):
            raise ValueError("xyz and t must be on cuda:%d, the cloud's device" % self.device)
        if xyz.dim() != 2 or xyz.shape[1] < 3 or xyz.stride(1) != 1 or xyz.dtype not in (torch.float32, torch.float64):
            raise ValueError("xyz must be an (N, >=3) float32 / float64 tensor with unit column stride")
        codes = _torch_dtype_codes(torch)
        if t is not None and (t.dim() != 1 or t.dtype not in codes or t.shape[0] != xyz.shape[0]):
            raise ValueError("t must be a 1-D tensor of a supported dtype, one entry per point")
        scan = abi.DeviceScan(xyz.data_ptr() if xyz.shape[0] else None, xyz.stride(0) * xyz.element_size(),
                              t.data_ptr() if t is not None and t.shape[0] else None,
                              t.stride(0) * t.element_size() if t is not None else 0, xyz.shape[0], codes[xyz.dtype],
                              codes[t.dtype] if t is not None else 0)
        return self.add_device(scan, trajectory, segments, torch.cuda.current_stream(self.device).cuda_stream)

    def add_odometry(self, odometry):
        """The odometry's last CTICP_POINTS_ALL_CORRECTED world points and timestamps, device to device"""
        st = abi.WorldCloudStats()
        self.b.check(self.b.fn("world_cloud_add_odometry")(self.h, odometry.h, C.byref(st)))
        return st

    def num_points(self):
        """what export returns (max_num_points applied)"""
        return self.b.check(self.b.fn("world_cloud_num_points")(self.h))

    def num_voxels(self):
        return self.b.check(self.b.fn("world_cloud_num_voxels")(self.h))

    def neighborhood(self):
        """A Neighborhood over the points export() returns, in that order (cticp_neighborhood_create_world_cloud)"""
        h = C.c_void_p()
        self.b.check(self.b.fn("neighborhood_create_world_cloud")(self.h, C.byref(h)))
        return Neighborhood(self.b, device=self.device, handle=h.value)

    def clear(self):
        self.b.check(self.b.fn("world_cloud_clear")(self.h))

    def export_sink(self, sink, src_index=None):
        """cticp_world_cloud_export into an abi.CloudSink in host memory; src_index: None or a uint64 array"""
        return self.b.check(self.b.fn("world_cloud_export")(self.h, C.byref(sink),
                                                            src_index.ctypes.data if src_index is not None else None))

    def export_device_sink(self, sink, src_index_ptr=None, stream=0):
        """cticp_world_cloud_export_device into an abi.CloudSink in device memory"""
        return self.b.check(self.b.fn("world_cloud_export_device")(self.h, C.byref(sink), src_index_ptr or None,
                                                                   C.c_void_p(stream or None)))

    def export(self, dtype=np.float64, with_timestamps=False, with_source_index=False, device=False):
        """The cloud as an (n, 3) array of `dtype` ((n, 4) with the timestamps); with_source_index: (points, source
        indices uint64). device=True: torch CUDA tensors on the cloud's device, written in order with torch's current
        stream (dtype torch.float32 / torch.float64 or the NumPy equivalents)."""
        n = self.num_points()
        cols = 4 if with_timestamps else 3
        if device:
            import torch
            tdtype = {np.dtype(np.float32): torch.float32, np.dtype(np.float64): torch.float64}.get(
                np.dtype(dtype) if not isinstance(dtype, torch.dtype) else None, dtype)
            if tdtype not in (torch.float32, torch.float64):
                raise ValueError("dtype must be float32 or float64")
            dev = torch.device("cuda", self.device)
            out = torch.empty((n, cols), dtype=tdtype, device=dev)
            src = torch.empty(n, dtype=torch.int64, device=dev) if with_source_index else None
            if n:
                code = abi.DTYPE["float32" if tdtype == torch.float32 else "float64"]
                size = out.element_size()
                sink = abi.CloudSink(out.data_ptr(), n, cols * size, 0, code, 3 * size, code if with_timestamps else 0, 1)
                self.export_device_sink(sink, src.data_ptr() if src is not None else None,
                                        torch.cuda.current_stream(self.device).cuda_stream)
            return (out, src) if with_source_index else out
        dtype = np.dtype(dtype)
        if dtype not in (np.dtype(np.float32), np.dtype(np.float64)):
            raise ValueError("dtype must be float32 or float64")
        out = np.zeros((n, cols), dtype=dtype)
        src = np.zeros(n, dtype=np.uint64) if with_source_index else None
        if n:
            code = abi.DTYPE[dtype.name]
            sink = abi.CloudSink(out.ctypes.data, n, cols * dtype.itemsize, 0, code, 3 * dtype.itemsize,
                                 code if with_timestamps else 0, 1)
            self.export_sink(sink, src)
        return (out, src) if with_source_index else out

    def export_ply(self, dtype=np.float32, with_timestamps=False, with_source_index=False, normals=None):
        """The cloud as one PLY file's bytes, encoded on the device: element vertex with x y z in `dtype` (float32 ->
        float, float64 -> double), then optionally timestamp (same type), source_index (uint: the low 32 bits of the
        uint64 index) and nx ny nz (float) from `normals`, a Neighborhood.describe result over the export order (a
        NumPy array of neighborhood_description_dtype() or the device variant's uint8 tensor). Everything stays on the
        device until the file's one copy to the host."""
        import torch
        dtype = np.dtype(dtype)
        if dtype not in (np.dtype(np.float32), np.dtype(np.float64)):
            raise ValueError("dtype must be float32 or float64")
        pts = self.export(np.float64, with_timestamps=True, with_source_index=with_source_index, device=True)
        xyzt, src = pts if with_source_index else (pts, None)
        n = xyzt.shape[0]
        ply = "float" if dtype == np.float32 else "double"
        cols = [("vertex", k, ply, xyzt[:, i]) for i, k in enumerate("xyz")]
        if with_timestamps:
            cols.append(("vertex", "timestamp", ply, xyzt[:, 3]))
        if with_source_index:
            cols.append(("vertex", "source_index", "uint", src))
        if normals is not None:
            dev = xyzt.device
            rec = normals if _is_cuda_tensor(normals) else torch.from_numpy(
                np.ascontiguousarray(normals).view(np.uint8).reshape(len(normals), -1)).to(dev)
            if rec.shape[0] != n:
                raise ValueError("normals has %d descriptions for %d points" % (rec.shape[0], n))
            off = abi.neighborhood_description_dtype().fields["normal"][1]
            nrm = rec.view(torch.float64)[:, off // 8:off // 8 + 3] if n else torch.zeros((0, 3), dtype=torch.float64,
                                                                                         device=dev)
            cols += [("vertex", k, "float", nrm[:, i]) for i, k in enumerate(("nx", "ny", "nz"))]
        out, _ = self.b.ply_write(cols, device=self.device, num_items=n)
        return out.cpu().numpy().tobytes()


class Neighborhood:
    """slam::TNeighborhood's k-nearest index and descriptions over one point set on one device (cticp_neighborhood_*).
    search / describe take queries as an (m, 3) NumPy array (the host path) or a torch CUDA tensor on the index's device
    (fp64, contiguous; the outputs are CUDA tensors written in order with torch's current stream); None: the indexed
    points themselves, in index order (host outputs)."""

    def __init__(self, binding, points=None, device=0, handle=None):
        self.b = binding
        self.device = device
        self.h = C.c_void_p(handle) if handle is not None else C.c_void_p()
        if handle is not None:
            return
        if _is_cuda_tensor(points):
            import torch
            if points.device.index != device:
                raise ValueError("points must be on cuda:%d" % device)
            if points.dim() != 2 or points.shape[1] < 3 or points.stride(1) != 1 or \
                    points.dtype not in (torch.float32, torch.float64):
                raise ValueError("points must be an (N, >=3) float32 / float64 tensor with unit column stride")
            scan = abi.DeviceScan(points.data_ptr() if points.shape[0] else None, points.stride(0) * points.element_size(),
                                  None, 0, points.shape[0], abi.DTYPE["float32" if points.dtype == torch.float32 else
                                                                     "float64"], 0)
            binding.check(binding.fn("neighborhood_create_device")(C.byref(scan),
                                                                   C.c_void_p(torch.cuda.current_stream(device).cuda_stream),
                                                                   device, C.byref(self.h)))
        else:
            xyz = _as_f64_rows(points, 3)
            binding.check(binding.fn("neighborhood_create")(xyz.ctypes.data if len(xyz) else None, 24, len(xyz), device,
                                                            C.byref(self.h)))

    def close(self):
        if self.h:
            self.b.fn("neighborhood_destroy")(self.h)
        self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def num_points(self):
        return self.b.check(self.b.fn("neighborhood_num_points")(self.h))

    def num_rejected(self):
        return self.b.check(self.b.fn("neighborhood_num_rejected")(self.h))

    def _queries(self, queries):
        if queries is None:
            return None, self.num_points()
        q = _as_f64_rows(queries, 3)
        return q, len(q)

    def search(self, queries=None, k=1, max_radius=np.finfo(np.float64).max):
        """NearestNeighborSearchResult(k, max_radius) + SearchNearestNeighbors for every query: (indices (m, k) uint64,
        d2 (m, k) float64, counts (m,) int32); row q ascending by d2 (ties: lower index first), ~0 / +inf past its count."""
        if _is_cuda_tensor(queries):
            return self._search_device(queries, k, max_radius)
        q, m = self._queries(queries)
        idx = np.zeros((m, max(k, 0)), dtype=np.uint64)
        d2 = np.zeros((m, max(k, 0)), dtype=np.float64)
        cnt = np.zeros(m, dtype=np.int32)
        self.b.check(self.b.fn("neighborhood_search")(self.h, q.ctypes.data if q is not None and m else None, m, int(k),
                                                      float(max_radius), idx.ctypes.data, d2.ctypes.data,
                                                      cnt.ctypes.data))
        return idx, d2, cnt

    def describe(self, queries=None, k=20, max_radius=np.finfo(np.float64).max, values=abi.NB["ALL"],
                 linearity_threshold=0.8, planarity_threshold=0.8):
        """ComputeNeighborhood(values) + ClassifyNeighborhood(linearity, planarity) of each query's k nearest: an array
        of abi.neighborhood_description_dtype() (a torch uint8 tensor of 160-byte records for CUDA queries)."""
        if _is_cuda_tensor(queries):
            return self._describe_device(queries, k, max_radius, values, linearity_threshold, planarity_threshold)
        q, m = self._queries(queries)
        out = np.zeros(m, dtype=abi.neighborhood_description_dtype())
        self.b.check(self.b.fn("neighborhood_describe")(self.h, q.ctypes.data if q is not None and m else None, m, int(k),
                                                        float(max_radius), int(values), float(linearity_threshold),
                                                        float(planarity_threshold), out.ctypes.data if m else None))
        return out

    def _device_queries(self, queries):
        import torch
        if queries.device.index != self.device or queries.dtype != torch.float64 or queries.dim() != 2 or \
                queries.shape[1] != 3 or not queries.is_contiguous():
            raise ValueError("queries must be a contiguous (m, 3) float64 tensor on cuda:%d" % self.device)
        return torch, queries.shape[0], torch.cuda.current_stream(self.device).cuda_stream

    def _search_device(self, queries, k, max_radius):
        torch, m, stream = self._device_queries(queries)
        dev = queries.device
        idx = torch.empty((m, max(k, 0)), dtype=torch.int64, device=dev)
        d2 = torch.empty((m, max(k, 0)), dtype=torch.float64, device=dev)
        cnt = torch.empty(m, dtype=torch.int32, device=dev)
        if m:
            self.b.check(self.b.fn("neighborhood_search_device")(self.h, queries.data_ptr(), m, int(k), float(max_radius),
                                                                 idx.data_ptr(), d2.data_ptr(), cnt.data_ptr(),
                                                                 C.c_void_p(stream)))
        return idx, d2, cnt

    def _describe_device(self, queries, k, max_radius, values, lin_t, plan_t):
        torch, m, stream = self._device_queries(queries)
        out = torch.empty((m, abi.neighborhood_description_dtype().itemsize), dtype=torch.uint8, device=queries.device)
        if m:
            self.b.check(self.b.fn("neighborhood_describe_device")(self.h, queries.data_ptr(), m, int(k),
                                                                   float(max_radius), int(values), float(lin_t),
                                                                   float(plan_t), out.data_ptr(), C.c_void_p(stream)))
        return out


class SyntheticScene:
    """slam::Scene with SyntheticSensorAcquisition::GenerateFrame behind the C ABI (include/cticp.h, "Synthetic scenes
    and sequences"): the distance of points to every primitive and the generation of points and frames."""

    def __init__(self, binding, triangles=(), lines=(), spheres=(), balls=(), device=0):
        self.b = binding
        self.device = device
        self._arrays = [np.ascontiguousarray(np.asarray(a, dtype=np.float64).reshape(-1, w))
                        for a, w in ((triangles, 9), (lines, 6), (spheres, 4), (balls, 4))]
        args = []
        for a in self._arrays:
            args += [a.ctypes.data if len(a) else None, len(a)]
        self.h = C.c_void_p()
        binding.check(binding.fn("synthetic_scene_create")(*args, device, C.byref(self.h)))

    def close(self):
        if self.h:
            self.b.fn("synthetic_scene_destroy")(self.h)
        self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def num_primitives(self):
        return self.b.check(self.b.fn("synthetic_scene_num_primitives")(self.h))

    def distance(self, points):
        """Distance of each point (m, 3) to every primitive: an (m, num_primitives) array"""
        q = _as_f64_rows(np.asarray(points, dtype=np.float64).reshape(-1, 3), 3)
        out = np.zeros((len(q), self.num_primitives()))
        self.b.check(self.b.fn("synthetic_scene_distance")(self.h, q.ctypes.data, len(q), out.ctypes.data))
        return out

    def generate_points(self, num_points_per_primitive, location=None, distance=0.0, seed=0):
        """GeneratePoints (location None) or GeneratePointsCloseToLocation: (xyz (N, 3), src_index (N, 2) uint32)"""
        f = self.b.fn("synthetic_generate_points")
        loc = None if location is None else np.ascontiguousarray(location, dtype=np.float64).reshape(3)
        lp = None if loc is None else loc.ctypes.data
        n = self.b.check(f(self.h, num_points_per_primitive, lp, float(distance), int(seed), None, 0, None))
        xyz = np.zeros((n, 3))
        src = np.zeros((n, 2), dtype=np.uint32)
        self.b.check(f(self.h, num_points_per_primitive, lp, float(distance), int(seed), xyz.ctypes.data, n,
                       src.ctypes.data))
        return xyz, src

    @staticmethod
    def _frames(frames):
        if isinstance(frames, np.ndarray) and frames.dtype == abi.synthetic_frame_dtype():
            return np.ascontiguousarray(frames)
        out = np.zeros(len(frames), dtype=abi.synthetic_frame_dtype())
        for k, (b, e, fid) in enumerate(frames):
            out[k] = (b, e, fid)
        return out

    def generate_frames_sink(self, trajectory, frames, num_points_per_primitive, distance, seed, sink, src_index=None,
                             frame_ends=None):
        """cticp_synthetic_generate_frames into an abi.CloudSink in host memory; src_index (N, 2) uint32 and frame_ends
        (m,) uint64 host arrays. Returns the count."""
        fr = self._frames(frames)
        ends = frame_ends if frame_ends is not None else np.zeros(len(fr), dtype=np.uint64)
        return self.b.check(self.b.fn("synthetic_generate_frames")(
            self.h, trajectory.h, fr.ctypes.data, len(fr), num_points_per_primitive, float(distance), int(seed),
            C.byref(sink), None if src_index is None else src_index.ctypes.data, ends.ctypes.data))

    def generate_frames_device(self, trajectory, frames, num_points_per_primitive, distance, seed, sink, src_index_ptr,
                               frame_ends_ptr, stream=0):
        """cticp_synthetic_generate_frames_device: an abi.CloudSink, src_index and frame_ends in device memory (pointers),
        ordered after and before `stream`"""
        fr = self._frames(frames)
        return self.b.check(self.b.fn("synthetic_generate_frames_device")(
            self.h, trajectory.h, fr.ctypes.data, len(fr), num_points_per_primitive, float(distance), int(seed),
            C.byref(sink), C.c_void_p(src_index_ptr or None), C.c_void_p(frame_ends_ptr or None),
            C.c_void_p(stream or None)))

    def generate_frames(self, trajectory, frames, num_points_per_primitive, distance, seed=0, world=False,
                        with_source_index=False, device=False):
        """GenerateFrame of every frame ((begin_ts, end_ts, frame_id) triples or a synthetic_frame_dtype() array): a dict
        with xyz (N, 3) float64 (raw, or world with world=True), t (N,), frame_ends (m,) uint64 and, when asked,
        src_index (N, 2) uint32. NumPy arrays, or torch CUDA tensors with device=True (generated on the device on torch's
        current stream: one pass counts the points, a second writes them)."""
        fr = self._frames(frames)
        if device:
            return self._generate_frames_tensors(trajectory, fr, num_points_per_primitive, distance, seed, world,
                                                 with_source_index)
        ends = np.zeros(len(fr), dtype=np.uint64)
        count = self.generate_frames_sink(trajectory, fr, num_points_per_primitive, distance, seed,
                                          abi.CloudSink(None, 0, 32, 0, abi.DTYPE["float64"], 24, abi.DTYPE["float64"],
                                                        int(world)), None, ends)
        rec = np.zeros((count, 4))
        src = np.zeros((count, 2), dtype=np.uint32)
        sink = abi.CloudSink(rec.ctypes.data if count else None, count, 32, 0, abi.DTYPE["float64"], 24,
                             abi.DTYPE["float64"], int(world))
        self.generate_frames_sink(trajectory, fr, num_points_per_primitive, distance, seed, sink,
                                  src if with_source_index else None, ends)
        out = {"xyz": rec[:, :3], "t": rec[:, 3], "frame_ends": ends}
        if with_source_index:
            out["src_index"] = src
        return out

    def _generate_frames_tensors(self, trajectory, fr, n, distance, seed, world, with_source_index):
        import torch
        dev = torch.device("cuda", self.device)
        stream = torch.cuda.current_stream(self.device).cuda_stream
        ends = torch.zeros(len(fr), dtype=torch.int64, device=dev)
        empty = abi.CloudSink(None, 0, 32, 0, abi.DTYPE["float64"], 24, abi.DTYPE["float64"], int(world))
        self.generate_frames_device(trajectory, fr, n, distance, seed, empty, None, ends.data_ptr(), stream)
        count = int(ends[-1].item()) if len(fr) else 0
        rec = torch.empty((count, 4), dtype=torch.float64, device=dev)
        src = torch.empty((count, 2), dtype=torch.int32, device=dev) if with_source_index else None
        sink = abi.CloudSink(rec.data_ptr() if count else None, count, 32, 0, abi.DTYPE["float64"], 24,
                             abi.DTYPE["float64"], int(world))
        self.generate_frames_device(trajectory, fr, n, distance, seed, sink,
                                    src.data_ptr() if src is not None and count else None, ends.data_ptr(), stream)
        out = {"xyz": rec[:, :3], "t": rec[:, 3], "frame_ends": ends}
        if with_source_index:
            out["src_index"] = src
        return out


def _lidar_sensor(sensor):
    """(abi.LidarSensor, the elevation array it points to) of a synthetic.SensorModel or an abi.LidarSensor-like object
    (n_rings, n_azimuth, period, min_range, max_range, elevations in degrees top to bottom, noise_sigma)"""
    table = getattr(sensor, "elev_table_deg", None)
    if table is None and hasattr(sensor, "elev_max_deg"):
        table = np.linspace(sensor.elev_max_deg, sensor.elev_min_deg, sensor.n_rings)   # synthetic.generate_scan's rings
    elif table is None:
        table = sensor.elevations_deg
    elev = np.ascontiguousarray(table, dtype=np.float64).reshape(-1)
    if len(elev) != int(sensor.n_rings):
        raise ValueError("the elevation table has %d rings, n_rings is %d" % (len(elev), sensor.n_rings))
    s = abi.LidarSensor(elev.ctypes.data, int(sensor.n_rings), int(sensor.n_azimuth), float(sensor.period),
                        float(sensor.min_range), float(sensor.max_range), float(getattr(sensor, "noise_sigma", 0.0)))
    return s, elev


class LidarScene:
    """A spinning-LiDAR ray-cast scene behind the C ABI (include/cticp.h, "Spinning-LiDAR sweeps"): the ranges of given
    rays, and sweeps of a sensor along a ContinuousTrajectory into host arrays or torch CUDA tensors."""

    def __init__(self, binding, boxes=(), cylinders=(), ground=True, device=0):
        self.b = binding
        self.device = device
        self.boxes = np.ascontiguousarray(np.asarray(boxes, dtype=np.float64).reshape(-1, 7))
        self.cylinders = np.ascontiguousarray(np.asarray(cylinders, dtype=np.float64).reshape(-1, 4))
        self.h = C.c_void_p()
        binding.check(binding.fn("lidar_scene_create")(
            self.boxes.ctypes.data if len(self.boxes) else None, len(self.boxes),
            self.cylinders.ctypes.data if len(self.cylinders) else None, len(self.cylinders), int(bool(ground)),
            device, C.byref(self.h)))

    def close(self):
        if self.h:
            self.b.fn("lidar_scene_destroy")(self.h)
        self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def raycast(self, o, d, max_range, seed=0):
        """The range of each ray (origins o and unit directions d, (n, 3)), +inf where nothing is hit: a float64 array,
        or a CUDA tensor for contiguous float64 CUDA tensors on the scene's device (ordered on torch's current stream)."""
        if _is_cuda_tensor(o) or _is_cuda_tensor(d):
            import torch
            for a in (o, d):
                if not _is_cuda_tensor(a) or a.device.index != self.device or a.dtype != torch.float64 or \
                        a.dim() != 2 or a.shape[1] != 3 or not a.is_contiguous():
                    raise ValueError("o and d must be contiguous (n, 3) float64 tensors on cuda:%d" % self.device)
            if o.shape[0] != d.shape[0]:
                raise ValueError("o and d must have the same length")
            out = torch.empty(o.shape[0], dtype=torch.float64, device=o.device)
            if o.shape[0]:
                stream = torch.cuda.current_stream(self.device).cuda_stream
                self.b.check(self.b.fn("lidar_scene_raycast_device")(self.h, o.data_ptr(), d.data_ptr(), o.shape[0],
                                                                     float(max_range), int(seed) & (2 ** 64 - 1),
                                                                     out.data_ptr(), C.c_void_p(stream)))
            return out
        o = _as_f64_rows(o, 3)
        d = _as_f64_rows(d, 3)
        if len(o) != len(d):
            raise ValueError("o and d must have the same length")
        out = np.empty(len(o))
        if len(o):
            self.b.check(self.b.fn("lidar_scene_raycast")(self.h, o.ctypes.data, d.ctypes.data, len(o), float(max_range),
                                                          int(seed) & (2 ** 64 - 1), out.ctypes.data))
        return out

    @staticmethod
    def _frames(frames):
        """an abi.lidar_frame_dtype() array of (t0, frame_id) pairs or such an array"""
        if isinstance(frames, np.ndarray) and frames.dtype == abi.lidar_frame_dtype():
            return np.ascontiguousarray(frames)
        out = np.zeros(len(frames), dtype=abi.lidar_frame_dtype())
        for k, (t0, fid) in enumerate(frames):
            out[k] = (t0, fid)
        return out

    def sweeps_sink(self, trajectory, sensor, frames, seed, sink, ray_index=None, frame_ends=None):
        """cticp_lidar_generate_sweeps into an abi.CloudSink in host memory; ray_index (N,) uint32 and frame_ends (m,)
        uint64 host arrays. Returns the count."""
        s, elev = _lidar_sensor(sensor)
        fr = self._frames(frames)
        ends = frame_ends if frame_ends is not None else np.zeros(len(fr), dtype=np.uint64)
        n = self.b.check(self.b.fn("lidar_generate_sweeps")(
            self.h, trajectory.h, C.byref(s), fr.ctypes.data if len(fr) else None, len(fr), int(seed) & (2 ** 64 - 1),
            C.byref(sink), None if ray_index is None else ray_index.ctypes.data, ends.ctypes.data if len(fr) else None))
        del elev
        return n

    def sweeps_device(self, trajectory, sensor, frames, seed, sink, ray_index_ptr, frame_ends_ptr, stream=0):
        """cticp_lidar_generate_sweeps_device: an abi.CloudSink, ray_index and frame_ends in device memory (pointers),
        ordered after and before `stream`"""
        s, elev = _lidar_sensor(sensor)
        fr = self._frames(frames)
        rc = self.b.check(self.b.fn("lidar_generate_sweeps_device")(
            self.h, trajectory.h, C.byref(s), fr.ctypes.data if len(fr) else None, len(fr), int(seed) & (2 ** 64 - 1),
            C.byref(sink), C.c_void_p(ray_index_ptr or None), C.c_void_p(frame_ends_ptr or None),
            C.c_void_p(stream or None)))
        del elev
        return rc

    def sweeps(self, trajectory, sensor, frames, seed=0, dtype=np.float64, world=False, device=True):
        """Sweeps of `sensor` (a synthetic.SensorModel, with noise_sigma 0 unless it has one) along `trajectory` for each
        frame ((t0, frame_id) pairs or an abi.lidar_frame_dtype() array): a dict with xyz (N, 3) of `dtype` (raw, or world
        with world=True), t (N,) float64, ray_index (N,) and frame_ends (m,). torch CUDA tensors generated on torch's
        current stream with device=True (one pass counts the points, a second writes them); NumPy arrays otherwise."""
        fr = self._frames(frames)
        dt = np.dtype(dtype)
        if dt not in (np.dtype(np.float32), np.dtype(np.float64)):
            raise ValueError("dtype must be float32 or float64")
        code = abi.DTYPE["float32" if dt == np.float32 else "float64"]
        size = dt.itemsize
        step = 3 * size + 8 + (4 if size == 4 else 0)   # x y z, pad to 8, t
        toff = step - 8
        if device:
            import torch
            dev = torch.device("cuda", self.device)
            stream = torch.cuda.current_stream(self.device).cuda_stream
            ends = torch.zeros(len(fr), dtype=torch.int64, device=dev)
            if len(fr) == 0:
                return {"xyz": torch.empty((0, 3), dtype=getattr(torch, dt.name), device=dev),
                        "t": torch.empty(0, dtype=torch.float64, device=dev),
                        "ray_index": torch.empty(0, dtype=torch.int32, device=dev), "frame_ends": ends}
            empty = abi.CloudSink(None, 0, step, 0, code, toff, abi.DTYPE["float64"], int(world))
            self.sweeps_device(trajectory, sensor, fr, seed, empty, None, ends.data_ptr(), stream)
            count = int(ends[-1].item())
            rec = torch.empty((count, step), dtype=torch.uint8, device=dev)
            idx = torch.empty(count, dtype=torch.int32, device=dev)
            sink = abi.CloudSink(rec.data_ptr() if count else None, count, step, 0, code, toff, abi.DTYPE["float64"],
                                 int(world))
            self.sweeps_device(trajectory, sensor, fr, seed, sink, idx.data_ptr() if count else None, ends.data_ptr(),
                               stream)
            xyz = rec[:, :3 * size].view(getattr(torch, dt.name))
            t = rec[:, toff:].view(torch.float64).reshape(-1)
            return {"xyz": xyz, "t": t, "ray_index": idx, "frame_ends": ends}
        ends = np.zeros(len(fr), dtype=np.uint64)
        empty = abi.CloudSink(None, 0, step, 0, code, toff, abi.DTYPE["float64"], int(world))
        count = self.sweeps_sink(trajectory, sensor, fr, seed, empty, None, ends)
        rec = np.zeros(count, dtype=np.dtype({"names": ["xyz", "t"], "formats": [(dt, 3), np.float64],
                                              "offsets": [0, toff], "itemsize": step}))
        idx = np.zeros(count, dtype=np.uint32)
        sink = abi.CloudSink(rec.ctypes.data if count else None, count, step, 0, code, toff, abi.DTYPE["float64"],
                             int(world))
        self.sweeps_sink(trajectory, sensor, fr, seed, sink, idx, ends)
        return {"xyz": np.ascontiguousarray(rec["xyz"]), "t": np.ascontiguousarray(rec["t"]), "ray_index": idx,
                "frame_ends": ends}


class NcltHits:
    """An indexed NCLT velodyne_hits.bin stream on one device (include/cticp.h, "Dataset sequences")."""

    def __init__(self, binding, data, num_aggregated=220, final=True, device=0):
        self.b = binding
        self.device = device
        self.h = C.c_void_p()
        if _is_cuda_tensor(data):
            import torch
            if data.dtype != torch.uint8 or not data.is_contiguous() or data.device.index != device:
                raise ValueError("data must be a contiguous uint8 tensor on cuda:%d" % device)
            stream = torch.cuda.current_stream(device).cuda_stream
            binding.check(binding.fn("nclt_open_device")(data.data_ptr() if data.numel() else None, data.numel(),
                                                         int(num_aggregated), int(bool(final)), device,
                                                         C.c_void_p(stream), C.byref(self.h)))
        else:
            buf = np.frombuffer(data, dtype=np.uint8) if not isinstance(data, np.ndarray) else \
                np.ascontiguousarray(data).view(np.uint8).reshape(-1)
            binding.check(binding.fn("nclt_open")(buf.ctypes.data if len(buf) else None, len(buf), int(num_aggregated),
                                                  int(bool(final)), device, C.byref(self.h)))

    def close(self):
        if self.h:
            self.b.fn("nclt_destroy")(self.h)
        self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    @property
    def num_frames(self):
        return self.b.check(self.b.fn("nclt_num_frames")(self.h))

    @property
    def num_packets(self):
        return self.b.check(self.b.fn("nclt_num_packets")(self.h))

    @property
    def num_hits(self):
        return self.b.check(self.b.fn("nclt_num_hits")(self.h))

    @property
    def bytes_used(self):
        return self.b.check(self.b.fn("nclt_bytes_used")(self.h))

    @property
    def index_walked(self):
        """True when the one-thread walk built the index (a chain link failed), False for the parallel chain check"""
        return bool(self.b.check(self.b.fn("nclt_index_walked")(self.h)))

    def frame_info(self, first=0, m=None):
        """frames [first, first + m): an array of abi.nclt_frame_dtype() (num_points, t_first, t_max)"""
        m = self.num_frames - first if m is None else m
        out = np.zeros(max(m, 0), dtype=abi.nclt_frame_dtype())
        self.b.check(self.b.fn("nclt_frame_info")(self.h, first, m, out.ctypes.data if m else None))
        return out

    def read_sink(self, first, m, sink, frame_ends):
        """cticp_nclt_read_frames into an abi.CloudSink in host memory; frame_ends a (m,) uint64 array. Returns the count."""
        return self.b.check(self.b.fn("nclt_read_frames")(self.h, first, m, C.byref(sink),
                                                          frame_ends.ctypes.data if m else None))

    def read_device(self, first, m, sink, frame_ends_ptr, stream=0):
        """cticp_nclt_read_frames_device: an abi.CloudSink and frame_ends in device memory, ordered after and before
        `stream`"""
        return self.b.check(self.b.fn("nclt_read_frames_device")(self.h, first, m, C.byref(sink),
                                                                 C.c_void_p(frame_ends_ptr or None),
                                                                 C.c_void_p(stream or None)))

    def read(self, first=0, m=None, dtype=np.float64, device=True):
        """Frames [first, first + m) as a dict: xyz (N, 3) of `dtype`, t (N,) float64 in microseconds and frame_ends
        (m,): torch CUDA tensors decoded on torch's current stream with device=True, NumPy arrays otherwise."""
        m = self.num_frames - first if m is None else m
        dt = np.dtype(dtype)
        if dt not in (np.dtype(np.float32), np.dtype(np.float64)):
            raise ValueError("dtype must be float32 or float64")
        code = abi.DTYPE[dt.name]
        size = dt.itemsize
        step = 3 * size + 8 + (4 if size == 4 else 0)   # x y z, pad to 8, t
        toff = step - 8
        info = self.frame_info(first, m)
        count = int(info["num_points"].sum())
        if device:
            import torch
            dev = torch.device("cuda", self.device)
            rec = torch.empty((count, step), dtype=torch.uint8, device=dev)
            ends = torch.zeros(m, dtype=torch.int64, device=dev)
            sink = abi.CloudSink(rec.data_ptr() if count else None, count, step, 0, code, toff, abi.DTYPE["float64"], 0)
            if m:
                self.read_device(first, m, sink, ends.data_ptr(), torch.cuda.current_stream(self.device).cuda_stream)
            return {"xyz": rec[:, :3 * size].view(getattr(torch, dt.name)),
                    "t": rec[:, toff:].view(torch.float64).reshape(-1), "frame_ends": ends}
        rec = np.zeros(count, dtype=np.dtype({"names": ["xyz", "t"], "formats": [(dt, 3), np.float64],
                                              "offsets": [0, toff], "itemsize": step}))
        ends = np.zeros(m, dtype=np.uint64)
        sink = abi.CloudSink(rec.ctypes.data if count else None, count, step, 0, code, toff, abi.DTYPE["float64"], 0)
        if m:
            self.read_sink(first, m, sink, ends)
        return {"xyz": np.ascontiguousarray(rec["xyz"]), "t": np.ascontiguousarray(rec["t"]), "frame_ends": ends}
