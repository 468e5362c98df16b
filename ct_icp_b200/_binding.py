"""Thin ctypes binding over a shared library that implements the include/cticp.h entry points.

`Binding(lib, prefix)` works for any library exporting `<prefix>odometry_create`, ... — the engine uses
prefix "cticp_"; the test-suite binds the CPU oracle (prefix "orc_") through the same class so both are
driven by identical calls. Nothing in this module computes anything: it marshals numpy arrays and PODs.
"""
import ctypes as C

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


def _snapshot_bytes(binding, fn, handle):
    n = binding.check(binding.fn(fn)(handle, None, 0))
    buf = C.create_string_buffer(n)
    m = binding.check(binding.fn(fn)(handle, buf, n))
    assert m == n, (m, n)
    return buf.raw


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
    def register_batch(self, odometries, scans, frame_ids, initial_estimates=None, motion_models=None):
        """One frame on each Odometry of `odometries` in one call (cticp_odometry_register_batch): the eligible
        Gauss-Newton loops run in one grouped launch, the eligible CERES / ROBUST loops in one grouped launch per LM mode
        (CERES nearest neighbour, CERES distance-based, ROBUST); the attempts of robust_registration frames run in rounds
        of such launches, apart from the plain frames; every result is that of the single-frame call.
        scans[i]: (xyz, timestamps) NumPy arrays (RegisterFrame's host path), (xyz, timestamps) torch CUDA tensors (read
        after the work queued on torch's current stream, as RegisterFrame), or an int staged slot (RegisterStaged).
        initial_estimates / motion_models: None or one entry (abi.Frame / abi.MotionPrior or None) per item.
        Returns the summaries; raises CticpError after the call when an item fails (.statuses: every item's status)."""
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
        if rc < 0:
            msg = self.fn("last_error")()
            raise CticpError(rc, msg.decode("utf-8", "replace") if msg else "", [items[i].status for i in range(B)])
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
