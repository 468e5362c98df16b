"""The reference's odometry runner (command/odometry_runner.cpp OdometryRunner::Run and SaveTrajectoryAndMetrics) over
the sequences of a dataset, on the device: every frame is read on the GPU (datasets.py), registered with
Odometry.register_device, its trajectory written as <sequence>.PLY (save_poses_ply) and scored against the ground truth
into metrics.yaml (ContinuousTrajectory.kitti_evaluate).

With RunnerOptions.concurrent_sequences = N > 1, up to N sequences run side by side: each round reads the next frame of
every active sequence and registers all of them in one cticp_odometry_register_batch call (CTICP_BATCH_DEVICE items).
A sequence that ends or fails leaves the batch and the next one joins; its reader is released when it leaves. The
files written are those of the serial run, up to summation order when the batch's problems do not fit on the device
together (DESIGN §5.13).
"""
import math
import os
import time

import numpy as np

from . import _abi as abi
from . import datasets
from ._binding import CticpError

METRIC_KEYS = ("MAX_APE", "MEAN_APE", "MEAN_RPE", "success", "finished", "MEAN_LOCAL_ERROR", "MAX_LOCAL_ERROR",
               "INDEX_MAX_LOCAL_ERROR", "Average(ms)", "AVG_NUM_ATTEMPTS")


def mid_frame_pose(begin, end):
    """begin.InterpolatePoseAlpha(end, 0.5, begin.dest_frame_id) (include/SlamCore/types.h:434-452): Eigen's slerp
    at alpha 0.5 (not renormalised) and the lerp of the translations and of the dest timestamps"""
    if begin.ref_frame_id != end.ref_frame_id:
        raise ValueError("Invalid operation: Cannot interpolate two frames not expressed in the same reference frame.")
    a = 0.5
    q0, q1 = begin.quat[:], end.quat[:]
    d = q0[0] * q1[0] + q0[1] * q1[1] + q0[2] * q1[2] + q0[3] * q1[3]
    if abs(d) >= 1.0 - np.finfo(np.float64).eps:
        s0, s1 = 1.0 - a, a
    else:
        theta = math.acos(abs(d))
        sin_theta = math.sin(theta)
        s0, s1 = math.sin((1.0 - a) * theta) / sin_theta, math.sin(a * theta) / sin_theta
    if d < 0:
        s1 = -s1
    p = abi.Pose()
    p.quat[:] = [s0 * q0[i] + s1 * q1[i] for i in range(4)]
    p.tr[:] = [(1.0 - a) * begin.tr[i] + a * end.tr[i] for i in range(3)]
    p.ref_frame_id, p.ref_timestamp = begin.ref_frame_id, begin.ref_timestamp
    p.dest_frame_id = begin.dest_frame_id
    p.dest_timestamp = (1.0 - a) * begin.dest_timestamp + a * end.dest_timestamp
    return p


def _yaml_double(x):
    if math.isnan(x):
        return ".nan"
    if math.isinf(x):
        return ".inf" if x > 0 else "-.inf"
    return "%.17g" % x


def metrics_yaml(metrics):
    """GenerateMetricYAMLNode (src/SlamCore/eval.cxx:114-133) as text: sequences in name order, each with the
    reference's keys in its insertion order. Doubles are written with 17 significant digits (.nan / .inf / -.inf),
    so they read back bit for bit; the layout is block YAML, not necessarily yaml-cpp's emitter's bytes."""
    import json
    lines = []
    for name in sorted(metrics):
        m = metrics[name]
        lines.append(json.dumps(name) + ":")
        for k in METRIC_KEYS:
            v = m[k]
            text = ("true" if v else "false") if isinstance(v, bool) else str(v) if isinstance(v, int) else \
                _yaml_double(float(v))
            lines.append("  %s: %s" % (json.dumps(k) if "(" in k else k, text))
    return "\n".join(lines) + "\n"


def read_metrics_yaml(path):
    """a metrics.yaml back as {sequence: {key: value}} with the reference's types (bool, int, double)"""
    from . import config
    out = {}
    for name, node in config.load_config(path).items():
        out[name] = {}
        for k in METRIC_KEYS:
            conv = config.as_bool if k in ("success", "finished") else \
                config.as_int if k == "INDEX_MAX_LOCAL_ERROR" else config.as_double
            out[name][k] = conv(node[k], k)
    return out


class _Run:
    """one sequence of the run: OdometryRunner's per-sequence locals and its Summary"""

    def __init__(self, order, name, sequence):
        self.order, self.name, self.seq = order, name, sequence
        self.od = None
        self.gt = None
        self.frame_id = 0
        self.sum_time = 0.0
        self.avg_time_ms = -1.0
        self.failed = False


def _register_device_batch(binding, runs, frames):
    """one cticp_odometry_register_batch call over CTICP_BATCH_DEVICE items (Binding.register_batch with CUDA tensors):
    (summary or None, message) per run, so an item the engine refuses fails its own sequence only"""
    statuses = []
    outs = binding.register_batch([r.od for r in runs], [(f["xyz"], f["t"]) for f in frames],
                                  [r.frame_id for r in runs], statuses=statuses)
    first_err = binding.fn("last_error")() if any(statuses) else None   # the first failing item's message
    res = []
    for out, st in zip(outs, statuses):
        if st == 0:
            res.append((out, None))
        else:
            res.append((None, first_err.decode("utf-8", "replace") if first_err else "status %d" % st))
            first_err = None
    return res


class OdometryRunner:
    """OdometryRunner(dataset) with its Options: `sequences` is a list of (label, sequence) as
    datasets.load_dataset_from_options returns it, `options` a config.RunnerOptions. Run() returns False when a frame
    failed with exit_early (as the reference, which stops there), True otherwise. After Run: summaries (per sequence:
    num_frames, avg_time_ms, trajectory of end poses, success), metrics (what metrics.yaml holds) and output_path."""

    def __init__(self, binding, sequences, options, device=0, log=None):
        self.b, self.sequences, self.options, self.device = binding, list(sequences), options, device
        self.log = log or (lambda msg: None)
        self.summaries, self.metrics, self.output_path = {}, {}, None

    # ---- SaveTrajectoryAndMetrics --------------------------------------------------------------------------------
    def _save(self, r, is_driving=True):
        frames = r.od.Trajectory()
        poses = []
        for f in frames:
            if not poses and not self.options.save_mid_frame:
                poses.append(f.begin_pose)
            poses.append(mid_frame_pose(f.begin_pose, f.end_pose) if self.options.save_mid_frame else f.end_pose)
        with open(os.path.join(self.output_path, r.name + ".PLY"), "wb") as f:
            f.write(self.b.save_poses_ply(poses, device=self.device))
        if r.gt is None:
            return
        # EvaluatePoses(poses, LinearContinuousTrajectory(gt), driving): the runner's poses sit in the ground-truth
        # slot, so pairs and distances come from them and the ground truth is interpolated at their timestamps
        traj = self.b.continuous_trajectory(datasets.pose_list(r.gt), device=self.device)
        try:
            e = traj.kitti_evaluate(poses, lengths="driving" if is_driving else "indoor")
        finally:
            traj.close()
        self.metrics[r.name] = {"MAX_APE": e["max_ape"], "MEAN_APE": e["mean_ape"], "MEAN_RPE": e["mean_rpe"],
                                "success": False, "finished": False, "MEAN_LOCAL_ERROR": e["mean_local_err"],
                                "MAX_LOCAL_ERROR": e["max_local_err"],
                                "INDEX_MAX_LOCAL_ERROR": int(e["index_max_local_err"]),
                                "Average(ms)": r.avg_time_ms, "AVG_NUM_ATTEMPTS": -1.0}
        self._write_metrics()

    def _write_metrics(self):
        with open(os.path.join(self.output_path, "metrics.yaml"), "w") as f:
            f.write(metrics_yaml(self.metrics))

    def _forget(self, r):
        """the outputs of a sequence the serial run would never have started (a concurrent run with exit_early)"""
        self.summaries.pop(r.name, None)
        if self.output_path is None:
            return
        path = os.path.join(self.output_path, r.name + ".PLY")
        if os.path.exists(path):
            os.remove(path)
        if self.metrics.pop(r.name, None) is not None:
            self._write_metrics()

    # ---- the per-sequence steps of Run ---------------------------------------------------------------------------
    def _start(self, r):
        self.log("Running the Odometry on the sequence named " + r.name)
        gt = r.seq.GroundTruth()
        r.gt = gt if gt is not None and len(gt) else None
        o = self.options.odometry_options.copy()
        if self.options.progress_bar or not self.options.debug_information:
            o.debug_print = 0
            o.ct_icp_options.debug_print = 0
        self.summaries[r.name] = {"num_frames": 0, "avg_time_ms": -1.0, "trajectory": [], "success": False}
        r.od = self.b.odometry(o, device=self.device)

    def _after_frame(self, r, summary, message, elapsed_ms):
        """the loop body after RegisterFrame: returns "next", "stop" (the sequence ends) or "exit" (exit_early)"""
        s = self.summaries[r.name]
        ok = summary is not None and bool(summary.success)
        if summary is not None:
            s["trajectory"].append(summary.frame.end_pose)
        if self.output_path is not None and r.frame_id > 0 and r.frame_id % self.options.compute_metrics_period == 0:
            self._save(r, bool(self.options.use_outdoor_evaluation))
        r.sum_time += elapsed_ms
        r.frame_id += 1
        r.avg_time_ms = s["avg_time_ms"] = r.sum_time / r.frame_id
        s["num_frames"] = r.frame_id
        if not ok:
            msg = message if summary is None else summary.error_message.decode("utf-8", "replace")
            self.log("Error while running SLAM for sequence %s, at frame index %d. Error Message: %s"
                     % (r.name, r.frame_id, msg))
            r.failed = True
            return "exit" if self.options.exit_early else "stop"
        return "next"

    def _finish(self, r, status):
        if status != "exit" and self.output_path is not None:
            self._save(r)   # the final save: driving lengths, the reference's default argument
        self.summaries[r.name]["success"] = not r.failed
        r.seq.close()
        if r.od is not None:
            r.od.close()
            r.od = None

    # ---- Run -------------------------------------------------------------------------------------------------------
    def Run(self):
        if not self.sequences:
            self.log("No sequence in the Dataset ! Returning early")
            return False
        if self.options.output_results:
            path = self.options.output_dir
            if self.options.generate_directory_prefix:
                path = os.path.join(path, time.strftime("%Y-%m-%d_%X", time.localtime()))
            os.makedirs(path or ".", exist_ok=True)
            self.output_path = path or "."
        runs, used = [], set()
        for i, (label, seq) in enumerate(self.sequences):
            name = label
            while name in used:
                name += "#"
            used.add(name)
            runs.append(_Run(i, name, seq))
        if self.options.concurrent_sequences <= 1:
            return self._run_serial(runs)
        return self._run_concurrent(runs)

    def _run_serial(self, runs):
        import torch
        stream = torch.cuda.current_stream(self.device).cuda_stream
        for r in runs:
            self._start(r)
            status = "next"
            while status == "next" and r.seq.HasNext():
                frame = r.seq.NextFrame()
                summary, message = None, None
                t0 = time.perf_counter()
                try:
                    summary = r.od.register_device(datasets.device_scan(frame), r.frame_id, stream=stream)
                except CticpError as e:   # an option combination the engine refuses fails the sequence
                    message = str(e)
                elapsed = (time.perf_counter() - t0) * 1e3
                status = self._after_frame(r, summary, message, elapsed)
            self._finish(r, status)
            if status == "exit":
                return False
        return True

    def _run_concurrent(self, runs):
        pending, active = list(runs), []
        stop_at = None   # the order of the first sequence that failed with exit_early
        while pending or active:
            while pending and len(active) < self.options.concurrent_sequences and stop_at is None:
                r = pending.pop(0)
                self._start(r)
                active.append(r)
            done = [r for r in active if not r.seq.HasNext()]
            for r in done:
                active.remove(r)
                self._finish(r, "stop")
            if not active:
                if stop_at is not None or not pending:
                    break
                continue
            frames = [r.seq.NextFrame() for r in active]
            t0 = time.perf_counter()
            results = _register_device_batch(self.b, active, frames)
            elapsed = (time.perf_counter() - t0) * 1e3
            for r, (summary, message) in list(zip(active, results)):
                status = self._after_frame(r, summary, message, elapsed)
                if status == "next":
                    continue
                active.remove(r)
                self._finish(r, status)
                if status == "exit" and (stop_at is None or r.order < stop_at):
                    stop_at = r.order
            if stop_at is not None:   # the serial run never starts the sequences after the one that failed
                for r in [r for r in active if r.order > stop_at]:
                    active.remove(r)
                    r.seq.close()
                    r.od.close()
                    self._forget(r)
                for r in [r for r in runs if r.order > stop_at and r.od is None and r.name in self.summaries]:
                    self._forget(r)
                pending = []
        return stop_at is None
