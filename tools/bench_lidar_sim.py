#!/usr/bin/env python
"""Throughput of spinning-LiDAR sweeps on the device (cticp_lidar_generate_sweeps_device).

Workloads, on the suburb scene of synthetic.UrbanScene(1234) along synthetic.Trajectory:
  * HDL-64E sweeps (64 x 2083 rays), 1 and 100 frames per call;
  * DENSE-128 sweeps (128 x 2400 rays), 1 and 100 frames per call.
For each: time per call (CUDA events, median of --reps calls after a warm-up), rays per second and microseconds per
sweep. Also: tools/raycast.c with
OpenMP on the same HDL-64E rays on this host (threads reported), and device generation plus
cticp_odometry_register_device per frame over a short HDL-64E sequence. Prints one JSON line with the card's name and
power limit.
usage: python tools/bench_lidar_sim.py [--reps 5]"""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import numpy as np  # noqa: E402
import torch  # noqa: E402

import ct_icp_b200  # noqa: E402
from ct_icp_b200 import _abi as abi  # noqa: E402
from ct_icp_b200 import synthetic as syn  # noqa: E402
import lidar_sim_ref as ref  # noqa: E402


def card():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True)
    return r.stdout.strip().splitlines()[0] if r.returncode == 0 and r.stdout.strip() else "unknown"


def time_sweeps(scene, traj, sensor, frames, reps):
    """median ms of one call into a device sink (x, y, z, t fp64, raw) with ray indices; the point count"""
    stream = torch.cuda.current_stream().cuda_stream
    ends = torch.zeros(len(frames), dtype=torch.int64, device="cuda")
    empty = abi.CloudSink(None, 0, 32, 0, abi.DTYPE["float64"], 24, abi.DTYPE["float64"], 0)
    scene.sweeps_device(traj, sensor, frames, 1, empty, None, ends.data_ptr(), stream)
    count = int(ends[-1].item())
    rec = torch.empty((max(count, 1), 4), dtype=torch.float64, device="cuda")
    idx = torch.empty(max(count, 1), dtype=torch.int32, device="cuda")
    sink = abi.CloudSink(rec.data_ptr(), count, 32, 0, abi.DTYPE["float64"], 24, abi.DTYPE["float64"], 0)
    times = []
    for r in range(reps + 1):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        scene.sweeps_device(traj, sensor, frames, 1, sink, idx.data_ptr(), ends.data_ptr(), stream)
        b.record()
        torch.cuda.synchronize()
        if r:
            times.append(a.elapsed_time(b))
    return float(np.median(times)), count


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("no CUDA device: this benchmark measures the GPU and has no CPU fallback")
    eng = ct_icp_b200.engine()
    urban = syn.UrbanScene(1234, profile="suburb")
    t_build = time.perf_counter()
    scene = eng.lidar_scene(urban.boxes, urban.cyl)
    t_build = time.perf_counter() - t_build
    traj = syn.Trajectory(height=1.73)
    tr = eng.continuous_trajectory(ref.trajectory_poses(traj, 11.0))
    out = {"card": card(), "boxes": len(urban.boxes), "cylinders": len(urban.cyl),
           "scene_create_ms": round(t_build * 1e3, 2), "workloads": {}}
    for sensor in (syn.HDL64E, syn.DENSE128):
        rays = sensor.n_rings * sensor.n_azimuth
        for m in (1, 100):
            frames = [(k * sensor.period, k) for k in range(m)]
            ms, count = time_sweeps(scene, tr, sensor, frames, args.reps)
            out["workloads"]["%s x%d" % (sensor.name, m)] = {
                "ms_per_call": round(ms, 3), "us_per_sweep": round(ms * 1e3 / m, 1),
                "rays_per_s": round(rays * m / (ms * 1e-3)), "points": count}
    # the host caster with OpenMP on the same HDL-64E rays (one sweep)
    sensor = syn.HDL64E
    quat, trn = ref.device_columns(tr, sensor, 0.0)
    j = np.tile(np.arange(sensor.n_azimuth), sensor.n_rings)
    o = trn[j]
    d = ref.qrot(ref.qnormalized(quat)[j], ref.sensor_directions(sensor))
    ref.raycast(urban.boxes, urban.cyl, o[:1000], d[:1000], sensor.max_range, 1)   # loads the library
    t = time.perf_counter()
    ref.raycast(urban.boxes, urban.cyl, o, d, sensor.max_range, 1234 * 1000003)
    t = time.perf_counter() - t
    out["raycast_c_openmp"] = {"threads": os.environ.get("OMP_NUM_THREADS") or os.cpu_count(),
                               "ms_per_sweep": round(t * 1e3, 1), "rays_per_s": round(len(o) / t)}
    # generation plus register_device per frame
    opts = eng.default_odometry_options()
    opts.ct_icp_options.solver = abi.SOLVER["GN"]
    opts.ct_icp_options.min_number_neighbors = 10
    opts.map_options = eng.legacy_map_options(1.0, 20, 0.1)
    opts.init_num_frames = 3
    opts.debug_print = 0
    od = eng.odometry(opts)
    noisy = syn.SensorModel(**{k: getattr(sensor, k) for k in syn.SensorModel.__dataclass_fields__})
    noisy.noise_sigma = 0.02
    stream = torch.cuda.current_stream().cuda_stream
    rec = torch.empty((sensor.n_rings * sensor.n_azimuth, 4), dtype=torch.float64, device="cuda")
    ends = torch.zeros(1, dtype=torch.int64, device="cuda")
    sink = abi.CloudSink(rec.data_ptr(), rec.shape[0], 32, 0, abi.DTYPE["float64"], 24, abi.DTYPE["float64"], 0)
    per = []
    for k in range(30):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        scene.sweeps_device(tr, noisy, [(k * sensor.period, k)], 1234, sink, None, ends.data_ptr(), stream)
        n = int(ends[0].item())
        scan = abi.DeviceScan(rec.data_ptr(), 32, rec.data_ptr() + 24, 32, n, abi.DTYPE["float64"], abi.DTYPE["float64"])
        s = od.register_device(scan, k, stream=stream)
        b.record()
        torch.cuda.synchronize()
        assert s.success, s.error_message
        if k >= 5:
            per.append(a.elapsed_time(b))
    out["generate_plus_register_ms_per_frame"] = round(float(np.median(per)), 3)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
