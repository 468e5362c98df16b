#!/usr/bin/env python
"""Throughput of synthetic frame generation on the device (cticp_synthetic_generate_frames_device).

Workloads:
  * courtyard: the whole reference sequence (tests/golden/synthetic_courtyard.json: 399 frames at 40 Hz, 300 points per
    primitive, 15 m), the workload of BASELINE.json configs[0];
  * scaled: ~10^4 random primitives spread over 200 m, 100 frames along a 100 m path, 100 points per primitive and a
    range that keeps every primitive: ~10^8 candidate points in one call.
For each: generation time (CUDA events, median of --reps calls after a warm-up), candidate and emitted points per
second, bytes written per second against the 3.35 TB/s HBM3 figure of the H100 SXM data sheet, and time per frame. On
the courtyard also: cticp_odometry_register_device time per frame (configs[0] options, first 30 frames), and the CPU
restatement (tests/oracle_synthetic) on the first 40 frames. Prints one JSON line with the card's name and power limit.
usage: python tools/bench_synthetic.py [--reps 5]"""
import argparse
import json
import math
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

HBM_BYTES_PER_S = 3.35e12


def card():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True)
    return r.stdout.strip().splitlines()[0] if r.returncode == 0 and r.stdout.strip() else "unknown"


def time_generation(scene, traj, frames, n, d, reps):
    """median ms of one device generation into a device sink (x, y, z, t fp64) with (primitive, point) pairs"""
    stream = torch.cuda.current_stream().cuda_stream
    ends = torch.zeros(len(frames), dtype=torch.int64, device="cuda")
    empty = abi.CloudSink(None, 0, 32, 0, abi.DTYPE["float64"], 24, abi.DTYPE["float64"], 0)
    scene.generate_frames_device(traj, frames, n, d, 1, empty, None, ends.data_ptr(), stream)
    count = int(ends[-1].item())
    rec = torch.empty((max(count, 1), 4), dtype=torch.float64, device="cuda")
    src = torch.empty((max(count, 1), 2), dtype=torch.int32, device="cuda")
    sink = abi.CloudSink(rec.data_ptr(), count, 32, 0, abi.DTYPE["float64"], 24, abi.DTYPE["float64"], 0)
    times = []
    for r in range(reps + 1):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        scene.generate_frames_device(traj, frames, n, d, 1, sink, src.data_ptr(), ends.data_ptr(), stream)
        b.record()
        torch.cuda.synchronize()
        if r:
            times.append(a.elapsed_time(b))
    return float(np.median(times)), count, rec, ends


def report(name, ms, count, frames, candidates):
    written = count * (32 + 8) + 8 * frames   # records, (primitive, point) pairs, frame ends
    s = ms / 1e3
    return {"workload": name, "frames": frames, "candidates": candidates, "emitted": count, "ms": round(ms, 3),
            "ms_per_frame": round(ms / frames, 4), "candidate_points_per_s": candidates / s, "emitted_points_per_s": count / s,
            "bytes_written_per_s": written / s, "hbm_share": written / s / HBM_BYTES_PER_S}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    args = ap.parse_args()
    eng = ct_icp_b200.engine()
    out = {"card": card(), "results": []}

    # courtyard
    with open(os.path.join(ROOT, "tests", "golden", "synthetic_courtyard.json")) as f:
        spec = json.load(f)
    seq = eng.synthetic_sequence(spec, num_frames=0)
    scene, traj = seq["scene"], seq["trajectory"]
    fr_all = np.zeros(len(seq["ground_truth"]) - 1, dtype=abi.synthetic_frame_dtype())
    ts = seq["ground_truth"]["dest_timestamp"]
    fr_all["begin_ts"], fr_all["end_ts"], fr_all["frame_id"] = ts[:-1], ts[1:], np.arange(len(fr_all))
    ms, count, rec, ends = time_generation(scene, traj, fr_all, 300, 15.0, args.reps)
    np_ = scene.num_primitives()
    r = report("courtyard", ms, count, len(fr_all), len(fr_all) * np_ * 300)
    # register_device per frame, configs[0] options
    o = eng.default_odometry_options()
    o.ct_icp_options.solver = abi.SOLVER["GN"]
    o.ct_icp_options.min_number_neighbors = 10
    o.ct_icp_options.num_iters_icp = 5
    o.map_options = eng.legacy_map_options(0.2, 20, 0.05)
    o.init_num_frames = 4
    o.debug_print = 0
    od = eng.odometry(o)
    e = ends.cpu().numpy().astype(np.int64)
    starts = np.concatenate([[0], e[:-1]])
    stream = torch.cuda.current_stream().cuda_stream
    reg = []
    for k in range(30):
        base = rec.data_ptr() + int(starts[k]) * 32
        scan = abi.DeviceScan(base, 32, base + 24, 32, int(e[k] - starts[k]), abi.DTYPE["float64"], abi.DTYPE["float64"])
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        sm = od.register_device(scan, k, stream=stream)
        reg.append(time.perf_counter() - t0)
        assert sm.success
    r["register_device_ms_per_frame_median"] = round(1e3 * float(np.median(reg[5:])), 3)
    # the CPU restatement on the first 40 frames
    from oracle_synthetic_lib import synthetic_oracle
    so = synthetic_oracle()
    so_seq = so.synthetic_sequence(spec, num_frames=0)
    t0 = time.perf_counter()
    so_seq["scene"].generate_frames(so_seq["trajectory"], fr_all[:40], 300, 15.0, seed=1)
    r["oracle_cpu_ms_per_frame"] = round(1e3 * (time.perf_counter() - t0) / 40, 3)
    out["results"].append(r)

    # scaled: ~10^4 primitives, ~10^8 candidates
    rng = np.random.default_rng(0)
    nt, nl, ns, nb = 6000, 2000, 1000, 1000
    tri = rng.uniform(-100, 100, (nt, 1, 3)) + rng.uniform(-2, 2, (nt, 3, 3))
    lines = rng.uniform(-100, 100, (nl, 1, 3)) + rng.uniform(-3, 3, (nl, 2, 3))
    sph = np.concatenate([rng.uniform(-100, 100, (ns, 3)), rng.uniform(0.2, 2, (ns, 1))], axis=1)
    ball = np.concatenate([rng.uniform(-100, 100, (nb, 3)), rng.uniform(0.2, 2, (nb, 1))], axis=1)
    big = eng.synthetic_scene(tri, lines, sph, ball)
    poses = []
    for k in range(11):
        a = 0.3 * k
        poses.append(abi.Pose.make([0, 0, math.sin(a / 2), math.cos(a / 2)], [10.0 * k - 50, 0.0, 1.5], float(k), k))
    btraj = eng.continuous_trajectory(poses)
    fr = np.zeros(100, dtype=abi.synthetic_frame_dtype())
    fr["begin_ts"], fr["end_ts"], fr["frame_id"] = np.arange(100) * 0.1, np.arange(1, 101) * 0.1, np.arange(100)
    ms, count, _, _ = time_generation(big, btraj, fr, 100, 400.0, args.reps)
    out["results"].append(report("scaled_1e4_primitives", ms, count, 100, 100 * (nt + nl + ns + nb) * 100))
    print(json.dumps(out))


if __name__ == "__main__":
    main()
