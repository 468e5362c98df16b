"""Scoring trajectories on the device against the CPU restatement of the reference (tests/oracle_eval).

Input: a KITTI-00-sized odometry-shaped ground truth (4541 poses, ~3.7 km) and B noisy estimates of it, B in {1, 16, 64};
kitti_evaluate with the driving lengths and trajectory_metrics with segment length 10. For each call: device time from
CUDA events recorded on the legacy default stream around the call (the engine's per-call stream is a blocking one, so
the events bracket its copies and kernels) and the wall clock of the synchronous call, both after a warm-up and over at
least --seconds of calls; then the wall clock of the oracle on the same input. Prints the GPU name and power limit and
one JSON line per (function, B).

    python tools/bench_eval.py [--seconds 1.0]
"""
import argparse
import json
import math
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import ct_icp_b200  # noqa: E402
from ct_icp_b200 import _abi as abi  # noqa: E402


def trajectory(rng, n, step=0.815):
    gt = np.zeros(n, dtype=abi.pose_dtype())
    yaw, tr = 0.0, np.zeros(3)
    for i in range(n):
        yaw += rng.normal(scale=0.02)
        q = np.array([rng.normal(scale=0.005), rng.normal(scale=0.005), math.sin(yaw / 2), math.cos(yaw / 2)])
        gt[i]["quat"] = q / np.linalg.norm(q)
        gt[i]["tr"] = tr
        gt[i]["dest_timestamp"] = 0.1 * i
        gt[i]["dest_frame_id"] = i
        tr = tr + step * np.array([math.cos(yaw), math.sin(yaw), 0.01 * rng.normal()])
    return gt


def noisy(rng, gt):
    e = gt.copy()
    q = e["quat"] + rng.normal(scale=0.002, size=(len(e), 4))
    e["quat"] = q / np.linalg.norm(q, axis=1, keepdims=True)
    e["tr"] = e["tr"] + np.cumsum(rng.normal(scale=0.02, size=(len(e), 3)), axis=0)
    return e


def timed(fn, seconds, torch):
    for _ in range(3):
        fn()
    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    dev, wall, t_end = [], [], time.perf_counter() + seconds
    while time.perf_counter() < t_end or len(dev) < 5:
        start.record()
        t0 = time.perf_counter()
        fn()
        t1 = time.perf_counter()
        end.record()
        end.synchronize()
        dev.append(start.elapsed_time(end))
        wall.append((t1 - t0) * 1e3)
    return float(np.median(dev)), float(np.median(wall)), len(dev)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--seconds", type=float, default=1.0)
    ap.add_argument("--n", type=int, default=4541)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        sys.exit("bench_eval: no CUDA device (this measurement has no CPU fallback)")
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True).stdout.strip().splitlines()
    print("GPU:", q[0] if q else torch.cuda.get_device_name(0))
    from oracle_eval_lib import eval_oracle
    eng, orc = ct_icp_b200.engine(), eval_oracle()
    rng = np.random.default_rng(2026)
    gt = trajectory(rng, args.n)
    ests = [noisy(rng, gt) for _ in range(64)]
    length = float(np.sum(np.linalg.norm(np.diff(gt["tr"], axis=0), axis=1)))
    for B in (1, 16, 64):
        e = ests[0] if B == 1 else ests[:B]
        for name, fn in (("kitti_evaluate", lambda b, x: b.kitti_evaluate(gt, x, "driving")),
                         ("trajectory_metrics", lambda b, x: b.trajectory_metrics(gt, x, 10.0))):
            dev_ms, wall_ms, calls = timed(lambda: fn(eng, e), args.seconds, torch)
            t0 = time.perf_counter()
            fn(orc, e)
            orc_ms = (time.perf_counter() - t0) * 1e3
            print(json.dumps({"function": name, "n": args.n, "length_m": round(length, 1), "B": B,
                              "device_event_ms": round(dev_ms, 4), "device_wall_ms": round(wall_ms, 4),
                              "calls": calls, "oracle_wall_ms": round(orc_ms, 3),
                              "gpu": q[0] if q else None}))


if __name__ == "__main__":
    main()
