#!/usr/bin/env python
"""Throughput of the odometry runner (ct_icp_b200/runner.py) over a dataset of many sequences, serial against
side-by-side registration (concurrent_sequences 1, 2, 4, 8).

Workload: K KITTI_raw-layout sequences (<root>/<NN>/frames/frame_%04d.ply, float x y z timestamp), each F HDL-64
sweeps of the lidar-sim suburb scene (synthetic.UrbanScene(1234)) along the same drive with its own noise seed, written
with datasets.write_ply_frames. The runner reads every frame on the device (PLY decode on the host, KITTI filter on the
GPU) and registers it with the odometry options of config/odometry/driving_config.yaml (--solver overrides the solver);
output_results is false, so no file is written. One warm-up run precedes the timed ones; each setting runs --reps
times, alternating settings, and the median is reported.

Reported per setting: frames/s over the whole run, and the split of its wall time into reading (NextFrame, ended by a
device synchronise) and registration (the rest: register_device or the batched call). Prints one JSON line with the
card's name and power limit.
usage: python tools/bench_run_config.py [--sequences 8] [--frames 60] [--reps 3] [--solver GN]"""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import numpy as np  # noqa: E402
import torch  # noqa: E402

import ct_icp_b200  # noqa: E402
from ct_icp_b200 import _abi as abi  # noqa: E402
from ct_icp_b200 import config, datasets, runner  # noqa: E402
from ct_icp_b200 import synthetic as syn  # noqa: E402
import lidar_sim_ref as lref  # noqa: E402


def card():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return r.stdout.strip().splitlines()[0] if r.returncode == 0 and r.stdout.strip() else "unknown"


def write_sequences(eng, root, K, F):
    scene, traj = syn.UrbanScene(1234, profile="suburb"), syn.Trajectory(height=1.0)
    sc = eng.lidar_scene(scene.boxes, scene.cyl)
    tr = eng.continuous_trajectory(lref.trajectory_poses(traj, F * 0.1 + 0.2))
    points = 0
    for k in range(K):
        out = sc.sweeps(tr, syn.HDL64, [(i * syn.HDL64.period, i) for i in range(F)], seed=k + 1, device=False)
        datasets.write_ply_frames(eng, out["xyz"], out["t"], out["frame_ends"], os.path.join(root, "%02d" % k,
                                                                                              "frames"))
        points += int(out["xyz"].shape[0])
    return points


class _Timed:
    """a sequence whose NextFrame is timed, ended by a device synchronise"""

    def __init__(self, seq, clock):
        self.seq, self.clock = seq, clock

    def NextFrame(self):
        t0 = time.perf_counter()
        f = self.seq.NextFrame()
        torch.cuda.synchronize()
        self.clock[0] += time.perf_counter() - t0
        return f

    def __getattr__(self, name):
        return getattr(self.seq, name)


def run_once(eng, root, K, F, options, concurrent):
    d = config.DatasetOptions()
    d.dataset, d.root_path, d.use_all_datasets = "KITTI_raw", root, False
    d.sequence_options = [config.SequenceOptions("%02d" % k, 0, F) for k in range(K)]
    clock = [0.0]
    seqs = [(label, _Timed(s, clock)) for label, s in datasets.load_dataset_from_options(eng, d)]
    options.concurrent_sequences = concurrent
    r = runner.OdometryRunner(eng, seqs, options)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    ok = r.Run()
    torch.cuda.synchronize()
    wall = time.perf_counter() - t0
    frames = sum(s["num_frames"] for s in r.summaries.values())
    failed = [n for n, s in r.summaries.items() if not s["success"]]
    return {"wall_s": wall, "read_s": clock[0], "frames": frames, "ok": ok, "failed": failed}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sequences", type=int, default=8)
    ap.add_argument("--frames", type=int, default=60)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--solver", choices=sorted(abi.SOLVER), default=None)
    ap.add_argument("--settings", default="1,2,4,8")
    args = ap.parse_args()
    eng = ct_icp_b200.engine()
    cfg = config.load_config(os.path.join(ROOT, "tests", "golden", "configs", "odometry", "driving_config.yaml"))
    options = config.load_runner_options(cfg, eng)
    options.output_results = False
    options.exit_early = False
    if args.solver:
        options.odometry_options.ct_icp_options.solver = abi.SOLVER[args.solver]
    settings = [int(s) for s in args.settings.split(",")]
    res = {"card": card(), "sequences": args.sequences, "frames_per_sequence": args.frames,
           "solver": [k for k, v in abi.SOLVER.items() if v == options.odometry_options.ct_icp_options.solver][0]}
    with tempfile.TemporaryDirectory() as root:
        res["points"] = write_sequences(eng, root, args.sequences, args.frames)
        run_once(eng, root, 2, 5, options, 2)   # warm-up: module loads, both paths
        runs = {n: [] for n in settings}
        for _ in range(args.reps):
            for n in settings:
                runs[n].append(run_once(eng, root, args.sequences, args.frames, options, n))
    out = {}
    for n, rs in runs.items():
        wall = float(np.median([r["wall_s"] for r in rs]))
        read = float(np.median([r["read_s"] for r in rs]))
        out[str(n)] = {"frames_per_s": round(rs[0]["frames"] / wall, 1), "wall_s": round(wall, 3),
                       "read_s": round(read, 3), "register_s": round(wall - read, 3), "frames": rs[0]["frames"],
                       "all_ok": all(r["ok"] for r in rs), "failed": rs[0]["failed"]}
    res["concurrent_sequences"] = out
    print(json.dumps(res))


if __name__ == "__main__":
    main()
