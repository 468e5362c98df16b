"""Aggregate scans/s of B odometry sequences served from one GPU: B single-frame calls per step (RegisterStaged, one
handle after the other) against one cticp_odometry_register_batch call per step on the same staged scans, for
B in {1, 2, 4, 8, 16}.

Workloads: the bench workload (BASELINE.json configs[1]: bench.py's GN options and KITTI-shape 64-beam scans, one seed
per sequence) and a small-scan one (the same options on 16-beam ~10k-pt scans); bench.py's kitti64_ceres workload
(BASELINE.json configs[2]: driving_config.yaml, solver CERES) on the same two scan kinds, and its options with solver
ROBUST (robust_registration off) on the small scans; and the kitti64_ceres options with robust_registration on (the
attempt ladder of RobustRegistration, run in rounds of grouped launches) on both scan kinds. Every sequence first registers
--preroll frames untimed (past init_num_frames), then --warmup frames, then --steps timed steps. A step is host-timed
and ends in a device synchronise. The two modes have their own handles over the same scans and take turns step by step.

Checks: each batched trajectory equals its sequential twin byte for byte when the batch's problems fit on the device
with their solo grids; otherwise a second batched run over the first frames must reproduce the first run byte for byte.
A separate run under torch.profiler gives the device time of the ICP launches per step (k_gn_persistent and
k_lm_persistent: B solo launches against one grouped launch). The card name and power limit come from a read-only nvidia-smi query in the same
run.

--single-frame: instead, for each workload, one handle with the device tail against one with CTICP_DEVICE_TAIL=0 (the
host-side tail), single-frame calls on the same staged scans, taking turns frame by frame; reports the median frame time
of each and the attempts per frame.

usage: python tools/bench_odometry_batch.py [--steps 20] [--warmup 3] [--preroll 20] [--sizes 1,2,4,8,16] [--out DIR]
                                            [--workloads a,b] [--single-frame]
"""
import argparse
import json
import multiprocessing
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import bench  # noqa: E402
import ct_icp_b200  # noqa: E402
from ct_icp_b200 import synthetic as syn  # noqa: E402

# name: (sensor, bench.py workload whose options the handles take, solver override, robust_registration)
WORKLOADS = {"kitti64_gn": ("HDL64E", "kitti64_gn", None, 0), "small16_gn": ("SMALL16", "kitti64_gn", None, 0),
             "kitti64_ceres": ("HDL64E", "kitti64_ceres", None, 0), "small16_ceres": ("SMALL16", "kitti64_ceres", None, 0),
             "small16_robust": ("SMALL16", "kitti64_ceres", "ROBUST", 0),
             "kitti64_ladder": ("HDL64E", "kitti64_ceres", None, 1), "small16_ladder": ("SMALL16", "kitti64_ceres", None, 1)}
KERNELS = ("k_gn_persistent", "k_lm_persistent")


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
        return out[0] if out else "unknown"
    except (OSError, subprocess.SubprocessError):
        return "unknown"


def make_options(eng, workload):
    _, bench_workload, solver, robust = WORKLOADS[workload]
    bench._WORKLOAD = bench_workload
    o = bench.make_options(eng)
    if solver:
        from ct_icp_b200 import _abi as abi
        o.ct_icp_options.solver = abi.SOLVER[solver]
    o.robust_registration = robust
    return o


def make_sequence(n_frames, sensor, seed):
    scene = syn.UrbanScene(1234, profile=bench.SCENE_PROFILE)
    return syn.make_sequence(n_frames, getattr(syn, sensor), seed=seed, scene=scene)


def trajectory_bytes(od, n=None):
    tr = od.Trajectory()
    return b"".join(bytes(memoryview(f)) for f in tr[:n])


class Arm:
    """B handles over B sequences, their scans staged on each handle"""

    def __init__(self, eng, seqs, workload):
        self.eng = eng
        self.seqs = seqs
        self.ods = [eng.odometry(make_options(eng, workload)) for _ in seqs]
        self.slots = [[od.stage_frame(s["xyz"], s["t"]) for s in seq] for od, seq in zip(self.ods, seqs)]

    def step(self, k, batched):
        if batched:
            self.eng.register_batch(self.ods, [slots[k] for slots in self.slots], [seq[k]["frame_idx"] for seq in self.seqs])
        else:
            for od, slots, seq in zip(self.ods, self.slots, self.seqs):
                od.RegisterStaged(slots[k], seq[k]["frame_idx"])

    def close(self):
        for od in self.ods:
            od.clear_staged()
            od.close()


def icp_device_ms(eng, seqs, workload, first, steps, batched, torch):
    """per ICP kernel (KERNELS): mean device time of its launches per step and launches per step, from a torch.profiler
    run of its own"""
    from torch.profiler import ProfilerActivity, profile
    arm = Arm(eng, seqs, workload)
    for k in range(first):
        arm.step(k, batched)
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for k in range(first, first + steps):
            arm.step(k, batched)
        torch.cuda.synchronize()
    out = {}
    for kernel in KERNELS:
        us = [e.device_time_total for e in prof.events() if kernel in e.name]
        out[kernel] = (sum(us) / 1000.0 / steps, len(us) / steps)
    arm.close()
    return out


def single_frame(eng, seqs, workload, args, torch):
    """device tail against host tail (CTICP_DEVICE_TAIL, read when a handle is created), one handle each, frame by frame
    in turns on the same staged scans"""
    arms = {}
    for mode, env in (("device_tail", "1"), ("host_tail", "0")):
        old = os.environ.get("CTICP_DEVICE_TAIL")
        os.environ["CTICP_DEVICE_TAIL"] = env
        try:
            arms[mode] = Arm(eng, seqs, workload)
        finally:
            if old is None:
                os.environ.pop("CTICP_DEVICE_TAIL")
            else:
                os.environ["CTICP_DEVICE_TAIL"] = old
    first = args.preroll + args.warmup
    frame_s = {m: [] for m in arms}
    attempts = {m: [] for m in arms}
    od = {m: arms[m].ods[0] for m in arms}
    for k in range(first + args.steps):
        for m in (("device_tail", "host_tail") if k % 2 == 0 else ("host_tail", "device_tail")):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            sm = od[m].RegisterStaged(arms[m].slots[0][k], seqs[0][k]["frame_idx"])
            torch.cuda.synchronize()
            if k >= first:
                frame_s[m].append(time.perf_counter() - t0)
                attempts[m].append(sm.number_of_attempts)
    same = trajectory_bytes(od["device_tail"]) == trajectory_bytes(od["host_tail"])
    row = {"workload": workload, "mode": "single_frame", "trajectories_identical": same}
    for m in arms:
        row[f"{m}_frame_ms_median"] = 1e3 * float(np.median(frame_s[m]))
        row[f"{m}_frame_ms_min"] = 1e3 * float(np.min(frame_s[m]))
        row[f"{m}_attempts_per_frame"] = float(np.mean(attempts[m]))
    row["host_over_device_tail"] = row["host_tail_frame_ms_median"] / row["device_tail_frame_ms_median"]
    for a in arms.values():
        a.close()
    return row


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--preroll", type=int, default=20)
    ap.add_argument("--sizes", default="1,2,4,8,16")
    ap.add_argument("--workloads", default=",".join(WORKLOADS))
    ap.add_argument("--out", default=None)
    ap.add_argument("--single-frame", action="store_true")
    args = ap.parse_args()
    import torch

    eng = ct_icp_b200.engine()
    sizes = [int(x) for x in args.sizes.split(",")]
    first = args.preroll + args.warmup
    n_frames = first + args.steps
    result = {"card": card(), "steps": args.steps, "warmup": args.warmup, "preroll": args.preroll, "rows": []}
    print("card (name, power limit):", result["card"], flush=True)
    for wl in args.workloads.split(","):
        with multiprocessing.get_context("fork").Pool(min(max(sizes), os.cpu_count() or 1)) as pool:
            all_seqs = pool.starmap(make_sequence, [(n_frames, WORKLOADS[wl][0], 1234 + b) for b in range(max(sizes))])
        if args.single_frame:
            row = single_frame(eng, all_seqs[:1], wl, args, torch)
            result["rows"].append(row)
            print(json.dumps(row), flush=True)
            continue
        for B in sizes:
            seqs = all_seqs[:B]
            arms = {"sequential": Arm(eng, seqs, wl), "batch": Arm(eng, seqs, wl)}
            step_s = {m: [] for m in arms}
            for k in range(n_frames):
                for m in (("sequential", "batch") if k % 2 == 0 else ("batch", "sequential")):
                    torch.cuda.synchronize()
                    t0 = time.perf_counter()
                    arms[m].step(k, m == "batch")
                    torch.cuda.synchronize()
                    if k >= first:
                        step_s[m].append(time.perf_counter() - t0)
            identical = all(trajectory_bytes(a) == trajectory_bytes(b)
                            for a, b in zip(arms["sequential"].ods, arms["batch"].ods))
            check = "bit-identical to sequential"
            if not identical:   # the problems share the device's CTAs: the batch must reproduce itself
                again = Arm(eng, seqs, wl)
                for k in range(args.preroll):
                    again.step(k, True)
                assert all(trajectory_bytes(a, args.preroll) == trajectory_bytes(b)
                           for a, b in zip(arms["batch"].ods, again.ods)), (wl, B, "batch not reproducible")
                again.close()
                check = "oversubscribed: differs from sequential, reproducible run to run"
            groups = arms["batch"].ods[0].last_timing().icp_batch_groups
            for a in arms.values():
                a.close()
            dev = {m: icp_device_ms(eng, seqs, wl, first, min(args.steps, 10), m == "batch", torch)
                   for m in ("sequential", "batch")}
            row = {"workload": wl, "B": B,
                   "sequential_scans_per_s": B / float(np.median(step_s["sequential"])),
                   "batch_scans_per_s": B / float(np.median(step_s["batch"])),
                   "sequential_step_ms_median": 1e3 * float(np.median(step_s["sequential"])),
                   "batch_step_ms_median": 1e3 * float(np.median(step_s["batch"])),
                   "icp_batch_groups": groups, "check": check}
            for m in dev:
                for kernel, (ms, n) in dev[m].items():
                    short = kernel.split("_")[1]   # gn / lm
                    row[f"{short}_device_ms_per_step_{m}"] = ms
                    row[f"{short}_launches_per_step_{m}"] = n
            row["speedup"] = row["batch_scans_per_s"] / row["sequential_scans_per_s"]
            result["rows"].append(row)
            print(json.dumps(row), flush=True)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "bench_odometry_batch.json"), "w") as f:
            json.dump(result, f, indent=1)


if __name__ == "__main__":
    main()
