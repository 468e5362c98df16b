"""Device time per launch of each kernel of a RegisterFrame step, from torch.profiler (needs a GPU).

    python tools/kernel_times.py [--workload kitti64_gn] [--frames 40] [--skip 25]

Registers `--frames` scans of the bench workload from staged device input (bench.py's timed path), profiles every
frame after the first `--skip`, and prints mean / min / max µs per launch and launches per frame of every kernel,
longest first. A run of its own: the profiler slows the host, so these are kernel times, not step times.
"""
import argparse
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import bench  # noqa: E402
import ct_icp_b200  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workload", default="kitti64_gn", choices=sorted(bench.WORKLOADS))
    ap.add_argument("--frames", type=int, default=40)
    ap.add_argument("--skip", type=int, default=25)
    args = ap.parse_args()
    import torch
    from torch.profiler import ProfilerActivity, profile
    eng = ct_icp_b200.engine()
    bench._WORKLOAD = args.workload
    seq = bench.make_scans(args.frames, bench.WORKLOADS[args.workload][0])
    od = eng.odometry(bench.make_options(eng))
    slots = [od.stage_frame(s["xyz"], s["t"]) for s in seq]
    for i in range(args.skip):
        od.RegisterStaged(slots[i], seq[i]["frame_idx"])
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for i in range(args.skip, args.frames):
            od.RegisterStaged(slots[i], seq[i]["frame_idx"])
        torch.cuda.synchronize()
    frames = args.frames - args.skip
    times = {}
    for e in prof.events():
        if e.device_time_total > 0:
            times.setdefault(e.name, []).append(e.device_time_total)
    print("%s, %d frames: us per launch mean / min / max, launches per frame" % (args.workload, frames))
    for name, us in sorted(times.items(), key=lambda kv: -sum(kv[1])):
        print("%8.2f %8.2f %8.2f  %5.2f  %s" % (sum(us) / len(us), min(us), max(us), len(us) / frames, name[:100]))
    return 0


if __name__ == "__main__":
    sys.exit(main())
