"""Profiling driver: registers `--frames` HDL-64 scans (device-resident input) so that ncu can list every launch
of steady-state RegisterFrame steps. Run under ncu; numbers printed under a profiler are
never bench values."""
import argparse
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import bench  # noqa: E402
import ct_icp_b200  # noqa: E402
from ct_icp_b200 import synthetic as syn  # noqa: E402

ap = argparse.ArgumentParser()
ap.add_argument("--frames", type=int, default=26)
ap.add_argument("--sensor", default="workload", help="workload (the bench workload's sensor on the suburb scene) | hdl64 (street scene) | dense128 (street scene)")
ap.add_argument("--workload", default="kitti64_gn", choices=sorted(bench.WORKLOADS))
args = ap.parse_args()
eng = ct_icp_b200.engine()
bench._WORKLOAD = args.workload
if args.sensor == "workload":
    seq = bench.make_scans(args.frames, bench.WORKLOADS[args.workload][0])
else:
    seq = syn.make_sequence(args.frames, {"hdl64": syn.HDL64, "dense128": syn.DENSE128}[args.sensor], seed=1234)
od = eng.odometry(bench.make_options(eng))
slots = [od.stage_frame(s["xyz"], s["t"]) for s in seq]
for i, s in enumerate(seq):
    sm = od.RegisterStaged(slots[i], s["frame_idx"])
    t = od.last_timing()
    print(i, "ok" if sm.success else "FAIL", "launches", t.kernel_launches, "total_ms %.3f ingest %.3f icp %.3f map %.3f" %
          (t.total_ms, t.ingest_ms, t.icp_ms, t.map_update_ms), "K", sm.num_keypoints, "F", sm.num_corrected_points)
