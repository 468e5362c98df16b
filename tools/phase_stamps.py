"""Phase split of the fused sampler (k_sample_fused) and the fused map update (k_map_update_fused), frame by frame.

Needs a -DCTICP_DEBUG_TIMERS build of the engine (csrc/Makefile BUILD=build_timers OUT=../libcticp_b200_timers.so
EXTRA=-DCTICP_DEBUG_TIMERS) and a GPU:

    CTICP_ENGINE_LIB=$PWD/ct_icp_b200/libcticp_b200_timers.so python tools/phase_stamps.py --frames 30

Runs tools/profile_step.py with CTICP_DEBUG_TIMERS=1 and reads the "[cticp] phase ends" lines the engine prints per
launch: the end of each phase as the latest %globaltimer over the CTAs, in µs after the first CTA started. Prints each
phase's length (its end minus the previous phase's end) per frame, then the median over the last `--last` frames.
The stamps add a CTA barrier per phase and a stream synchronisation per launch: compare them between builds, not with
bench.py's times.
"""
import argparse
import os
import re
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LINE = re.compile(r"\[cticp\] phase ends (\S+) \(us\):(.*)")


def parse(text):
    """[(kernel, [(label, end_us), ...])] in launch order"""
    out = []
    for line in text.splitlines():
        m = LINE.search(line)
        if m:
            out.append((m.group(1), [(k, float(v)) for k, v in (kv.split("=") for kv in m.group(2).split())]))
    return out


def spans(ends):
    """phase lengths from cumulative ends; a phase the launch skipped (end 0) has no length"""
    prev, res = 0.0, []
    for label, t in ends:
        res.append((label, t - prev if t > 0 else None))
        if t > 0:
            prev = t
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=30)
    ap.add_argument("--workload", default="kitti64_gn")
    ap.add_argument("--last", type=int, default=10, help="frames in the median")
    args = ap.parse_args()
    env = dict(os.environ, CTICP_DEBUG_TIMERS="1")
    r = subprocess.run([sys.executable, os.path.join(ROOT, "tools", "profile_step.py"), "--frames", str(args.frames),
                        "--workload", args.workload], env=env, capture_output=True, text=True)
    if r.returncode != 0:
        sys.stderr.write(r.stdout[-2000:] + r.stderr[-4000:])
        return r.returncode
    launches = parse(r.stderr)
    if not launches:
        sys.stderr.write("no phase stamps: is CTICP_ENGINE_LIB a -DCTICP_DEBUG_TIMERS build?\n")
        return 1
    per_kernel = {}
    for kernel, ends in launches:
        sp = spans(ends)
        per_kernel.setdefault(kernel, []).append(sp)
        print("%-20s total %7.2f  " % (kernel, max(t for _, t in ends)) +
              "  ".join("%s %s" % (k, "-" if v is None else "%.2f" % v) for k, v in sp))
    print("\nmedian over the last %d launches (us)" % args.last)
    for kernel, rows in per_kernel.items():
        rows = rows[-args.last:]
        labels = [k for k, _ in rows[-1]]
        cells = []
        for i, k in enumerate(labels):
            vals = [row[i][1] for row in rows if i < len(row) and row[i][1] is not None]
            cells.append("%s %s" % (k, "%.2f" % statistics.median(vals) if vals else "-"))
        print("%-20s " % kernel + "  ".join(cells))
    return 0


if __name__ == "__main__":
    sys.exit(main())
