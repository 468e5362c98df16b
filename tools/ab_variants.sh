#!/bin/bash
# A/B of experiment builds of the engine (compile-time variants of the kernels) against the default build.
#
#   tools/ab_variants.sh build            # here (no GPU needed): nvcc cross-compiles ct_icp_b200/libcticp_b200_<name>.so
#   tools/ab_variants.sh run [outdir]     # on the GPU box (inside ONE gpurun call): GN parity tests + bench per build
#
# Variants (name:flags). A variant's bench line only counts if its parity tests pass.
#   bulk        -DCTICP_SEL_BULK            the stencil's point runs staged in shared memory by cp.async.bulk + mbarrier
#                                           (UBLKCP / SYNCS: the north star's "TMA staging") instead of per-lane loads
#   prefetch2/6 -DCTICP_SEL_PREFETCH=2 / 6  2 / 6 chunks of 32 point loads in flight per batch (default 4)
#   warps8      -DCTICP_GATHER_WARPS=8      8 warps per gather CTA (two CTAs per SM) instead of 16
#   warps20/24  -DCTICP_GATHER_WARPS=20/24  20 / 24 warps per gather CTA (96 / 80 registers per thread, smaller staging areas):
#                                           2940 / 3528 warps in the grid instead of 2352 — one keypoint per warp up to that K
#   timers      -DCTICP_DEBUG_TIMERS        clock64 stamps in the solver CTA of k_gn_persistent (built here, not benchmarked)
#   selv1       -DCTICP_SEL_V1              the selection's first cut (owner by binary search over shuffles, separate histogram
#                                           pass, butterfly sums): what the default path of gather_select.cuh replaced
#   gridsync    -DCTICP_GN_GRID_BARRIERS    k_gn_persistent with two cg::grid.sync() per iteration around the tagged hand-off words
#   noprune     -DCTICP_NO_VOXEL_PRUNE      the gather loads every voxel of the stencil (no box-vs-radius prune)
set -u
ROOT="$(cd "$(dirname "$0")/.." && pwd)"
VARIANTS=("selv1:-DCTICP_SEL_V1" "bulk:-DCTICP_SEL_BULK" "prefetch2:-DCTICP_SEL_PREFETCH=2" "prefetch6:-DCTICP_SEL_PREFETCH=6 -DCTICP_SEL_CAP=224"
          "warps8:-DCTICP_GATHER_WARPS=8" "warps20:-DCTICP_GATHER_WARPS=20 -DCTICP_SEL_CAP=128 -DCTICP_SEL_PREFETCH=2"
          "warps24:-DCTICP_GATHER_WARPS=24 -DCTICP_SEL_CAP=96 -DCTICP_SEL_PREFETCH=2" "timers:-DCTICP_DEBUG_TIMERS"
          "gridsync:-DCTICP_GN_GRID_BARRIERS" "noprune:-DCTICP_NO_VOXEL_PRUNE")
case "${1:-}" in
build)
    for v in "${VARIANTS[@]}"; do
        name="${v%%:*}"; flags="${v#*:}"
        make -C "$ROOT/ct_icp_b200/csrc" -j8 BUILD="build_$name" OUT="../libcticp_b200_$name.so" EXTRA="$flags" \
            > /dev/null || { echo "build of $name failed"; exit 1; }
        echo "built libcticp_b200_$name.so ($flags)"
    done ;;
run)
    out="${2:-$ROOT/gpurun_out/ab}"; mkdir -p "$out"
    cd "$ROOT"
    timeout 600 python bench.py --no-cpu-baseline --no-extras > "$out/bench_default.json" 2> "$out/bench_default.err"
    for v in "${VARIANTS[@]}"; do
        name="${v%%:*}"
        lib="$ROOT/ct_icp_b200/libcticp_b200_$name.so"
        [ -f "$lib" ] || continue
        [ "$name" = "timers" ] && continue   # instrumented build (tools/gpu_check.sh prints its stamps), not a candidate
        CTICP_ENGINE_LIB="$lib" timeout 900 python -m pytest tests -m gpu -q -n 6 -k "gn or neighborhoods or small or suburb" \
            > "$out/pytest_$name.log" 2>&1
        echo "rc=$?" >> "$out/pytest_$name.log"
        CTICP_ENGINE_LIB="$lib" timeout 600 python bench.py --no-cpu-baseline --no-extras > "$out/bench_$name.json" 2> "$out/bench_$name.err"
    done
    python - "$out" <<'PY'
import glob, json, os, sys
rows = []
for f in sorted(glob.glob(os.path.join(sys.argv[1], "bench_*.json"))):
    name = os.path.basename(f)[6:-5]
    try:
        d = json.loads(open(f).read().strip().splitlines()[-1])
        log = os.path.join(sys.argv[1], "pytest_%s.log" % name)
        tests = " ".join(open(log).read().strip().splitlines()[-2:]) if os.path.exists(log) else "(default build)"
        rows.append({"variant": name, "ms_per_step": d["ms_per_step"], "gn_loop_us": d["roofline"]["us_per_launch"],
                     "e2e_ms": d["e2e"]["ms_per_step"], "tests": tests})
        print("%-12s step %.4f ms  GN loop %.1f us  e2e %.4f ms  | %s" % (name, d["ms_per_step"], d["roofline"]["us_per_launch"],
                                                                        d["e2e"]["ms_per_step"], tests))
    except Exception as e:
        print(f, "unreadable:", e)
json.dump(rows, open(os.path.join(sys.argv[1], "summary.json"), "w"), indent=1)
PY
    ;;
*) echo "usage: $0 build | run [outdir]"; exit 2 ;;
esac
