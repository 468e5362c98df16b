#!/bin/bash
# A/B of k_gn_persistent's loop hand-off against an earlier revision of the engine.
#
#   tools/gn_handoff_ab.sh build [rev]     # no GPU needed: the engine of `rev` (default HEAD; HEAD~1 once this change is
#                                          # committed) from a git worktree as ct_icp_b200/libcticp_b200_parent.so, and the
#                                          # -DCTICP_DEBUG_TIMERS builds of both (libcticp_b200_parent_timers.so / _timers.so)
#   tools/gn_handoff_ab.sh run [outdir]    # on the GPU: bench.py five times per build and the hand-off floor
#                                          # (CTICP_DEBUG_FLAGS=3: no gather work, no solve) three times per build,
#                                          # the builds alternating; card, power limit and SM clock of the same session
#   tools/gn_handoff_ab.sh outputs [outdir]  # on the GPU: --dump-outputs of kitti64_gn, dense128_gn and kitti64_ceres from
#                                          # both builds compared byte for byte, dense128_gn timing, the solver / warp stamps
#                                          # of the timers builds, tools/bench_icp_batch.py per build
# Results go to outdir (default: under $TMPDIR). run and outputs are separate so that each takes under ten minutes.
set -u
ROOT="$(cd "$(dirname "$0")/.." && pwd)"
LIB="$ROOT/ct_icp_b200"
summ() {   # ms_per_step and the GN launch of bench.py result lines
    python - "$@" <<'PY'
import json, sys
for f in sys.argv[1:]:
    try:
        d = json.loads(open(f).read().strip().splitlines()[-1])
        print("%-40s ms_per_step %.4f  GN launch %.1f us  serial share %.3f" % (f.rsplit("/", 1)[-1], d["ms_per_step"],
              d["roofline"]["us_per_launch"], d["roofline"].get("serial_reduce_and_solve_share", float("nan"))))
    except Exception as e:
        print(f, "unreadable:", e)
PY
}
case "${1:-}" in
build)
    rev="${2:-HEAD}"
    wt="$(mktemp -d)"
    git -C "$ROOT" worktree add --detach "$wt" "$rev" > /dev/null || exit 1
    make -C "$wt/ct_icp_b200/csrc" -j8 OUT="$LIB/libcticp_b200_parent.so" > /dev/null &&
    make -C "$wt/ct_icp_b200/csrc" -j8 BUILD=build_timers OUT="$LIB/libcticp_b200_parent_timers.so" EXTRA=-DCTICP_DEBUG_TIMERS > /dev/null
    rc=$?
    git -C "$ROOT" worktree remove --force "$wt"
    [ $rc -eq 0 ] || { echo "build of $rev failed"; exit 1; }
    make -C "$LIB/csrc" -j8 > /dev/null &&
    make -C "$LIB/csrc" -j8 BUILD=build_timers OUT=../libcticp_b200_timers.so EXTRA=-DCTICP_DEBUG_TIMERS > /dev/null || exit 1
    echo "built libcticp_b200_parent.so ($rev), libcticp_b200.so, and their timers builds" ;;
run)
    out="${2:-${TMPDIR:-/tmp}/gn_handoff_ab/run}"; mkdir -p "$out"; cd "$ROOT"
    nvidia-smi --query-gpu=name,power.limit,clocks.max.sm --format=csv > "$out/gpu.txt"
    for i in 1 2 3 4 5; do
        for b in parent branch; do
            lib="$LIB/libcticp_b200.so"; [ $b = parent ] && lib="$LIB/libcticp_b200_parent.so"
            CTICP_ENGINE_LIB="$lib" timeout 300 python bench.py --no-extras --no-cpu-baseline > "$out/bench_${b}_$i.json" 2> "$out/bench_${b}_$i.err"
        done
    done
    for i in 1 2 3; do
        for b in parent branch; do
            lib="$LIB/libcticp_b200.so"; [ $b = parent ] && lib="$LIB/libcticp_b200_parent.so"
            CTICP_DEBUG_FLAGS=3 CTICP_ENGINE_LIB="$lib" timeout 300 python bench.py --no-extras --no-cpu-baseline \
                > "$out/floor_${b}_$i.json" 2> "$out/floor_${b}_$i.err"
        done
    done
    nvidia-smi --query-gpu=name,power.limit,clocks.sm --format=csv >> "$out/gpu.txt"
    summ "$out"/bench_*.json "$out"/floor_*.json | tee "$out/summary.txt" ;;
outputs)
    out="${2:-${TMPDIR:-/tmp}/gn_handoff_ab/outputs}"; mkdir -p "$out"; cd "$ROOT"
    nvidia-smi --query-gpu=name,power.limit,clocks.max.sm --format=csv > "$out/gpu.txt"
    for wl in kitti64_gn dense128_gn kitti64_ceres; do
        for b in parent branch; do
            lib="$LIB/libcticp_b200.so"; [ $b = parent ] && lib="$LIB/libcticp_b200_parent.so"
            CTICP_ENGINE_LIB="$lib" timeout 300 python bench.py --no-extras --no-cpu-baseline --workload $wl \
                --dump-outputs "$out/dump_${b}_$wl" > "$out/wl_${b}_$wl.json" 2> "$out/wl_${b}_$wl.err"
        done
        for f in "$out/dump_parent_$wl"/*; do
            cmp "$f" "$out/dump_branch_$wl/$(basename "$f")" && echo "identical $wl/$(basename "$f")" || echo "DIFFERENT $wl/$(basename "$f")"
        done | tee -a "$out/cmp.txt"
    done
    for b in parent branch; do
        lib="$LIB/libcticp_b200_timers.so"; [ $b = parent ] && lib="$LIB/libcticp_b200_parent_timers.so"
        CTICP_ENGINE_LIB="$lib" CTICP_DEBUG_TIMERS=1 timeout 300 python tools/profile_step.py --frames 30 > "$out/timers_$b.txt" 2>&1
        lib="$LIB/libcticp_b200.so"; [ $b = parent ] && lib="$LIB/libcticp_b200_parent.so"
        CTICP_ENGINE_LIB="$lib" timeout 300 python tools/bench_icp_batch.py --batches 1,4,16 > "$out/batch_$b.txt" 2>&1
    done
    summ "$out"/wl_*.json | tee "$out/summary.txt" ;;
*) echo "usage: $0 build [rev] | run [outdir] | outputs [outdir]"; exit 2 ;;
esac
