#!/bin/bash
# A/B of the loop synchronisation of k_gn_persistent (tagged hand-off words = default build, grid barriers = libcticp_b200_gridsync.so),
# alternating, same box: does it move the end-to-end numbers (e2e, e2e_dropin)? usage: bash tools/gpu_ab_sync.sh <tag>
TAG=${1:-x}; mkdir -p gpurun_out
for round in 1 2; do
  for b in flags gridsync; do
    lib=$PWD/ct_icp_b200/libcticp_b200.so; [ $b = gridsync ] && lib=$PWD/ct_icp_b200/libcticp_b200_gridsync.so
    CTICP_ENGINE_LIB=$lib timeout 600 python bench.py --no-extras --no-cpu-baseline > gpurun_out/${TAG}_${b}_${round}.json 2> gpurun_out/${TAG}_${b}_${round}.err
    python - gpurun_out/${TAG}_${b}_${round}.json $b $round <<'PY'
import json, sys
d = json.loads(open(sys.argv[1]).read().strip().splitlines()[-1])
e, p = d["e2e"], d["e2e_dropin"]
print("%-9s #%s step %.4f GN %.1f us | e2e mean %.4f med %.4f | dropin mean %.4f med %.4f max %.4f" % (sys.argv[2], sys.argv[3], d["ms_per_step"],
      d["roofline"]["us_per_launch"], e["ms_per_step"], e["ms_per_step_median"], p["ms_per_step"], p["ms_per_step_median"], p["ms_per_step_max"]))
PY
  done
done
