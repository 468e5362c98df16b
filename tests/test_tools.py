"""tools/summarize_ncu.py on a stored Nsight Compute launch list (tests/golden/ncu_launches_steady_state.csv, a parser
fixture: one capture of steady-state frames of an earlier build) against the per-frame launch shares stored beside it."""
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden")


def test_launch_shares_from_the_committed_capture(tmp_path):
    out = tmp_path / "shares.json"
    r = subprocess.run([sys.executable, os.path.join(ROOT, "tools", "summarize_ncu.py"), "launches",
                        os.path.join(GOLDEN, "ncu_launches_steady_state.csv"), str(out)],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    d = json.loads(out.read_text())
    assert len(d["launches"]) == 11                      # launches per steady-state frame of the captured build
    assert abs(sum(x["share"] for x in d["launches"]) - 1.0) < 1e-9
    top = max(d["share_by_kernel"], key=d["share_by_kernel"].get)
    assert "k_gn_persistent" in top and d["share_by_kernel"][top] > 0.5
    committed = json.load(open(os.path.join(GOLDEN, "ncu_launch_shares.json")))
    assert abs(committed["sum_us"] - d["sum_us"]) < 1e-6
