"""The robust ladder's decision (csrc/frame_policy.h robust_attempt_decide: AssessRegistration with the robust branch,
the acceptance rule of RobustRegistration, the robust branch of UpdateMap, the insert overrides) built with plain g++ and
checked against a restatement of the reference's control flow over thresholds just below, at and above their values,
ICP failure flags, attempt positions, attempt budgets, consecutive failures, minimal levels and room_for."""
import os
import subprocess

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_robust_attempt_decision(tmp_path):
    cxx = "/usr/bin/g++" if os.path.exists("/usr/bin/g++") else "g++"
    exe = str(tmp_path / "robust_policy_test")
    r = subprocess.run([cxx, "-std=c++17", "-O2", "-Wall", "-Wno-unknown-pragmas", "-I", "/usr/local/cuda/include", "-I",
                        os.path.join(ROOT, "ct_icp_b200", "csrc"), "-I", os.path.join(ROOT, "include"),
                        os.path.join(ROOT, "tests", "cpp", "robust_policy_test.cpp"), "-o", exe], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    r = subprocess.run([exe], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0 and "ROBUST POLICY OK" in r.stdout, r.stdout + r.stderr
