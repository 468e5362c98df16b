"""The snapshot format of cticp_odometry_save / cticp_map_save (csrc/snapshot_format.h) built with plain g++: synthetic
odometry and map snapshots round-trip; every truncation, random single-bit flips, a wrong magic or version and
structural faults that carry a valid checksum (slot index out of range, repeated or decreasing, count > B, totals that
disagree with the counters, non-finite offsets, unknown frame ordinals) are refused."""
import os
import subprocess

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_snapshot_format(tmp_path):
    cxx = "/usr/bin/g++" if os.path.exists("/usr/bin/g++") else "g++"
    exe = str(tmp_path / "snapshot_format_test")
    r = subprocess.run([cxx, "-std=c++17", "-O2", "-Wall", "-I", os.path.join(ROOT, "ct_icp_b200", "csrc"),
                        os.path.join(ROOT, "tests", "cpp", "snapshot_format_test.cpp"), "-o", exe],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    r = subprocess.run([exe], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0 and "SNAPSHOT FORMAT OK" in r.stdout, r.stdout + r.stderr
