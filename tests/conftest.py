import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs an H100 (sm_90) CUDA device: pytest -m gpu")


@pytest.fixture(scope="session")
def orc():
    """CPU oracle binding (test infrastructure)."""
    from oracle_lib import oracle
    return oracle()


@pytest.fixture(scope="session")
def eng():
    """Engine binding (CUDA). GPU tests only."""
    import ct_icp_b200
    return ct_icp_b200.engine()


_SEQ_CACHE = {}


def get_sequence(name, n_frames):
    """Seeded synthetic sequences (generated once per session)."""
    from ct_icp_b200 import synthetic as syn
    key = (name, n_frames)
    if key not in _SEQ_CACHE:
        sensor = {"hdl64": syn.HDL64, "hdl32": syn.HDL32, "small16": syn.SMALL16, "dense128": syn.DENSE128}[name]
        _SEQ_CACHE[key] = syn.make_sequence(n_frames, sensor, seed=1234)
    return _SEQ_CACHE[key]


@pytest.fixture(scope="session")
def seq_small():
    return get_sequence("small16", 8)


@pytest.fixture(scope="session")
def seq_hdl64():
    return get_sequence("hdl64", 26)


def quat_angle(qa, qb):
    """Rotation angle (rad) between two quaternions (x,y,z,w)."""
    qa = np.asarray(qa, dtype=np.float64) / np.linalg.norm(qa)
    qb = np.asarray(qb, dtype=np.float64) / np.linalg.norm(qb)
    d = abs(float(np.dot(qa, qb)))
    return 2.0 * np.arccos(min(1.0, d))


# worst pose difference seen by each test (every parity assertion goes through frame_diff): written at session end to
# $CTICP_PARITY_LOG_DIR (default gpurun_out/) as parity_worst.<pid>.json, merged by tools/summarize_parity.py into the
# table of DESIGN.md §4 — so the numbers quoted there are the ones the assertions saw
_PARITY_WORST = {}


def frame_diff(fa, fb, log=True):
    """(max translation diff [m], max rotation diff [rad]) over begin and end poses of two cticp_frame.
    log=False: a comparison that is not a parity statement (e.g. "the registration moved the pose")."""
    dt = max(np.linalg.norm(np.array(fa.begin_pose.tr) - np.array(fb.begin_pose.tr)),
             np.linalg.norm(np.array(fa.end_pose.tr) - np.array(fb.end_pose.tr)))
    dr = max(quat_angle(fa.begin_pose.quat, fb.begin_pose.quat), quat_angle(fa.end_pose.quat, fb.end_pose.quat))
    if log:
        test = os.environ.get("PYTEST_CURRENT_TEST", "?").split(" ")[0]
        w = _PARITY_WORST.setdefault(test, [0.0, 0.0, 0])
        w[0], w[1], w[2] = max(w[0], float(dt)), max(w[1], float(dr)), w[2] + 1
    return dt, dr


def pytest_sessionfinish(session, exitstatus):
    if not _PARITY_WORST:
        return
    out = os.environ.get("CTICP_PARITY_LOG_DIR", os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "gpurun_out"))
    try:
        os.makedirs(out, exist_ok=True)
        import json
        with open(os.path.join(out, "parity_worst.%d.json" % os.getpid()), "w") as f:
            json.dump({k: {"max_translation_m": v[0], "max_rotation_rad": v[1], "frames_compared": v[2]}
                       for k, v in _PARITY_WORST.items()}, f, indent=1)
    except OSError:
        pass
