"""The spinning-LiDAR sweeps without a GPU: the layouts of cticp_lidar_sensor and cticp_lidar_frame in include/cticp.h,
_abi.LidarSensor / LidarFrame and lidar_frame_dtype() agree, the engine exports every entry point, and the NumPy
restatement the GPU tests use (tests/lidar_sim_ref.py) reproduces synthetic.generate_scan with noise_sigma = 0."""
import ctypes as C

import numpy as np
import pytest

from ct_icp_b200 import _abi as abi
from ct_icp_b200 import synthetic as syn
import lidar_sim_ref as ref


def test_lidar_struct_layouts():
    import ct_icp_b200
    eng = ct_icp_b200.engine()
    assert eng.fn("abi_sizeof")(b"cticp_lidar_sensor") == C.sizeof(abi.LidarSensor) == 48
    assert eng.fn("abi_sizeof")(b"cticp_lidar_frame") == C.sizeof(abi.LidarFrame) == 16
    assert abi.LidarSensor.period.offset == 16 and abi.LidarSensor.noise_sigma.offset == 40
    assert abi.lidar_frame_dtype().itemsize == 16
    assert abi.LidarFrame.frame_id.offset == abi.lidar_frame_dtype().fields["frame_id"][1] == 8


def test_lidar_entry_points_exported():
    import ct_icp_b200
    eng = ct_icp_b200.engine()
    for name in ("lidar_scene_create", "lidar_scene_destroy", "lidar_scene_raycast", "lidar_scene_raycast_device",
                 "lidar_generate_sweeps", "lidar_generate_sweeps_device"):
        assert eng.has(name), name


def test_lidar_scene_creation_without_a_device_reports_no_device():
    import torch
    import ct_icp_b200
    if torch.cuda.is_available():
        pytest.skip("a CUDA device is present")
    eng = ct_icp_b200.engine()
    h = C.c_void_p()
    box = np.array([0, 0, 0, 1, 1, 1, 0], dtype=np.float64)
    assert eng.fn("lidar_scene_create")(box.ctypes.data, 1, None, 0, 1, 0, C.byref(h)) == abi.ERR_NO_DEVICE


def _f32_step(v):
    return np.spacing(np.abs(v).astype(np.float32)).astype(np.float64)


@pytest.mark.parametrize("sensor", [syn.SMALL16, syn.HDL64E], ids=lambda s: s.name)
def test_restatement_reproduces_generate_scan_without_noise(sensor):
    """generate_scan's own analytic poses per column, fed to the restatement: the same kept rays (a ray may flip only when
    its range lies within 1e-9 m of a keep bound: the rotations differ, matrix against quaternion), the same timestamps,
    and xyz within one float32 rounding step of generate_scan's float32-rounded points."""
    from scipy.spatial.transform import Rotation
    scene = syn.UrbanScene(1234, profile="suburb")
    traj = syn.Trajectory(height=sensor.height)
    frame = 7
    scan = syn.generate_scan(scene, traj, sensor, frame, seed=1234, noise_sigma=0.0)
    t0 = frame * sensor.period
    tc = ref.column_times(t0, sensor)
    quat = Rotation.from_matrix(traj.rotation(tc)).as_quat()   # x y z w
    out = ref.sweep(scene.boxes, scene.cyl, sensor, t0, frame, 1234, quat, traj.position(tc))
    # generate_scan's kept rays: rebuild its ray indices from the ray timestamps and ranges it kept
    ours = set(out["ray_index"].tolist())
    naz = sensor.n_azimuth
    j_of_t = {float(t): j for j, t in enumerate(tc)}
    ring_dir = ref.sensor_directions(sensor).reshape(sensor.n_rings, naz, 3)
    theirs = []
    for p, t in zip(scan["xyz"], scan["t"]):
        j = j_of_t[float(t)]
        u = p / np.linalg.norm(p)
        theirs.append(int(np.argmax(ring_dir[:, j] @ u)) * naz + j)
    theirs_set = set(theirs)
    assert len(theirs_set) == len(theirs)
    flipped = sorted(ours ^ theirs_set)
    r = out["all_r"]
    bounds = np.minimum(np.abs(r[flipped] - sensor.min_range), np.abs(r[flipped] - sensor.max_range)) if flipped else []
    print("%s: %d kept, flipped rays %s (distance to a keep bound %s)" % (sensor.name, len(ours), flipped, list(bounds)))
    assert all(b <= 1e-9 for b in bounds), (flipped, bounds)
    both = np.array(sorted(ours & theirs_set))
    mine = {int(i): k for k, i in enumerate(out["ray_index"])}
    theirs_at = {i: k for k, i in enumerate(theirs)}
    a = out["raw"][[mine[i] for i in both]]
    b = scan["xyz"][[theirs_at[i] for i in both]]
    assert np.all(np.abs(a - b) <= _f32_step(b) + 1e-9), np.abs(a - b).max()
    np.testing.assert_array_equal(out["t"][[mine[i] for i in both]], scan["t"][[theirs_at[i] for i in both]])
