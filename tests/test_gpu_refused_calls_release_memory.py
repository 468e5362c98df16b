"""A call the engine refuses with CTICP_ERR_INVALID_ARGUMENT leaves the device's free memory where it was, even when it
had already allocated large buffers before the check that refused it: eight refused calls of each kind may not take
1 GiB (each one allocates at least 512 MiB before it is refused)."""
import ctypes as C

import numpy as np
import pytest

import ct_icp_b200
from ct_icp_b200 import _abi as abi

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

CALLS = 8
GIB = 1 << 30


def _free_bytes():
    torch.cuda.synchronize()
    return torch.cuda.mem_get_info(0)[0]


def _refused_neighborhoods(eng):
    m = eng.voxel_map(eng.legacy_map_options(1.0, 20, 0.1))
    rng = np.random.default_rng(7)
    m.insert(rng.uniform(-20, 20, size=(20000, 3)))
    m.compute_neighborhoods(rng.uniform(-20, 20, size=(64, 3)), 20)   # warm-up: the same entry, accepted
    n = 1 << 20   # n x 33 neighbours x 24 bytes: 792 MiB of output on the device
    q = np.zeros((n, 3))
    pts = np.empty((n, 33, 3))
    cnt = np.empty(n, dtype=np.int32)
    call = eng.fn("map_compute_neighborhoods")
    return lambda: call(m.h, q.ctypes.data, n, 33, pts.ctypes.data, cnt.ctypes.data), m.close


def _refused_odometry(eng):
    o = eng.default_odometry_options()
    eng.odometry(o).close()   # warm-up
    o.max_points_per_frame = 4 * (1 << 20) + 1   # one point past what the samplers' tiles cover
    h = C.c_void_p()
    return lambda: eng.fn("odometry_create")(C.byref(o), 0, C.byref(h)), lambda: None


def _refused_map(eng):
    o = eng.legacy_map_options(1.0, 20, 0.1)
    eng.voxel_map(o).close()   # warm-up
    o.capacity_voxels = 1 << 21   # level 0: 2^21 voxels x 20 points x 16 bytes = 640 MiB of points alone
    o.num_resolutions = 2
    o.resolutions[1] = o.resolutions[0]
    o.resolutions[1].max_num_points = 65   # level 1 is refused after level 0 was allocated
    h = C.c_void_p()
    return lambda: eng.fn("map_create")(C.byref(o), 0, C.byref(h)), lambda: None


@pytest.mark.parametrize("kind", [_refused_neighborhoods, _refused_odometry, _refused_map],
                         ids=["map_compute_neighborhoods", "odometry_create", "map_create"])
def test_refused_calls_release_memory(kind):
    eng = ct_icp_b200.engine()
    call, close = kind(eng)
    before = _free_bytes()
    for _ in range(CALLS):
        assert call() == abi.ERR_INVALID_ARGUMENT, eng.fn("last_error")()
    lost = before - _free_bytes()
    close()
    assert lost < GIB, "%d refused calls took %.2f GiB of device memory" % (CALLS, lost / GIB)
