"""cticp_odometry_register_batch without a GPU: the item's layout against the library, and the argument checks the
Python binding makes before it calls into the library."""
import ctypes as C

import numpy as np
import pytest

from ct_icp_b200 import _abi as abi
from ct_icp_b200._binding import Binding


def test_batch_frame_layout(eng):
    assert eng.fn("abi_sizeof")(b"cticp_batch_frame") == C.sizeof(abi.BatchFrame) == 112
    offsets = {"handle": 0, "kind": 8, "frame_id": 12, "xyz": 16, "xyz_stride_bytes": 24, "t": 32, "t_stride_bytes": 40,
               "n": 48, "device_scan": 56, "stream": 64, "staged_slot": 72, "initial_estimate": 80,
               "motion_model": 88, "out": 96, "status": 104}
    for name, off in offsets.items():
        assert getattr(abi.BatchFrame, name).offset == off, name
    # the renamed padding of the timing record: same size, same place
    assert eng.fn("abi_sizeof")(b"cticp_device_timing") == C.sizeof(abi.DeviceTiming)
    assert abi.DeviceTiming.icp_batch_groups.offset == C.sizeof(abi.DeviceTiming) - 4


class _NoCalls:
    """A library whose every entry point fails the test when called."""

    def __getattr__(self, name):
        if not name.startswith("cticp_"):
            raise AttributeError(name)

        def call(*args):
            raise AssertionError("called into the library: " + name)
        return call


@pytest.mark.parametrize("field", ["scans", "frame_ids", "initial_estimates", "motion_models"])
def test_register_batch_checks_list_lengths(field):
    b = Binding.__new__(Binding)
    b.lib, b.prefix = _NoCalls(), "cticp_"
    scan = (np.zeros((4, 3)), np.zeros(4))
    args = {"scans": [scan, scan], "frame_ids": [0, 0], "initial_estimates": [None, None], "motion_models": [None, None]}
    args[field] = args[field][:1]
    with pytest.raises(ValueError, match=field):
        b.register_batch([object(), object()], args["scans"], args["frame_ids"], args["initial_estimates"],
                         args["motion_models"])
