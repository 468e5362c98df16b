"""The layout of cticp_synthetic_frame in include/cticp.h, _abi.SyntheticFrame and synthetic_frame_dtype() agree, and
the engine exports every synthetic entry point. No GPU."""
import ctypes as C

from ct_icp_b200 import _abi as abi


def test_synthetic_frame_layout():
    import ct_icp_b200
    eng = ct_icp_b200.engine()
    assert eng.fn("abi_sizeof")(b"cticp_synthetic_frame") == C.sizeof(abi.SyntheticFrame) == 24
    assert abi.synthetic_frame_dtype().itemsize == 24
    assert abi.SyntheticFrame.frame_id.offset == abi.synthetic_frame_dtype().fields["frame_id"][1] == 16


def test_synthetic_entry_points_exported():
    import ct_icp_b200
    eng = ct_icp_b200.engine()
    for name in ("synthetic_scene_create", "synthetic_scene_destroy", "synthetic_scene_num_primitives",
                 "synthetic_scene_distance", "synthetic_generate_points", "synthetic_generate_frames",
                 "synthetic_generate_frames_device", "synthetic_generate_poses", "apply_uniform_noise"):
        assert eng.has(name), name


def test_scene_creation_without_a_device_reports_no_device():
    import torch
    import ct_icp_b200
    if torch.cuda.is_available():
        return
    eng = ct_icp_b200.engine()
    h = C.c_void_p()
    assert eng.fn("synthetic_scene_create")(None, 0, None, 0, None, 0, None, 0, 0, C.byref(h)) == abi.ERR_NO_DEVICE
