"""CPU test of rgbdslam_b200_octomap_filter_clouds (include/rgbdslam_b200/octomap.h): the library exports it with a prototype,
and before rgbdslam_b200_init it returns ERR_STATE with a message of its own (no CPU fallback)."""
import ctypes as C

import numpy as np
import pytest


def test_filter_clouds_is_exported_and_refuses_without_a_device(built):
    import torch
    from rgbdslam_v2_b200 import _capi
    lib = _capi.load_library()
    fn = lib.rgbdslam_b200_octomap_filter_clouds
    assert fn.argtypes
    if torch.cuda.is_available():
        pytest.skip("GPU present: the library may already be initialised in this process")
    assert lib.rgbdslam_b200_set_hamming_path(7) == 1  # leaves a known message in last_error
    sentinel = lib.rgbdslam_b200_last_error()
    hs = np.zeros(1, np.uint64)
    s7 = np.array([0, 0, 0, 1, 0, 0, 0], np.float32)
    counts = np.zeros(1, np.int32)
    assert fn(C.c_uint64(1), 1, hs.ctypes.data, s7.ctypes.data, 0.9, counts.ctypes.data) == 3  # ERR_STATE
    msg = lib.rgbdslam_b200_last_error()
    assert msg and msg != sentinel
    lib.rgbdslam_b200_set_hamming_path(1)
