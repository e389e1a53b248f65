"""CPU tests of the C-ABI boundary: the library builds, loads, exports every declared symbol, has the
declared struct layouts, and fails loudly (no CPU fallback) when no CUDA device is present."""
import ctypes as C

import numpy as np
import pytest


def test_library_exports_every_declared_symbol(built):
    from rgbdslam_v2_b200 import _capi
    lib = _capi.load_library()
    names = _capi.declared_symbols()
    assert len(names) >= 15
    for n in names:
        assert hasattr(lib, n), n


def test_struct_layouts_match_reference_types(built):
    from rgbdslam_v2_b200 import _capi
    assert C.sizeof(_capi.KeyPoint) == 28  # cv::KeyPoint
    assert C.sizeof(_capi.DMatch) == 16    # cv::DMatch
    assert _capi.PAIR_RESULT_DTYPE.itemsize == C.sizeof(_capi.PairResult)
    for name in _capi.PAIR_RESULT_DTYPE.names:
        assert _capi.PAIR_RESULT_DTYPE.fields[name][1] == getattr(_capi.PairResult, name).offset


def test_default_params_are_the_reference_defaults(built):
    """src/parameter_server.cpp:83-101."""
    from rgbdslam_v2_b200 import _capi
    p = _capi.default_params()
    assert (p.max_keypoints, p.min_matches, p.max_matches, p.ransac_iterations) == (600, 20, 300, 200)
    assert p.max_dist_for_inliers == 3.0 and p.sigma_depth == 0.01
    assert p.detector_grid_resolution == 3 and p.adjuster_max_iterations == 5
    assert p.nn_distance_ratio == 0.95 and p.use_root_sift == 1


def test_no_cpu_fallback(built):
    import torch
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    from rgbdslam_v2_b200 import _capi
    lib = _capi.load_library()
    p = _capi.default_params()
    rc = lib.rgbdslam_b200_init(0, C.byref(p))
    assert rc == 2  # RGBDSLAM_B200_ERR_CUDA
    assert b"CUDA" in lib.rgbdslam_b200_last_error()
    q = np.zeros((4, 32), np.uint8)
    idx = np.zeros(4, np.int32)
    rc = lib.rgbdslam_b200_brute_force_orb(q.ctypes.data, 4, q.ctypes.data, 4, idx.ctypes.data, idx.ctypes.data)
    assert rc == 3  # ERR_STATE: not initialised, nothing computed on the CPU
    with pytest.raises(_capi.B200Error):
        _capi.Frontend(0)


def test_missing_library_fails_loudly(tmp_path):
    from rgbdslam_v2_b200 import _capi
    with pytest.raises(_capi.LibraryMissingError):
        _capi.load_library(tmp_path / "nope.so")


# Return code of every entry point called before rgbdslam_b200_init with zero / NULL arguments.  Entry points that need an
# initialised library return ERR_STATE (3); the ones below work without init.  init itself: test_no_cpu_fallback.
_NO_INIT_RC = {
    "rgbdslam_b200_launch_count": 0, "rgbdslam_b200_depth_cov_z0": 0, "rgbdslam_b200_set_hamming_path": 0,
    "rgbdslam_b200_set_sift_matcher": 0, "rgbdslam_b200_shutdown": 0,
    "rgbdslam_b200_comm_destroy": 1, "rgbdslam_b200_detector_create": 1, "rgbdslam_b200_detector_destroy": 1,
    "rgbdslam_b200_detector_thresholds": 1, "rgbdslam_b200_get_params": 1, "rgbdslam_b200_graph_from_pairs": 1,
    "rgbdslam_b200_node_destroy": 1, "rgbdslam_b200_node_num_features": 1,
    "rgbdslam_b200_comm_unique_id": (1, 4),  # 4 = ERR_NCCL when libnccl.so.2 cannot be loaded
}
_NOT_CALLED = {"rgbdslam_b200_init", "rgbdslam_b200_default_params", "rgbdslam_b200_last_error"}


def test_every_entry_point_before_init(built):
    """Every declared entry point, called before init with zero / NULL arguments, returns its documented code, and every
    non-zero return replaces last_error (no stale message from the previous call)."""
    import torch
    if torch.cuda.is_available():
        pytest.skip("GPU present: the library may already be initialised in this process")
    from rgbdslam_v2_b200 import _capi
    lib = _capi.load_library()
    names = [n for n in _capi.declared_symbols() if n not in _NOT_CALLED]
    assert len(names) == 49
    for name in names:
        fn = getattr(lib, name)
        assert lib.rgbdslam_b200_set_hamming_path(7) == 1  # leaves a known message in last_error
        sentinel = lib.rgbdslam_b200_last_error()
        args = [None if t is C.c_void_p or issubclass(t, C._Pointer) else 0.0 if t is C.c_double else 0 for t in fn.argtypes]
        rc = fn(*args)
        want = _NO_INIT_RC.get(name, 3)
        if name == "rgbdslam_b200_depth_cov_z0":
            assert rc == 0.0, name
            continue
        assert rc in (want if isinstance(want, tuple) else (want,)), (name, rc)
        if rc != 0:
            msg = lib.rgbdslam_b200_last_error()
            assert msg and msg != sentinel, (name, msg)
    lib.rgbdslam_b200_set_hamming_path(1)  # the default
