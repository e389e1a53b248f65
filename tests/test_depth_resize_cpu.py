"""CPU tests of the Node constructor for depth images of another size than the visual (include/rgbdslam_b200/depth_resize.h):
the two entry points are exported and need an initialised library, the Python methods check shapes before the library is
called, and the nearest-neighbour index rule the library builds its tables with equals cv2.resize(INTER_NEAREST)."""
import numpy as np
import pytest

ENTRY_POINTS = ("rgbdslam_b200_nodes_create_resized", "rgbdslam_b200_nodes_create_sharded_resized")


def test_resized_entry_points_are_declared_in_their_own_header(built):
    from rgbdslam_v2_b200 import _capi
    txt = (_capi.header_path().parent / "rgbdslam_b200" / "depth_resize.h").read_text()
    lib = _capi.load_library()
    for name in ENTRY_POINTS:
        assert name + "(" in txt and hasattr(lib, name)
        assert name not in _capi.header_path().read_text()  # the main header's entry points stay as they are


def test_resized_entry_points_need_init(built):
    import torch
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    from rgbdslam_v2_b200 import _capi
    lib = _capi.load_library()
    gray = np.zeros((1, 480, 640), np.uint8)
    depth = np.zeros((1, 240, 320), np.float32)
    K4 = np.array([525.0, 525.0, 319.5, 239.5], np.float32)
    handles = np.zeros(1, np.uint64)
    nf = np.zeros(1, np.int32)
    rc = lib.rgbdslam_b200_nodes_create_resized(1, 1, gray.ctypes.data, depth.ctypes.data, 320, 240, None, 640, 480, K4.ctypes.data,
                                                None, 0, handles.ctypes.data, nf.ctypes.data)
    assert rc == 3  # ERR_STATE
    rc = lib.rgbdslam_b200_nodes_create_sharded_resized(1, 1, 1, gray.ctypes.data, depth.ctypes.data, 320, 240, None, 640, 480,
                                                        K4.ctypes.data, None, 0, handles.ctypes.data, nf.ctypes.data)
    assert rc == 3
    assert b"init" in lib.rgbdslam_b200_last_error().lower()


class _NoLibrary:
    """a Frontend's library that fails the test when any entry point is called"""

    def __getattr__(self, name):
        raise AssertionError(f"{name} called")


def _frontend():
    from rgbdslam_v2_b200._capi import Frontend
    fe = Frontend.__new__(Frontend)
    fe.lib = _NoLibrary()
    fe._nodes = []
    return fe


@pytest.mark.parametrize("method", ["nodes_create_resized", "nodes_create_sharded_resized"])
def test_python_shape_checks_raise_before_the_library(method):
    fe = _frontend()
    K4 = (525.0, 525.0, 319.5, 239.5)
    gray = np.zeros((2, 480, 640), np.uint8)

    def call(g, d):
        if method == "nodes_create_resized":
            return fe.nodes_create_resized(1, g, d, None, K4)
        return fe.nodes_create_sharded_resized(1, 1, 2, g, d, None, K4)
    for depth in (np.zeros((2, 240, 320, 8), np.float32), np.zeros((2, 240, 320, 4), np.float32)):  # clouds
        with pytest.raises(ValueError, match="depth image"):
            call(gray, depth)
    with pytest.raises(ValueError, match="depth image"):
        call(gray, np.zeros((240, 320), np.float32))
    for depth in (np.zeros((3, 240, 320), np.float32), np.zeros((1, 240, 320), np.uint16)):  # another frame count
        with pytest.raises(ValueError, match="frames"):
            call(gray, depth)
    with pytest.raises(ValueError, match=r"\(F,H,W,3\)"):
        call(np.zeros((2, 480, 640, 4), np.uint8), np.zeros((2, 240, 320), np.float32))


def test_nodes_create_keeps_refusing_another_size():
    fe = _frontend()
    with pytest.raises(ValueError, match="image size"):
        fe.nodes_create(1, np.zeros((1, 480, 640), np.uint8), np.zeros((1, 240, 320), np.float32), None, (1, 1, 1, 1))


def _nn_index(n, dn):
    """the library's table rule (nn_resize_tables): min((int)floor(x * (1.0 / ((double)n / dn))), dn - 1)"""
    ifx = 1.0 / (n / dn)
    return np.minimum(np.floor(np.arange(n) * ifx).astype(np.int64), dn - 1)


@pytest.mark.parametrize("w,h,dw,dh", [(640, 480, 320, 240), (640, 480, 1280, 960), (640, 480, 512, 424), (640, 480, 97, 61),
                                       (1280, 1024, 640, 480), (1920, 1080, 512, 424), (1280, 720, 640, 480),
                                       (1279, 1023, 320, 240), (4095, 4095, 1, 1), (333, 4095, 4094, 7)])
def test_index_rule_equals_cv2_nearest(w, h, dw, dh):
    import cv2
    rng = np.random.default_rng(w * 7 + dh)
    d16 = rng.integers(0, 65536, (dh, dw)).astype(np.uint16)
    d32 = rng.random((dh, dw)).astype(np.float32)
    d32[rng.random((dh, dw)) < 0.1] = np.nan
    rows, cols = _nn_index(h, dh), _nn_index(w, dw)
    assert np.array_equal(cv2.resize(d16, (w, h), interpolation=cv2.INTER_NEAREST), d16[rows][:, cols])
    r32 = cv2.resize(d32, (w, h), interpolation=cv2.INTER_NEAREST)
    assert np.array_equal(r32.view(np.uint32), d32[rows][:, cols].view(np.uint32))


def test_shorter_index_form_differs_somewhere():
    """cv2's double arithmetic is not the exact quotient: floor(x * dw / w) in integers picks another source pixel for some
    sizes, so the tables must be built with cv2's form"""
    diffs = 0
    for w in range(96, 1400):
        for dw in (97, 320, 424, 480, 512, 640):
            x = np.arange(w)
            diffs += int((np.minimum(x * dw // w, dw - 1) != _nn_index(w, dw)).sum())
    assert diffs > 0
