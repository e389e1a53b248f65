"""CPU tests of the map's C ABI (include/rgbdslam_b200/map.h): the library exports both entry points, and before
rgbdslam_b200_init each returns ERR_STATE with a message of its own (no CPU fallback)."""
import ctypes as C
import re
from pathlib import Path

import pytest

MAP_H = Path(__file__).resolve().parent.parent / "include" / "rgbdslam_b200" / "map.h"


def _declared():
    txt = re.sub(r"/\*.*?\*/", "", MAP_H.read_text(), flags=re.S)
    return sorted(set(re.findall(r"\b(rgbdslam_b200_[a-z0-9_]+)\s*\(", txt)))


def test_map_entry_points_are_exported(built):
    from rgbdslam_v2_b200 import _capi
    lib = _capi.load_library()
    names = _declared()
    assert names == ["rgbdslam_b200_node_download_cloud", "rgbdslam_b200_render_cloud"]
    for n in names:
        assert hasattr(lib, n), n
        assert getattr(lib, n).argtypes, n  # load_library sets the prototype


def test_map_entry_points_before_init(built):
    import torch
    if torch.cuda.is_available():
        pytest.skip("GPU present: the library may already be initialised in this process")
    from rgbdslam_v2_b200 import _capi
    lib = _capi.load_library()
    for name in _declared():
        fn = getattr(lib, name)
        assert lib.rgbdslam_b200_set_hamming_path(7) == 1  # leaves a known message in last_error
        sentinel = lib.rgbdslam_b200_last_error()
        args = [None if t is C.c_void_p or issubclass(t, C._Pointer) else 0.0 if t is C.c_double else 0 for t in fn.argtypes]
        assert fn(*args) == 3, name  # ERR_STATE
        msg = lib.rgbdslam_b200_last_error()
        assert msg and msg != sentinel, (name, msg)
    lib.rgbdslam_b200_set_hamming_path(1)
