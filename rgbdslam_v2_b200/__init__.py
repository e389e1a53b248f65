"""rgbdslam_v2_b200 -- H100-native (sm_90a) re-implementation of the rgbdslam_v2 frame-pair hot path.

The product is the C-ABI shared library ``librgbdslam_b200.so`` (see ``include/rgbdslam_b200.h``) built from
``csrc/``.  This package is the thin Python host mirror used by tests and ``bench.py``; it binds the library
with ctypes and FAILS LOUDLY if the library is missing -- there is no CPU fallback.
"""
from .build import build_library, library_path  # noqa: F401
from ._capi import (  # noqa: F401
    Params, PairResult, DMatch, KeyPoint, Frontend, load_library, LibraryMissingError, B200Error,
)
