"""The ctypes wrapper of the C oracle of ColorOctomapServer::occupancyFilter (tests/octomap_filter_oracle.c, DESIGN.md
4.15).  That library includes the OctoMap oracle (tests/octomap_oracle.c), so FilterOracle is an octomap_exact.Oracle whose
map the filter reads."""
import ctypes as C
import functools
import subprocess
import tempfile
from pathlib import Path

import numpy as np

import octomap_exact as ox

HERE = Path(__file__).resolve().parent
F32 = np.float32


@functools.lru_cache(maxsize=None)
def lib() -> C.CDLL:
    """tests/octomap_filter_oracle.c built into a temporary directory (the source tree may be read-only)."""
    out = Path(tempfile.mkdtemp(prefix="octomap_filter_oracle_")) / "liboctomap_filter_oracle.so"
    subprocess.run(["gcc", "-O2", "-fPIC", "-shared", "-ffp-contract=off", "-Wall", f"-I{HERE}", "-o", str(out),
                    str(HERE / "octomap_filter_oracle.c"), "-lm"], check=True, capture_output=True)
    L = C.CDLL(str(out))
    L.om_create.restype = C.c_void_p
    L.om_create.argtypes = [C.c_double] * 5
    for f in ("om_clear", "om_destroy"):
        getattr(L, f).argtypes = [C.c_void_p]
        getattr(L, f).restype = None
    L.om_insert.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_long, C.c_void_p, C.c_double]
    L.om_insert.restype = C.c_long
    L.om_write.argtypes = [C.c_void_p, C.c_void_p, C.c_long]
    L.om_write.restype = C.c_long
    L.om_stats.argtypes = [C.c_void_p, C.POINTER(C.c_long), C.POINTER(C.c_long)]
    L.om_stats.restype = None
    L.om_occupancy_filter.argtypes = [C.c_void_p, C.c_void_p, C.c_long, C.c_void_p, C.c_void_p, C.c_double, C.c_void_p]
    L.om_occupancy_filter.restype = C.c_long
    L.om_sensor_transform.argtypes = [C.c_void_p] * 4
    L.om_sensor_transform.restype = None
    return L


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


class FilterOracle(ox.Oracle):
    """One ColorOcTree of the oracle, in the library that also holds the filter."""

    def __init__(self, resolution=0.05, prob_hit=0.9, prob_miss=0.4, clamping_min=0.001, clamping_max=0.999):
        self.h = lib().om_create(resolution, prob_hit, prob_miss, clamping_min, clamping_max)

    def __del__(self):
        if getattr(self, "h", None):
            lib().om_destroy(self.h)

    def insert(self, xyz, rgb, origin, max_range=-1.0):
        xyz = np.ascontiguousarray(xyz, F32).reshape(-1, 3)
        rgb = np.ascontiguousarray(rgb, np.uint32).reshape(-1)
        o = np.ascontiguousarray(origin, F32).reshape(3)
        return lib().om_insert(self.h, _p(xyz), _p(rgb), len(xyz), _p(o), float(max_range))

    def write(self) -> bytes:
        n = lib().om_write(self.h, None, 0)
        buf = np.zeros(n, np.uint8)
        lib().om_write(self.h, _p(buf), n)
        return buf.tobytes()

    def stats(self):
        a, b = C.c_long(), C.c_long()
        lib().om_stats(self.h, C.byref(a), C.byref(b))
        return a.value, b.value

    def clear(self):
        lib().om_clear(self.h)

    def occupancy_filter(self, xyz, q, t, threshold=0.9):
        """ColorOctomapServer::occupancyFilter: the keep mask of the points xyz ((n, 3) float32, as stored) under the sensor
        pose q (x, y, z, w) / t (float32)"""
        xyz = np.ascontiguousarray(xyz, F32).reshape(-1, 3)
        q = np.ascontiguousarray(q, F32).reshape(4)
        t = np.ascontiguousarray(t, F32).reshape(3)
        keep = np.zeros(len(xyz), np.uint8)
        n = lib().om_occupancy_filter(self.h, _p(xyz), len(xyz), _p(q), _p(t), float(threshold), _p(keep))
        assert n == int(keep.sum())
        return keep.astype(bool)


def sensor_transform(q, t, p):
    """q * p + t as occupancyFilter forms it (the oracle's float32 result)"""
    q, t, p = (np.ascontiguousarray(a, F32) for a in (q, t, p))
    out = np.zeros(3, F32)
    lib().om_sensor_transform(_p(q), _p(t), _p(p), _p(out))
    return out
