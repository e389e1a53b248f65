"""The ctypes wrapper of the C oracle of the colour OctoMap (tests/octomap_oracle.c, rules 2-8 of DESIGN.md 4.14), and the
scans the reference builds from a node's stored cloud: the cloud transformed as map_point does (R p summed
(r0 p0 + r1 p1) + r2 p2, plus t, in float32), the ray origin the transform's translation.  Rule 1, the pose chain, is
rgbdslam_v2_b200._capi.octomap_pose."""
import ctypes as C
import functools
import subprocess
import tempfile
from pathlib import Path

import numpy as np

HERE = Path(__file__).resolve().parent
F32 = np.float32
HEADER = (b"# Octomap OcTree file\n# (feel free to add / change comments, but leave the first line as it is!)\n#\n"
          b"id ColorOcTree\n")
RECORD = np.dtype([("lo", "<f4"), ("r", "u1"), ("g", "u1"), ("b", "u1"), ("children", "u1")])


@functools.lru_cache(maxsize=None)
def lib() -> C.CDLL:
    """tests/octomap_oracle.c built into a temporary directory (the source tree may be read-only)."""
    out = Path(tempfile.mkdtemp(prefix="octomap_oracle_")) / "liboctomap_oracle.so"
    subprocess.run(["gcc", "-O2", "-fPIC", "-shared", "-ffp-contract=off", "-Wall", "-o", str(out), str(HERE / "octomap_oracle.c"), "-lm"],
                   check=True, capture_output=True)
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
    L.om_ray_keys.argtypes = [C.c_double, C.c_void_p, C.c_void_p, C.c_void_p, C.c_long]
    L.om_ray_keys.restype = C.c_long
    return L


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


class Oracle:
    """One ColorOcTree of the oracle."""

    def __init__(self, resolution=0.05, prob_hit=0.9, prob_miss=0.4, clamping_min=0.001, clamping_max=0.999):
        self.h = lib().om_create(resolution, prob_hit, prob_miss, clamping_min, clamping_max)

    def __del__(self):
        if getattr(self, "h", None):
            lib().om_destroy(self.h)

    def insert(self, xyz, rgb, origin, max_range=-1.0):
        """one scan: xyz (n, 3) float32 map points, rgb (n,) colour words, origin (3,) float32; returns its ray and occupied
        cells before deduplication"""
        xyz = np.ascontiguousarray(xyz, F32).reshape(-1, 3)
        rgb = np.ascontiguousarray(rgb, np.uint32).reshape(-1)
        o = np.ascontiguousarray(origin, F32).reshape(3)
        return lib().om_insert(self.h, _p(xyz), _p(rgb), len(xyz), _p(o), float(max_range))

    def insert_cloud(self, pc, T34, max_range=-1.0):
        """the scan of a stored cloud (a map_cloud_exact cloud dict) under the float 3 x 4 T34"""
        xyz = transform(pc, T34)
        return self.insert(xyz, pc["rgb"], np.asarray(T34, F32)[:, 3], max_range)

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


def ray_keys(origin, end, resolution=0.05):
    """computeRayKeys: (n, 3) uint16 keys, or None when a key is out of range"""
    o = np.ascontiguousarray(origin, F32)
    e = np.ascontiguousarray(end, F32)
    out = np.zeros((1 << 16, 3), np.uint16)
    n = lib().om_ray_keys(resolution, _p(o), _p(e), _p(out), len(out))
    return None if n < 0 else out[:n].copy()


def transform(pc, T34):
    """map_point without the depth filter: every point of the cloud, NaN points untransformed"""
    M = np.asarray(T34, F32)
    x, y, z = pc["x"], pc["y"], pc["z"]
    with np.errstate(all="ignore"):
        t = [(((M[r, 0] * x) + (M[r, 1] * y)) + (M[r, 2] * z)) + M[r, 3] for r in range(3)]
    nanp = np.isnan(x) | np.isnan(y) | np.isnan(z)
    return np.stack([np.where(nanp, c, tc).astype(F32) for c, tc in zip((x, y, z), t)], 1)


def parse(data: bytes):
    """(size, res text, records) of an .ot file, checking the fixed header lines"""
    assert data.startswith(HEADER), data[:120]
    rest = data[len(HEADER):]
    size_line, rest = rest.split(b"\n", 1)
    res_line, rest = rest.split(b"\n", 1)
    data_line, body = rest.split(b"\n", 1)
    assert size_line.startswith(b"size ") and res_line.startswith(b"res ") and data_line == b"data"
    size = int(size_line[5:])
    assert len(body) == 8 * size
    return size, res_line[4:].decode(), np.frombuffer(body, RECORD)


def tree(records):
    """the pre-order records as nested (record, [children]) -- checks that the child bits account for every record"""
    pos = 0

    def rec():
        nonlocal pos
        r = records[pos]
        pos += 1
        kids = [(c, rec()) for c in range(8) if (int(r["children"]) >> c) & 1]
        return r, kids

    root = rec() if len(records) else None
    assert pos == len(records)
    return root
