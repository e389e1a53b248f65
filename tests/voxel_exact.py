"""numpy restatement of the voxel filter of a node's stored cloud (Node::reducePointCloud, node.cpp:1448-1460:
pcl::VoxelGrid<PointXYZRGB> with a cubic leaf, all fields downsampled), and the ctypes wrapper of its C oracle
(tests/voxel_oracle.c).  Clouds are the dicts of tests/map_cloud_exact.py (flat x, y, z float32, rgb / w16 uint32, raster w, h).
Every float operation is one numpy float32 operation; the sums inside a voxel run point after point in raster order (a stable
sort by voxel index keeps it), and the mean multiplies by the float reciprocal of the count (DESIGN.md 4.11).
"""
import ctypes as C
import functools
import subprocess
import tempfile
from pathlib import Path

import numpy as np

HERE = Path(__file__).resolve().parent
F32 = np.float32
INT32_MAX = 2**31 - 1


def _cloud(x, y, z, rgb):
    rgb = np.asarray(rgb, np.uint32)
    return dict(x=np.asarray(x, F32), y=np.asarray(y, F32), z=np.asarray(z, F32), rgb=rgb, w16=rgb.copy(), w=len(rgb), h=1)


def grid(pc, vfs):
    """(finite mask, inv, min_b, div_b) of the cloud's voxel grid; min_b None when no point is finite, div_b None when the leaf
    size is too small for the cloud (more than INT32_MAX cells: PCL copies its input)"""
    inv = F32(1.0) / F32(vfs)
    P = np.stack([pc["x"], pc["y"], pc["z"]])
    fin = np.isfinite(P).all(0)
    if not fin.any():
        return fin, inv, None, None
    mn, mx = P[:, fin].min(1), P[:, fin].max(1)
    min_b = np.floor(mn * inv).astype(np.int64)
    div_b = np.floor(mx * inv).astype(np.int64) - min_b + 1
    guard = ((mx - mn) * inv).astype(np.int64) + 1  # the float product, truncated
    too_small = any(int(d[0]) * int(d[1]) * int(d[2]) > INT32_MAX for d in (guard, div_b))
    return fin, inv, min_b, None if too_small else div_b


def reduce_cloud(pc, vfs):
    """The reduced cloud (n x 1), or None when the leaf size is too small and the cloud stays as it is."""
    fin, inv, min_b, div_b = grid(pc, vfs)
    if min_b is None:
        return _cloud([], [], [], [])
    if div_b is None:
        return None
    P = np.stack([pc["x"], pc["y"], pc["z"]])[:, fin]
    ijk = (np.floor(P * inv) - min_b.astype(F32)[:, None]).astype(np.int64)
    idx = ijk[0] + ijk[1] * div_b[0] + ijk[2] * (div_b[0] * div_b[1])
    order = np.argsort(idx, kind="stable")
    sidx = idx[order]
    rgb = pc["rgb"][fin][order]
    vals = np.concatenate([P[:, order], np.stack([(rgb >> s) & 255 for s in (16, 8, 0)]).astype(F32)])
    starts = np.flatnonzero(np.concatenate([[True], sidx[1:] != sidx[:-1]]))
    lens = np.diff(np.concatenate([starts, [len(sidx)]]))
    # sequential float32 sums: step t adds the t-th point of every voxel that has one (the longest voxels first in `by_len`)
    by_len = np.argsort(-lens, kind="stable")
    sorted_lens = lens[by_len]
    acc = np.zeros((6, len(starts)), F32)
    for t in range(int(lens.max())):
        sel = by_len[:np.searchsorted(-sorted_lens, -t, side="left")]
        acc[:, sel] = acc[:, sel] + vals[:, starts[sel] + t]
    mean = acc * (F32(1.0) / lens.astype(F32))
    r, g, b = (mean[c].astype(np.int64).astype(np.uint32) for c in (3, 4, 5))  # truncated toward zero
    return _cloud(mean[0], mean[1], mean[2], (r << 16) | (g << 8) | b)


# ---- the C oracle ----------------------------------------------------------------------------------------------------------

@functools.lru_cache(maxsize=None)
def _oracle_lib() -> C.CDLL:
    """tests/voxel_oracle.c built into a temporary directory (the source tree may be read-only)."""
    out = Path(tempfile.mkdtemp(prefix="voxel_oracle_")) / "libvoxel_oracle.so"
    subprocess.run(["gcc", "-O2", "-fPIC", "-shared", "-ffp-contract=off", "-Wall", "-o", str(out), str(HERE / "voxel_oracle.c"), "-lm"],
                   check=True, capture_output=True)
    lib = C.CDLL(str(out))
    lib.voxel_grid_filter.restype = C.c_long
    return lib


def oracle_reduce_cloud(pc, vfs):
    """the C oracle of reduce_cloud"""
    x, y, z = (np.ascontiguousarray(pc[k], F32) for k in "xyz")
    rgb = np.ascontiguousarray(pc["rgb"], np.uint32)
    n = len(x)
    ox, oy, oz, orgb = np.zeros(n, F32), np.zeros(n, F32), np.zeros(n, F32), np.zeros(n, np.uint32)
    p = lambda a: a.ctypes.data_as(C.c_void_p)
    m = _oracle_lib().voxel_grid_filter(p(x), p(y), p(z), p(rgb), C.c_long(n), C.c_float(vfs), p(ox), p(oy), p(oz), p(orgb))
    return None if m < 0 else _cloud(ox[:m], oy[:m], oz[:m], orgb[:m])
