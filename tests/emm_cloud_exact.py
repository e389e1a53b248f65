"""Exact restatement of the environment measurement model on the organised clouds that point-cloud nodes keep
(RGBDSLAM_B200_KEEP_CLOUD; the `EmmPoints::kCloud` instantiations of `k_emm_pairs` / `k_emm_single` in csrc/emm.cu), and
the ctypes wrapper of its C oracle (tests/emm_cloud_oracle.c).

observationLikelihood (misc.cpp:814-969) with clouds as input differs from the depth-image case of tests/emm_exact.py:
- the points are taken as stored, every skip_step-th point of the full-resolution cloud; no cloud step (the intrinsics are
  not divided, sigma is not scaled);
- pcl::transformPointCloud on a cloud that is not dense leaves a point with a non-finite coordinate untransformed: a +inf z
  stays +inf and is judged at (round(cx), round(cy));
- round() as x86-64 evaluates it: NaN, +-inf and out-of-range values become INT_MIN, outside the raster;
- a direction whose two clouds differ in width contributes nothing, not even to `all`.
As in observationLikelihood's else branch, a comparison whose p is NaN (inf / inf in the cdf argument) marks a bad point.
The float chain is float32 with one rounding per operation in the reference's order, the sigma sums float64; loose samples
(p within LOOSE of a cut) are marked as in tests/emm_exact.py.
"""
from __future__ import annotations

import ctypes as C
import functools
import subprocess
import tempfile
from pathlib import Path

import numpy as np
from scipy.special import erf

from emm_exact import CUTS, LOOSE, _cov, affine_inverse_f

F32, F64 = np.float32, np.float64
HERE = Path(__file__).resolve().parent


def direction_cloud(T, src, dst, dstK, *, skip_step=8, sigma_depth=0.01, czc=None):
    """One direction: src / dst organised clouds (h, w, >= 3) float32 with x, y, z first, T (float32 4x4 row-major, src
    frame -> dst frame), dstK = (fx, fy, cx, cy) of the camera the direction projects into, czc = constant depth covariance
    (None = per point).  Returns dict(counts=[good, bad, occluded, all], loose=bool per sample, margin=smallest |p / cut - 1|
    per sample)."""
    T = np.asarray(T, F32)
    R, t = T[:3, :3], T[:3, 3]
    src, dst = np.asarray(src, F32), np.asarray(dst, F32)
    sh, sw = src.shape[:2]
    dh, dw = dst.shape[:2]
    if dw != sw:  # misc.cpp:844-847
        return dict(counts=np.zeros(4, np.int64), loose=np.zeros(0, bool), margin=np.zeros(0))
    dst_z = dst[:, :, 2]
    ry, rx = np.meshgrid(np.arange(0, sh, skip_step), np.arange(0, sw, skip_step), indexing="ij")
    p = src[ry.ravel(), rx.ravel(), :3]
    px, py, pz = p[:, 0], p[:, 1], p[:, 2]
    finite = np.isfinite(p).all(1)
    with np.errstate(invalid="ignore", over="ignore"):
        q = [(((R[r, 0] * px + R[r, 1] * py) + R[r, 2] * pz) + t[r]).astype(F32) for r in range(3)]
    qx, qy, qz = (np.where(finite, a, b).astype(F32) for a, b in zip(q, (px, py, pz)))
    fx, fy, cx, cy = (F32(k) for k in dstK)
    n_all = len(qz)
    with np.errstate(invalid="ignore", divide="ignore", over="ignore"):
        live = ~np.isnan(qz) & ~(qz < 0)
        xc = ((qx / qz) * fx + cx).astype(F32)
        yc = ((qy / qz) * fy + cy).astype(F32)
        ocx = np.floor(xc.astype(F64) + 0.5)   # misc.cpp:804-807; NaN / inf / out of range -> INT_MIN -> outside
        ocy = np.floor(yc.astype(F64) + 0.5)
        live &= np.isfinite(ocx) & np.isfinite(ocy) & (ocx >= 0) & (ocx < dw) & (ocy >= 0) & (ocy < dh)
    idx = np.nonzero(live)[0]
    cxi, cyi = ocx[idx].astype(np.int64), ocy[idx].astype(np.int64)
    qzl = qz[idx].astype(F64)
    good = np.zeros(len(idx), bool)
    occl = np.zeros(len(idx), bool)
    bad = np.zeros(len(idx), bool)
    margin = np.full(len(idx), np.inf)
    startx, starty = np.maximum(0, cxi - 2), np.maximum(0, cyi - 2)
    endx, endy = np.minimum(dw, cxi + 3), np.minimum(dh, cyi + 3)
    with np.errstate(invalid="ignore", over="ignore"):
        new_sigma = _cov(qzl, sigma_depth, czc)
    for jy in range(3):
        oy = starty + 2 * jy
        for jx in range(3):
            ox = startx + 2 * jx
            inside = (oy < endy) & (ox < endx)
            oz = np.full(len(idx), np.nan, F32)
            oz[inside] = dst_z[oy[inside], ox[inside]]
            ok = inside & ~np.isnan(oz)
            oz64 = oz.astype(F64)
            with np.errstate(invalid="ignore", over="ignore"):
                joint = _cov(oz64, sigma_depth, czc) + new_sigma
                pr = 0.5 * (1 + erf((oz64 - qzl) / (np.sqrt(joint) * 1.41421)))
            occl |= ok & (pr < CUTS[0])
            good |= ok & (pr >= CUTS[0]) & (pr < CUTS[1])
            bad |= ok & ~(pr < CUTS[0]) & ~(pr < CUTS[1])   # the else branch: a NaN p is bad
            for c in CUTS:
                margin = np.where(ok, np.minimum(margin, np.abs(pr / c - 1)), margin)
    g = int(good.sum())
    o = int((~good & occl).sum())
    b = int((~good & ~occl & bad).sum())
    m_all = np.full(n_all, np.inf)
    m_all[idx] = margin
    return dict(counts=np.array([g, b, o, n_all], np.int64), loose=m_all < LOOSE, margin=m_all)


def pairwise_cloud(T, newer, newerK, older, olderK, **kw):
    """pairwiseObservationLikelihood (node.cpp:1520-1554) on kept clouds: newer -> older under T, older -> newer under the
    float cofactor inverse of T; K = the camera each direction projects into (the older node's for newer -> older)."""
    a = direction_cloud(T, newer, older, olderK, **kw)
    b = direction_cloud(affine_inverse_f(T), older, newer, newerK, **kw)
    return dict(counts=a["counts"] + b["counts"], loose=np.concatenate([a["loose"], b["loose"]]),
                margin=np.concatenate([a["margin"], b["margin"]]))


# ---- the C oracle ---------------------------------------------------------------------------------------------------------

@functools.lru_cache(maxsize=1)
def _oracle_lib() -> C.CDLL:
    """tests/emm_cloud_oracle.c built into a temporary directory (the source tree may be read-only)."""
    out = Path(tempfile.mkdtemp(prefix="emm_cloud_oracle_")) / "libemm_cloud_oracle.so"
    subprocess.run(["gcc", "-O2", "-fPIC", "-shared", "-ffp-contract=off", "-Wall", "-o", str(out),
                    str(HERE / "emm_cloud_oracle.c"), "-lm"], check=True, capture_output=True)
    lib = C.CDLL(str(out))
    lib.emm_cloud_pairwise_observation.restype = None
    return lib


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


def oracle_pairwise_cloud(T4x4, newer_pc, newerK, older_pc, olderK, skip_step=8, sigma_depth=0.01, z0=None):
    """The C oracle of pairwise_cloud: z0 = latched depth for the covariance, None = per point.  Returns int64[4]."""
    T = np.ascontiguousarray(np.asarray(T4x4, F32).T)  # column-major Matrix4f
    nc, oc = np.ascontiguousarray(newer_pc, F32), np.ascontiguousarray(older_pc, F32)
    assert nc.ndim == 3 and oc.ndim == 3 and nc.shape[2] == oc.shape[2]
    nk, ok = np.ascontiguousarray(newerK, F32), np.ascontiguousarray(olderK, F32)
    out = np.zeros(4, np.uint32)
    _oracle_lib().emm_cloud_pairwise_observation(
        C.c_double(sigma_depth), C.c_double(-1.0 if z0 is None else z0), _p(T), _p(nc), C.c_int(nc.shape[1]),
        C.c_int(nc.shape[0]), _p(nk), _p(oc), C.c_int(oc.shape[1]), C.c_int(oc.shape[0]), _p(ok), C.c_int(nc.shape[2]),
        C.c_int(skip_step), _p(out))
    return out.astype(np.int64)
