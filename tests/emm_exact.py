"""Exact restatement of the environment measurement model (`k_emm_pairs`, `k_emm_single` in csrc/emm.cu).

- `cloud_z`: the z-plane of createXYZRGBPointCloud (misc.cpp:467-556) for a depth map, a cloud step, a scaling and a minimum
  depth.
- `direction`: observationLikelihood (misc.cpp:814-969) vectorised over the samples, in float32 with one rounding per
  operation in the reference's order (the reference is built without FMA contraction), the sigma sums in float64.  Besides
  the four counts it returns, for every sample, how far each depth comparison of its neighbourhood is from the 0.001 and
  0.999 cuts in p.  Those are the only decisions a few-ulp difference between two erf implementations can move.
- `pairwise`: pairwiseObservationLikelihood (node.cpp:1520-1554): one direction under T, the other under the float cofactor
  inverse of T.
- `loose`: a sample whose p lies within LOOSE (relative) of a cut; every other sample is decided the same way by any erf
  that is within a few ulps of the exact one.
"""
from __future__ import annotations

import numpy as np
from scipy.special import erf

F32, F64 = np.float32, np.float64
LOOSE = 1e-12
CUTS = (0.001, 0.999)


def cloud_z(depth, step=2, scaling=1.0, min_depth=0.1):
    """misc.cpp:467-556: every step-th pixel of the depth map times the (float) scaling, NaN where !(Z >= min_depth)."""
    d = np.asarray(depth, F32)
    h, w = d.shape
    z = (d[::step, ::step] * F32(scaling)).astype(F32)
    with np.errstate(invalid="ignore"):
        z = np.where(z >= F32(min_depth), z, F32(np.nan)).astype(F32)
    assert z.shape == ((h + step - 1) // step, (w + step - 1) // step)
    return z


def cov_const(sigma_depth, z0):
    """depth_covariance with its function-static latched at z0 (misc2.h:20-35)"""
    sd = sigma_depth * z0 * z0
    return sd * sd


def _cov(z, sigma_depth, czc):
    if czc is not None:
        return np.full(np.shape(z), czc, F64)
    sd = sigma_depth * z * z
    return sd * sd


def direction(T, src_z, srcK, dst_z, dstK, *, cloud_step=2, skip_step=8, sigma_depth=0.01, czc=None):
    """One direction: the `src` cloud under the float32 4x4 T (row-major numpy, src frame -> dst frame) projected into the
    `dst` raster.  K = (fx, fy, cx, cy) of the full-resolution camera.  czc: constant depth covariance (None = per point).
    Returns dict(counts=[good, bad, occluded, all], loose=bool per sample, margin=smallest |p / cut - 1| per sample)."""
    T = np.asarray(T, F32)
    R, t = T[:3, :3], T[:3, 3]
    src_z, dst_z = np.asarray(src_z, F32), np.asarray(dst_z, F32)
    sfx, sfy, scx, scy = (F32(k) for k in srcK)
    dfx, dfy, dcx, dcy = (F32(k) for k in dstK)
    sfxinv, sfyinv = F32(1.0 / F64(sfx)), F32(1.0 / F64(sfy))  # misc.cpp:64-69
    cs = F32(cloud_step)
    fx, fy, cx, cy = dfx / cs, dfy / cs, dcx / cs, dcy / cs   # misc.cpp:854-861
    sch, scw = src_z.shape
    dch, dcw = dst_z.shape
    ry, rx = np.meshgrid(np.arange(0, sch, skip_step), np.arange(0, scw, skip_step), indexing="ij")
    ry, rx = ry.ravel(), rx.ravel()
    n_all = len(rx)
    Z = src_z[ry, rx]
    u, v = (rx * cloud_step).astype(F32), (ry * cloud_step).astype(F32)
    zs = np.where(np.isnan(Z), F32(1), Z).astype(F32)
    px = ((u - scx) * zs) * sfxinv
    py = ((v - scy) * zs) * sfyinv
    pz = Z
    q = [((R[r, 0] * px + R[r, 1] * py) + R[r, 2] * pz) + t[r] for r in range(3)]  # pcl::transformPointCloud
    qx, qy, qz = (a.astype(F32) for a in q)
    with np.errstate(invalid="ignore", divide="ignore", over="ignore"):
        live = ~np.isnan(qz) & ~(qz < 0)
        xc = ((qx / qz) * fx + cx).astype(F32)
        yc = ((qy / qz) * fy + cy).astype(F32)
        ocx = np.floor(xc.astype(F64) + 0.5)   # misc.cpp:804-807
        ocy = np.floor(yc.astype(F64) + 0.5)
        live &= np.isfinite(ocx) & np.isfinite(ocy) & (ocx >= 0) & (ocx < dcw) & (ocy >= 0) & (ocy < dch)
    idx = np.nonzero(live)[0]
    cxi, cyi = ocx[idx].astype(np.int64), ocy[idx].astype(np.int64)
    qzl = qz[idx].astype(F64)
    good = np.zeros(len(idx), bool)
    occl = np.zeros(len(idx), bool)
    bad = np.zeros(len(idx), bool)
    margin = np.full(len(idx), np.inf)
    startx, starty = np.maximum(0, cxi - 2), np.maximum(0, cyi - 2)
    endx, endy = np.minimum(dcw, cxi + 3), np.minimum(dch, cyi + 3)
    new_sigma = cloud_step * _cov(qzl, sigma_depth, czc)
    for jy in range(3):
        oy = starty + 2 * jy
        for jx in range(3):
            ox = startx + 2 * jx
            inside = (oy < endy) & (ox < endx)
            oz = np.full(len(idx), np.nan, F32)
            oz[inside] = dst_z[oy[inside], ox[inside]]
            ok = inside & ~np.isnan(oz)
            oz64 = oz.astype(F64)
            with np.errstate(invalid="ignore"):
                joint = cloud_step * _cov(oz64, sigma_depth, czc) + new_sigma
                p = 0.5 * (1 + erf((oz64 - qzl) / (np.sqrt(joint) * 1.41421)))
            occl |= ok & (p < CUTS[0])
            good |= ok & (p >= CUTS[0]) & (p < CUTS[1])
            bad |= ok & (p >= CUTS[1])
            for c in CUTS:
                margin = np.where(ok, np.minimum(margin, np.abs(p / c - 1)), margin)
    g = int(good.sum())
    o = int((~good & occl).sum())
    b = int((~good & ~occl & bad).sum())
    m_all = np.full(n_all, np.inf)
    m_all[idx] = margin
    return dict(counts=np.array([g, b, o, n_all], np.int64), loose=m_all < LOOSE, margin=m_all)


def affine_inverse_f(T):
    """Matrix4f::inverse() of an affine transform as the float cofactor inverse, one rounding per operation."""
    T = np.asarray(T, F32)
    R = T[:3, :3]
    t = T[:3, 3]
    m = lambda a, b: F32(F32(a) * F32(b))
    c00 = F32(m(R[1, 1], R[2, 2]) - m(R[1, 2], R[2, 1]))
    c01 = F32(m(R[1, 2], R[2, 0]) - m(R[1, 0], R[2, 2]))
    c02 = F32(m(R[1, 0], R[2, 1]) - m(R[1, 1], R[2, 0]))
    det = F32(F32(m(R[0, 0], c00) + m(R[0, 1], c01)) + m(R[0, 2], c02))
    i = F32(F32(1) / det)
    Ri = np.array([
        [m(c00, i), m(F32(m(R[0, 2], R[2, 1]) - m(R[0, 1], R[2, 2])), i), m(F32(m(R[0, 1], R[1, 2]) - m(R[0, 2], R[1, 1])), i)],
        [m(c01, i), m(F32(m(R[0, 0], R[2, 2]) - m(R[0, 2], R[2, 0])), i), m(F32(m(R[0, 2], R[1, 0]) - m(R[0, 0], R[1, 2])), i)],
        [m(c02, i), m(F32(m(R[0, 1], R[2, 0]) - m(R[0, 0], R[2, 1])), i), m(F32(m(R[0, 0], R[1, 1]) - m(R[0, 1], R[1, 0])), i)],
    ], F32)
    Ti = np.eye(4, dtype=F32)
    Ti[:3, :3] = Ri
    for r in range(3):
        Ti[r, 3] = -F32(F32(m(Ri[r, 0], t[0]) + m(Ri[r, 1], t[1])) + m(Ri[r, 2], t[2]))
    return Ti


def pairwise(T, newer_z, newerK, older_z, olderK, **kw):
    """pairwiseObservationLikelihood: T maps the newer frame into the older one.  Returns dict(counts, loose) with the loose
    flags of both directions concatenated (newer samples first)."""
    a = direction(T, newer_z, newerK, older_z, olderK, **kw)
    b = direction(affine_inverse_f(T), older_z, olderK, newer_z, newerK, **kw)
    return dict(counts=a["counts"] + b["counts"], loose=np.concatenate([a["loose"], b["loose"]]),
                margin=np.concatenate([a["margin"], b["margin"]]))


def criterion(counts, threshold):
    """observation_criterion_met (misc.cpp:1136-1148) as the kernel evaluates it: quality and certainty in float64."""
    g, b, o = (int(x) for x in counts[:3])
    with np.errstate(invalid="ignore", divide="ignore"):
        quality = F64(g) / F64(g + b)
        certainty = F64(g) / F64(o + g + b)
    return bool(quality > threshold and certainty > 0.25), float(quality), float(certainty)


# ---- scenes ---------------------------------------------------------------------------------------------------------------

def plane_depth(w, h, K, n, d):
    """Depth of the plane n . X = d seen by a camera with intrinsics K (NaN where the ray misses or hits behind)."""
    fx, fy, cx, cy = K
    u, v = np.meshgrid(np.arange(w), np.arange(h))
    rx, ry = (u - cx) / fx, (v - cy) / fy
    den = n[0] * rx + n[1] * ry + n[2]
    with np.errstate(divide="ignore", invalid="ignore"):
        z = d / den
    return np.where(z > 0, z, np.nan).astype(F32)


def block_scene(rng, w, h, K, z=(0.6, 4.0), nblocks=(12, 9), holes=0.05):
    """Fronto-parallel blocks of random depth over a slanted background, with a few NaN holes: good, bad and occluded
    samples in every direction."""
    bg = plane_depth(w, h, K, np.array([0.1, -0.15, 1.0]), rng.uniform(*z))
    out = bg.copy()
    for _ in range(nblocks[0] * nblocks[1] // 3):
        x0, y0 = rng.integers(0, w - 20), rng.integers(0, h - 20)
        out[y0:y0 + rng.integers(10, max(11, h // 4)), x0:x0 + rng.integers(10, max(11, w // 4))] = rng.uniform(*z)
    out[rng.random(out.shape) < holes] = np.nan
    out += rng.normal(0, 0.004, out.shape).astype(F32)
    return out.astype(F32)


def rigid(rng, rot_deg, trans):
    axis = rng.normal(size=3)
    axis /= np.linalg.norm(axis)
    a = np.deg2rad(rot_deg)
    Kx = np.array([[0, -axis[2], axis[1]], [axis[2], 0, -axis[0]], [-axis[1], axis[0], 0]])
    T = np.eye(4)
    T[:3, :3] = np.eye(3) + np.sin(a) * Kx + (1 - np.cos(a)) * (Kx @ Kx)
    T[:3, 3] = trans
    return T.astype(F32)
