"""Exact restatements and input generators for the RANSAC stage (`ransac_hyp_kernel`, `ransac_select_kernel`).

- `scores_f64`: the float64 errorFunction2 decision (misc.cpp:697-770) of every correspondence under one float transform, with
  the z == 0 rule of computeInliersAndError (node.cpp:994), the shortcut of misc.cpp:726-735 and NaN rejection, for the
  constant (latched, misc2.h:30-35) and per-point depth covariance.  It also returns how far each correspondence is from the
  two cuts, so a test can tell a decision that float rounding could flip from one it cannot.
- `screen_f32`: a numpy emulation of the kernel's float32 screen (`mahal_screen`): every fmaf as an exact float64 product plus
  an add rounded to float32, `__fdividef` as a correctly rounded division.  The kernel trusts the screen only outside a 1e-3
  relative band around each cut and re-evaluates the rest in float64; `screen_envelope` measures how far the screen can be
  from the float64 value.
- `plant_near_cut`: correspondences planted at m = sq_max (1 +- delta) or at dsq = lim (1 +- delta).
- `pair_descriptors`: ORB descriptors whose Hamming matching yields a chosen correspondence order, so that tests decide which
  correspondences the distance-biased sampler (node.cpp:1024-1047) draws first.
- `scenario_pair`: noise-free-ish inliers and gross outliers arranged so that a chosen set of hypotheses draws all-inlier
  samples and every other hypothesis draws at least one outlier; this sets the path of the reference loop (node.cpp:1130-1190).
- `identity_planted_pair`: every hypothesis draws an outlier, so the pair ends in the identity fallback and rows planted near
  both cuts under T = I keep their margins in the transform the kernel returns.
- `degenerate_pair`: hypothesis 0 draws a rank-deficient sample (many-to-one matches or collinear from-points).
- `kabsch_f64`: the float64 weighted rigid fit (getTransformFromMatches): weights 1/(z_from z_to), NaN-depth rows skipped,
  R = U diag(1, 1, d) V^T of the weighted centred covariance C = sum w (to - m2)(from - m1)^T, d = sign(det U det V).
- `fit_f32`: a numpy emulation of the kernel's float32 fit (`fit_moments` + `fit_solve`, csrc/frontend_kernels.cu) in its
  operation order: the centroid the fit is centred on, per-lane sequential fmaf sums, the butterfly of `wsum16`, the Jacobi
  sweeps with their early exit, the column choice and the cross products.  MUFU steps (rsqrtf, __fdividef) are taken as IEEE
  operations, and products nvcc may contract into an fma are rounded separately.
- `fit_bound`: the error bound of that fit against `kabsch_f64`, derived below; `fit_cases`: the conditioning edges it is
  checked on.

The fit's error bound.  u = 2^-24.  The kernel centres every row on the pair's float centroid c (one rounding per coordinate,
relative to the centred value) and sums the 16 moments per lane (ceil(M/32) sequential fmaf adds) and then over a 5-level
butterfly, so with L = ceil(M/32) + 5 every moment carries at most L u of the sum of its terms' magnitudes.  The weight (two
roundings), the weighted to-point (one) and the centring (two) add 5 u per term, and fit_solve's 1/W, means and the
subtraction C = S/W - m2 m1^T add 5 u more.  With A = E_w[|b~| |a~|] + |m2~| |m1~| (a~, b~ the rows centred on c, E_w the
weighted mean: A >= ||C||_F, and A is the size of the float sums C is formed from, which exceeds ||C||_F when the weighted
mean lies far from c)
    ||dC||_F <= (L + 10) u A.
The one-sided Jacobi applies at most 6 sweeps x 3 rotations; a rotation from the 2-ulp rsqrtf / __fdividef and two rounded
products is orthogonal to 6 u, so the sweeps add at most 18 x 6 u ||C||_F <= 108 u A of backward error.  The rotation factor
of C moves by at most 2 ||dC||_F / (s2 + d s3) (s1 >= s2 >= s3 the singular values of C).  The exit test leaves columns at most
4e-7 (7 u) from orthogonal, and the normalisation (2-ulp rsqrtf), the cross products and the three-term sums of R add about
8 u more: 30 u in all, absolute, which is at most 60 u A / (s2 + d s3) because s2 + d s3 <= 2 s1 <= 2 A.  So
    ||R_gpu - R64||_max <= K u A / (s2 + d s3),   K = 2 (L + 10 + 108) + 60 = 2 L + 296.
The translation t = (m2 + c_to) - R (m1 + c_from) adds the means' error ((L + 3) u of E_w|a~|, E_w|b~|), the centroid add-back
and the 3-term product (4 u of |g1|) and the final subtraction (u of |g2| + |g1|):
    |t_gpu - t64 + (R_gpu - R64) g1| <= K u (|g2| + |g1| + E_w|a~| + E_w|b~|)
with g1, g2 the weighted centroids: the translation is the one R_gpu implies (t64 = g2 - R64 g1), which bounds
|t_gpu - t64| by ||R_gpu - R64||_2 |g1| plus the same term without letting a rotation error hide a translation error.  Separately, |det R - 1| and ||R^T R - I||_max stay below 1e-5 (SHAPE_TOL).
"""
from __future__ import annotations

import ctypes as C

import numpy as np

_ax = 58.0 / 180.0 * np.pi
_ay = 45.0 / 180.0 * np.pi
RCX = (3 * np.tan(_ax / 640)) ** 2  # misc.cpp:702-709
RCY = (3 * np.tan(_ay / 480)) ** 2
F32, F64 = np.float32, np.float64


def sq_max_of(max_dist: float) -> float:
    """node.cpp:1105,1152: a float max_dist_m squared in float, promoted to double."""
    m = F32(max_dist)
    return float(F64(F32(m * m)))


def cov_const(sigma_depth: float, z0: float) -> float:
    """misc2.h:20-35 with the function-static latched at depth z0."""
    sd = sigma_depth * z0 * z0
    return sd * sd


def _cz(z, sigma_depth, czc):
    if czc is not None:
        return np.full(z.shape, czc, F64)
    sd = sigma_depth * (z * z)
    return sd * sd


def _mahal(R, d, z1, z2, cz1, cz2):
    """d^T S^-1 d, S = R^T diag(rcx z1, rcy z1, cz1) R + diag(rcx z2, rcy z2, cz2), by the adjugate (as the kernel does)."""
    c1 = np.stack([RCX * z1, RCY * z1, cz1], 1)
    S = np.einsum("ki,nk,kj->nij", R, c1, R)
    S[:, 0, 0] += RCX * z2
    S[:, 1, 1] += RCY * z2
    S[:, 2, 2] += cz2
    s00, s01, s02, s11, s12, s22 = S[:, 0, 0], S[:, 0, 1], S[:, 0, 2], S[:, 1, 1], S[:, 1, 2], S[:, 2, 2]
    A00, A01, A02 = s11 * s22 - s12 * s12, s02 * s12 - s01 * s22, s01 * s12 - s02 * s11
    A11, A12, A22 = s00 * s22 - s02 * s02, s01 * s02 - s00 * s12, s00 * s11 - s01 * s01
    det = s00 * A00 + s01 * A01 + s02 * A02
    d0, d1, d2 = d[:, 0], d[:, 1], d[:, 2]
    num = d0 * (A00 * d0 + A01 * d1 + A02 * d2) + d1 * (A01 * d0 + A11 * d1 + A12 * d2) + d2 * (A02 * d0 + A12 * d1 + A22 * d2)
    with np.errstate(invalid="ignore", divide="ignore"):
        return num / det


def scores_f64(T, frm, to, *, max_dist=3.0, sigma_depth=0.01, czc=None):
    """The float64 inlier decision of every correspondence (frm[i] -> to[i], (x, y, z, w) float32 rows) under the float32
    4x4 transform T (row-major numpy; cast to double like node.cpp:984).  czc: constant depth covariance (latched z0), None
    for the per-point model.  Returns a dict:
      inl       bool mask (node.cpp:994-1005)
      cnt, esum number of inliers and the float64 sum of their errors; rmse = sqrt(esum / cnt) (1e9 below 3 inliers)
      m, dsq, lim  float64 error, squared distance and shortcut limit (m is inf where a rule rejects before the solve)
      m_margin  |m / sq_max - 1| (inf where m is not evaluated)      s_margin  |dsq / lim - 1|
      scored    the rows errorFunction2 is called for (both z non-zero)."""
    T = np.asarray(T, F32).astype(F64)
    R, t = T[:3, :3], T[:3, 3]
    a = np.asarray(frm, F32).reshape(-1, 4)
    b = np.asarray(to, F32).reshape(-1, 4)
    scored = ~((a[:, 2] == 0) | (b[:, 2] == 0))
    a64, b64 = a.astype(F64), b.astype(F64)
    mu = a64[:, :3] @ R.T + a64[:, 3:4] * t
    d = mu - b64[:, :3]
    z1, z2 = a64[:, 2], b64[:, 2]
    nan = np.isnan(z1) | np.isnan(z2)
    cz1, cz2 = _cz(z1, sigma_depth, czc), _cz(z2, sigma_depth, czc)
    dsq = (d * d).sum(1)
    lim = 2.0 * (np.maximum(RCX, cz1) + np.maximum(RCX, cz2))
    with np.errstate(invalid="ignore"):
        short = dsq > lim
    m = _mahal(R, d, z1, z2, cz1, cz2)
    sq_max = sq_max_of(max_dist)
    with np.errstate(invalid="ignore"):
        ok = scored & ~nan & ~short & (m >= 0)
        inl = ok & (m <= sq_max)
        m_margin = np.where(scored & ~nan & ~short & (m >= 0), np.abs(m / sq_max - 1), np.inf)
        s_margin = np.where(scored & ~nan & np.isfinite(dsq), np.abs(dsq / lim - 1), np.inf)
    cnt = int(inl.sum())
    esum = float(m[inl].sum())
    rmse = 1e9 if cnt < 3 else float(np.sqrt(esum / cnt))
    return dict(inl=inl, cnt=cnt, esum=esum, rmse=rmse, m=np.where(ok, m, np.inf), dsq=dsq, lim=lim, m_margin=m_margin,
                s_margin=s_margin, scored=scored, sq_max=sq_max)


# ---- the float32 screen ---------------------------------------------------------------------------------------------------

def _fma(a, b, c):
    return (F64(a) * F64(b) + F64(c)).astype(F32) if np.ndim(a) or np.ndim(b) or np.ndim(c) else F32(F64(a) * F64(b) + F64(c))


def screen_f32(T, frm, to, *, max_dist=3.0, sigma_depth=0.01, czc=None):
    """mahal_screen (csrc/frontend_kernels.cu) step for step in float32.  Returns (m, dsq, lim, det) as float32 arrays."""
    T = np.asarray(T, F32)
    R, t = T[:3, :3], T[:3, 3]
    x1 = np.asarray(frm, F32).reshape(-1, 4)
    x2 = np.asarray(to, F32).reshape(-1, 4)
    f = _fma
    d = [f(R[r, 0], x1[:, 0], f(R[r, 1], x1[:, 1], f(R[r, 2], x1[:, 2], (t[r] * x1[:, 3]).astype(F32)))) - x2[:, r]
         for r in range(3)]
    d0, d1, d2 = (x.astype(F32) for x in d)
    rcx, rcy = F32(RCX), F32(RCY)
    I, J = (0, 0, 0, 1, 1, 2), (0, 1, 2, 1, 2, 2)
    Pf = [f((rcx * R[0, I[k]]).astype(F32), R[0, J[k]], ((rcy * R[1, I[k]]).astype(F32) * R[1, J[k]]).astype(F32)) for k in range(6)]
    O2f = [F32(R[2, I[k]] * R[2, J[k]]) for k in range(6)]
    dsq = f(d0, d0, f(d1, d1, (d2 * d2).astype(F32)))
    a2, b2 = x1[:, 2], x2[:, 2]
    if czc is not None:
        c = F32(czc)
        # `czc * O2f[k] + (k == 5 ? czc : 0.f)`: nvcc (--fmad=true by default) contracts it into one fmaf
        Cc = [f(c, O2f[k], c if k == 5 else F32(0)) for k in range(6)]
        lim = np.full(len(x1), F32(2) * (max(rcx, c) + max(rcx, c)), F32)
        S00 = f(a2, Pf[0], f(rcx, b2, Cc[0]))
        S01 = f(a2, Pf[1], Cc[1])
        S02 = f(a2, Pf[2], Cc[2])
        S11 = f(a2, Pf[3], f(rcy, b2, Cc[3]))
        S12 = f(a2, Pf[4], Cc[4])
        S22 = f(a2, Pf[5], Cc[5])
    else:
        sg = F32(sigma_depth)
        sd1 = (sg * (a2 * a2).astype(F32)).astype(F32)
        sd2 = (sg * (b2 * b2).astype(F32)).astype(F32)
        cz1, cz2 = (sd1 * sd1).astype(F32), (sd2 * sd2).astype(F32)
        lim = (F32(2) * (np.maximum(rcx, cz1) + np.maximum(rcx, cz2)).astype(F32)).astype(F32)
        S00 = f(a2, Pf[0], f(cz1, O2f[0], (rcx * b2).astype(F32)))
        S01 = f(a2, Pf[1], (cz1 * O2f[1]).astype(F32))
        S02 = f(a2, Pf[2], (cz1 * O2f[2]).astype(F32))
        S11 = f(a2, Pf[3], f(cz1, O2f[3], (rcy * b2).astype(F32)))
        S12 = f(a2, Pf[4], (cz1 * O2f[4]).astype(F32))
        S22 = f(a2, Pf[5], f(cz1, O2f[5], cz2))
    k = F32(1024)
    s00, s01, s02, s11, s12, s22 = ((x * k).astype(F32) for x in (S00, S01, S02, S11, S12, S22))
    neg = lambda x: (-x).astype(F32)
    A00 = f(s11, s22, neg(s12 * s12)); A01 = f(s02, s12, neg(s01 * s22)); A02 = f(s01, s12, neg(s02 * s11))
    A11 = f(s00, s22, neg(s02 * s02)); A12 = f(s01, s02, neg(s00 * s12)); A22 = f(s00, s11, neg(s01 * s01))
    det = f(s00, A00, f(s01, A01, (s02 * A02).astype(F32)))
    e0 = f(A00, d0, f(A01, d1, (A02 * d2).astype(F32)))
    e1 = f(A01, d0, f(A11, d1, (A12 * d2).astype(F32)))
    e2 = f(A02, d0, f(A12, d1, (A22 * d2).astype(F32)))
    num = (f(d0, e0, f(d1, e1, (d2 * e2).astype(F32))) * k).astype(F32)
    with np.errstate(invalid="ignore", divide="ignore"):
        m = (num.astype(F64) / det.astype(F64)).astype(F32)
    return m, dsq, lim, det


def screen_codes(m, dsq, lim, det, x1z, x2z, sq_max):
    """The screen's three-way outcome (mahal_screen's return): +1 certain inlier, -1 certain reject, 0 undecided."""
    sq = F32(sq_max)
    with np.errstate(invalid="ignore"):
        reject1 = np.isnan(x1z) | np.isnan(x2z) | (dsq > lim * F32(1.001))
        unsure = ~(dsq < lim * F32(0.999)) | ~(m >= 0) | ~(det > 0)
        r = np.where(m > sq * F32(1.001), -1, np.where(m < sq * F32(0.999), 1, 0))
    return np.where(reject1, -1, np.where(unsure, 0, r))


def screen_envelope(T, frm, to, band=3e-3, **kw):
    """Largest relative error of the screen's m and dsq/lim against float64 over the correspondences within `band` of a cut
    (those are the ones where an error could change a decision), plus the number of decisions the screen gets wrong
    (certain inlier / certain reject where float64 decides the other way)."""
    ref = scores_f64(T, frm, to, **kw)
    m, dsq, lim, det = screen_f32(T, frm, to, **kw)
    x1, x2 = np.asarray(frm, F32), np.asarray(to, F32)
    near_m = np.isfinite(ref["m"]) & (ref["m_margin"] < band)
    near_s = ref["s_margin"] < band
    with np.errstate(invalid="ignore", divide="ignore"):
        em = np.abs(m[near_m].astype(F64) / ref["m"][near_m] - 1)
        es = np.abs((dsq[near_s].astype(F64) / lim[near_s]) / (ref["dsq"][near_s] / ref["lim"][near_s]) - 1)
    code = screen_codes(m, dsq, lim, det, x1[:, 2], x2[:, 2], ref["sq_max"])
    sc = ref["scored"]
    wrong = int((sc & (code == 1) & ~ref["inl"]).sum() + (sc & (code == -1) & ref["inl"]).sum())
    return dict(m_err=float(em.max(initial=0.0)), s_err=float(es.max(initial=0.0)), n_m=int(near_m.sum()),
                n_s=int(near_s.sum()), wrong=wrong, undecided=int((sc & (code == 0)).sum()))


# ---- the rigid fit --------------------------------------------------------------------------------------------------------

U32 = 2.0 ** -24
SHAPE_TOL = 1e-5


def _fit_rows(frm, to, sel=None):
    """float64 copies of the selected rows whose depth is finite on both sides (transformation_estimation_euclidean.cpp:22)."""
    a = np.asarray(frm, F32).reshape(-1, 4).astype(F64)
    b = np.asarray(to, F32).reshape(-1, 4).astype(F64)
    keep = ~(np.isnan(a[:, 2]) | np.isnan(b[:, 2]))
    if sel is not None:
        m = np.zeros(len(a), bool)
        m[sel] = True
        keep &= m
    return a[keep], b[keep]


def kabsch_f64(frm, to, sel=None):
    """The weighted rigid fit of getTransformFromMatches in float64: R, t minimising sum w |R from + t - to|^2 with
    w = 1/(z_from z_to) over the rows (of `sel`, indices or a mask) with a finite depth on both sides.  Returns
    (R, t, s, d): s the singular values of the weighted centred covariance C = sum w (to - m2)(from - m1)^T / W, descending,
    and d = sign(det U det V), so R = U diag(1, 1, d) V^T."""
    a, b = _fit_rows(frm, to, sel)
    w = 1.0 / (a[:, 2] * b[:, 2])  # :25
    w = w / w.sum()
    m1, m2 = w @ a[:, :3], w @ b[:, :3]
    Cm = ((b[:, :3] - m2) * w[:, None]).T @ (a[:, :3] - m1)
    U, S, Vt = np.linalg.svd(Cm)
    d = 1.0 if np.linalg.det(U) * np.linalg.det(Vt) >= 0 else -1.0
    R = U @ np.diag([1.0, 1.0, d]) @ Vt
    return R, m2 - R @ m1, S, d


def _bfly(x):
    """wsum / wsum16: the xor butterfly over 32 lanes (offsets 16, 8, 4, 2, 1); every lane ends with the same float."""
    x = np.asarray(x, F32)
    idx = np.arange(32)
    for o in (16, 8, 4, 2, 1):
        x = (x + x[idx ^ o]).astype(F32)
    return x[0]


def centroid_f32(frm, to):
    """The centroid ransac_hyp_kernel centres the fit on: kCenWarps = 8 virtual warps, virtual lane v sums rows v, v + 256
    (rows with a NaN coordinate left out), each warp's butterfly, the 8 warp sums in order, divided by M."""
    a = np.asarray(frm, F32).reshape(-1, 4)
    b = np.asarray(to, F32).reshape(-1, 4)
    M = len(a)
    x = np.concatenate([a[:, :3], b[:, :3]], 1)
    ok = ~np.isnan(x.sum(1))
    cs = np.zeros((256, 6), F32)
    for i in range(M):
        if ok[i]:
            cs[i % 256] = (cs[i % 256] + x[i]).astype(F32)
    tot = np.zeros(6, F32)
    for w in range(8):
        part = np.array([_bfly(cs[w * 32:(w + 1) * 32, k]) for k in range(6)], F32)
        tot = (tot + part).astype(F32)
    return (tot / F32(M)).astype(F32)


def _fmaf(a, b, c):
    return F32(F64(a) * F64(b) + F64(c))


def _rsq(x):
    return F32(1.0 / np.sqrt(F64(x)))


def fit_f32(frm, to, sel, *, sweeps=6):
    """fit_moments + fit_solve in float32 on the pair's rows frm / to ((M, 4) float32, the fit's centroid is taken over all M
    rows) for the rows of `sel` (indices or a mask).  Returns (R, t, ok) with R (3, 3) and t (3,) float32; ok is False where
    the kernel reports a failed fit (no weight, rank < 2, or a non-finite result)."""
    a = np.asarray(frm, F32).reshape(-1, 4)
    b = np.asarray(to, F32).reshape(-1, 4)
    M = len(a)
    cen = centroid_f32(a, b)
    ca = np.concatenate([(a[:, :3] - cen[:3]).astype(F32), a[:, 2:3]], 1)
    cb = np.concatenate([(b[:, :3] - cen[3:]).astype(F32), b[:, 2:3]], 1)
    mask = np.zeros(M, bool)
    mask[sel] = True
    # fit_moments: lane l adds rows l, l + 32, ... in order
    acc = np.zeros((32, 16), F32)
    for w in range((M + 31) // 32):
        for lane in range(32):
            i = w * 32 + lane
            if i >= M or not mask[i]:
                continue
            p, q = ca[i], cb[i]
            if np.isnan(p[3]) or np.isnan(q[3]):
                continue
            m = acc[lane]
            wt = F32(F32(1.0) / F32(p[3] * q[3]))
            m[0] = F32(m[0] + wt)
            for k in range(3):
                m[1 + k] = _fmaf(wt, p[k], m[1 + k])
            bw = [F32(wt * q[k]) for k in range(3)]
            for k in range(3):
                m[4 + k] = F32(m[4 + k] + bw[k])
            for r in range(3):
                for k in range(3):
                    m[7 + 3 * r + k] = _fmaf(bw[r], p[k], m[7 + 3 * r + k])
    mom = np.array([_bfly(acc[:, j]) for j in range(16)], F32)
    # fit_solve
    W = mom[0]
    if not W > 0:
        return np.eye(3, dtype=F32), np.zeros(3, F32), False
    iW = F32(F32(1.0) / W)
    m1 = [F32(mom[1 + k] * iW) for k in range(3)]
    m2 = [F32(mom[4 + k] * iW) for k in range(3)]
    A = np.array([[F32(F32(mom[7 + 3 * r + k] * iW) - F32(m2[r] * m1[k])) for k in range(3)] for r in range(3)], F32)
    V = np.eye(3, dtype=F32)

    def dot(x, y):
        return F32(F32(F32(x[0] * y[0]) + F32(x[1] * y[1])) + F32(x[2] * y[2]))

    for _ in range(sweeps):
        rotated = False
        for pp, qq in ((0, 1), (0, 2), (1, 2)):
            al, be, ga = dot(A[:, pp], A[:, pp]), dot(A[:, qq], A[:, qq]), dot(A[:, pp], A[:, qq])
            if not F32(ga * ga) > F32(F32(1.6e-13) * F32(al * be)):
                continue
            if F32(ga * ga) > F32(F32(1e-7) * F32(al * be)):
                rotated = True
            dd, g2 = F32(be - al), F32(F32(2) * ga)
            hh = F32(np.sqrt(_fmaf(dd, dd, F32(g2 * g2))))
            sg = F32(-1) if (dd < 0) != (g2 < 0) else F32(1)
            tt = F32(sg * F32(abs(g2) / F32(abs(dd) + hh)))
            cs = _rsq(_fmaf(tt, tt, F32(1)))
            sn = F32(cs * tt)
            for X in (A, V):
                x, y = X[:, pp].copy(), X[:, qq].copy()
                X[:, pp] = (F32(cs) * x - F32(sn) * y).astype(F32)
                X[:, qq] = (F32(sn) * x + F32(cs) * y).astype(F32)
        if not rotated:
            break
    n = [dot(A[:, k], A[:, k]) for k in range(3)]
    ip = 0
    if n[1] > n[0]:
        ip = 1
    if n[2] > n[ip]:
        ip = 2
    iq = {0: 2 if n[2] > n[1] else 1, 1: 2 if n[2] > n[0] else 0, 2: 1 if n[1] > n[0] else 0}[ip]
    if not (n[ip] > 0) or not (n[iq] > F32(F32(1e-24) * n[ip])):
        return np.eye(3, dtype=F32), np.zeros(3, F32), False
    p = (A[:, ip] * _rsq(n[ip])).astype(F32)
    q = (A[:, iq] * _rsq(n[iq])).astype(F32)
    vp, vq = V[:, ip], V[:, iq]

    def cross(x, y):
        return np.array([F32(x[1] * y[2]) - F32(x[2] * y[1]), F32(x[2] * y[0]) - F32(x[0] * y[2]),
                         F32(x[0] * y[1]) - F32(x[1] * y[0])], F32)

    u3, v3 = cross(p, q), cross(vp, vq)
    R = np.array([[F32(F32(F32(p[r] * vp[k]) + F32(q[r] * vq[k])) + F32(u3[r] * v3[k])) for k in range(3)] for r in range(3)],
                 F32)
    g1 = [F32(m1[k] + cen[k]) for k in range(3)]
    t = np.array([F32(F32(m2[r] + cen[3 + r]) - dot(R[r], g1)) for r in range(3)], F32)
    ok = bool(np.isfinite(R).all() and np.isfinite(t).all())
    return R, t, ok


def fit_K(M):
    """K of the rotation bound (module docstring) for a pair of M rows."""
    return 2 * (-(-M // 32) + 5) + 296


def fit_bound(frm, to, sel=None):
    """The bound of the module docstring for the fit of the rows `sel` of a pair (frm, to: all M rows, which set the
    centroid).  Returns a dict: rot and trans, the bounds on ||R_gpu - R64||_max and |t_gpu - t64 + (R_gpu - R64) g1|_max;
    R, t, s, d of kabsch_f64, the conditioning ratio cond = A / (s2 + d s3), K and the weighted from-centroid g1."""
    R, t, s, d = kabsch_f64(frm, to, sel)
    M = len(np.asarray(frm).reshape(-1, 4))
    c = centroid_f32(frm, to).astype(F64)
    a, b = _fit_rows(frm, to, sel)
    w = 1.0 / (a[:, 2] * b[:, 2])
    w = w / w.sum()
    at, bt = a[:, :3] - c[:3], b[:, :3] - c[3:]
    na, nb = np.linalg.norm(at, axis=1), np.linalg.norm(bt, axis=1)
    A = w @ (na * nb) + np.linalg.norm(w @ at) * np.linalg.norm(w @ bt)
    K = fit_K(M)
    cond = A / (s[1] + d * s[2])
    g1, g2 = w @ a[:, :3], w @ b[:, :3]
    tmag = np.linalg.norm(g1) + np.linalg.norm(g2) + w @ na + w @ nb
    return dict(rot=K * U32 * cond, trans=K * U32 * tmag, R=R, t=t, s=s, d=d, cond=cond, K=K, g1=g1)


def fit_errors(R, t, ref):
    """(rotation error, translation error, shape error) of a fit (R, t) against fit_bound's ref: ||R - R64||_max,
    |t - t64 + (R - R64) g1|_max (bounded by ref["trans"]) and max(|det R - 1|, ||R^T R - I||_max)."""
    R64, t64 = np.asarray(R, F64), np.asarray(t, F64)
    dR = R64 - ref["R"]
    shape = max(abs(np.linalg.det(R64) - 1), np.abs(R64.T @ R64 - np.eye(3)).max())
    return float(np.abs(dR).max()), float(np.abs(t64 - ref["t"] + dR @ ref["g1"]).max()), float(shape)


# ---- generators -----------------------------------------------------------------------------------------------------------

FX = FY = 525.0
CX, CY = 319.5, 239.5


def frustum_points(rng, n, zlo, zhi):
    u = rng.uniform(31, 609, n)
    v = rng.uniform(31, 449, n)
    z = rng.uniform(zlo, zhi, n)
    return np.stack([(u - CX) * z / FX, (v - CY) * z / FY, z], 1)


def small_motion(rng, max_trans=0.05, max_rot_deg=2.0):
    axis = rng.normal(size=3)
    axis /= np.linalg.norm(axis)
    ang = np.deg2rad(rng.uniform(0.2, 1.0) * max_rot_deg)
    K = np.array([[0, -axis[2], axis[1]], [axis[2], 0, -axis[0]], [-axis[1], axis[0], 0]])
    T = np.eye(4)
    T[:3, :3] = np.eye(3) + np.sin(ang) * K + (1 - np.cos(ang)) * (K @ K)
    t = rng.normal(size=3)
    T[:3, 3] = t * rng.uniform(0.2, 1.0) * max_trans / np.linalg.norm(t)
    return T


def to4(p):
    return np.concatenate([p, np.ones((len(p), 1))], 1).astype(F32)


def _m_of(T, p, q, sigma_depth, czc):
    R = np.asarray(T, F32).astype(F64)[:3, :3]
    d = p @ R.T + np.asarray(T, F32).astype(F64)[:3, 3] - q
    cz1, cz2 = _cz(p[:, 2], sigma_depth, czc), _cz(q[:, 2], sigma_depth, czc)
    return _mahal(R, d, p[:, 2], q[:, 2], cz1, cz2), (d * d).sum(1), 2.0 * (np.maximum(RCX, cz1) + np.maximum(RCX, cz2))


def plant_near_cut(rng, T, p, kind, delta, *, max_dist=3.0, sigma_depth=0.01, czc=None):
    """To-points for from-points p (n x 3, float64) that sit at m = sq_max (1 + delta) (kind 'm', random direction) or at
    dsq = lim (1 + delta) (kind 's', along the direction of least Mahalanobis weight, so that the shortcut and not the
    threshold decides).  T is the float transform the points are planted under.  Returns (to+e, to-e): the two mirrored
    to-points of each from-point; displacements of +e and -e cancel in the weighted covariance of the fit."""
    Tf = np.asarray(T, F32).astype(F64)
    base = p @ Tf[:3, :3].T + Tf[:3, 3]
    n = len(p)
    delta = np.broadcast_to(np.asarray(delta, F64), (n,)).copy()
    if kind == "m":  # in the image plane: both mirrored plants keep the depth, so their fit weights 1/(z1 z2) are equal
        u = rng.normal(size=(n, 3))
        u[:, 2] = 0.0
    else:  # z-ish direction: the depth covariance dominates S there
        u = np.zeros((n, 3))
        u[:, 2] = 1.0
        u += rng.normal(scale=0.002, size=(n, 3))
    u /= np.linalg.norm(u, axis=1, keepdims=True)

    def solve(sign, delta):
        target_m = sq_max_of(max_dist) * (1 + delta)
        ss = np.full(n, 1e-3)
        for _ in range(60):
            q = base - sign * ss[:, None] * u  # d = T p - q = sign * s * u
            m, dsq, lim = _m_of(T, p, q, sigma_depth, czc)
            ratio = target_m / m if kind == "m" else lim * (1 + delta) / dsq
            ss = ss * np.sqrt(np.clip(ratio, 0.25, 4.0))
            if np.abs(ratio - 1).max() < 1e-13:
                break
        return base - sign * ss[:, None] * u

    if kind == "m":
        return solve(1.0, delta), solve(-1.0, delta)
    # Shortcut plants move along the depth axis.  With a constant covariance the plant at the limit moves away from the camera;
    # with the per-point model (limit ~ z^4, no fixed point far from the camera) towards it.  Its partner is a balancer on the
    # other side, displaced so that the two weighted displacements cancel in the fit: c_b = -c_a z / (z + 2 c_a).
    a = solve(-1.0 if czc is not None else 1.0, delta)
    ca = a[:, 2] - base[:, 2]
    bad = base[:, 2] + 2 * ca < 0.2 * base[:, 2]
    if bad.any():  # no balancer with a positive depth: plant outside the limit (rejected, so it does not enter the fit)
        delta[bad] = np.abs(delta[bad])
        a = np.where(bad[:, None], solve(1.0, delta), a)
        ca = a[:, 2] - base[:, 2]
    scale = np.where(bad, 1.0, -base[:, 2] / (base[:, 2] + 2 * ca))
    return a, base + (a - base) * scale[:, None]


def log_uniform_delta(rng, n, lo=1e-5, hi=3e-2):
    """delta log-uniform in [lo, hi] with a random sign"""
    return np.exp(rng.uniform(np.log(lo), np.log(hi), n)) * rng.choice([-1.0, 1.0], n)


def pair_descriptors(rng, M, n_extra_train=1):
    """ORB descriptors for M queries that match train rows 0..M-1 (query k = train k with 0..60 bits flipped: every other
    train row is ~128 bits away) plus `n_extra_train` unmatched train rows at the end (bruteForceSearchORB never examines the
    last row, features.cpp:172).  The sort order of the matches is fixed by the Hamming distances and the jitter of
    node.cpp:573; the caller reads it from the oracle's match list and places the correspondences by rank."""
    t = rng.integers(0, 256, (M + n_extra_train, 32), dtype=np.uint8)
    q = t[:M].copy()
    hd = rng.integers(0, 61, M)
    for k in range(M):
        bits = rng.permutation(256)[:hd[k]]
        flip = np.zeros(256, np.uint8)
        flip[bits] = 1
        q[k] ^= np.packbits(flip, bitorder="little")
    return q, t


def place_by_rank(oracle_mod, q, t, frm, to, seed, pair, max_matches):
    """xyz arrays (newer = query side, older = train side) such that the match of sort rank j carries correspondence
    frm[j] -> to[j].  Returns (xyz_newer, xyz_older, matches)."""
    mlist = oracle_mod.feature_matching_orb(q, t, max_matches, seed, pair)
    M = len(frm)
    assert len(mlist) == M and np.array_equal(np.sort(mlist["queryIdx"]), np.arange(M))
    assert np.array_equal(mlist["queryIdx"], mlist["trainIdx"]), "a query matched the wrong train row"
    xn = np.zeros((len(q), 4), F32)
    xo = np.zeros((len(t), 4), F32)
    xo[:, 3] = 1
    xo[M:, 2] = 1.0
    xn[mlist["queryIdx"]] = frm
    xo[mlist["trainIdx"]] = to
    return xn, xo, mlist


def concat_batch(pairs, first_id=0):
    """Host buffers of match_pairs_host / oracle.match_pairs from a list of (desc_newer, xyz_newer, desc_older, xyz_older)."""
    cat = lambda k: np.ascontiguousarray(np.concatenate([p[k] for p in pairs]))
    n = len(pairs)
    return dict(desc_newer=cat(0), xyz_newer=cat(1), desc_older=cat(2), xyz_older=cat(3),
                n_newer=np.array([len(p[0]) for p in pairs], np.int32), n_older=np.array([len(p[2]) for p in pairs], np.int32),
                id_newer=np.arange(n, dtype=np.int32) + first_id + 1000, id_older=np.arange(n, dtype=np.int32) + first_id)


def hypothesis_samples(oracle_mod, M, H, seed, pair):
    """The 4 match indices hypothesis n draws (sample_matches_prefer_by_distance, node.cpp:1024-1047), n < H."""
    fn = oracle_mod.lib().oracle_sample_matches_prefer_by_distance
    fn.restype = C.c_int
    fn.argtypes = [C.c_int, C.c_int, C.c_uint64, C.c_uint64, C.c_uint32, C.c_void_p]
    out = np.zeros((H, 4), np.int32)
    ids = np.zeros(4, np.int32)
    for n in range(H):
        k = fn(4, M, seed, pair, n, ids.ctypes.data)
        assert k == 4
        out[n] = ids
    return out


def plan_outliers(samples, valid, M, n_out, rng):
    """An outlier mask over M ranks with n_out outliers such that sample n is all-inlier exactly for n in `valid` (a set of
    hypothesis indices) and holds an outlier for every other n < len(samples).  Greedy cover: the rank that appears in the
    most uncovered samples becomes an outlier first.  Returns None when the samples make that impossible."""
    forced_in = np.zeros(M, bool)
    for n in valid:
        if n < len(samples):
            forced_in[samples[n]] = True
    out = np.zeros(M, bool)
    todo = [samples[n] for n in range(len(samples)) if n not in valid]
    while True:
        todo = [s for s in todo if not out[s].any()]
        if not todo:
            break
        hits = np.zeros(M)
        for s in todo:
            free = s[~forced_in[s]]
            if len(free) == 0:
                return None
            hits[free] += 1 + 1e-3 * rng.random(len(free))
        out[int(np.argmax(hits))] = True
    if out.sum() > n_out:
        return None
    rest = np.nonzero(~out & ~forced_in)[0]
    if len(rest) < n_out - out.sum():
        return None
    out[rng.choice(rest, n_out - int(out.sum()), replace=False)] = True
    return out


def scenario_pair(oracle_mod, rng, M, H, valid, n_out, seed, pair, *, T=None, max_matches=300, noise=0.002, z=(1.0, 3.0),
                  outliers_last=False):
    """One pair of M matches whose hypotheses [0, H) draw all-inlier samples exactly for n in `valid` (noisy inliers that sit
    far inside the threshold; gross outliers that the shortcut rejects).  outliers_last: no plan, the n_out outliers take the
    last ranks (most samples are then all-inlier).  Returns (desc_newer, xyz_newer, desc_older, xyz_older, T_true)."""
    if outliers_last:
        out = np.zeros(M, bool)
        out[M - n_out:] = True
    else:
        # the plan covers the first 40 hypotheses (a > 80 % pair breaks before; the plans with jumps use H <= 40)
        samples = hypothesis_samples(oracle_mod, M, min(H, 40), seed, pair) if M >= 4 else np.zeros((0, 4), np.int32)
        out = plan_outliers(samples, set(valid), M, n_out, rng)
        if out is None:
            raise RuntimeError(f"no outlier placement satisfies the plan (M={M}, H={H}, valid={valid}, n_out={n_out})")
    T = small_motion(rng) if T is None else T
    p = frustum_points(rng, M, *z)
    q = p @ T[:3, :3].T + T[:3, 3]
    q[:, :2] += np.clip(rng.normal(scale=noise, size=(M, 2)), -2.5 * noise, 2.5 * noise)
    q[:, 2] += np.clip(rng.normal(scale=noise, size=M), -2.5 * noise, 2.5 * noise)
    q[out] = _gross(rng, q[out])
    qd, td = pair_descriptors(rng, M)
    xn, xo, _ = place_by_rank(oracle_mod, qd, td, to4(p), to4(q), seed, pair, max_matches)
    return qd, xn, td, xo, T


def _gross(rng, q, scale=1.0):
    """gross outliers: dsq far above any shortcut limit, and a 4-sample with one of them fits nothing; depths stay positive"""
    k = len(q)
    q = q + rng.choice([-1.0, 1.0], (k, 3)) * rng.uniform(1.5, 3.0, (k, 3)) * np.array([scale, scale, 0.0])
    q[:, 2] += scale * rng.uniform(1.5, 3.0, k)
    return q


def identity_planted_pair(oracle_mod, rng, zr, czc, seed, pair, H, *, max_dist=3.0, n_base=40, n_m=100, n_s=20, n_out=20,
                          zfar=None):
    """A pair of 2 (n_m + n_s) + n_base + n_out = 300 matches whose hypotheses [0, H) all draw a gross outlier, so that no
    hypothesis is valid and the identity fallback (node.cpp:1192-1215) scores the pair under T = I exactly.  Rows planted
    under T = I therefore keep their margins in the returned transform: n_m mirrored pairs at m = sq_max (1 +- delta) and
    n_s pairs at the shortcut limit, delta log-uniform in [1e-8, 3e-2] (below ~1e-6 the float32 rounding of the points and
    the screen's own error decide which side a row lands on), plus n_base exact inliers.  zfar: the first sorted match gets
    this from-depth (the correspondence the library latches z0 from)."""
    M = n_base + 2 * n_m + 2 * n_s + n_out
    samples = hypothesis_samples(oracle_mod, M, H, seed, pair)
    out = plan_outliers(samples, set(), M, n_out, rng)
    if out is None:
        raise RuntimeError("no outlier placement covers every sample")
    T = np.eye(4)
    base = frustum_points(rng, n_base, *zr)
    frm, to = [base], [base.copy()]
    for kind, n in (("m", n_m), ("s", n_s)):
        p = frustum_points(rng, n, *zr)
        a, c = plant_near_cut(rng, T, p, kind, log_uniform_delta(rng, n, lo=1e-8), max_dist=max_dist, czc=czc)
        frm += [p, p]
        to += [a, c]
    frm, to = np.concatenate(frm), np.concatenate(to)
    perm = rng.permutation(len(frm))
    P = np.zeros((M, 3))
    Q = np.zeros((M, 3))
    P[~out], Q[~out] = frm[perm], to[perm]
    po = frustum_points(rng, n_out, *zr)
    # a large depth covariance (latched far z0, or far points) lets a fit from a sample with one outlier still collect inliers (its rotated depth variance
    # accepts errors up to the shortcut limit) and converge: the outliers then move further than 10x that limit
    lim = 4 * (czc if czc is not None else (0.01 * zr[1] ** 2) ** 2)
    P[out], Q[out] = po, _gross(rng, po, max(1.0, 10 * np.sqrt(lim)))
    if zfar is not None:
        s = zfar / P[0, 2]
        Q[0] = Q[0] + P[0] * (s - 1) if out[0] else P[0] * s
        P[0] = P[0] * s
    qd, td = pair_descriptors(rng, M)
    xn, xo, _ = place_by_rank(oracle_mod, qd, td, to4(P), to4(Q), seed, pair, 300)
    return qd, xn, td, xo


def degenerate_pair(oracle_mod, rng, kind, seed, pair, *, H=8, M=300, n_out=40):
    """A > 80 % pair whose hypothesis 0 draws a rank-deficient sample and whose first later hypothesis with a sample disjoint
    from it (k) draws a clean one; hypotheses 1..k-1 draw an outlier.  kind 'many-to-one': the four queries of sample 0 are
    noisy copies of ONE train row (bruteForceSearchORB maps them all to it: the fit's covariance is 0, rank 0); kind
    'collinear': the four from-points of sample 0 lie on a line (rank 1).  Returns (desc_newer, xyz_newer, desc_older,
    xyz_older, k, n_in, sample 0 ranks)."""
    samples = hypothesis_samples(oracle_mod, M, H, seed, pair)
    k = next(n for n in range(1, H) if not set(samples[n]) & set(samples[0]))
    out = plan_outliers(samples[:k + 1], {0, k}, M, n_out, rng)
    if out is None:
        raise RuntimeError("no outlier placement satisfies the plan")
    T = small_motion(rng)
    p = frustum_points(rng, M, 1.0, 3.0)
    s0 = samples[0]
    if kind == "collinear":
        c, u = p[s0[0]], rng.normal(size=3)
        p[s0] = c + np.outer([0.0, 0.2, 0.45, 0.7], u / np.linalg.norm(u))
    q = p @ T[:3, :3].T + T[:3, 3]
    # 2 mm of noise, so that rmse is a residual and not the float32 fit's noise floor
    q += np.clip(rng.normal(scale=0.002, size=(M, 3)), -0.005, 0.005)
    q[out] = _gross(rng, q[out])
    qd, td = pair_descriptors(rng, M)
    order = oracle_mod.feature_matching_orb(qd, td, 300, seed, pair)
    assert np.array_equal(order["queryIdx"], order["trainIdx"])
    if kind == "many-to-one":  # same number of flipped bits, so the same Hamming distance and the same sort order
        X = int(order["trainIdx"][s0[0]])
        for r in s0[1:]:
            qi = int(order["queryIdx"][r])
            hd = int(np.unpackbits(qd[qi] ^ td[qi]).sum())
            flip = np.zeros(256, np.uint8)
            flip[rng.permutation(256)[:hd]] = 1
            qd[qi] = td[X] ^ np.packbits(flip, bitorder="little")
    m = oracle_mod.feature_matching_orb(qd, td, 300, seed, pair)
    assert np.array_equal(m["queryIdx"], order["queryIdx"])
    xn = np.zeros((len(qd), 4), F32)
    xo = np.zeros((len(td), 4), F32)
    xo[:, 2:] = 1
    xn[m["queryIdx"]] = to4(p)
    xo[m["trainIdx"][::-1]] = to4(q)[::-1]  # a shared train row keeps the to-point of its lowest rank
    n_in = M - n_out - (3 if kind == "many-to-one" else 0)
    if kind == "many-to-one":
        assert (m["trainIdx"][s0] == m["trainIdx"][s0[0]]).all()
    return qd, xn, td, xo, k, n_in, s0


def expected_path(valid, H, M, n_in, min_matches):
    """The sequential loop (node.cpp:1130-1190) over a plan in which exactly the hypotheses in `valid` reach n_in inliers
    and the others none: returns (real_iterations, valid_iterations, broke)."""
    thr = min_matches if min_matches <= 0.75 * M else int(0.75 * M)
    real = nvalid = 0
    n = 0
    while n < H and M >= 4:
        real += 1
        if n in valid and n_in >= thr:
            nvalid += 1
            if nvalid == 1:  # the first valid hypothesis always improves; the plans never visit a second one
                if n_in > M * 0.5:
                    n += 10
                if n_in > M * 0.75:
                    n += 10
                if n_in > M * 0.8:
                    return real, nvalid, True
        n += 1
    return real, nvalid, False


# Scenarios of the reference loop's bookkeeping.  Each entry: name, parameters (min_matches, max_matches, ransac_iterations),
# M, the hypotheses that draw all-inlier samples, the number of outliers, and whether T_true is the identity (for the
# identity fallback of node.cpp:1192-1215).  Hypotheses listed after the first valid one lie in the range its jump skips, so
# a kernel that does not honour the jump sees a second valid hypothesis.
SCENARIOS = [
    # > 80 % inliers: break at the first valid hypothesis
    *[(f"break@{k}", (20, 300, 40), 300, (k,), 40, False) for k in (0, 3, 4, 5, 11, 12, 19, 20)],
    ("break@H-1", (20, 300, 24), 300, (23,), 40, False),
    # 50-75 %: one +10 jump that lands across kPhase1 = 4 or a phase-2 CTA edge (hypotheses 4-11, 12-19, ...); no break
    *[(f"jump1@{k}", (20, 300, 40), 300, (k, k + 4, k + 10), 100, False) for k in (0, 1, 2, 3, 5, 9)],
    # 75-80 %: two jumps, no break
    *[(f"jump2@{k}", (20, 300, 40), 300, (k, k + 7, k + 15, k + 20), 62, False) for k in (0, 3, 7)],
    # no valid hypothesis: identity fallback accepted / rejected
    ("identity-accepted", (20, 300, 8), 100, (), 30, True),
    ("identity-rejected", (20, 300, 8), 100, (), 30, False),
    # M < 4 with min_matches < 3: no hypothesis at all, straight to the identity fallback
    ("M3-identity", (2, 300, 40), 3, (), 0, True),
    ("M3-rejected", (2, 300, 40), 3, (), 0, False),
    # 0.75 M clamp of min_inlier_threshold: 19 inliers of 24 pass a threshold of 18 (min_matches 20)
    ("clamp", (20, 300, 8), 24, (2,), 5, False),
    # M around multiples of 32 (mask-word edges)
    *[(f"M{m}", (20, 300, 8), m, (1,), max(1, m // 8), False) for m in (31, 32, 33, 63, 64, 65)],
    # max_matches around the two kernel instantiations (10 and 16 mask words)
    *[(f"maxm{mm}", (20, mm, 16), mm, (2,), mm // 8, False) for mm in (300, 320, 321, 512)],
    # ransac_iterations
    *[(f"H{h}", (20, 300, h), 300, (h - 1,), 40, False) for h in (1, 3, 4, 5, 8, 12)],
    ("H200", (20, 300, 200), 300, (0,), 40, False),
]


def scenario_batches(oracle_mod, seed=7, names=None):
    """The scenarios grouped by parameters: {(min_matches, max_matches, H): (batch dict, [(name, M, valid, n_in)], seed)}.
    Each scenario pair is placed at its own pair index, which the sampler is keyed on."""
    groups = {}
    for name, cfg, M, valid, n_out, ident in SCENARIOS:
        if names is not None and name not in names:
            continue
        groups.setdefault(cfg, []).append((name, M, valid, n_out, ident))
    out = {}
    for cfg, items in groups.items():
        _, mm, H = cfg
        pairs, meta = [], []
        for i, (name, M, valid, n_out, ident) in enumerate(items):
            rng = np.random.default_rng(sum(map(ord, name)) * 7919 + M)
            T = np.eye(4) if ident else None
            if not ident and not valid:  # a motion the identity fallback cannot explain
                T = np.eye(4)
                T[:3, 3] = [0.08, -0.06, 0.05]
            qd, xn, td, xo, _ = scenario_pair(oracle_mod, rng, M, H, valid, n_out, seed, i, T=T, max_matches=mm)
            pairs.append((qd, xn, td, xo))
            meta.append((name, M, valid, M - n_out))
        out[cfg] = (concat_batch(pairs), meta, seed)
    return out


# ---- conditioning edges of the rigid fit ----------------------------------------------------------------------------------

def rot_axis(axis, deg):
    """Rotation by `deg` degrees about `axis` (Rodrigues)."""
    k = np.asarray(axis, F64) / np.linalg.norm(axis)
    K = np.array([[0, -k[2], k[1]], [k[2], 0, -k[0]], [-k[1], k[0], 0]])
    a = np.deg2rad(deg)
    return np.eye(3) + np.sin(a) * K + (1 - np.cos(a)) * (K @ K)


def _moved(P, R, shift=(0.0, 0.0, 0.0), zmin=0.3):
    """R about the cloud's centre plus `shift`, and a z-shift that keeps every to-point at z >= zmin."""
    c = P.mean(0)
    Q = (P - c) @ R.T + c + np.asarray(shift, F64)
    lo = Q[:, 2].min()
    if lo < zmin:
        Q[:, 2] += zmin + 0.2 - lo
    return Q


def _noisy(rng, Q, sd):
    return Q + np.clip(rng.normal(scale=sd, size=Q.shape), -2.5 * sd, 2.5 * sd)


def _case(family, name, P, Q, noisy=False, nan=None):
    """One pair's rows: frm (from = query / newer side), to (train / older side), float32 (x, y, z, 1); nan: (rows, side)
    with side 'from', 'to' or 'both' gets a NaN depth."""
    frm, to = to4(P), to4(Q)
    if nan is not None:
        rows, side = nan
        if side in ("from", "both"):
            frm[rows, 2] = np.nan
        if side in ("to", "both"):
            to[rows, 2] = np.nan
    return dict(family=family, name=name, frm=frm, to=to, noisy=noisy, M=len(frm))


OBLIQUE = (1.0, -2.0, 0.7)


def fit_cases():
    """The fit's conditioning edges, one dict per pair (see `_case`; `noisy`: 0.5-2 mm of noise on every to-point, so that the
    refit over all rows is a strictly better model than any 4-point sample's)."""
    rng = np.random.default_rng(2024)
    cases = []
    # trivial motions
    P4 = np.array([[-0.4, -0.3, 1.2], [0.5, -0.2, 1.9], [0.1, 0.45, 2.6], [-0.3, 0.35, 1.6]])
    P40 = frustum_points(rng, 40, 1.0, 3.0)
    for nm, sh in (("identity", (0, 0, 0)), ("t=1cm", (0.01, 0, 0)), ("t=5m-lateral", (3.0, -4.0, 0)), ("t=5m-depth", (0, 0, 5.0))):
        cases.append(_case("trivial", f"{nm}-M4", P4, P4 + sh))
        cases.append(_case("trivial", f"{nm}-M40", P40, P40 + sh))
    # rotations about x, y, z and an oblique axis
    for ax_name, ax in (("x", (1, 0, 0)), ("y", (0, 1, 0)), ("z", (0, 0, 1)), ("oblique", OBLIQUE)):
        for deg in (1.0, 30.0, 90.0, 179.9, 180.0):
            R = rot_axis(ax, deg)
            cases.append(_case("rotation", f"{ax_name}{deg:g}-M4", P4, _moved(P4, R, (0.1, -0.05, 0.2))))
            P = frustum_points(rng, 40, 1.0, 3.0)
            cases.append(_case("rotation", f"{ax_name}{deg:g}-M40-noisy", P,
                               _noisy(rng, _moved(P, R, (0.1, -0.05, 0.2)), rng.uniform(5e-4, 2e-3)), noisy=True))
    # coplanar sets (exact rank 2): a fronto-parallel wall at z = 2 and an oblique plane; rotations about the normal and
    # about in-plane axes
    wall = lambda n: np.concatenate([rng.uniform(-1, 1, (n, 2)), np.full((n, 1), 2.0)], 1)
    nrm = np.array([0.3, -0.5, 0.8]) / np.linalg.norm([0.3, -0.5, 0.8])
    e1 = np.cross(nrm, [1.0, 0, 0]); e1 /= np.linalg.norm(e1)
    e2 = np.cross(nrm, e1)
    oblique = lambda n: np.array([0.0, 0.0, 2.5]) + rng.uniform(-1, 1, (n, 1)) * e1 + rng.uniform(-1, 1, (n, 1)) * e2
    for pl_name, gen, normal, inplane in (("wall", wall, (0, 0, 1.0), (1.0, 0.3, 0)), ("oblique", oblique, nrm, e1)):
        for rot_name, ax, deg in (("normal30", normal, 30.0), ("normal180", normal, 180.0), ("inplane30", inplane, 30.0),
                                  ("inplane90", inplane, 90.0), ("inplane180", inplane, 180.0)):
            R = rot_axis(ax, deg)
            for M in (4, 40):
                P = gen(M)
                cases.append(_case("coplanar", f"{pl_name}-{rot_name}-M{M}", P, _moved(P, R, (0.05, 0.1, 0.3))))
    # the reflection case: noisy coplanar sets whose unconstrained Kabsch has d = -1 (test_oracle's reflection case)
    found = 0
    while found < 4:
        M = 4 if found < 2 else 6
        P = np.concatenate([rng.uniform(-1, 1, (M, 2)), np.full((M, 1), 2.0)], 1)
        Q = P + np.array([0.1, -0.05, 0.02]) + rng.normal(size=P.shape) * 1e-4
        if kabsch_f64(to4(P), to4(Q))[3] < 0 and (M == 4 or kabsch_f64(to4(P), to4(Q), np.arange(4))[3] < 0):
            cases.append(_case("reflection", f"reflection-{found}-M{M}", P, Q))
            found += 1
    # near-collinear strips: 1 m long, lateral spread 1e-2, 1e-3, 1e-4 of the length
    u = np.array(OBLIQUE) / np.linalg.norm(OBLIQUE)
    for s in (1e-2, 1e-3, 1e-4):
        for M in (4, 40):
            lat = rng.normal(size=(M, 3))
            lat -= np.outer(lat @ u, u)
            P = np.array([0.0, 0.0, 2.0]) + np.outer(np.linspace(-0.5, 0.5, M), u) + s * lat
            cases.append(_case("collinear", f"strip{s:g}-M{M}", P, _moved(P, rot_axis((0.2, 1, 0.4), 20.0), (0.05, 0, 0.1))))
    # isotropic sets: equal singular values (exact ties when the motion keeps C diagonal)
    h = 0.25
    cube = np.array([[x, y, z] for x in (-h, h) for y in (-h, h) for z in (-h, h)])
    tetra = np.array([[1, 1, 1], [1, -1, -1], [-1, 1, -1], [-1, -1, 1]]) * (h / np.sqrt(3))
    octa = np.concatenate([np.eye(3), -np.eye(3)]) * h
    square = np.array([[h, 0, 0], [-h, 0, 0], [0, h, 0], [0, -h, 0]])
    for nm, S in (("cube", cube), ("tetrahedron", tetra), ("octahedron", octa), ("square", square)):
        P = S + np.array([0.0, 0.0, 2.5])
        cases.append(_case("isotropic", f"{nm}-identity", P, P.copy()))
        cases.append(_case("isotropic", f"{nm}-shift", P, P + np.array([0.25, -0.5, 0.5])))
        cases.append(_case("isotropic", f"{nm}-rot", P, _moved(P, rot_axis(OBLIQUE, 30.0), (0.1, 0.0, 0.2))))
    # scale: 4-point clouds of 0.1 mm to 1 cm, 10 m clouds, 2 cm clouds 8 m away
    for size in (1e-4, 3e-4, 1e-3, 1e-2):
        P = np.array([0.2, -0.1, 1.0]) + P4 / 0.9 * size
        for z_name, zoff in (("z1", 0.0), ("z3", 2.0)):
            Pz = P + np.array([0, 0, zoff])
            cases.append(_case("scale", f"{size:g}m-{z_name}-M4", Pz, _moved(Pz, rot_axis(OBLIQUE, 10.0), (0.03, 0.01, 0.02))))
    P = np.concatenate([rng.uniform(-5, 5, (40, 2)), rng.uniform(1.0, 11.0, (40, 1))], 1)
    cases.append(_case("scale", "10m-M40-noisy", P, _noisy(rng, _moved(P, rot_axis(OBLIQUE, 10.0), (0.2, 0, 0.3)), 1e-3),
                       noisy=True))
    for M in (4, 40):
        P = np.array([0.5, -0.3, 8.0]) + rng.uniform(-0.01, 0.01, (M, 3))
        cases.append(_case("scale", f"2cm-at-8m-M{M}", P, _moved(P, rot_axis(OBLIQUE, 10.0), (0.05, 0.02, -0.1))))
    # weight spread: depths from 0.3 m to 15 m on both sides (weights over four decades)
    zz = np.array([0.3, 1.0, 5.0, 15.0])
    P = np.stack([(np.array([100.0, 500.0, 250.0, 400.0]) - CX) * zz / FX, (np.array([300.0, 100.0, 400.0, 200.0]) - CY) * zz / FY, zz], 1)
    cases.append(_case("weights", "z0.3-15-M4", P, P @ rot_axis((0, 1, 0), 0.5).T))
    for k in range(2):
        z = np.exp(rng.uniform(np.log(0.3), np.log(15.0), 40))
        z[:2] = (0.3, 15.0)
        P = np.stack([rng.uniform(-0.5, 0.5, 40) * z, rng.uniform(-0.4, 0.4, 40) * z, z], 1)
        Q = P @ rot_axis((0.1, 1, 0.2), 0.5).T + np.array([0.0, 0.0, 0.01])
        assert Q[:, 2].min() >= 0.3
        cases.append(_case("weights", f"z0.3-15-M40-{k}", P, _noisy(rng, Q, 5e-4), noisy=True))
    # NaN depths among finite rows
    for side in ("from", "to", "both"):
        P = frustum_points(rng, 40, 1.0, 3.0)
        Q = _noisy(rng, _moved(P, rot_axis(OBLIQUE, 5.0), (0.05, 0.0, 0.02)), 1e-3)
        cases.append(_case("nan", f"nan-{side}", P, Q, noisy=True, nan=(np.array([5, 17, 33]), side)))
    # M around the mask words and the two kernel instantiations (10 words up to max_matches 320, 16 above)
    for M in (4, 5, 31, 32, 33, 63, 64, 65, 300, 320, 321, 512):
        P = frustum_points(rng, M, 1.0, 3.0)
        Q = _noisy(rng, _moved(P, rot_axis(OBLIQUE, 3.0), (0.04, -0.02, 0.03)), 1e-3)
        cases.append(_case("M", f"M{M}", P, Q, noisy=True))
    return cases
