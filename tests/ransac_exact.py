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
