"""numpy float32 restatement of rgbdslam_b200_icp_align_ex(..., RGBDSLAM_B200_ICP_METHOD_ICP_NL) (csrc/icp_nl.cu) in the
device's exact operation order: PCL 1.7's IterativeClosestPointNonLinear, whose increments come from
TransformationEstimationLM (Eigen's LevenbergMarquardt over NumericalDiff, WarpPointRigid6D).  The rules and the decisions
taken where PCL and Eigen leave the order open are those of include/rgbdslam_b200/icp.h.  Every float operation is one
correctly rounded float32 operation, so the device and this file agree bit for bit.

The length-m work (residuals, the Jacobian, column norms, the Householder tails, Q^T f) is vectorised; the 6 x 6 work
(pivots, lmpar, qrsolv, the LM bookkeeping) is scalar, as on the device's thread 0."""
import numpy as np

import icp_exact as ix
from icp_exact import MAX_ITERATIONS, block_sum, filter_cloud, transform

F32 = np.float32
N = 6  # WarpPointRigid6D's parameters (tx, ty, tz, qx, qy, qz)
MIN_CORRESPONDENCES = 4
EPS = F32(2.0 ** -23)  # NumTraits<float>::epsilon()
SQRT_EPS = np.sqrt(EPS, dtype=F32)  # ftol, xtol and NumericalDiff's step factor
FACTOR = F32(100.0)
MAXFEV = 400
FLT_MIN = F32(2.0 ** -126)
FLT_MAX = F32(np.finfo(F32).max)
STABLE_BLOCK = 4096  # stableNorm's block size
# blueNorm's constants for float (radix 2, 24 digits, exponents -125 ... 128)
B1, B2, S1M, S2M = F32(2.0 ** -63), F32(2.0 ** 52), F32(2.0 ** 63), F32(2.0 ** -76)
RELERR = np.sqrt(EPS, dtype=F32)
# Eigen's LevenbergMarquardtSpace::Status
IMPROPER, REL_REDUCTION, REL_ERROR, REL_ERROR_AND_REDUCTION, COSINUS, MAXFEV_REACHED, FTOL, XTOL, GTOL = range(9)
ZERO, ONE, HALF, TENTH = F32(0.0), F32(1.0), F32(0.5), F32(0.1)


def _max(a, b):
    """std::max: (a < b) ? b : a"""
    return b if a < b else a


def _min(a, b):
    """std::min: (b < a) ? b : a"""
    return b if b < a else a


def _dot(a, b):
    """a length-n dot product: the first product, then each further product added in index order"""
    s = F32(a[0] * b[0])
    for i in range(1, len(a)):
        s = F32(s + F32(a[i] * b[i]))
    return s


def _amax(v):
    """max |v_i|, NaN when any v_i is NaN, 0 for an empty vector"""
    a = np.abs(np.asarray(v, F32))
    if a.size == 0:
        return ZERO
    if np.isnan(a).any():
        return F32(np.nan)
    return F32(a.max())


def stable_norm(v):
    """Eigen 3.3's stableNorm: blocks of 4096 in index order, each block's sum of squares by block_sum"""
    v = np.asarray(v, F32)
    scale, inv, ssq = ZERO, ONE, ZERO
    with np.errstate(over="ignore", invalid="ignore", under="ignore"):
        for b in range(0, len(v), STABLE_BLOCK):
            bl = v[b:b + STABLE_BLOCK]
            mx = _amax(bl)
            if mx > scale:
                r = F32(scale / mx)
                ssq = F32(ssq * F32(r * r))
                tmp = F32(ONE / mx)
                if tmp > FLT_MAX:
                    inv = FLT_MAX
                    scale = F32(ONE / inv)
                elif mx > FLT_MAX:
                    inv = ONE
                    scale = mx
                else:
                    scale = mx
                    inv = tmp
            elif mx != mx:
                scale = mx
            if scale > ZERO:
                w = (bl * inv).astype(F32)
                ssq = F32(ssq + block_sum((w * w).astype(F32)))
        return F32(scale * np.sqrt(ssq, dtype=F32))


def blue_norm(v):
    """Eigen's blueNorm (Blue's algorithm); each of the three accumulators is a block_sum"""
    v = np.asarray(v, F32)
    with np.errstate(over="ignore", invalid="ignore", under="ignore"):
        ab2 = F32(B2 / F32(len(v)))
        ax = np.abs(v)
        big = ax > ab2
        sml = ~big & (ax < B1)
        med = ~big & ~sml
        zb, zs = (ax * S2M).astype(F32), (ax * S1M).astype(F32)
        abig = block_sum(np.where(big, (zb * zb).astype(F32), ZERO))
        asml = block_sum(np.where(sml, (zs * zs).astype(F32), ZERO))
        amed = block_sum(np.where(med, (ax * ax).astype(F32), ZERO))
        sq = lambda a: np.sqrt(a, dtype=F32)  # noqa: E731
        if amed != amed:
            return amed
        if abig > ZERO:
            abig = sq(abig)
            if abig > FLT_MAX:
                return abig
            if amed > ZERO:
                abig = F32(abig / S2M)
                amed = sq(amed)
            else:
                return F32(abig / S2M)
        elif asml > ZERO:
            if amed > ZERO:
                abig = sq(amed)
                amed = F32(sq(asml) / S1M)
            else:
                return F32(sq(asml) / S1M)
        else:
            return sq(amed)
        asml = _min(abig, amed)
        abig = _max(abig, amed)
        if asml <= F32(abig * RELERR):
            return abig
        r = F32(asml / abig)
        return F32(abig * sq(F32(ONE + F32(r * r))))


# ---- WarpPointRigid6D and the residuals -------------------------------------------------------------------------------------

def warp_transform(x):
    """WarpPointRigid6D::setParam(x).getTransform(): t = x[0:3], q = (x[3], x[4], x[5]), w = sqrt(1 - q.q) with
    q.q = (qx qx + qz qz) + qy qy (the order of Eigen's SSE Vector4 reduction), not renormalised; the rotation is
    Quaternion::toRotationMatrix.  q.q > 1 makes w and the rotation NaN."""
    x = np.asarray(x, F32)
    qx, qy, qz = x[3], x[4], x[5]
    with np.errstate(invalid="ignore", over="ignore"):
        qq = F32(F32(F32(qx * qx) + F32(qz * qz)) + F32(qy * qy))
        w = np.sqrt(F32(ONE - qq), dtype=F32)
        two = F32(2.0)
        tx, ty, tz = F32(two * qx), F32(two * qy), F32(two * qz)
        twx, twy, twz = F32(tx * w), F32(ty * w), F32(tz * w)
        txx, txy, txz = F32(tx * qx), F32(ty * qx), F32(tz * qx)
        tyy, tyz, tzz = F32(ty * qy), F32(tz * qy), F32(tz * qz)
        T = np.eye(4, dtype=F32)
        T[0] = [F32(ONE - F32(tyy + tzz)), F32(txy - twz), F32(txz + twy), x[0]]
        T[1] = [F32(txy + twz), F32(ONE - F32(txx + tzz)), F32(tyz - twx), x[1]]
        T[2] = [F32(txz - twy), F32(tyz + twx), F32(ONE - F32(txx + tyy)), x[2]]
    return T


def residuals(x, src, dst):
    """fvec_i = |warp(src_i) - dst_i|: the warp ((r0 x + r1 y) + r2 z) + t, then sqrt((dx dx + dz dz) + dy dy) (the
    Vector4 norm with w = 0, in the order of Eigen's SSE reduction)"""
    p = transform(warp_transform(x), src)
    with np.errstate(invalid="ignore", over="ignore"):
        dx, dy, dz = ((p[c] - dst[c]).astype(F32) for c in range(3))
        s = ((dx * dx).astype(F32) + (dz * dz).astype(F32)).astype(F32)
        return np.sqrt((s + (dy * dy).astype(F32)).astype(F32), dtype=F32)


# ---- ColPivHouseholderQR (Eigen 3.2's squared-norm downdate) and Q^T f -------------------------------------------------------

def qr(J):
    """ColPivHouseholderQR of the m x 6 Jacobian given as its 6 columns J (6, m).  Returns (A, perm, hc, rank): A[c] holds
    column c of matrixQR() (R above the diagonal, the Householder essentials below it), perm = colsPermutation().indices()."""
    A = np.array(J, F32, copy=True)
    m = A.shape[1]
    rows = np.arange(m)
    sq = [block_sum((A[c] * A[c]).astype(F32)) for c in range(N)]
    mx = sq[0]
    for c in range(1, N):
        if sq[c] > mx:
            mx = sq[c]
    thr = F32(F32(mx * F32(EPS * EPS)) / F32(m))
    perm = list(range(N))
    hc = [ZERO] * N
    nonzero, maxpivot = N, ZERO
    with np.errstate(over="ignore", invalid="ignore", divide="ignore", under="ignore"):
        for k in range(N):
            big = k
            for c in range(k + 1, N):
                if sq[c] > sq[big]:
                    big = c
            col = A[big]
            bsq = block_sum(np.where(rows >= k, (col * col).astype(F32), ZERO))
            sq[big] = bsq
            if nonzero == N and bsq < F32(thr * F32(m - k)):
                nonzero = k
            if big != k:
                A[[k, big]] = A[[big, k]]
                sq[k], sq[big] = sq[big], sq[k]
                perm[k], perm[big] = perm[big], perm[k]
            # makeHouseholderInPlace
            c0 = A[k, k]
            tail = rows > k
            tsq = block_sum(np.where(tail, (A[k] * A[k]).astype(F32), ZERO))
            if tsq <= FLT_MIN:
                tau, beta = ZERO, c0
                A[k, k + 1:] = ZERO
            else:
                beta = np.sqrt(F32(F32(c0 * c0) + tsq), dtype=F32)
                if c0 >= ZERO:
                    beta = F32(-beta)
                A[k, k + 1:] = (A[k, k + 1:] / F32(c0 - beta)).astype(F32)
                tau = F32(F32(beta - c0) / beta)
            A[k, k] = beta
            hc[k] = tau
            if abs(beta) > maxpivot:
                maxpivot = F32(abs(beta))
            # applyHouseholderOnTheLeft to the remaining columns
            if tau != ZERO:
                ess = np.where(tail, A[k], ZERO)
                te = (tau * A[k, k + 1:]).astype(F32)
                for c in range(k + 1, N):
                    tmp = F32(block_sum((ess * A[c]).astype(F32)) + A[c, k])
                    A[c, k] = F32(A[c, k] - F32(tau * tmp))
                    A[c, k + 1:] = (A[c, k + 1:] - (te * tmp).astype(F32)).astype(F32)
            for c in range(k + 1, N):
                sq[c] = F32(sq[c] - F32(A[c, k] * A[c, k]))
    pthr = F32(maxpivot * F32(EPS * F32(min(m, N))))
    rank = sum(1 for i in range(nonzero) if abs(A[i, i]) > pthr)
    return A, perm, hc, rank


def apply_qt(A, hc, f):
    """householderQ().adjoint() * f: H_0 first"""
    f = np.array(f, F32, copy=True)
    rows = np.arange(len(f))
    with np.errstate(over="ignore", invalid="ignore"):
        for k in range(N):
            if hc[k] == ZERO:
                continue
            tau = hc[k]
            ess = np.where(rows > k, A[k], ZERO)
            tmp = F32(block_sum((ess * f).astype(F32)) + f[k])
            f[k] = F32(f[k] - F32(tau * tmp))
            f[k + 1:] = (f[k + 1:] - ((tau * A[k, k + 1:]).astype(F32) * tmp).astype(F32)).astype(F32)
    return f


# ---- lmpar2 and qrsolv (6 x 6, thread 0 on the device) -----------------------------------------------------------------------

def _givens(p, q):
    """JacobiRotation::makeGivens(p, q) for real scalars: (c, s)"""
    if q == ZERO:
        return (F32(-1.0) if p < ZERO else ONE), ZERO
    if p == ZERO:
        return ZERO, (ONE if q < ZERO else F32(-1.0))
    if abs(p) > abs(q):
        t = F32(q / p)
        u = np.sqrt(F32(ONE + F32(t * t)), dtype=F32)
        if p < ZERO:
            u = F32(-u)
        c = F32(ONE / u)
        return c, F32(F32(-t) * c)
    t = F32(p / q)
    u = np.sqrt(F32(ONE + F32(t * t)), dtype=F32)
    if q < ZERO:
        u = F32(-u)
    s = F32(F32(-1.0) / u)
    return F32(F32(-t) * s), s


def qrsolv(S, perm, d, qtb):
    """qrsolv: S is the 6 x 6 working copy (R above the diagonal; its lower triangle and diagonal are overwritten and the
    diagonal restored).  Returns (x, sdiag)."""
    x_save = [S[i][i] for i in range(N)]
    wa = list(qtb)
    for i in range(N):
        for j in range(i):
            S[i][j] = S[j][i]
    sdiag = [ZERO] * N
    for j in range(N):
        l = perm[j]
        if d[l] == ZERO:
            break
        for i in range(j, N):
            sdiag[i] = ZERO
        sdiag[j] = d[l]
        qtbpj = ZERO
        for k in range(j, N):
            c, s = _givens(F32(-S[k][k]), sdiag[k])
            S[k][k] = F32(F32(c * S[k][k]) + F32(s * sdiag[k]))
            temp = F32(F32(c * wa[k]) + F32(s * qtbpj))
            qtbpj = F32(F32(F32(-s) * wa[k]) + F32(c * qtbpj))
            wa[k] = temp
            for i in range(k + 1, N):
                temp = F32(F32(c * S[i][k]) + F32(s * sdiag[i]))
                sdiag[i] = F32(F32(F32(-s) * S[i][k]) + F32(c * sdiag[i]))
                S[i][k] = temp
    sdiag = [S[i][i] for i in range(N)]
    nsing = 0
    while nsing < N and sdiag[nsing] != ZERO:
        nsing += 1
    for i in range(nsing, N):
        wa[i] = ZERO
    for i in range(nsing - 1, -1, -1):  # the transposed lower triangle, backwards (row-major upper solve)
        if i < nsing - 1:
            wa[i] = F32(wa[i] - _dot([S[l][i] for l in range(i + 1, nsing)], wa[i + 1:nsing]))
        wa[i] = F32(wa[i] / S[i][i])
    for i in range(N):
        S[i][i] = x_save[i]
    x = [ZERO] * N
    for j in range(N):
        x[perm[j]] = wa[j]
    return x, sdiag


def lmpar(R, perm, rank, diag, qtb, delta, par):
    """lmpar2: returns (par, x), x the step before LevenbergMarquardt negates it"""
    wa1 = [qtb[i] if i < rank else ZERO for i in range(N)]
    for i in range(rank - 1, -1, -1):  # column-major upper back substitution; a zero right-hand side is skipped
        if wa1[i] != ZERO:
            wa1[i] = F32(wa1[i] / R[i][i])
            for r in range(i):
                wa1[r] = F32(wa1[r] - F32(wa1[i] * R[r][i]))
    x = [ZERO] * N
    for i in range(N):
        x[perm[i]] = wa1[i]
    wa2 = [F32(diag[i] * x[i]) for i in range(N)]
    dxnorm = blue_norm(wa2)
    fp = F32(dxnorm - delta)
    if fp <= F32(TENTH * delta):
        return ZERO, x
    parl = ZERO
    if rank == N:
        wa1 = [F32(F32(diag[perm[i]] * wa2[perm[i]]) / dxnorm) for i in range(N)]
        for i in range(N):  # R^T lower, forwards (row-major lower solve)
            if i > 0:
                wa1[i] = F32(wa1[i] - _dot([R[s][i] for s in range(i)], wa1[:i]))
            wa1[i] = F32(wa1[i] / R[i][i])
        temp = blue_norm(wa1)
        parl = F32(F32(F32(fp / delta) / temp) / temp)
    wa1 = [F32(_dot([R[i][j] for i in range(j + 1)], qtb[:j + 1]) / diag[perm[j]]) for j in range(N)]
    gnorm = stable_norm(wa1)
    paru = F32(gnorm / delta)
    if paru == ZERO:
        paru = F32(FLT_MIN / _min(delta, TENTH))
    par = _max(par, parl)
    par = _min(par, paru)
    if par == ZERO:
        par = F32(gnorm / dxnorm)
    S = [[R[i][j] for j in range(N)] for i in range(N)]
    it = 0
    while True:
        it += 1
        if par == ZERO:
            par = _max(FLT_MIN, F32(F32(0.001) * paru))
        sp = np.sqrt(par, dtype=F32)
        x, sdiag = qrsolv(S, perm, [F32(sp * diag[i]) for i in range(N)], qtb)
        wa2 = [F32(diag[i] * x[i]) for i in range(N)]
        dxnorm = blue_norm(wa2)
        temp = fp
        fp = F32(dxnorm - delta)
        if abs(fp) <= F32(TENTH * delta) or (parl == ZERO and fp <= temp and temp < ZERO) or it == 10:
            break
        wa1 = [F32(diag[perm[i]] * F32(wa2[perm[i]] / dxnorm)) for i in range(N)]
        for j in range(N):
            wa1[j] = F32(wa1[j] / sdiag[j])
            temp = wa1[j]
            for i in range(j + 1, N):
                wa1[i] = F32(wa1[i] - F32(S[i][j] * temp))
        temp = blue_norm(wa1)
        parc = F32(F32(F32(fp / delta) / temp) / temp)
        if fp > ZERO:
            parl = _max(parl, par)
        if fp < ZERO:
            paru = _min(paru, par)
        par = _max(parl, F32(par + parc))
    return par, x


# ---- LevenbergMarquardt::minimize --------------------------------------------------------------------------------------------

def lm_estimate(src, dst):
    """TransformationEstimationLM over the correspondences (src_i, dst_i), i in order.  Returns (T_inc 4 x 4 float32, status,
    nfev, iterations): Eigen's status, the function evaluations counted as Eigen counts them (7 per Jacobian), and the LM
    iterations (Jacobians computed)."""
    src = np.asarray(src, F32)
    dst = np.asarray(dst, F32)
    m = src.shape[1]
    x = np.zeros(N, F32)
    if m < N:
        return warp_transform(x), IMPROPER, 0, 0
    with np.errstate(over="ignore", invalid="ignore", divide="ignore", under="ignore"):
        fvec = residuals(x, src, dst)
        nfev, iterations = 1, 0
        fnorm = stable_norm(fvec)
        par, it = ZERO, 1
        diag = [ZERO] * N
        xnorm = delta = temp = ZERO
        while True:
            # the forward-difference Jacobian; f(x) is fvec (NumericalDiff evaluates it again: counted, same bits)
            J = np.empty((N, m), F32)
            for j in range(N):
                h = F32(SQRT_EPS * abs(x[j]))
                if h == ZERO:
                    h = SQRT_EPS
                xp = x.copy()
                xp[j] = F32(x[j] + h)
                J[j] = ((residuals(xp, src, dst) - fvec).astype(F32) / h).astype(F32)
            nfev += N + 1
            iterations += 1
            wa2 = [blue_norm(J[j]) for j in range(N)]
            A, perm, hc, rank = qr(J)
            R = [[A[j][i] for j in range(N)] for i in range(N)]  # R[i][j] = matrixQR()(i, j)
            if it == 1:
                diag = [ONE if w == ZERO else w for w in wa2]
                xnorm = stable_norm([F32(diag[i] * x[i]) for i in range(N)])
                delta = F32(FACTOR * xnorm)
                if delta == ZERO:
                    delta = FACTOR
            qtf = list(apply_qt(A, hc, fvec)[:N])
            gnorm = ZERO
            if fnorm != ZERO:
                for j in range(N):
                    w = wa2[perm[j]]
                    if w != ZERO:
                        q = [F32(qtf[i] / fnorm) for i in range(j + 1)]
                        gnorm = _max(gnorm, F32(abs(F32(_dot([R[i][j] for i in range(j + 1)], q) / w))))
            if gnorm <= ZERO:  # gtol
                return warp_transform(x), COSINUS, nfev, iterations
            diag = [_max(diag[i], wa2[i]) for i in range(N)]
            while True:
                par, wa1 = lmpar(R, perm, rank, diag, qtf, delta, par)
                wa1 = np.array([F32(-v) for v in wa1], F32)
                wa2 = (x + wa1).astype(F32)
                pnorm = stable_norm([F32(diag[i] * wa1[i]) for i in range(N)])
                if it == 1:
                    delta = _min(delta, pnorm)
                wa4 = residuals(wa2, src, dst)
                nfev += 1
                fnorm1 = stable_norm(wa4)
                actred = F32(-1.0)
                if F32(TENTH * fnorm1) < fnorm:
                    q = F32(fnorm1 / fnorm)
                    actred = F32(np.float64(1.0) - np.float64(F32(q * q)))  # 1. - abs2(...) in double
                v = [wa1[perm[j]] for j in range(N)]
                wa3 = []
                for r in range(N):
                    s = ZERO
                    for i in range(r, N):
                        s = F32(s + F32(v[i] * R[r][i]))
                    wa3.append(s)
                q = F32(stable_norm(wa3) / fnorm)
                temp1 = F32(q * q)
                q = F32(F32(np.sqrt(par, dtype=F32) * pnorm) / fnorm)
                temp2 = F32(q * q)
                prered = F32(temp1 + F32(temp2 / HALF))
                dirder = F32(-F32(temp1 + temp2))
                ratio = ZERO
                if prered != ZERO:
                    ratio = F32(actred / prered)
                if ratio <= F32(0.25):
                    if actred >= ZERO:
                        temp = HALF
                    if actred < ZERO:
                        temp = F32(F32(HALF * dirder) / F32(dirder + F32(HALF * actred)))
                    if F32(TENTH * fnorm1) >= fnorm or temp < TENTH:
                        temp = TENTH
                    delta = F32(temp * _min(delta, F32(pnorm / TENTH)))
                    par = F32(par / temp)
                elif not (par != ZERO and ratio < F32(0.75)):
                    delta = F32(pnorm / HALF)
                    par = F32(HALF * par)
                if ratio >= F32(1e-4):
                    x = wa2
                    xnorm = stable_norm([F32(diag[i] * x[i]) for i in range(N)])
                    fvec = wa4
                    fnorm = fnorm1
                    it += 1
                small = abs(actred) <= SQRT_EPS and prered <= SQRT_EPS and F32(HALF * ratio) <= ONE
                status = None
                if small and delta <= F32(SQRT_EPS * xnorm):
                    status = REL_ERROR_AND_REDUCTION
                elif small:
                    status = REL_REDUCTION
                elif delta <= F32(SQRT_EPS * xnorm):
                    status = REL_ERROR
                elif nfev >= MAXFEV:
                    status = MAXFEV_REACHED
                elif abs(actred) <= EPS and prered <= EPS and F32(HALF * ratio) <= ONE:
                    status = FTOL
                elif delta <= F32(EPS * xnorm):
                    status = XTOL
                elif gnorm <= EPS:
                    status = GTOL
                if status is not None:
                    return warp_transform(x), status, nfev, iterations
                if not ratio < F32(1e-4):
                    break


def align_points(src, tgt, max_iterations=MAX_ITERATIONS):
    """IterativeClosestPointNonLinear::align: icp_exact.align_points with lm_estimate, plus the estimator's (status, nfev,
    iterations) per ICP iteration in `lm`"""
    lm = []

    def estimate(ws, dst, ok):
        T, *record = lm_estimate(ws[:, ok], dst[:, ok])
        lm.append(tuple(record))
        return T
    return dict(ix.align_points(src, tgt, max_iterations, estimate, MIN_CORRESPONDENCES), lm=lm)


def align(source_pc, target_pc, max_cloud_size=10000):
    """icpAlignment with icp_method "icp_nl": IterativeClosestPointNonLinear of filterCloud(source), filterCloud(target)"""
    return align_points(filter_cloud(source_pc, max_cloud_size), filter_cloud(target_pc, max_cloud_size))
