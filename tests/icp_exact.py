"""numpy float32 restatement of rgbdslam_b200_icp_align (csrc/icp.cu) in the device's exact operation order: filterCloud's
index walk, brute-force nearest neighbours (lowest target index on ties), the fixed-order Umeyama sums, the 3 x 3 Jacobi SVD,
the float transform chain and PCL 1.7's convergence test.  Every float operation is one correctly rounded float32 operation,
so the device and this file agree bit for bit."""
import numpy as np

F32 = np.float32
THREADS = 256  # the partial sums of the device: thread t owns source points t, t + 256, ...
MAX_D2 = 0.05 * 0.05  # max correspondence distance 0.05, squared in double
MAX_ITERATIONS = 50
TRANSFORM_EPS = 1e-8
FITNESS_EPS = 1.0
SVD_SWEEPS = 32
DBL_MAX = np.finfo(np.float64).max
CRITERIA = ("too few correspondences", "iterations", "transform", "absolute MSE", "relative MSE")


def filter_indices(z, desired):
    """filterCloud (icp.cpp:20-45): the kept indices of a cloud whose z plane is `z`, in storage order."""
    idx = np.flatnonzero(~np.isnan(np.asarray(z, F32)))
    n = len(idx)
    step = F32(F32(n) / F32(desired))
    step = F32(1.0) if step < 1.0 else step
    if step == F32(1.0):  # i runs through 0, 1, ..., n - 1 exactly (n < 2^24)
        return idx
    ranks = []
    i = F32(0.0)
    while i < F32(n):
        ranks.append(int(i))
        i = F32(i + step)
    return idx[np.asarray(ranks, np.int64)]


def filter_cloud(pc, desired):
    """(x, y, z) float32 planes of the points filterCloud keeps of pc (a dict with planes x, y, z in storage order)"""
    k = filter_indices(pc["z"], desired)
    return np.stack([np.asarray(pc[c], F32)[k] for c in "xyz"])


def _dot3(a0, b0, a1, b1, a2, b2):
    return F32(F32(F32(a0 * b0) + F32(a1 * b1)) + F32(a2 * b2))


def block_sum(v):
    """the device's float sum of v (one value per source point, 0 where the point has no correspondence): thread t adds
    v[t], v[t + 256], ... in order from +0, then a pairwise tree over the 256 partials (p[t] += p[t + s], s = 128 ... 1)"""
    v = np.asarray(v, F32)
    R = -(-len(v) // THREADS)
    pad = np.zeros(max(R, 1) * THREADS, F32)
    pad[:len(v)] = v
    m = pad.reshape(-1, THREADS)
    acc = np.zeros(THREADS, F32)
    for r in range(len(m)):
        acc = (acc + m[r]).astype(F32)
    s = THREADS // 2
    while s >= 1:
        acc[:s] = (acc[:s] + acc[s:2 * s]).astype(F32)
        s //= 2
    return F32(acc[0])


def nearest(src, tgt):
    """per source point (index of the nearest finite target, its float squared distance ((dx dx + dy dy) + dz dz)); -1 / inf
    for a non-finite source point or when no target is finite.  Ties go to the lowest target index."""
    n = src.shape[1]
    idx = np.full(n, -1, np.int64)
    dist = np.full(n, np.inf, F32)
    tf = np.isfinite(tgt).all(0)
    sf = np.isfinite(src).all(0)
    if not tf.any():
        return idx, dist
    tj = np.flatnonzero(tf)
    T = tgt[:, tj]
    q = np.flatnonzero(sf)
    with np.errstate(over="ignore", invalid="ignore"):
        for a in range(0, len(q), 512):
            qq = q[a:a + 512]
            S = src[:, qq]
            dx = (S[0][:, None] - T[0][None, :]).astype(F32)
            dy = (S[1][:, None] - T[1][None, :]).astype(F32)
            dz = (S[2][:, None] - T[2][None, :]).astype(F32)
            d = ((dx * dx + dy * dy).astype(F32) + dz * dz).astype(F32)
            j = np.argmin(d, 1)  # the first minimum: the lowest index
            idx[qq] = tj[j]
            dist[qq] = d[np.arange(len(qq)), j]
    return idx, dist


def _rot(x, y, c, s):
    """(c x + s y, -s x + c y)"""
    return F32(F32(c * x) + F32(s * y)), F32(F32(F32(-s) * x) + F32(c * y))


def svd3(A):
    """two-sided cyclic Jacobi SVD of a 3 x 3 float matrix: U, singular values (descending), V with A = U diag(s) V^T"""
    W = [[F32(A[i][j]) for j in range(3)] for i in range(3)]
    U = [[F32(1.0 if i == j else 0.0) for j in range(3)] for i in range(3)]
    V = [[F32(1.0 if i == j else 0.0) for j in range(3)] for i in range(3)]
    one, two = F32(1.0), F32(2.0)
    zero_lim, prec = F32(2.0 ** -148), F32(2.0 ** -22)
    for _ in range(SVD_SWEEPS):
        finished = True
        for p, q in ((1, 0), (2, 0), (2, 1)):
            thr = max(zero_lim, F32(prec * max(abs(W[p][p]), abs(W[q][q]))))
            if not max(abs(W[p][q]), abs(W[q][p])) > thr:
                continue
            finished = False
            m00, m01, m10, m11 = W[p][p], W[p][q], W[q][p], W[q][q]
            t = F32(m00 + m11)
            d = F32(m10 - m01)
            if t == 0:
                c1, s1 = F32(0.0), (one if d > 0 else F32(-1.0))
            else:
                u = F32(d / t)
                c1 = F32(one / np.sqrt(F32(one + F32(u * u)), dtype=F32))
                s1 = F32(c1 * u)
            a00, a10 = _rot(m00, m10, c1, s1)
            a01, a11 = _rot(m01, m11, c1, s1)
            if a01 == 0:
                c2, s2 = one, F32(0.0)
            else:
                tau = F32(F32(a00 - a11) / F32(two * abs(a01)))
                w = np.sqrt(F32(F32(tau * tau) + one), dtype=F32)
                tt = F32(one / F32(tau + w)) if tau > 0 else F32(one / F32(tau - w))
                n = F32(one / np.sqrt(F32(F32(tt * tt) + one), dtype=F32))
                mag = F32(abs(tt) * n)
                s2 = F32(-mag) if (tt > 0) == (a01 > 0) else mag
                c2 = n
            cl = F32(F32(c1 * c2) + F32(s1 * s2))
            sl = F32(F32(s1 * c2) - F32(c1 * s2))
            for k in range(3):
                W[p][k], W[q][k] = _rot(W[p][k], W[q][k], cl, sl)
            for k in range(3):
                U[k][p], U[k][q] = _rot(U[k][p], U[k][q], cl, sl)
            for k in range(3):
                W[k][p], W[k][q] = _rot(W[k][p], W[k][q], c2, F32(-s2))
            for k in range(3):
                V[k][p], V[k][q] = _rot(V[k][p], V[k][q], c2, F32(-s2))
        if finished:
            break
    s = [abs(W[i][i]) for i in range(3)]
    for i in range(3):
        if W[i][i] < 0:
            for k in range(3):
                U[k][i] = F32(-U[k][i])
    for i in range(3):
        pos = max(range(i, 3), key=lambda j: (s[j], -j))
        if s[pos] == 0:
            break
        if pos != i:
            s[i], s[pos] = s[pos], s[i]
            for M in (U, V):
                for k in range(3):
                    M[k][i], M[k][pos] = M[k][pos], M[k][i]
    return U, s, V


def det3(M):
    a = F32(F32(M[1][1] * M[2][2]) - F32(M[1][2] * M[2][1]))
    b = F32(F32(M[1][0] * M[2][2]) - F32(M[1][2] * M[2][0]))
    c = F32(F32(M[1][0] * M[2][1]) - F32(M[1][1] * M[2][0]))
    return F32(F32(F32(M[0][0] * a) - F32(M[0][1] * b)) + F32(M[0][2] * c))


def umeyama(src, dst, mask):
    """the rigid transform (4 x 4 float32) of TransformationEstimationSVD for the source points with mask, paired with dst"""
    n = int(mask.sum())
    inv_n = F32(F32(1.0) / F32(n))
    z = F32(0.0)
    sm = [F32(block_sum(np.where(mask, src[c], z)) * inv_n) for c in range(3)]
    dm = [F32(block_sum(np.where(mask, dst[c], z)) * inv_n) for c in range(3)]
    with np.errstate(over="ignore", invalid="ignore"):
        sd = [(src[c] - sm[c]).astype(F32) for c in range(3)]
        dd = [(dst[c] - dm[c]).astype(F32) for c in range(3)]
        sigma = [[F32(inv_n * block_sum(np.where(mask, (dd[i] * sd[j]).astype(F32), z))) for j in range(3)] for i in range(3)]
    U, _, V = svd3(sigma)
    neg = F32(det3(U) * det3(V)) < 0
    if neg:
        for k in range(3):
            U[k][2] = F32(-U[k][2])
    T = np.eye(4, dtype=F32)
    for i in range(3):
        for j in range(3):
            T[i, j] = _dot3(U[i][0], V[j][0], U[i][1], V[j][1], U[i][2], V[j][2])
    for i in range(3):
        T[i, 3] = F32(dm[i] - _dot3(T[i, 0], sm[0], T[i, 1], sm[1], T[i, 2], sm[2]))
    return T


def transform(T, pts):
    """((r0 x + r1 y) + r2 z) + t of every finite point; the others stay"""
    fin = np.isfinite(pts).all(0)
    out = pts.copy()
    with np.errstate(over="ignore", invalid="ignore"):
        for r in range(3):
            v = ((((T[r, 0] * pts[0]).astype(F32) + (T[r, 1] * pts[1]).astype(F32)).astype(F32) + (T[r, 2] * pts[2]).astype(F32))
                 .astype(F32) + T[r, 3]).astype(F32)
            out[r] = np.where(fin, v, pts[r])
    return out


def matmul4(A, B):
    C = np.zeros((4, 4), F32)
    for i in range(4):
        for j in range(4):
            C[i, j] = F32(F32(F32(F32(A[i, 0] * B[0, j]) + F32(A[i, 1] * B[1, j])) + F32(A[i, 2] * B[2, j])) + F32(A[i, 3] * B[3, j]))
    return C


def align_points(src, tgt, max_iterations=MAX_ITERATIONS, estimate=umeyama, min_correspondences=3):
    """IterativeClosestPoint::align of filtered (3, n) float32 clouds with an identity guess, with the transformation
    estimator estimate(source, dst, mask) -> T_inc, where dst holds at the masked source points their corresponding target
    points.  Returns a dict with the fields of rgbdslam_b200_icp_result (T as a 4 x 4 row-major matrix) and the
    per-iteration correspondences `corr`."""
    src = np.asarray(src, F32)
    tgt = np.asarray(tgt, F32)
    ws = src.copy()
    final = np.eye(4, dtype=F32)
    prev = DBL_MAX
    it, mse, cnt, crit = 0, 0.0, 0, 0
    corr = []
    while True:
        idx, dist = nearest(ws, tgt)
        ok = (idx >= 0) & (dist.astype(np.float64) <= MAX_D2)
        cnt = int(ok.sum())
        corr.append(np.where(ok, idx, -1))
        if cnt < min_correspondences:
            crit = 0
            break
        dst = np.zeros_like(ws)
        dst[:, ok] = tgt[:, idx[ok]]
        Tinc = estimate(ws, dst, ok)
        ws = transform(Tinc, ws)
        final = matmul4(Tinc, final)
        it += 1
        acc = 0.0
        for d in dist[ok]:
            acc += float(d)
        mse = acc / cnt
        if it >= max_iterations:
            crit = 1
            break
        cos = 0.5 * float(F32(F32(F32(Tinc[0, 0] + Tinc[1, 1]) + Tinc[2, 2]) - F32(1.0)))
        tr = float(F32(F32(F32(Tinc[0, 3] * Tinc[0, 3]) + F32(Tinc[1, 3] * Tinc[1, 3])) + F32(Tinc[2, 3] * Tinc[2, 3])))
        if cos >= 1.0 - TRANSFORM_EPS and tr <= TRANSFORM_EPS:
            crit = 2
            break
        with np.errstate(divide="ignore", invalid="ignore"):
            if abs(mse - prev) < 1e-12:
                crit = 3
                break
            if np.float64(abs(mse - prev)) / np.float64(prev) < FITNESS_EPS:
                crit = 4
                break
        prev = mse
    converged = crit != 0
    return dict(T=final if converged else np.eye(4, dtype=F32), converged=int(converged), iterations=it, criterion=crit,
                n_source=src.shape[1], n_target=tgt.shape[1], n_correspondences=cnt, mse=mse, corr=corr)


def align(source_pc, target_pc, max_cloud_size=10000):
    """icpAlignment(filterCloud(source), filterCloud(target), Identity) of two stored clouds (dicts with x, y, z planes)"""
    return align_points(filter_cloud(source_pc, max_cloud_size), filter_cloud(target_pc, max_cloud_size))
