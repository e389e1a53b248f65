"""The icp_nl restatement (tests/icp_nl_exact.py): its estimator against scipy's MINPACK (an independent Levenberg-Marquardt in
float64) on well-conditioned correspondence sets, a noise-free motion, Eigen's edge cases (too few rows, a rank-deficient
Jacobian, a zero residual, a trial step with q.q > 1, the maxfev bound), and ICP's criteria with 3, 4 and 5 correspondences."""
import re

import numpy as np
import pytest
from scipy.optimize import leastsq

import icp_exact as ix
import icp_nl_exact as nx
from test_icp_exact_cpu import ROOT, _rot, _scene

F32 = np.float32


def _residuals64(x, src, dst):
    """the same residual in float64: WarpPointRigid6D's rotation from (qx, qy, qz) and w = sqrt(1 - q.q)"""
    qx, qy, qz = x[3:]
    w = np.sqrt(1.0 - (qx * qx + qy * qy + qz * qz))
    R = np.array([[1 - 2 * (qy * qy + qz * qz), 2 * (qx * qy - w * qz), 2 * (qx * qz + w * qy)],
                  [2 * (qx * qy + w * qz), 1 - 2 * (qx * qx + qz * qz), 2 * (qy * qz - w * qx)],
                  [2 * (qx * qz - w * qy), 2 * (qy * qz + w * qx), 1 - 2 * (qx * qx + qy * qy)]])
    return np.sqrt(((R @ src + x[:3, None] - dst) ** 2).sum(0))


def _x_of(T):
    """(t, q) of a rotation with w >= 0, as WarpPointRigid6D parametrises it"""
    R = T[:3, :3].astype(np.float64)
    w = np.sqrt(max(0.0, 1.0 + np.trace(R))) / 2
    q = np.array([R[2, 1] - R[1, 2], R[0, 2] - R[2, 0], R[1, 0] - R[0, 1]]) / (4 * w)
    return np.concatenate([T[:3, 3].astype(np.float64), q])


def _pairs(seed, n=300, noise=1e-4):
    """well-conditioned correspondences: a cloud centred on its origin (no lever arm between rotation and translation),
    moved by up to 3 cm and 0.05 rad, with 0.1 mm noise.  Returns src, dst and the motion (R, t)."""
    rng = np.random.default_rng(seed)
    src = rng.uniform(-1, 1, (3, n))
    R = _rot(rng.normal(size=3), rng.uniform(0.005, 0.05))
    t = rng.uniform(-0.03, 0.03, 3)
    dst = R @ src + t[:, None] + rng.normal(0, noise, src.shape)
    return src.astype(F32), dst.astype(F32), R, t


@pytest.mark.parametrize("seed", range(6))
def test_lm_estimate_agrees_with_minpack(seed):
    """scipy's leastsq is MINPACK lmdif in float64 with the same factor, ftol, xtol and gtol, epsfcn = FLT_EPSILON (the same
    forward-difference step), started from 0.  On these sets both stop once the trust region is below xtol * ||D x|| (xtol
    about 3.5e-4), so each is within about xtol |x| of the true minimiser: the parameters must agree to 2 xtol |x|, plus
    1e-6 for the float32 residuals (their rounding, 1e-7 of 1 m, moves a 300-point least-squares fit by far less)."""
    src, dst, _, _ = _pairs(seed)
    T, status, nfev, its = nx.lm_estimate(src, dst)
    assert status in (nx.REL_REDUCTION, nx.REL_ERROR, nx.REL_ERROR_AND_REDUCTION) and nfev <= nx.MAXFEV
    assert nfev == 1 + 7 * its + (nfev - 1 - 7 * its) and nfev - 1 - 7 * its >= its  # at least one trial per Jacobian
    x64, _, info, _, ier = leastsq(_residuals64, np.zeros(6), args=(src.astype(np.float64), dst.astype(np.float64)),
                                   full_output=True, factor=100, ftol=float(nx.SQRT_EPS), xtol=float(nx.SQRT_EPS), gtol=0.0,
                                   epsfcn=float(nx.EPS))
    assert ier in (1, 2, 3)
    x32 = _x_of(T)
    tol = 2 * float(nx.SQRT_EPS) * np.abs(x64).max() + 1e-6
    assert np.abs(x32 - x64).max() <= tol, (x32, x64, tol)


def test_noise_free_motion_is_recovered():
    for seed in range(3):
        src, dst, R, t = _pairs(seed, n=200, noise=0.0)
        T, status, _, _ = nx.lm_estimate(src, dst)
        assert np.abs(T[:3, :3] - R).max() < 2e-5 and np.abs(T[:3, 3] - t).max() < 2e-5, (T, R, t)


def test_warp_and_residuals():
    x = np.array([0.1, -0.2, 0.3, 0.0, 0.0, 0.0], F32)
    T = nx.warp_transform(x)
    assert np.array_equal(T[:3, :3], np.eye(3, dtype=F32)) and np.array_equal(T[:3, 3], x[:3])
    q = np.array([0.0, 0.0, 0.0, 0.1, -0.2, 0.05], F32)
    R = nx.warp_transform(q)[:3, :3].astype(np.float64)
    assert np.abs(R.T @ R - np.eye(3)).max() < 1e-6 and abs(np.linalg.det(R) - 1) < 1e-6
    R = nx.warp_transform(np.array([0, 0, 0, 0.8, 0.7, 0.0], F32))[:3, :3]  # q.q > 1: w is NaN, and so is every term with w
    assert np.isnan(R[~np.eye(3, dtype=bool)]).all() and np.isfinite(np.diag(R)).all()
    src = np.array([[1.0, 0.0], [0.0, 2.0], [0.0, 0.0]], F32)
    assert np.array_equal(nx.residuals(np.zeros(6, F32), src, src + F32(0.0)), np.zeros(2, F32))
    p = ix.transform(T, src)
    d = [F32(p[c, 0] - src[c, 0]) for c in range(3)]  # the order: (dx dx + dz dz) + dy dy
    assert nx.residuals(x, src, src)[0] == np.sqrt(F32(F32(F32(d[0] * d[0]) + F32(d[2] * d[2])) + F32(d[1] * d[1])), dtype=F32)


def test_norms_equal_their_definitions():
    rng = np.random.default_rng(3)
    for n in (6, 100, 4096, 4097, 10000):
        v = rng.normal(size=n).astype(F32)
        ref = np.sqrt(np.sum(v.astype(np.float64) ** 2))
        assert abs(float(nx.stable_norm(v)) - ref) <= 1e-6 * ref
        assert abs(float(nx.blue_norm(v)) - ref) <= 1e-6 * ref
    tiny = np.array([1e-30, 2e-30, 3.0], F32)  # blueNorm's small and medium ranges
    assert abs(float(nx.blue_norm(tiny)) - 3.0) < 1e-6
    assert nx.blue_norm(np.array([1e-30, 2e-30], F32)) == F32(np.sqrt(5.0) * 1e-30) or \
        abs(float(nx.blue_norm(np.array([1e-30, 2e-30], F32))) / (np.sqrt(5.0) * 1e-30) - 1) < 1e-6
    assert np.isnan(nx.stable_norm(np.array([1.0, np.nan], F32))) and np.isnan(nx.blue_norm(np.array([1.0, np.nan], F32)))


def test_qr_reconstructs_the_jacobian():
    rng = np.random.default_rng(4)
    J = rng.normal(size=(6, 50)).astype(F32)
    A, perm, hc, rank = nx.qr(J)
    assert rank == 6 and sorted(perm) == list(range(6))
    Rm = np.triu(np.array([[A[j][i] for j in range(6)] for i in range(6)], np.float64))
    # Q^T J P = [R; 0]: apply Q^T column by column
    QtJ = np.stack([nx.apply_qt(A, hc, J[perm[j]]) for j in range(6)], 1).astype(np.float64)
    assert np.abs(QtJ[:6] - Rm).max() < 1e-5 and np.abs(QtJ[6:]).max() < 1e-5
    assert all(abs(Rm[i, i]) >= abs(Rm[i + 1, i + 1]) * (1 - 1e-6) for i in range(5))  # column pivoting


def test_too_few_rows_leave_x_at_zero():
    src, dst, _, _ = _pairs(1, n=6)
    for m in (4, 5):
        T, status, nfev, its = nx.lm_estimate(src[:, :m], dst[:, :m])
        assert (status, nfev, its) == (nx.IMPROPER, 0, 0) and np.array_equal(T, np.eye(4, dtype=F32))
    T, status, _, _ = nx.lm_estimate(src[:, :6], dst[:, :6])
    assert status != nx.IMPROPER and not np.array_equal(T, np.eye(4, dtype=F32))


def test_icp_with_four_five_and_three_correspondences():
    src, tgt = _scene(2)
    idx, dist = ix.nearest(src, tgt)
    ok = np.flatnonzero((idx >= 0) & (dist.astype(np.float64) <= ix.MAX_D2))
    for m in (4, 5):  # identity increment: the transform criterion ends ICP after one iteration, converged
        r = nx.align_points(src[:, ok[:m]], tgt)
        assert (r["criterion"], r["iterations"], r["converged"], r["n_correspondences"]) == (2, 1, 1, m)
        assert np.array_equal(r["T"], np.eye(4, dtype=F32)) and r["lm"] == [(nx.IMPROPER, 0, 0)]
    r = nx.align_points(src[:, ok[:3]], tgt)  # plain ICP would run with 3
    assert (r["criterion"], r["iterations"], r["converged"], r["n_correspondences"]) == (0, 0, 0, 3)
    assert ix.align_points(src[:, ok[:3]], tgt)["criterion"] != 0


def test_icp_nl_on_a_planted_scene():
    src, tgt = _scene(2)
    r = nx.align_points(src, tgt)
    assert r["converged"] == 1 and r["criterion"] in (2, 3, 4) and r["iterations"] >= 1
    assert all(s in (1, 2, 3) for s, _, _ in r["lm"])
    far = (tgt + F32(0.5)).astype(F32)
    r = nx.align_points(far, tgt)
    assert (r["criterion"], r["converged"], r["iterations"], r["mse"]) == (0, 0, 0, 0.0)


def test_rank_deficient_jacobian_of_collinear_points():
    """points on the x axis: a rotation about it leaves them where they are, bit for bit, so the Jacobian has rank < 6"""
    t = np.linspace(0.0, 1.0, 20)
    src = np.stack([t, np.zeros(20), np.zeros(20)]).astype(F32)
    dst = (src + np.array([[0.01], [-0.02], [0.005]], F32)).astype(F32)
    fvec = nx.residuals(np.zeros(6, F32), src, dst)
    h = nx.SQRT_EPS
    J = np.stack([((nx.residuals(np.eye(6, dtype=F32)[j] * h, src, dst) - fvec) / h).astype(F32) for j in range(6)])
    assert nx.qr(J)[3] < 6
    T, status, nfev, its = nx.lm_estimate(src, dst)
    assert np.isfinite(T).all() and status in range(1, 9)
    moved = ix.transform(T, src)
    assert np.abs(moved - dst).max() < np.abs(src - dst).max()


def test_zero_residual_start_ends_on_the_gradient_test():
    src, _, _, _ = _pairs(0, n=40)
    T, status, nfev, its = nx.lm_estimate(src, src)
    assert (status, nfev, its) == (nx.COSINUS, 8, 1) and np.array_equal(T, np.eye(4, dtype=F32))


def _record_qq(monkeypatch):
    hits = []
    orig = nx.warp_transform

    def warp(x):
        x = np.asarray(x, F32)
        hits.append(F32(F32(F32(x[3] * x[3]) + F32(x[5] * x[5])) + F32(x[4] * x[4])) > 1)
        return orig(x)
    monkeypatch.setattr(nx, "warp_transform", warp)
    return hits


def _turned(seed, ang):
    """30 points turned by ang radians about a random axis and moved by 0.1 m"""
    rng = np.random.default_rng(seed)
    src = rng.normal(size=(3, 30)).astype(F32)
    R = _rot(rng.normal(size=3), ang)
    return src, (R @ src.astype(np.float64) + 0.1).astype(F32), R


def test_a_trial_step_with_qq_above_one_is_rejected(monkeypatch):
    """a 2.5 rad rotation: a trial step leaves the unit ball of q; its residuals are NaN, the step is refused (actred -1)
    and the LM goes on to the rotation"""
    hits = _record_qq(monkeypatch)
    src, dst, R = _turned(0, 2.5)
    T, status, nfev, its = nx.lm_estimate(src, dst)
    assert any(hits) and np.isfinite(T).all() and status in (1, 2, 3)
    assert np.abs(T[:3, :3].astype(np.float64) - R).max() < 1e-4


def test_maxfev_bounds_the_minimisation():
    """a rotation of 3 rad (w near 0, where WarpPointRigid6D's parametrisation is singular) exhausts 400 evaluations; the
    test runs after a trial step, so a Jacobian's 7 can carry nfev past 400"""
    src, dst, _ = _turned(0, 3.0)
    T, status, nfev, its = nx.lm_estimate(src, dst)
    assert status == nx.MAXFEV_REACHED and nx.MAXFEV <= nfev < nx.MAXFEV + 8


def test_icp_align_ex_is_declared_and_exported(built):
    from rgbdslam_v2_b200 import _capi
    txt = (ROOT / "include" / "rgbdslam_b200" / "icp.h").read_text()
    assert "int rgbdslam_b200_icp_align_ex(int n, const uint64_t* source, const uint64_t* target, int max_cloud_size, int method," in txt
    assert re.search(r"#define RGBDSLAM_B200_ICP_METHOD_ICP 0\b", txt) and re.search(r"#define RGBDSLAM_B200_ICP_METHOD_ICP_NL 1\b", txt)
    assert _capi.ICP_METHODS == {"icp": 0, "icp_nl": 1}
    assert hasattr(_capi.load_library(), "rgbdslam_b200_icp_align_ex")


def test_frontend_rejects_an_unknown_method_before_the_library():
    from rgbdslam_v2_b200._capi import Frontend

    class _NoLib:  # icp_align must raise before it touches the library
        lib = None
    for bad in ("gicp", "ICP", ""):
        with pytest.raises(ValueError):
            Frontend.icp_align(_NoLib(), [], [], method=bad)
