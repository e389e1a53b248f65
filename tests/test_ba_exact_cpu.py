"""The float64 restatement of the landmark bundle adjustment (tests/ba_exact.py) checked before it checks the GPU: its algebra
against the dense full-system oracle (oracle/landmark_oracle.py), its solver steps against each other, and its problem
generator against the boundaries each configuration is named for."""
import numpy as np
import pytest

import ba_exact as bx
from oracle import landmark_oracle as lo
from rgbdslam_v2_b200 import synth


def _oracle_problem(d, edges=True):
    kw = dict(ij=d["ij"], meas=d["meas"], info=d["info"]) if edges else {}
    return lo.Problem(d["poses"], d["fixed"], d["points"], d["obs_cam"], d["obs_point"], d["obs_uvd"], d["obs_info3"], d["K4"], **kw)


def test_observation_jacobians_match_central_differences(oracle_mod):
    d = bx.make_ba_corridor(**bx.CASES["c17_p129_topology"])
    P = bx.Problem.from_dict(d)
    sel = np.arange(0, len(P.oc), 7)
    e, Jc, Jp = bx.obs_terms(P.poses, P.points, P.oc[sel], P.op[sel], P.uvd[sel], P.K4)
    eps = 1e-6
    for n, o in enumerate(sel):
        c, p = P.oc[o], P.op[o]
        f = lambda pose, pw: lo.obs_error(pose, pw, P.uvd[o], P.K4)
        assert np.allclose(e[n], f(P.poses[c], P.points[p]), rtol=1e-12, atol=1e-9)
        for a in range(6):
            dv = np.zeros(6); dv[a] = eps
            fd = (f(lo.pose_oplus(P.poses[c], dv), P.points[p]) - f(lo.pose_oplus(P.poses[c], -dv), P.points[p])) / (2 * eps)
            assert np.abs(Jc[n, :, a] - fd).max() <= 1e-6 * max(1.0, np.abs(fd).max())
        for a in range(3):
            dv = np.zeros(3); dv[a] = eps
            fd = (f(P.poses[c], P.points[p] + dv) - f(P.poses[c], P.points[p] - dv)) / (2 * eps)
            assert np.abs(Jp[n, :, a] - fd).max() <= 1e-6 * max(1.0, np.abs(fd).max())


@pytest.mark.parametrize("edges", [False, True])
@pytest.mark.parametrize("shape", [(5, 40, 9), (6, 60, 5)])
def test_normal_equations_match_dense_oracle(oracle_mod, shape, edges):
    nc, npt, seed = shape
    d = synth.make_ba_problem(n_cams=nc, n_points=npt, seed=seed)
    d["fixed"][2] = 1
    P = bx.Problem.from_dict(d, edges=edges)
    O = _oracle_problem(d, edges)
    assert abs(P.chi2() - O.chi2()) <= 1e-12 * O.chi2()
    A, b, free = P.full_system(P.linearize(), 0.0)
    H, bo = O.normal_equations()
    f = np.ix_(free, free)
    assert np.abs(A[f] - H[f]).max() <= 1e-6 * np.abs(H[f]).max()
    assert np.abs(b[free] + bo[free]).max() <= 1e-6 * np.abs(bo[free]).max()   # the oracle's b is J'We, the solver's -J'We


@pytest.mark.parametrize("case", ["c17_p129_topology", "c171_topology", "pose_edges_only", "no_pose_edges"])
def test_pcg_and_schur_steps_match_direct_solves(oracle_mod, case):
    P = bx.Problem.from_dict(bx.make_ba_corridor(**bx.CASES[case]))
    L = P.linearize()
    lam = 1e-5 * P.max_diag(L)
    t = bx.trial(P, L, lam)
    assert t["pcg_status"] == "converged" and t["pcg_certified"]
    # PCG stops at r'M^-1 r <= 1e-18 r0'M^-1 r0: the step is that close to the direct solve of the same reduced system
    assert np.abs(t["xc"] - t["xc_dir"]).max() <= 1e-6 * np.abs(t["xc_dir"]).max()
    if case == "c171_topology":
        return  # the dense full system below is (6 * 171 + 3 * 2021)^2: the smaller cases cover the elimination
    # the reduced system's direct step and its back-substitution solve the full damped system
    A, b, free = P.full_system(L, lam)
    x = np.zeros(len(b))
    x[free] = np.linalg.solve(A[np.ix_(free, free)], b[free])
    nc6 = 6 * P.nc
    assert np.abs(x[:nc6] - t["xc_dir"]).max() <= 1e-9 * max(np.abs(x[:nc6]).max(), 1e-300)
    if P.np_:
        assert np.abs(x[nc6:].reshape(-1, 3) - t["dp_dir"]).max() <= 1e-9 * np.abs(x[nc6:]).max()


@pytest.mark.parametrize("edges", [False, True])
def test_lm_reaches_the_dense_oracles_optimum(oracle_mod, edges):
    d = synth.make_ba_problem(n_cams=6, n_points=60, seed=5)
    r = bx.optimize(bx.Problem.from_dict(d, edges=edges), 12)
    O = _oracle_problem(d, edges)
    c1 = O.optimize(iterations=12)
    assert abs(r["chi2"] - c1) <= 1e-6 * c1
    assert np.abs(r["poses"][:, :3] - O.poses[:, :3]).max() < 1e-6
    assert np.abs(r["poses"][:, 3:] - O.poses[:, 3:]).max() < 1e-6
    assert np.abs(r["points"] - O.points).max() < 1e-6


def test_lm_first_iteration_matches_the_dense_oracle(oracle_mod):
    d = synth.make_ba_problem(n_cams=5, n_points=40, seed=9)
    r = bx.optimize(bx.Problem.from_dict(d), 1)
    O = _oracle_problem(d)
    c1 = O.optimize(iterations=1)
    assert r["lm_iterations"] == 1
    # the oracle's central-difference Jacobians (h = 1e-6) limit the agreement, as in test_gpu_landmark_ba.py
    assert abs(r["chi2"] - c1) <= 1e-7 * c1
    assert np.abs(r["poses"] - O.poses).max() < 1e-7 and np.abs(r["points"] - O.points).max() < 1e-6


def test_generator_reaches_every_boundary():
    cv = {k: bx.coverage(bx.make_ba_corridor(**kw)) for k, kw in bx.CASES.items()}
    # points per CTA of 128 in ba_points / ba_pt_gather / ba_pt_update
    assert [cv[k]["n_points"] for k in ("c8_p127", "c9_p128_loops", "c17_p129_topology", "c17_p257")] == [127, 128, 129, 257]
    # cameras per CTA of 8 in ba_cams / ba_cam_apply; ba_cg_step's second strided pass (6 * 171 > 1024)
    assert [cv[k]["n_cams"] for k in ("c8_p127", "c9_p128_loops", "c17_p129_topology", "c171_topology", "c200")] == \
        [8, 9, 17, 171, 200]
    # a warp per camera: 31 / 32 / 33 observations, and one camera above 1000
    for k in ("c8_p127", "c17_p257"):
        assert {31, 32, 33} <= set(cv[k]["per_cam"].tolist())
    assert cv["c171_topology"]["per_cam"].max() > 1000 and cv["c200"]["per_cam"].max() > 1000
    # pose-edge incidences: a hub above one warp, loop closures, cameras in both roles, edges into fixed cameras
    for k in ("c171_topology", "c200"):
        assert cv[k]["max_incidences"] > 32
        assert cv[k]["n_obs"] > 256 and cv[k]["n_edges"] > 256      # more than one chi2 block of each
    for k in ("c9_p128_loops", "c17_p129_topology", "c171_topology", "c200", "pose_edges_only"):
        assert cv[k]["loop_edges"] > 0 and cv[k]["both_roles"] > 0
    for k in ("c17_p129_topology", "c171_topology"):
        c = cv[k]
        fixed = np.nonzero(bx.make_ba_corridor(**bx.CASES[k])["fixed"])[0]
        assert len(fixed) >= 3 and fixed[-1] == c["n_cams"] - 1 and 0 < fixed[1] < c["n_cams"] - 1
        assert c["fixed_in_edges"] >= 3
        assert c["duplicates"] > 0 and c["seen_once"] > 0 and c["fixed_only"] > 0 and c["unobserved"] > 0
        assert len(c["isolated"]) == 1 and len(c["edges_only"]) >= 1
    # Huber active on the outlier edges at the start
    for k in ("c17_p129_topology", "c171_topology"):
        P = bx.Problem.from_dict(bx.make_ba_corridor(**bx.CASES[k]))
        e2 = [t[3] for t in P.edge_terms(P.poses, jac=False)]
        assert sum(v > 10 * P.delta ** 2 for v in e2) >= 2
    assert cv["pose_edges_only"]["n_obs"] == 0 and cv["pose_edges_only"]["n_edges"] > 0
    assert cv["no_pose_edges"]["n_edges"] == 0 and cv["no_pose_edges"]["n_cams"] > 1


def test_cases_give_certified_decisions():
    """The GPU tests compare decisions only where they are certain: every case's first LM iteration must be, and the case
    named for it must reject its first trial at lambda_0 (the pop path with ni doubling)."""
    for k, kw in bx.CASES.items():
        r = bx.optimize(bx.Problem.from_dict(bx.make_ba_corridor(**kw)), 3 if k in ("c171_topology", "c200") else 12)
        assert bx.certified_prefix(r) >= (3 if k in ("c171_topology", "c200") else 3), k
    r = bx.optimize(bx.Problem.from_dict(bx.make_ba_corridor(**bx.CASES["first_trial_rejected"])), 1)
    assert [t["accepted"] for t in r["iters"][0]][:2] == [False, False] and r["iters"][0][-1]["accepted"]
