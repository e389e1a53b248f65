"""rgbdslam_b200_landmark_ba against the float64 restatement (tests/ba_exact.py) at multi-CTA shapes and every pose-edge
topology: chi2 to rounding, one LM iteration re-seeded from the restatement's state, full runs on certified decisions, and the
solver's invariants (fixed / unobserved / isolated variables, determinism, grow-only buffers, observation order)."""
import functools
import math

import numpy as np
import pytest

import ba_exact as bx
from rgbdslam_v2_b200 import _capi

pytestmark = pytest.mark.gpu

EPS = np.finfo(np.float64).eps
SHAPES = list(bx.CASES)
LARGE = ("c171_topology", "c200")


@pytest.fixture(scope="module")
def fe(oracle_mod):
    f = _capi.Frontend(0)
    yield f
    f.close()


@functools.lru_cache(maxsize=None)
def problem(case):
    d = bx.make_ba_corridor(**bx.CASES[case])
    return d, bx.Problem.from_dict(d)


def gpu(fe, P, iterations, poses=None, points=None, order=None):
    """landmark_ba on P's arrays (optionally another state, optionally the observations permuted)"""
    o = np.arange(len(P.oc)) if order is None else order
    kw = dict(ij=P.ij, meas=P.meas, info=P.info) if len(P.ij) else {}
    return fe.landmark_ba(P.poses if poses is None else poses, P.fixed.astype(np.uint8), P.points if points is None else points,
                          P.oc[o], P.op[o], P.uvd[o], P.w3[o], P.K4, iterations=iterations, huber_delta=P.delta, **kw)


def pose_bound(bc, poses):
    """A camera step difference of bc (max norm) moves t + R dt by at most sqrt(3) bc and q * (v, sqrt(1 - |v|^2)), normalised,
    by at most sqrt(3) bc (1 + |v|^2) for the small |v| of an LM step: 2 bc; plus the float64 rounding of the update, a few
    ulps of the pose's largest entry."""
    return 2 * bc + 8 * EPS * max(1.0, float(np.abs(poses).max()))


def point_bound(bp, points):
    return bp + 4 * EPS * max(1.0, float(np.abs(points).max(initial=0.0)))


def check_state(x, pts, ref_poses, ref_points, bc, bp, what):
    dpose = float(np.abs(x - ref_poses).max(initial=0.0))
    dpt = float(np.abs(pts - ref_points).max(initial=0.0))
    assert dpose <= pose_bound(bc, ref_poses), (what, dpose, pose_bound(bc, ref_poses))
    assert dpt <= point_bound(bp, ref_points), (what, dpt, point_bound(bp, ref_points))
    return dpose, dpt


def check_pcg(got, trials):
    want = sum(t["pcg_iterations"] for t in trials)
    if all(t["pcg_certified"] for t in trials):
        assert got == want, (got, want)
    else:
        assert abs(got - want) <= len(trials), (got, want)


@pytest.mark.parametrize("case", SHAPES)
def test_zero_iterations_return_the_input_and_its_chi2(fe, case):
    d, P = problem(case)
    x, pts, c0, c1, it, cg = gpu(fe, P, 0)
    assert c0 == c1 and it == 0 and cg == 0
    want = P.chi2()
    # the kernels sum per-observation / per-edge terms in blocks of 256, then the blocks: a few hundred float64 additions of
    # positive terms, relative error below 1e-13; 1e-11 leaves room for the 3-term error expressions
    assert abs(c0 - want) <= 1e-11 * want, (c0, want)
    assert np.array_equal(x, P.poses) and np.array_equal(pts, P.points)


@pytest.mark.parametrize("case", SHAPES)
def test_one_iteration_reseeded(fe, case):
    """iterations = 1 from the restatement's state, three times: every kernel at every shape without accumulated path
    differences.  Decisions are compared only while they are certified (tests/test_ba_exact_cpu.py requires the first few)."""
    d, P = problem(case)
    state = P
    for k in range(3):
        r = bx.optimize(state, 1)
        if not bx.certified_prefix(r):
            assert k > 0, "the first iteration of every case is certified"
            break
        x, pts, c0, c1, it, cg = gpu(fe, state, 1)
        assert it == r["lm_iterations"]
        check_pcg(cg, r["trials"])
        bc, bp = bx.iteration_bound(r["iters"][0])
        dpose, dpt = check_state(x, pts, r["poses"], r["points"], bc, bp, (case, k))
        assert abs(c1 - r["chi2"]) <= 1e-10 * r["chi2"], (c1, r["chi2"])
        print(f"{case} it{k}: pose diff {dpose:.3g} (bound {pose_bound(bc, r['poses']):.3g}) point diff {dpt:.3g} "
              f"(bound {point_bound(bp, r['points']):.3g}) chi2 rel {abs(c1 - r['chi2']) / r['chi2']:.3g} pcg {cg}")
        state = state.with_state(r["poses"], r["points"])


@pytest.mark.parametrize("case", ["c17_p129_topology", "c17_p257", "first_trial_rejected", "pose_edges_only", "c200"])
def test_full_run_on_certified_decisions(fe, case):
    """Up to 12 iterations, as long as every trial's decision is certified: the state after each iteration (hence the same
    accepted / rejected sequence), lm_iterations and pcg_iterations.  The bound compounds by summing the per-iteration bounds:
    to first order an LM iteration maps a difference in its start state through I - (H + lambda I)^-1 H, whose eigenvalues
    lie in [0, 1), so earlier differences do not grow."""
    d, P = problem(case)
    r = bx.optimize(P, 12)
    k = bx.certified_prefix(r)
    assert k >= 3
    bc = bp = 0.0
    pcg = 0
    for j in range(1, k + 1):
        b = bx.iteration_bound(r["iters"][j - 1])
        bc, bp = bc + b[0], bp + b[1]
        pcg += sum(t["pcg_iterations"] for t in r["iters"][j - 1])
        if case in LARGE and j not in (1, k):
            continue
        x, pts, c0, c1, it, cg = gpu(fe, P, j)
        assert it == j
        assert cg == pcg, (j, cg, pcg)
        poses, points, chi2 = r["states"][j - 1]
        check_state(x, pts, poses, points, bc, bp, (case, j))
        assert abs(c1 - chi2) <= 1e-10 * chi2 * j, (j, c1, chi2)
    if case == "first_trial_rejected":
        assert [t["accepted"] for t in r["iters"][0]][:3] == [False, False, False]


def test_fixed_unobserved_and_isolated_variables_stay(fe):
    d, P = problem("c17_p129_topology")
    x, pts, *_ = gpu(fe, P, 8)
    cv = bx.coverage(d)
    for c in np.nonzero(P.fixed)[0]:
        assert np.array_equal(x[c], P.poses[c])
    un = cv["per_pt"] == 0
    assert un.sum() > 0 and np.array_equal(pts[un], P.points[un])
    iso = cv["isolated"][0]
    # its step is exactly 0 (r = g = 0): only the quaternion's renormalisation may round
    assert np.abs(x[iso] - P.poses[iso]).max() <= 1e-15
    assert np.abs(x[~P.fixed] - P.poses[~P.fixed]).max() > 1e-4


def test_same_call_twice_is_bit_identical(fe):
    d, P = problem("c171_topology")
    a = gpu(fe, P, 3)
    b = gpu(fe, P, 3)
    assert np.array_equal(a[0], b[0]) and np.array_equal(a[1], b[1]) and a[2:] == b[2:]


def test_large_then_small_problem_is_bit_identical(fe):
    """the solver's buffers are grow-only: a small problem after a large one must not read the large one's leftovers"""
    _, small = problem("c9_p128_loops")
    _, large = problem("c200")
    a = gpu(fe, small, 4)
    gpu(fe, large, 2)
    b = gpu(fe, small, 4)
    assert np.array_equal(a[0], b[0]) and np.array_equal(a[1], b[1]) and a[2:] == b[2:]


def test_pose_graph_solve_in_between_changes_nothing(fe):
    _, P = problem("c17_p129_topology")
    a = gpu(fe, P, 4)
    fe.optimize_graph(P.poses, P.fixed.astype(np.uint8), P.ij.astype(np.int32), P.meas, P.info)
    b = gpu(fe, P, 4)
    assert np.array_equal(a[0], b[0]) and np.array_equal(a[1], b[1]) and a[2:] == b[2:]


@pytest.mark.parametrize("case", ["c17_p129_topology", "c171_topology"])
def test_observation_order_changes_only_rounding(fe, case):
    d, P = problem(case)
    r = bx.optimize(P, 1)
    assert bx.certified_prefix(r) == 1
    order = np.random.default_rng(11).permutation(len(P.oc))
    x, pts, c0, c1, it, cg = gpu(fe, P, 1, order=order)
    assert it == 1
    assert abs(cg - r["pcg_iterations"]) <= len(r["trials"])
    bc, bp = bx.iteration_bound(r["iters"][0])
    check_state(x, pts, r["poses"], r["points"], bc, bp, case)
    assert abs(c0 - r["chi2_before"]) <= 1e-11 * r["chi2_before"]
    assert math.isclose(c1, r["chi2"], rel_tol=1e-10)
