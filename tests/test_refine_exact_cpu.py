"""The restatement of the refinement's bookkeeping (tests/refine_exact.py) against the C oracle's node.cpp:1225-1268
(`oracle.refine_g2o`), and the margin band that makes a decision firm."""
import numpy as np
import pytest

import ransac_exact as rx
import refine_exact as rf

DMATCH = np.dtype([("queryIdx", "<i4"), ("trainIdx", "<i4"), ("imgIdx", "<i4"), ("distance", "<f4")])


def _cases():
    """(name, kind, n, iterations, depth_cov_z0 parameter, rotation / translation error of the RANSAC transform)"""
    out = []
    for k, (kind, n) in enumerate([("clean", 80), ("noisy", 90), ("skewed", 70), ("outliers", 100), ("few", 26),
                                   ("noisy", 60), ("clean", 40), ("skewed", 110)]):
        for iters, z0 in ((1, 2.0), (5, -1.0), (20, 3.25)):
            for err in (0.0, 0.012):
                out.append((f"{kind}{n}-it{iters}-z0{z0}-e{err}", kind, n, iters, z0, err, 100 * k + iters))
    return out


CASES = _cases()


def _case(oracle_mod, case):
    name, kind, n, iters, z0, err, seed = case
    rng = np.random.default_rng(seed)
    dn, xn, kn, de, xe, ke = rf.refine_pair(rng, kind, n)
    m = np.zeros(n, DMATCH)
    m["queryIdx"] = m["trainIdx"] = np.arange(n)
    prm = oracle_mod.make_params(depth_cov_z0=z0)
    czc = None if z0 < 0 else rx.cov_const(0.01, z0)
    # the RANSAC transform: the least-squares fit of the scene, moved by a small error
    T0 = oracle_mod.get_transform_from_matches(xn, xe, m).astype(np.float64)
    T0 = (rx.small_motion(rng, err, 20 * err) @ T0 if err else T0).astype(np.float32)
    frm, to = rf.rows(xn, xe, m)
    s0 = rx.scores_f64(T0, frm, to, czc=czc)
    return prm, czc, iters, (xn, kn, xe, ke, m), T0, s0


def test_restatement_equals_the_oracle(oracle_mod):
    """The restated branch, transform, count, rmse and inlier mask equal oracle.refine_g2o wherever every decision is firm,
    and the cases visit every branch but the rare rejection after a second pass."""
    branches = {b: 0 for b in rf.BRANCHES}
    n_firm = 0
    for case in CASES:
        prm, czc, iters, (xn, kn, xe, ke, m), T0, s0 = _case(oracle_mod, case)
        r = rf.restate(oracle_mod, prm, iters, xn, kn, xe, ke, m, T0, np.float32(s0["rmse"]), s0["cnt"], czc=czc)
        T, rmse, inl, n_inl, vi = oracle_mod.refine_g2o(prm, iters, xn, kn, xe, ke, m, T0, np.float32(s0["rmse"]),
                                                         s0["inl"].astype(np.uint8), 0)
        branches[r["branch"]] += 1
        if not r["firm"]:
            continue
        n_firm += 1
        accepted = r["branch"] in ("equal", "second")
        assert vi == int(accepted), (case[0], r["branch"], vi)
        assert np.array_equal(T, r["T"]), case[0]
        assert n_inl == r["cnt"] and np.array_equal(inl.astype(bool), r["inl"]), (case[0], n_inl, r["cnt"])
        assert np.float32(rmse) == np.float32(r["rmse"]), case[0]
    assert n_firm >= 0.8 * len(CASES), n_firm
    assert min(branches[b] for b in ("skipped", "rejected", "equal", "second")) >= 3, branches


def _ulp_moves(T, rng, k):
    """T with every entry moved by up to 2 float ulps (k random sign / size patterns, plus all +2 and all -2)"""
    T = np.asarray(T, np.float32)
    out = [np.nextafter(np.nextafter(T, np.float32(np.inf)), np.float32(np.inf)),
           np.nextafter(np.nextafter(T, np.float32(-np.inf)), np.float32(-np.inf))]
    for _ in range(k):
        steps = rng.integers(-2, 3, T.shape)
        X = T.copy()
        for s in (1, 2):
            X = np.where(steps >= s, np.nextafter(X, np.float32(np.inf)), X)
            X = np.where(steps <= -s, np.nextafter(X, np.float32(-np.inf)), X)
        out.append(X.astype(np.float32))
    return out


def test_two_ulp_moves_flip_no_firm_row(oracle_mod):
    """The band of refine_exact.firm_rows: no transform of a refinement step, moved by 2 float ulps per entry, changes the
    decision of a firm row.  Also checks the band is not vacuous: rows inside it exist."""
    rng = np.random.default_rng(0)
    inside, checked = 0, 0
    for case in CASES[::3]:
        prm, czc, iters, (xn, kn, xe, ke, m), T0, s0 = _case(oracle_mod, case)
        r = rf.restate(oracle_mod, prm, iters, xn, kn, xe, ke, m, T0, np.float32(s0["rmse"]), s0["cnt"], czc=czc)
        frm, to = rf.rows(xn, xe, m)
        for T, s in r["steps"]:
            firm = rf.firm_rows(s)
            inside += int((~firm).sum())
            for X in _ulp_moves(T, rng, 6):
                sx = rx.scores_f64(X, frm, to, czc=czc)
                assert np.array_equal(sx["inl"][firm], s["inl"][firm]), case[0]
                checked += 1
    assert checked > 100
    print("rows inside the band:", inside)


def test_oracle_solve_leaves_its_input_alone(oracle_mod):
    """The oracle writes its result into a column-major buffer; a transposed view of a result row (the layout the library
    returns) must not be that buffer, or the caller's RANSAC transform silently becomes the refined one."""
    prm, czc, iters, (xn, kn, xe, ke, m), T0, s0 = _case(oracle_mod, CASES[1])
    row = np.zeros(1, [("ransac_trafo", "<f4", (16,))])
    row["ransac_trafo"][0] = T0.T.reshape(-1)
    view = row[0]["ransac_trafo"].reshape(4, 4).T
    before = view.copy()
    T1 = oracle_mod.get_transform_from_matches_g2o(prm, xn, kn, xe, ke, m, np.nonzero(s0["inl"])[0], view, iters)
    T2, *_ = oracle_mod.refine_g2o(prm, iters, xn, kn, xe, ke, m, view, np.float32(s0["rmse"]), s0["inl"].astype(np.uint8))
    assert not np.array_equal(T1, before)
    assert np.array_equal(view, before)
