"""CPU self-tests of tests/ransac_exact.py: the float64 scoring restatement against the C oracle, the error envelope of the
kernel's float32 screen over the covariance regimes the product reaches, the near-threshold generator and the oracle paths of
the bookkeeping scenarios."""
import ctypes as C

import numpy as np
import pytest

import ransac_exact as rx

# (name, depth covariance: z0 of the latch or None for the per-point model, point depth range, max_dist_for_inliers).
# cond(S) runs from ~1e2 (the synthetic batches of the older tests: z 0.8-4 m, z0 = 2) to ~1e5 (latched far z0 / far points).
REGIMES = [
    ("z0=2, z 0.8-4", 2.0, (0.8, 4.0), 3.0),
    ("z0=2, z 0.3-0.8", 2.0, (0.3, 0.8), 3.0),
    ("z0=2, z 0.3-0.8, 1.5 m", 2.0, (0.3, 0.8), 1.5),
    ("latched z0=8, z 0.4-1", 8.0, (0.4, 1.0), 3.0),
    ("latched z0=5, z 0.4-1", 5.0, (0.4, 1.0), 3.0),
    ("per-point, z 4-10", None, (4.0, 10.0), 3.0),
    ("per-point, z 10-30", None, (10.0, 30.0), 3.0),
    ("per-point, z 4-10, 1.5 m", None, (4.0, 10.0), 1.5),
]


def _kw(z0, md):
    return dict(max_dist=md, sigma_depth=0.01, czc=None if z0 is None else rx.cov_const(0.01, z0))


def _planted(rng, z0, zr, md, n_m=600, n_s=300, T=None):
    """frm / to rows: n_m +- pairs at the threshold, n_s +- pairs at the shortcut limit, 100 plain inliers."""
    T = rx.small_motion(rng) if T is None else T
    kw = _kw(z0, md)
    frm, to = [], []
    for kind, n in (("m", n_m), ("s", n_s)):
        p = rx.frustum_points(rng, n, *zr)
        delta = rx.log_uniform_delta(rng, n)
        a, b = rx.plant_near_cut(rng, T, p, kind, delta, **kw)
        frm += [p, p]
        to += [a, b]
    p = rx.frustum_points(rng, 100, *zr)
    frm.append(p)
    to.append(p @ T[:3, :3].T + T[:3, 3])
    return np.asarray(T, np.float32), rx.to4(np.concatenate(frm)), rx.to4(np.concatenate(to))


def _oracle_inliers(oracle_mod, prm, T, frm, to, sq_max):
    """oracle_compute_inliers_and_error (node.cpp:968-1020) over frm[i] -> to[i]."""
    n = len(frm)
    m = np.zeros(n, oracle_mod.DMATCH_DTYPE)
    m["queryIdx"] = m["trainIdx"] = np.arange(n)
    inl = np.zeros(n, np.uint8)
    err = C.c_double()
    Tc = np.ascontiguousarray(np.asarray(T, np.float32).T.reshape(-1))
    fn = oracle_mod.lib().oracle_compute_inliers_and_error
    fn.restype = C.c_int
    cnt = fn(C.byref(prm), oracle_mod._p(m), C.c_int(n), oracle_mod._p(Tc), oracle_mod._p(np.ascontiguousarray(frm)),
             oracle_mod._p(np.ascontiguousarray(to)), oracle_mod._p(inl), C.byref(err), C.c_double(sq_max))
    return cnt, inl.astype(bool), err.value


@pytest.mark.parametrize("regime", REGIMES, ids=[r[0] for r in REGIMES])
def test_scores_f64_matches_oracle(oracle_mod, regime):
    """scores_f64 == errorFunction2 of the C oracle (LLT solve) on planted near-threshold rows, NaN and zero depths."""
    _, z0, zr, md = regime
    rng = np.random.default_rng(len(regime[0]))
    T, frm, to = _planted(rng, z0, zr, md, n_m=150, n_s=80)
    frm[3, 2] = np.nan
    to[7, 2] = np.nan
    frm[11, :3] = 0.0
    to[13, 2] = 0.0
    prm = oracle_mod.make_params(max_dist_for_inliers=md, depth_cov_z0=-1.0 if z0 is None else z0)
    r = rx.scores_f64(T, frm, to, **_kw(z0, md))
    cnt, inl, err = _oracle_inliers(oracle_mod, prm, T, frm, to, r["sq_max"])
    # decisions within 1e-12 of a cut may legitimately differ between two float64 solves; the planted ones are >= 1e-5 away
    firm = (r["m_margin"] > 1e-12) & (r["s_margin"] > 1e-12)
    assert firm.sum() >= len(frm) - 2
    assert np.array_equal(inl[firm], r["inl"][firm])
    assert cnt == r["cnt"] and err == pytest.approx(r["rmse"], rel=1e-12)
    assert not r["inl"][[3, 7, 11, 13]].any() and not r["scored"][[11, 13]].any()
    Td = np.asarray(T, np.float64)
    for i in rng.choice(np.nonzero(r["scored"])[0], 60, replace=False):
        e = oracle_mod.error_function2(prm, frm[i], to[i], Td)
        if np.isfinite(r["m"][i]):
            assert e == pytest.approx(r["m"][i], rel=1e-11), i
        else:
            assert e == np.finfo(np.float64).max, i
    near_m = r["m_margin"] < 3e-2
    assert (near_m & r["inl"]).sum() > 30 and (near_m & ~r["inl"]).sum() > 30


@pytest.mark.parametrize("regime", REGIMES, ids=[r[0] for r in REGIMES])
def test_screen_envelope(regime):
    """The float32 screen of mahal_screen stays >= 10x inside its 1e-3 fall-back band in every regime, and never decides a
    correspondence the float64 formula decides the other way."""
    _, z0, zr, md = regime
    rng = np.random.default_rng(1000 + len(regime[0]))
    worst_m = worst_s = 0.0
    n_m = n_s = 0
    for _ in range(4):
        T, frm, to = _planted(rng, z0, zr, md)
        env = rx.screen_envelope(T, frm, to, **_kw(z0, md))
        assert env["wrong"] == 0
        worst_m, worst_s = max(worst_m, env["m_err"]), max(worst_s, env["s_err"])
        n_m += env["n_m"]
        n_s += env["n_s"]
    assert n_m >= 1000 and n_s >= 500
    assert worst_m < 1e-4 and worst_s < 1e-4, (worst_m, worst_s)


def test_condition_numbers_cover_the_product_range():
    """The regimes above reach condition numbers of S from ~1e2 up to >= 1e4 (the old argument assumed < 1e2)."""
    conds = []
    for _, z0, zr, md in REGIMES:
        rng = np.random.default_rng(5)
        T = rx.small_motion(rng).astype(np.float32).astype(np.float64)
        p = rx.frustum_points(rng, 400, *zr)
        q = p @ T[:3, :3].T + T[:3, 3]
        czc = None if z0 is None else rx.cov_const(0.01, z0)
        cz1 = rx._cz(p[:, 2], 0.01, czc)
        cz2 = rx._cz(q[:, 2], 0.01, czc)
        c1 = np.stack([rx.RCX * p[:, 2], rx.RCY * p[:, 2], cz1], 1)
        S = np.einsum("ki,nk,kj->nij", T[:3, :3], c1, T[:3, :3]) + np.stack(
            [np.diag([rx.RCX * a, rx.RCY * a, b]) for a, b in zip(q[:, 2], cz2)])
        conds.append(np.linalg.cond(S).max())
    assert min(conds) < 200 and max(conds) > 1e4, conds


def test_plant_generator_hits_both_sides_of_both_cuts():
    """Planted rows under the planting transform: >= 200 inside the fall-back band, >= 200 in [1e-3, 3e-2], >= 50 within 1e-3
    of the shortcut limit, inliers and rejects on both cuts."""
    for _, z0, zr, md in REGIMES:
        rng = np.random.default_rng(77)
        T, frm, to = _planted(rng, z0, zr, md, n_m=300, n_s=120)
        r = rx.scores_f64(T, frm, to, **_kw(z0, md))
        mm, sm = r["m_margin"], r["s_margin"]
        assert (mm < 1e-3).sum() >= 200 and ((mm >= 1e-3) & (mm < 3e-2)).sum() >= 200
        assert (sm < 1e-3).sum() >= 50
        near_m = mm < 3e-2
        assert (near_m & r["inl"]).sum() and (near_m & ~r["inl"]).sum()
        inside_s = (sm < 3e-2) & (r["dsq"] < r["lim"])
        outside_s = (sm < 3e-2) & (r["dsq"] > r["lim"])
        assert outside_s.sum() >= 50 and (inside_s & r["inl"]).sum() >= 50, (z0, zr)


def test_expected_path_matches_the_sequential_loop():
    assert rx.expected_path({0}, 40, 300, 260, 20) == (1, 1, True)
    assert rx.expected_path({5}, 40, 300, 260, 20) == (6, 1, True)
    assert rx.expected_path({2, 6, 12}, 40, 300, 200, 20) == (40 - 10, 1, False)
    assert rx.expected_path({3, 10, 18, 23}, 40, 300, 238, 20) == (40 - 20, 1, False)
    assert rx.expected_path(set(), 8, 100, 70, 20) == (8, 0, False)
    assert rx.expected_path(set(), 40, 3, 3, 2) == (0, 0, False)


def test_scenarios_take_their_path_in_the_oracle(oracle_mod):
    """Every bookkeeping scenario takes the planned path through the reference loop: real / valid iterations, the break, the
    identity fallback and the final edge decision."""
    for cfg, (b, meta, seed) in rx.scenario_batches(oracle_mod).items():
        mn, mm, H = cfg
        prm = oracle_mod.make_params(min_matches=mn, max_matches=mm, ransac_iterations=H, depth_cov_z0=2.0)
        res, allm, inl = oracle_mod.match_pairs(prm, b["desc_newer"], b["xyz_newer"], b["n_newer"], b["desc_older"],
                                                b["xyz_older"], b["n_older"], b["id_newer"], b["id_older"], seed=seed)
        for i, (name, M, valid, n_in) in enumerate(meta):
            r = res[i]
            assert r["n_all_matches"] == M, name
            real, nvalid, broke = rx.expected_path(set(valid), H, M, n_in, mn)
            assert r["real_iterations"] == real, (name, r["real_iterations"], real)
            if not valid:
                accepted = name.endswith("accepted") or name == "M3-identity"
                assert r["used_identity"] == int(accepted) and r["valid_iterations"] == int(accepted), name
                assert (r["id1"] >= 0) == accepted, name
                if accepted:
                    assert r["n_inliers"] == n_in, name
            else:
                assert r["valid_iterations"] == nvalid == 1 and r["used_identity"] == 0, name
                assert r["n_inliers"] == n_in and r["id1"] >= 0, name


def _oracle_batch(oracle_mod, b, seed, **kw):
    prm = oracle_mod.make_params(**kw)
    return oracle_mod.match_pairs(prm, b["desc_newer"], b["xyz_newer"], b["n_newer"], b["desc_older"], b["xyz_older"],
                                  b["n_older"], b["id_newer"], b["id_older"], seed=seed)


def _rows(b, allm, i, n):
    on, oo = int(np.sum(b["n_newer"][:i])), int(np.sum(b["n_older"][:i]))
    m = allm[i, :n]
    return b["xyz_newer"][on + m["queryIdx"]], b["xyz_older"][oo + m["trainIdx"]]


def test_identity_planted_batches_reach_the_fallback_and_fill_the_band(oracle_mod):
    """The near-threshold batches of the GPU test: in the oracle every pair ends in the accepted identity fallback, and under
    T = I the planted rows fill the screen's fall-back band on both sides of both cuts."""
    import test_gpu_ransac_exact as g
    for regime in g.PLANTED:
        name, z0p, zr, md, zfar = regime
        b, z0 = g.planted_batch(oracle_mod, regime)
        res, allm, _ = _oracle_batch(oracle_mod, b, 3, max_dist_for_inliers=md, ransac_iterations=g.PLANTED_H,
                                     depth_cov_z0=-1.0 if z0 is None else z0)
        czc = None if z0 is None else rx.cov_const(0.01, z0)
        for i in range(len(res)):
            frm, to = _rows(b, allm, i, int(res[i]["n_all_matches"]))
            s = rx.scores_f64(res[i]["ransac_trafo"].reshape(4, 4).T, frm, to, max_dist=md, czc=czc)
            assert s["cnt"] == res[i]["n_inliers"], name
        g.assert_not_vacuous(g.identity_margins(b, res, allm, md, czc))


def test_degenerate_pairs_take_their_path_in_the_oracle(oracle_mod):
    import test_gpu_ransac_exact as g
    b, meta = g.degenerate_batch(oracle_mod)
    res, _, _ = _oracle_batch(oracle_mod, b, 11, ransac_iterations=8, depth_cov_z0=2.0)
    for i, (kind, k, n_in, _) in enumerate(meta):
        assert res[i]["real_iterations"] == k + 1 and res[i]["valid_iterations"] == 1, (kind, k, res[i]["real_iterations"])
        assert res[i]["n_inliers"] == n_in, kind
