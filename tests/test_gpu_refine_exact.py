"""Exact gates on the pairwise g2o refinement (refine_g2o_kernel, node.cpp:1225-1268), run with -m gpu on an H100.

One batch of feature pairs (tests/refine_exact.refine_pair: clean, noisy, skewed keypoints, outliers, RANSAC-rejected, too
few inliers) is matched twice with the same seed, refinement off and on, at max_matches 300 and 512 (both kernel
instantiations), under the constant, latched and per-point depth covariance and 1, 5 and 20 iterations.
- Identical inputs: the match lists agree; a pair that is skipped or whose refinement is rejected returns the RANSAC result
  byte for byte, with the same inlier rows.
- Scoring invariant: an accepted pair's inlier list is the float64 errorFunction2 decision under the returned transform,
  n_inliers its size, rmse the float64 value to the float32 envelope, info_scale bit for bit.
- Bookkeeping: where every decision of the restatement (tests/refine_exact.restate, run from the GPU's own RANSAC result)
  is firm, the branch, valid_iterations, n_inliers and the inlier list equal the restatement's, and the returned transform
  is within 1 float ulp (or 1e-12) of the oracle's, entry by entry.
"""
import ctypes as C

import numpy as np
import pytest

import ransac_exact as rx
import refine_exact as rf

pytestmark = pytest.mark.gpu

# (max_matches, depth_cov_z0 parameter (0 = latched), iterations)
CONFIGS = [(300, 2.0, 5), (300, 0.0, 20), (300, -1.0, 1), (512, 2.0, 1), (512, -1.0, 5), (512, 0.0, 5)]
TALLY = {"branches": {b: 0 for b in rf.BRANCHES}, "identical": 0, "compared": 0, "unfirm": 0}


@pytest.fixture(scope="module")
def fe(built):
    from rgbdslam_v2_b200 import Frontend
    from rgbdslam_v2_b200._capi import default_params
    p = default_params()
    p.depth_cov_z0 = 2.0
    f = Frontend(0, p)
    yield f
    f.close()
    print("\nrefinement branches:", TALLY)


def _reinit(fe, **kw):
    from rgbdslam_v2_b200._capi import default_params
    p = default_params()
    for k, v in kw.items():
        setattr(p, k, v)
    fe.params = p
    fe._check(fe.lib.rgbdslam_b200_init(0, C.byref(p)))
    return p


@pytest.fixture(scope="module")
def batch(fe):
    """~200 pairs: every kind at sizes 24..160, plus a few above 320 correspondences (only the 16-word instantiation sees
    all of them)."""
    from rgbdslam_v2_b200._capi import KEYPOINT_DTYPE
    rng = np.random.default_rng(2024)
    kinds = rf.KINDS + ("noisy", "noisy")   # noisy pairs are the ones that reach a second pass
    specs = [(kinds[k % len(kinds)], int(rng.integers(24, 161))) for k in range(192)]
    specs += [("clean", 340), ("noisy", 360), ("skewed", 330), ("outliers", 380)]
    nodes, data = [], []
    for i, (kind, n) in enumerate(specs):
        if kind == "few":
            n = int(rng.integers(24, 40))
        dn, xn, kn, de, xe, ke = rf.refine_pair(rng, kind, n)
        a = fe.node_from_features(2 * i + 1, dn, xn)
        b = fe.node_from_features(2 * i, de, xe)
        for h, k in ((a, kn), (b, ke)):
            kp = np.zeros(len(k), KEYPOINT_DTYPE)
            kp["x"], kp["y"] = k[:, 0], k[:, 1]
            fe.node_set_keypoints(h, kp)
        nodes.append((a, b))
        data.append((kind, xn, kn, xe, ke))
    return nodes, data


def _ulps(a, b):
    a, b = np.asarray(a, np.float32), np.asarray(b, np.float32)
    return np.abs(a.astype(np.float64) - b.astype(np.float64)) / np.spacing(np.maximum(np.abs(a), np.abs(b)))


def _check_invariant(r, frm, to, inl_rows, allm_rows, prm, czc, tie=1e-10):
    s = rx.scores_f64(r["ransac_trafo"].reshape(4, 4).T, frm, to, max_dist=prm.max_dist_for_inliers,
                      sigma_depth=prm.sigma_depth, czc=czc)
    firm = (s["m_margin"] > tie) & (s["s_margin"] > tie)
    ni = int(r["n_inliers"])
    got = np.zeros(len(frm), bool)
    pos = {(int(q), int(t)): k for k, (q, t) in enumerate(zip(allm_rows["queryIdx"], allm_rows["trainIdx"]))}
    got[[pos[(int(q), int(t))] for q, t in zip(inl_rows["queryIdx"], inl_rows["trainIdx"])]] = True
    assert got.sum() == ni
    assert np.array_equal(got[firm], s["inl"][firm])
    assert abs(ni - s["cnt"]) <= (~firm).sum()
    if firm.all():
        assert np.array_equal(inl_rows, allm_rows[s["inl"]])
    assert abs(float(r["rmse"]) / s["rmse"] - 1) < 5e-5, (float(r["rmse"]), s["rmse"])
    if r["id1"] >= 0:
        assert r["info_scale"] == np.float64(np.float32(ni) / (np.float32(r["rmse"]) * np.float32(r["rmse"])))


@pytest.mark.parametrize("cfg", CONFIGS, ids=[f"maxm{c[0]}-z0{c[1]}-it{c[2]}" for c in CONFIGS])
def test_refinement_is_exact(fe, oracle_mod, batch, cfg):
    mm, z0p, iters = cfg
    nodes, data = batch
    newer, older = [a for a, _ in nodes], [b for _, b in nodes]
    _reinit(fe, max_matches=mm, depth_cov_z0=z0p)
    res0, allm0, inl0 = fe.match_node_pairs(newer, older, seed=17)
    _reinit(fe, max_matches=mm, depth_cov_z0=z0p, g2o_transformation_refinement=iters)
    res1, allm1, inl1 = fe.match_node_pairs(newer, older, seed=17)
    z0 = fe.depth_cov_z0 if z0p >= 0 else -1.0
    assert z0p != 0.0 or z0 > 0
    czc = None if z0 < 0 else rx.cov_const(fe.params.sigma_depth, z0)
    prm = oracle_mod.make_params(max_matches=mm, depth_cov_z0=z0)
    seen = {b: 0 for b in rf.BRANCHES}
    big = 0
    for i, (kind, xn, kn, xe, ke) in enumerate(data):
        r0, r1 = res0[i], res1[i]
        M = int(r0["n_all_matches"])
        big += M > 320
        assert np.array_equal(allm0[i, :M], allm1[i, :M]) and int(r1["n_all_matches"]) == M, i
        m = allm0[i, :M]
        st = rf.restate(oracle_mod, prm, iters, xn, kn, xe, ke, m, r0["ransac_trafo"].reshape(4, 4).T, r0["rmse"],
                        int(r0["n_inliers"]), czc=czc)
        seen[st["branch"]] += 1
        accepted = r1["valid_iterations"] == r0["valid_iterations"] + 1
        assert r1["valid_iterations"] in (r0["valid_iterations"], r0["valid_iterations"] + 1), i
        if st["branch"] == "skipped" or not accepted:
            # skipped, rejected, rejected by RANSAC: the refinement-off result, byte for byte
            assert r1.tobytes() == r0.tobytes(), (i, kind, st["branch"])
            assert np.array_equal(inl1[i, :r1["n_inliers"]], inl0[i, :r0["n_inliers"]]), i
        else:
            frm, to = rf.rows(xn, xe, m)
            _check_invariant(r1, frm, to, inl1[i, :r1["n_inliers"]], m, prm, czc)
        if not st["firm"]:
            TALLY["unfirm"] += 1
            continue
        assert accepted == (st["branch"] in ("equal", "second")), (i, kind, st["branch"])
        if accepted:
            assert int(r1["n_inliers"]) == st["cnt"], (i, kind, st["branch"], int(r1["n_inliers"]), st["cnt"])
            assert np.array_equal(inl1[i, :st["cnt"]], m[st["inl"]]), i
            T1 = r1["ransac_trafo"].reshape(4, 4).T
            d = _ulps(T1, st["T"])
            ok = (d <= 1) | (np.abs(T1.astype(np.float64) - st["T"]) <= 1e-12)
            assert ok.all(), (i, kind, st["branch"], d.max())
            TALLY["compared"] += 1
            TALLY["identical"] += int(np.array_equal(T1, st["T"]))
    for b, n in seen.items():
        TALLY["branches"][b] += n
    if mm == 512:
        assert big >= 3, big
    # every branch the reference has is visited (a rejection after a second pass is rare); a single Gauss-Newton step from
    # the RANSAC transform loses inliers on these scenes, so with 1 iteration every refinement that runs is rejected
    assert seen["skipped"] >= 3 and seen["rejected"] >= 3, seen
    if iters > 1:
        assert seen["equal"] >= 3 and seen["second"] >= 3, seen
    _reinit(fe)
