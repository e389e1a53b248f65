"""The RANSAC rigid fit (`fit_moments` + `fit_solve` in csrc/frontend_kernels.cu) against the float64 weighted Kabsch
(tests/ransac_exact.kabsch_f64) at its conditioning edges (run with -m gpu on an H100).

Every pair is built so that hypothesis 0 draws an all-inlier sample, every correspondence is an inlier under both candidate
fits (asserted in float64) and the > 80 % break ends the loop there.  The returned transform is then either the fit of
hypothesis 0's 4-sample or the refit over every finite row (node.cpp:1140-1166), and is held to the bound of
tests/ransac_exact.py against the float64 fit of that set:
- M = 4: both sets are the same.
- noisy data: the float64 error sums of the two fits are asserted to differ by >= 1e-3 relative, so the loop's choice
  (the refit unless its error is larger) is certain; the comparison is with the float64 fit of the set it keeps (for most
  pairs the refit over all finite rows; the Mahalanobis error is not the Kabsch objective, so a 4-sample can win).
- noise-free data: both candidates are the same motion up to the rounding of the input; the comparison is with the fit over
  all finite rows, under the bound of the worse-conditioned of the two sets.
The case families (ransac_exact.fit_cases) run as one batched call per max_matches setting: 320 (10 mask words) and 512 (16);
the pairs with M > 320 run at 512 only.
"""
import numpy as np
import pytest

import ransac_exact as rx

pytestmark = pytest.mark.gpu

SEED = 13
Z0 = 2.0  # depth_cov_z0: the constant depth covariance of the inlier test
PARAMS = dict(min_matches=3, ransac_iterations=8, g2o_transformation_refinement=0, depth_cov_z0=Z0, max_dist_for_inliers=3.0,
              sigma_depth=0.01, min_translation_meter=0.0, min_rotation_degree=0.0, max_translation_meter=1e10,
              max_rotation_degree=360.0)


def _params(max_matches):
    from rgbdslam_v2_b200._capi import default_params
    p = default_params()
    for k, v in dict(PARAMS, max_matches=max_matches).items():
        setattr(p, k, v)
    return p


def _inliers(T, c):
    return rx.scores_f64(T, c["frm"], c["to"], max_dist=PARAMS["max_dist_for_inliers"], czc=rx.cov_const(PARAMS["sigma_depth"], Z0))


def _as_T(R, t):
    T = np.eye(4)
    T[:3, :3], T[:3, 3] = R, t
    return T


def fit_batch(oracle_mod, max_matches):
    """The batch of every case with M <= max_matches, and per pair the reference fit and bounds.  Asserts the premises of the
    module docstring in float64."""
    pairs, refs = [], []
    cases = [c for c in rx.fit_cases() if c["M"] <= max_matches]
    for i, c in enumerate(cases):
        rng = np.random.default_rng(1000 + i)
        M = c["M"]
        qd, td = rx.pair_descriptors(rng, M)
        sample = rx.hypothesis_samples(oracle_mod, M, 1, SEED, i)[0]
        finite = ~(np.isnan(c["frm"][:, 2]) | np.isnan(c["to"][:, 2]))
        if not finite.all():  # one NaN-depth row inside hypothesis 0's sample (its fit has 3 rows), the others outside it
            rest = np.setdiff1d(np.arange(M), sample)
            slots = np.concatenate([sample[:1], rest[::-1][:(~finite).sum() - 1]])
            perm = np.full(M, -1)
            perm[slots] = np.nonzero(~finite)[0]
            perm[perm < 0] = np.nonzero(finite)[0]
            c = dict(c, frm=c["frm"][perm], to=c["to"][perm])
            finite = finite[perm]
        xn, xo, _ = rx.place_by_rank(oracle_mod, qd, td, c["frm"], c["to"], SEED, i, max_matches)
        pairs.append((qd, xn, td, xo))
        assert finite.sum() > 0.8 * M, c["name"]  # the > 80 % break at hypothesis 0
        f_all = rx.fit_bound(c["frm"], c["to"])
        f_smp = rx.fit_bound(c["frm"], c["to"], sample)
        s_all, s_smp = (_inliers(_as_T(f["R"], f["t"]), c) for f in (f_all, f_smp))
        for s in (s_all, s_smp):
            assert np.array_equal(s["inl"], finite), c["name"]
        ref = dict(f_all)
        if c["noisy"] and M > 4:  # the loop keeps the refit unless its error is larger (node.cpp:1160)
            gap = s_all["esum"] / s_smp["esum"] - 1
            assert abs(gap) > 1e-3, (c["name"], s_all["esum"], s_smp["esum"])
            if gap > 0:
                ref = dict(f_smp)
        elif M > 4:
            ref["rot"] = max(f_all["rot"], f_smp["rot"])
            ref["trans"] = max(f_all["trans"], f_smp["trans"])
        refs.append((c, ref))
    return rx.concat_batch(pairs), refs


def check_fits(b, res, allm, refs):
    """Every pair against its reference; returns the failures as (family, case, what)."""
    bad = []
    on = oo = 0
    for i, (c, ref) in enumerate(refs):
        M = c["M"]
        r = res[i]
        m = allm[i, :M]
        frm, to = b["xyz_newer"][on + m["queryIdx"]], b["xyz_older"][oo + m["trainIdx"]]
        on += int(b["n_newer"][i])
        oo += int(b["n_older"][i])
        assert r["n_all_matches"] == M and np.array_equal(frm, c["frm"], equal_nan=True) and \
            np.array_equal(to, c["to"], equal_nan=True), c["name"]  # rank j carries correspondence j
        if r["id1"] < 0:
            bad.append((c["family"], c["name"], f"no edge (n_inliers {int(r['n_inliers'])}, used_identity {int(r['used_identity'])})"))
            continue
        T = r["ransac_trafo"].reshape(4, 4).T
        eR, et, shape = rx.fit_errors(T[:3, :3], T[:3, 3], ref)
        if not (eR <= ref["rot"] and et <= ref["trans"] and shape <= rx.SHAPE_TOL):
            bad.append((c["family"], c["name"], f"rot {eR:.2e} / {ref['rot']:.2e}, trans {et:.2e} / {ref['trans']:.2e}, "
                                                f"shape {shape:.1e}"))
    return bad


@pytest.mark.parametrize("max_matches", [320, 512])
def test_fit_inside_the_float64_bound(built, oracle_mod, max_matches):
    from rgbdslam_v2_b200 import Frontend
    b, refs = fit_batch(oracle_mod, max_matches)
    fe = Frontend(0, _params(max_matches))
    try:
        res, allm, _ = fe.match_pairs_host(b["desc_newer"], b["xyz_newer"], b["n_newer"], b["desc_older"], b["xyz_older"],
                                           b["n_older"], b["id_newer"], b["id_older"], seed=SEED)
    finally:
        fe.close()
    bad = check_fits(b, res, allm, refs)
    assert not bad, f"{len(bad)} of {len(refs)} pairs outside the bound:\n" + "\n".join(map(str, bad))
