"""Exact restatement of the pairwise g2o refinement's bookkeeping (`refine_g2o_kernel`, node.cpp:1225-1268).

- `restate`: the refinement of one pair on top of a RANSAC result.  The solve step is the oracle's dense Gauss-Newton
  (`oracle.get_transform_from_matches_g2o`), the scoring step the float64 errorFunction2 decision (`ransac_exact.scores_f64`).
  It returns the branch taken (skipped, rejected, accepted with an equal count, accepted after a second pass, rejected after a
  second pass) with every intermediate transform, count, error and per-row margin.
- `firm`: a decision whose every row lies more than BAND (relative) from both cuts, and whose rmse comparison (node.cpp:1241)
  lies more than ERR_BAND from a tie.  Moving each entry of the transform by 2 float ulps cannot flip a firm row
  (tests/test_refine_exact_cpu.py checks this), so a GPU result within an ulp of the oracle's must take the same branch.
- `refine_pair`: feature pairs from `synth.make_refine_scene` variants that reach every branch.
"""
from __future__ import annotations

import numpy as np

import ransac_exact as rx

F32 = np.float32
BAND = 2e-3
ERR_BAND = 1e-4
BRANCHES = ("skipped", "rejected", "equal", "second", "second-rejected")


def min_thr(min_matches, M):  # node.cpp:1094-1099
    return min_matches if min_matches <= 0.75 * M else int(0.75 * M)


def rows(xyz_n, xyz_e, matches):
    return np.asarray(xyz_n, F32)[matches["queryIdx"]], np.asarray(xyz_e, F32)[matches["trainIdx"]]


def firm_rows(s, band=BAND):
    return (s["m_margin"] > band) & (s["s_margin"] > band)


def restate(oracle_mod, prm, iterations, xyz_n, kp_n, xyz_e, kp_e, matches, T0, rmse0, n_inliers, *, czc):
    """node.cpp:1225-1268 for one pair: matches (DMATCH rows of the pair, length M), T0 / rmse0 / n_inliers the RANSAC result
    (T0 row-major float32).  prm: oracle params (min_matches, max_dist_for_inliers, sigma_depth, depth_cov_z0 of the run).
    Returns dict(branch, T, cnt, rmse, inl, steps=[(T, scores)], firm) where T / cnt / rmse / inl are the final result."""
    M = len(matches)
    thr = min_thr(prm.min_matches, M)
    frm, to = rows(xyz_n, xyz_e, matches)
    score = lambda T: rx.scores_f64(T, frm, to, max_dist=prm.max_dist_for_inliers, sigma_depth=prm.sigma_depth, czc=czc)
    T0 = np.asarray(T0, F32)
    s0 = score(T0)
    out = dict(branch="skipped", T=T0, cnt=int(n_inliers), rmse=float(rmse0), inl=s0["inl"], steps=[(T0, s0)], firm=True)
    if not (M > prm.min_matches and M >= 4 and n_inliers > thr):  # :1226
        return out
    g2o = lambda sel, T: np.asarray(oracle_mod.get_transform_from_matches_g2o(prm, xyz_n, kp_n, xyz_e, kp_e, matches,
                                                                               np.nonzero(sel)[0], T, iterations), F32)
    cnt0 = s0["cnt"]
    T1 = g2o(s0["inl"], T0)
    s1 = score(T1)
    out["steps"].append((T1, s1))
    firm = True
    err_used = not (s1["cnt"] >= cnt0) and s1["cnt"] >= thr   # the rmse comparison decides
    if err_used:
        firm &= abs(s1["rmse"] / float(F32(rmse0)) - 1) > ERR_BAND
    final = None
    if s1["cnt"] >= cnt0 or (s1["cnt"] >= thr and s1["rmse"] < float(F32(rmse0))):  # :1241
        final = (T1, s1)
        if s1["cnt"] > cnt0:                                                           # :1243-1251
            T2 = g2o(s1["inl"], T1)
            s2 = score(T2)
            out["steps"].append((T2, s2))
            final = (T2, s2)
            out["branch"] = "second" if s2["cnt"] >= cnt0 else "second-rejected"
        else:
            out["branch"] = "equal" if s1["cnt"] >= cnt0 else "rejected"
    else:
        out["branch"] = "rejected"
    out["firm"] = bool(firm and all(firm_rows(s).all() for _, s in out["steps"]))
    if out["branch"] in ("equal", "second"):
        T, s = final
        out.update(T=T, cnt=s["cnt"], rmse=float(F32(s["rmse"])), inl=s["inl"])
    return out


# ---- scenes ---------------------------------------------------------------------------------------------------------------

KINDS = ("clean", "noisy", "skewed", "outliers", "ransac-reject", "few")


def refine_pair(rng, kind, n):
    """One pair (desc_newer, xyz_newer, kp_newer, desc_older, xyz_older, kp_older) of n correspondences; the older node gets an
    extra dummy row (the brute-force matcher never examines the last train row).
      clean          make_refine_scene defaults
      noisy          3-4x the noise: many rows near the cut, so the refined transform gains or loses inliers
      skewed         the older keypoints sheared and shifted: the 2-D terms pull the pose away from the 3-D fit
      outliers       a fifth of the correspondences with swapped geometry
      ransac-reject  the older points shuffled: no transformation explains them
      few            fewer than min_matches inliers"""
    from rgbdslam_v2_b200 import synth
    if kind == "noisy":
        X1, kp_n, xyz_n, kp_e, xyz_e = synth.make_refine_scene(rng, n, noise_px=rng.uniform(0.8, 1.5),
                                                               noise_z=rng.uniform(0.006, 0.012))
    else:
        X1, kp_n, xyz_n, kp_e, xyz_e = synth.make_refine_scene(rng, n)
    if kind == "skewed":
        kp_e = kp_e.copy()
        kp_e[:, 0] += rng.uniform(0.01, 0.04) * (kp_e[:, 1] - 239.5) + rng.uniform(1.0, 4.0)
    if kind in ("outliers", "few"):
        bad = rng.permutation(n)[:n // 5 if kind == "outliers" else max(1, n // 3)]
        xyz_e[bad] = xyz_e[np.roll(bad, 1)]
    if kind == "ransac-reject":
        xyz_e = xyz_e[rng.permutation(n)]
        xyz_e[:, :3] += rng.normal(0, 0.2, (n, 3)).astype(F32)
    desc_e = rng.integers(0, 256, (n + 1, 32), dtype=np.uint8)
    desc_n = desc_e[:n].copy()
    for i in range(n):  # a few flipped bits: unique nearest neighbour
        for b in rng.permutation(256)[:3]:
            desc_n[i, b // 8] ^= 1 << (b % 8)
    xyz_e = np.concatenate([xyz_e, [[0, 0, 1, 1]]]).astype(F32)
    kp_e = np.concatenate([kp_e, [[0, 0]]]).astype(F32)
    return desc_n, xyz_n.astype(F32), kp_n.astype(F32), desc_e, xyz_e, kp_e
