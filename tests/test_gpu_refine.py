"""Pairwise g2o refinement on the GPU (refine_g2o_kernel: Schur-complement Gauss-Newton + the accept logic of
node.cpp:1225-1268) against the oracle's dense full-system solve (oracle/refine_oracle.c)."""
import numpy as np
import pytest

import ransac_exact as rx
import refine_exact as rf

pytestmark = pytest.mark.gpu


def _scene_nodes(fe, rng, n, outliers, seed):
    from rgbdslam_v2_b200 import synth
    from rgbdslam_v2_b200._capi import KEYPOINT_DTYPE
    X1, kp_n, xyz_n, kp_e, xyz_e = synth.make_refine_scene(rng, n)
    desc_e = rng.integers(0, 256, (n, 32), dtype=np.uint8)
    desc_n = desc_e.copy()
    flip = rng.integers(0, 256, (n, 3))
    for i in range(n):                       # a few flipped bits: unique nearest neighbour, hd << 128
        for b in flip[i]:
            desc_n[i, b // 8] ^= 1 << (b % 8)
    if outliers:
        bad = rng.permutation(n)[:outliers]
        xyz_e[bad] = xyz_e[np.roll(bad, 1)]  # geometry of these correspondences is wrong
    # the brute-force matcher never examines the last train row: append a dummy
    desc_e2 = np.concatenate([desc_e, np.zeros((1, 32), np.uint8)]); xyz_e2 = np.concatenate([xyz_e, [[0, 0, 1, 1]]]).astype(np.float32)
    kp_e2 = np.concatenate([kp_e, [[0, 0]]]).astype(np.float32)
    a = fe.node_from_features(1, desc_n, xyz_n); b = fe.node_from_features(0, desc_e2, xyz_e2)
    ka = np.zeros(n, KEYPOINT_DTYPE); ka["x"], ka["y"] = kp_n[:, 0], kp_n[:, 1]
    kb = np.zeros(n + 1, KEYPOINT_DTYPE); kb["x"], kb["y"] = kp_e2[:, 0], kp_e2[:, 1]
    fe.node_set_keypoints(a, ka); fe.node_set_keypoints(b, kb)
    return a, b, (xyz_n, kp_n, xyz_e2, kp_e2), X1


@pytest.mark.parametrize("n,outliers,iters", [(150, 0, 5), (280, 40, 3), (60, 10, 10)])
def test_refinement_matches_the_oracle(built, oracle_mod, n, outliers, iters):
    import ctypes as C
    from rgbdslam_v2_b200 import Frontend
    from rgbdslam_v2_b200._capi import default_params
    rng = np.random.default_rng(n + outliers)
    p = default_params(); p.depth_cov_z0 = 2.0
    fe = Frontend(0, p)
    a, b, (xyz_n, kp_n, xyz_e, kp_e), X1 = _scene_nodes(fe, rng, n, outliers, 0)
    res0, allm0, inl0 = fe.match_node_pairs([a], [b], seed=11)
    assert res0[0]["id1"] == 0 and res0[0]["n_inliers"] >= n - outliers - 5
    p.g2o_transformation_refinement = iters
    fe._check(fe.lib.rgbdslam_b200_init(0, C.byref(p)))      # same library state, refinement switched on
    res1, allm1, inl1 = fe.match_node_pairs([a], [b], seed=11)
    # expected: the oracle's refinement applied to the GPU's own RANSAC result
    M = int(res0[0]["n_all_matches"]); m = allm0[0, :M]
    mask = np.zeros(M, np.uint8)
    keyset = {(int(q), int(t)) for q, t in zip(inl0[0, :res0[0]["n_inliers"]]["queryIdx"], inl0[0, :res0[0]["n_inliers"]]["trainIdx"])}
    for k in range(M):
        mask[k] = (int(m[k]["queryIdx"]), int(m[k]["trainIdx"])) in keyset
    prm = oracle_mod.make_params(depth_cov_z0=2.0)
    T0 = res0[0]["ransac_trafo"].reshape(4, 4).T
    T, rmse, mask2, n_inl, vi = oracle_mod.refine_g2o(prm, iters, xyz_n, kp_n, xyz_e, kp_e, m, T0, float(res0[0]["rmse"]), mask,
                                                       int(res0[0]["valid_iterations"]))
    st = rf.restate(oracle_mod, prm, iters, xyz_n, kp_n, xyz_e, kp_e, m, T0, res0[0]["rmse"], int(res0[0]["n_inliers"]),
                    czc=rx.cov_const(0.01, 2.0))
    T1 = res1[0]["ransac_trafo"].reshape(4, 4).T
    assert np.array_equal(allm0[0, :M], allm1[0, :M])
    assert int(res1[0]["valid_iterations"]) == vi
    assert res1[0]["rmse"] == pytest.approx(rmse, rel=5e-5)
    if st["firm"]:  # no decision within refine_exact.BAND of a cut: the oracle's result exactly
        assert int(res1[0]["n_inliers"]) == n_inl == st["cnt"]
        assert np.array_equal(T, st["T"])
        # Schur complement vs dense full-system solve in float64, rounded to float: within one float ulp
        assert (np.abs(T1.astype(np.float64) - T) <= np.spacing(np.maximum(np.abs(T1), np.abs(T)))).all(), np.abs(T1 - T).max()
    if vi > res0[0]["valid_iterations"]:                          # accepted: the pose moved towards the truth
        T_true = np.linalg.inv(X1)
        assert np.abs(T1[:3, 3] - T_true[:3, 3]).max() <= np.abs(T0[:3, 3] - T_true[:3, 3]).max() + 2e-3
        if st["firm"]:
            assert np.array_equal(inl1[0, :res1[0]["n_inliers"]], m[mask2.astype(bool)])
        assert res1[0]["info_scale"] == np.float64(np.float32(n_inl) / (np.float32(res1[0]["rmse"]) * np.float32(res1[0]["rmse"])))
    fe.close()


def test_refinement_needs_keypoints(built):
    from rgbdslam_v2_b200 import Frontend, synth
    from rgbdslam_v2_b200._capi import B200Error, default_params
    p = default_params(); p.depth_cov_z0 = 2.0; p.g2o_transformation_refinement = 3
    fe = Frontend(0, p)
    b = synth.make_pair(3, 300)
    x, y = fe.node_from_features(1, b["desc_newer"], b["xyz_newer"]), fe.node_from_features(0, b["desc_older"], b["xyz_older"])
    with pytest.raises(B200Error):
        fe.match_node_pairs([x], [y])
    fe.close()
