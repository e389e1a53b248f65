"""Environment measurement model on the GPU (csrc/emm.cu) vs oracle/emm_oracle.c: pairwiseObservationLikelihood counts for
explicit transformations, and the gate it puts on accepted RANSAC transformations (node.cpp:1340-1342)."""
import ctypes as C

import numpy as np
import pytest

import emm_exact as ee

pytestmark = pytest.mark.gpu


def _frames(ks):
    from oracle import orb_oracle
    from rgbdslam_v2_b200 import synth
    poses = synth.trajectory(240)
    fr = [synth.render_frame(poses[k], seed=k) for k in ks]
    gray = np.stack([f[0] for f in fr]); depth = np.stack([f[1] for f in fr])
    mask = np.stack([orb_oracle.depth_to_mask(d) for d in depth])
    return [poses[k] for k in ks], gray, depth, mask, (synth.FX, synth.FY, synth.CX, synth.CY)


def _assert_exact(got, exp, T, zn, Kn, zo, Ko):
    """the oracle's counts exactly, unless the restatement finds a sample whose p lies within 1e-12 of a cut"""
    rs = ee.pairwise(T, zn, Kn, zo, Ko, czc=ee.cov_const(0.01, 2.0))
    assert np.array_equal(rs["counts"], np.asarray(exp, np.int64))
    n_loose = int(rs["loose"].sum())
    assert np.abs(np.asarray(got, np.int64) - rs["counts"]).max() <= n_loose, (got, exp, n_loose)


def test_observation_likelihood_counts_match_the_oracle(built, oracle_mod):
    from rgbdslam_v2_b200 import Frontend, synth
    from rgbdslam_v2_b200._capi import default_params
    poses, gray, depth, mask, K4 = _frames([0, 30])
    p = default_params(); p.depth_cov_z0 = 2.0
    fe = Frontend(0, p)
    b = synth.make_pair(1, 50)
    older = fe.node_from_features(0, b["desc_older"], b["xyz_older"]); newer = fe.node_from_features(1, b["desc_newer"], b["xyz_newer"])
    fe.node_set_depth(older, depth[0], K4); fe.node_set_depth(newer, depth[1], K4)
    prm = oracle_mod.make_params(depth_cov_z0=2.0)
    z_old, z_new = oracle_mod.create_cloud_z(depth[0]), oracle_mod.create_cloud_z(depth[1])
    T = np.linalg.inv(poses[0]) @ poses[1]      # newer -> older
    seen_bad = False
    for dz in (0.0, 0.05, 0.3, -0.6):
        Tb = T.copy(); Tb[2, 3] += dz
        got = fe.observation_likelihood(newer, older, Tb)
        exp = oracle_mod.pairwise_observation(prm, Tb, z_new, K4, z_old, K4)
        assert got[3] == exp[3] == 2 * 40 * 30                       # every sampled raster cell counts
        _assert_exact(got, exp, Tb, z_new, K4, z_old, K4)
        ok, q = oracle_mod.observation_criterion_met(got[0], got[1], got[2], 0.75)
        assert ok == (abs(dz) < 0.1)
        seen_bad |= not ok
    assert seen_bad
    fe.close()


def test_emm_gates_accepted_transformations(built, oracle_mod):
    from rgbdslam_v2_b200 import Frontend
    from rgbdslam_v2_b200._capi import B200Error, default_params
    poses, gray, depth, mask, K4 = _frames([0, 4, 8])
    p = default_params(); p.depth_cov_z0 = 2.0; p.max_keypoints = 600; p.observability_threshold = 0.75
    fe = Frontend(0, p)
    det = fe.detector_create()
    handles, _ = fe.nodes_create(det, gray, depth, mask, K4, ids=np.arange(3, dtype=np.int32))
    res, _, _ = fe.match_node_pairs([handles[1], handles[2], handles[2]], [handles[0], handles[1], handles[0]], seed=2)
    prm = oracle_mod.make_params(depth_cov_z0=2.0)
    zs = [oracle_mod.create_cloud_z(d) for d in depth]
    for r, (a, b) in zip(res, [(1, 0), (2, 1), (2, 0)]):
        assert r["id1"] == b and r["id2"] == a                         # good geometry passes the model
        exp = oracle_mod.pairwise_observation(prm, r["ransac_trafo"].reshape(4, 4).T, zs[a], K4, zs[b], K4)
        got = np.array([r["inlier_points"], r["outlier_points"], r["occluded_points"], r["all_points"]])
        _assert_exact(got, exp, r["ransac_trafo"].reshape(4, 4).T, zs[a], K4, zs[b], K4)
        assert got[0] / max(got[0] + got[1], 1) > 0.75
    # a threshold nothing can meet rejects every pair: ids -1 like node.cpp:1420, the rest of the result stays
    p.observability_threshold = 1.5
    fe._check(fe.lib.rgbdslam_b200_init(0, C.byref(p)))
    res2, _, _ = fe.match_node_pairs([handles[1]], [handles[0]], seed=2)
    assert res2[0]["id1"] == -1 and res2[0]["id2"] == -1 and res2[0]["n_inliers"] == res[0]["n_inliers"]
    # nodes without a cloud cannot be judged
    from rgbdslam_v2_b200 import synth
    bb = synth.make_pair(5, 300)
    x, y = fe.node_from_features(7, bb["desc_newer"], bb["xyz_newer"]), fe.node_from_features(6, bb["desc_older"], bb["xyz_older"])
    with pytest.raises(B200Error):
        fe.match_node_pairs([x], [y])
    fe.close()


def test_refinement_and_emm_together_on_image_nodes(built, oracle_mod):
    """Every optional stage of matchNodePair switched on at once (g2o refinement, then the measurement model) on nodes built
    from images: the stages compose, the result stays close to the ground truth and to the plain RANSAC result."""
    from rgbdslam_v2_b200 import Frontend
    from rgbdslam_v2_b200._capi import default_params
    poses, gray, depth, mask, K4 = _frames([0, 5])
    outs = []
    for refine, emm in ((0, -0.6), (4, 0.75)):
        p = default_params(); p.depth_cov_z0 = 2.0; p.max_keypoints = 600
        p.g2o_transformation_refinement = refine; p.observability_threshold = emm
        fe = Frontend(0, p)
        det = fe.detector_create()
        handles, _ = fe.nodes_create(det, gray, depth, mask, K4, ids=np.arange(2, dtype=np.int32))
        res, allm, inl = fe.match_node_pairs([handles[1]], [handles[0]], seed=8)
        outs.append((res[0].copy(), inl[0, :res[0]["n_inliers"]].copy()))
        fe.close()
    (r0, i0), (r1, i1) = outs
    assert r0["id1"] == 0 and r1["id1"] == 0 and r1["id2"] == 1
    assert r0["all_points"] == 0 and r1["all_points"] == 2400 and r1["inlier_points"] > 0.75 * (r1["inlier_points"] + r1["outlier_points"])
    assert r1["n_inliers"] >= r0["n_inliers"] and r1["valid_iterations"] in (r0["valid_iterations"], r0["valid_iterations"] + 1)
    T_true = np.linalg.inv(poses[0]) @ poses[1]
    T0, T1 = r0["ransac_trafo"].reshape(4, 4).T, r1["ransac_trafo"].reshape(4, 4).T
    assert np.abs(T1[:3, 3] - T_true[:3, 3]).max() < 0.01 and np.abs(T1 - T0).max() < 0.01
    assert len(i1) == r1["n_inliers"]
