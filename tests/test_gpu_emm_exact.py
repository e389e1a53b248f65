"""Exact gates on the environment measurement model (csrc/emm.cu) against the numpy restatement (tests/emm_exact.py).

- observation_likelihood: all four counts equal the restatement wherever no sample is loose (p within 1e-12 of a cut), on
  rendered frames and on synthetic depth maps given to node_set_depth: block scenes with good, bad and occluded samples,
  different intrinsics and frame sizes for the two nodes (sizes that are not a multiple of the steps), other cloud and EMM
  steps, depth scaling and minimum depth, constant, latched and per-point covariance, transforms that put points behind the
  camera or off the raster.
- match_node_pairs: on a batch mixing accepted, RANSAC-rejected and refined pairs, each judged pair's counts equal the
  restatement under its returned transform, and the gate is exact: a threshold equal to the realised quality rejects (strict
  >), one ulp below accepts; a certainty of exactly 0.25 rejects; an all-occluded pair (NaN quality) rejects; a rejected pair
  keeps every field but the ids.
"""
import ctypes as C

import numpy as np
import pytest

import emm_exact as ee

pytestmark = pytest.mark.gpu

K_A = (525.0, 525.0, 319.5, 239.5)
K_B = (481.2, 479.7, 305.25, 251.5)
K_C = (300.0, 301.0, 166.0, 124.5)
LOOSE_SEEN = []


@pytest.fixture(scope="module", autouse=True)
def _report_loose():
    yield
    print(f"\nEMM comparisons: {len(LOOSE_SEEN)}, loose samples: {sum(LOOSE_SEEN)}")


@pytest.fixture(scope="module")
def fe(built):
    from rgbdslam_v2_b200 import Frontend
    from rgbdslam_v2_b200._capi import default_params
    p = default_params()
    p.depth_cov_z0 = 2.0
    f = Frontend(0, p)
    yield f
    f.close()


def _reinit(fe, **kw):
    from rgbdslam_v2_b200._capi import default_params
    p = default_params()
    p.depth_cov_z0 = 2.0
    for k, v in kw.items():
        setattr(p, k, v)
    fe.params = p
    fe._check(fe.lib.rgbdslam_b200_init(0, C.byref(p)))
    return p


def _czc(fe):
    return None if fe.params.depth_cov_z0 < 0 else ee.cov_const(fe.params.sigma_depth, fe.depth_cov_z0)


def _assert_counts(got, exp, what):
    """all four counts equal unless a sample is loose (then the pair is counted and skipped)"""
    n_loose = int(exp["loose"].sum())
    LOOSE_SEEN.append(n_loose)
    if n_loose == 0:
        assert np.array_equal(np.asarray(got, np.int64), exp["counts"]), (what, got, exp["counts"])
    else:
        assert np.abs(np.asarray(got, np.int64) - exp["counts"]).max() <= n_loose, (what, got, exp["counts"], n_loose)


def _feature_node(fe, node_id, n=40):
    from rgbdslam_v2_b200 import synth
    b = synth.make_pair(node_id + 1, n)
    return fe.node_from_features(node_id, b["desc_newer"], b["xyz_newer"])


def _observe(fe, dn, Kn, do, Ko, transforms, what):
    p = fe.params
    a, b = _feature_node(fe, 1), _feature_node(fe, 0)
    fe.node_set_depth(a, dn, Kn)
    fe.node_set_depth(b, do, Ko)
    step, scale, md = p.cloud_creation_skip_step, p.depth_scaling_factor, p.minimum_depth
    zn, zo = ee.cloud_z(dn, step, scale, md), ee.cloud_z(do, step, scale, md)
    seen = np.zeros(3, np.int64)
    for k, T in enumerate(transforms):
        T = np.asarray(T, np.float32)
        got = fe.observation_likelihood(a, b, T)
        exp = ee.pairwise(T, zn, Kn, zo, Ko, cloud_step=step, skip_step=p.emm_skip_step, sigma_depth=p.sigma_depth,
                          czc=_czc(fe))
        _assert_counts(got, exp, (what, k))
        seen += exp["counts"][:3]
    return seen


def _frames(ks):
    from rgbdslam_v2_b200 import synth
    poses = synth.trajectory(240)
    return [poses[k] for k in ks], [synth.render_frame(poses[k], seed=k)[1] for k in ks]


def test_rendered_frames(fe):
    _reinit(fe)
    poses, depth = _frames([0, 30])
    T = (np.linalg.inv(poses[0]) @ poses[1]).astype(np.float32)
    rng = np.random.default_rng(2)
    Ts = []
    for dz in (0.0, 0.01, 0.05, 0.3, -0.6):
        Tb = T.copy()
        Tb[2, 3] += dz
        Ts.append(Tb)
    Ts += [(T.astype(np.float64) @ ee.rigid(rng, 0.3, rng.normal(0, 0.002, 3))).astype(np.float32) for _ in range(8)]
    seen = _observe(fe, depth[1], K_A, depth[0], K_A, Ts, "rendered")
    assert seen.min() > 0, seen


def _block_pair(seed, shape_n, Kn, shape_o, Ko):
    rng = np.random.default_rng(seed)
    return ee.block_scene(rng, *shape_n, Kn), ee.block_scene(rng, *shape_o, Ko)


TRANSFORMS = {
    "small": lambda rng: [ee.rigid(rng, 1.0, rng.normal(0, 0.02, 3)) for _ in range(4)],
    "big": lambda rng: [ee.rigid(rng, 20.0, rng.normal(0, 0.3, 3))],
    "behind": lambda rng: [np.array([[-1, 0, 0, 0.1], [0, 1, 0, 0], [0, 0, -1, 1.5], [0, 0, 0, 1]], np.float32)],
    "off-raster": lambda rng: [ee.rigid(rng, 0.5, [2.5, 0.0, 0.0]), ee.rigid(rng, 0.5, [0.0, -1.8, 0.2])],
}

# (name, params, newer (w, h), newer K, older (w, h), older K, depth multiplier)
CONFIGS = [
    ("defaults", dict(), (640, 480), K_A, (640, 480), K_A, 1.0),
    ("other-K-size", dict(), (640, 480), K_A, (517, 389), K_B, 1.0),
    ("other-K-size-rev", dict(), (333, 250), K_C, (640, 480), K_A, 1.0),
    ("steps-3-5", dict(cloud_creation_skip_step=3, emm_skip_step=5), (517, 389), K_B, (640, 480), K_A, 1.0),
    ("steps-1-7", dict(cloud_creation_skip_step=1, emm_skip_step=7), (333, 250), K_C, (517, 389), K_B, 1.0),
    ("steps-4-3", dict(cloud_creation_skip_step=4, emm_skip_step=3), (640, 480), K_A, (333, 250), K_C, 1.0),
    ("scaling-mm", dict(depth_scaling_factor=0.001), (640, 480), K_A, (517, 389), K_B, 1000.0),
    ("scaling-1.03", dict(depth_scaling_factor=1.03), (517, 389), K_B, (517, 389), K_B, 1.0),
    ("min-depth-1.7", dict(minimum_depth=1.7), (640, 480), K_A, (517, 389), K_B, 1.0),
    ("per-point", dict(depth_cov_z0=-1.0), (640, 480), K_A, (517, 389), K_B, 1.0),
    ("per-point-steps-3-5", dict(depth_cov_z0=-1.0, cloud_creation_skip_step=3, emm_skip_step=5), (333, 250), K_C,
     (640, 480), K_A, 1.0),
    ("z0-0.7", dict(depth_cov_z0=0.7), (640, 480), K_A, (517, 389), K_B, 1.0),
]


@pytest.mark.parametrize("cfg", CONFIGS, ids=[c[0] for c in CONFIGS])
def test_synthetic_depth_maps(fe, cfg):
    name, params, sn, Kn, so, Ko, mult = cfg
    _reinit(fe, **params)
    dn, do = _block_pair(sum(map(ord, name)), sn, Kn, so, Ko)
    rng = np.random.default_rng(len(name))
    seen = np.zeros(3, np.int64)
    for tname, gen in TRANSFORMS.items():
        s = _observe(fe, (dn * mult).astype(np.float32), Kn, (do * mult).astype(np.float32), Ko, gen(rng), (name, tname))
        if tname == "small":
            assert s.min() > 0, (name, s)   # good, bad and occluded samples all occur
        seen += s
    _reinit(fe)


def test_latched_covariance(fe):
    """depth_cov_z0 = 0: the first match_pairs call latches z0 from its first usable correspondence; the model then uses
    that constant."""
    from rgbdslam_v2_b200 import synth
    _reinit(fe, depth_cov_z0=0.0)
    b = synth.make_pair(3, 300)
    x, y = fe.node_from_features(1, b["desc_newer"], b["xyz_newer"]), fe.node_from_features(0, b["desc_older"], b["xyz_older"])
    fe.match_node_pairs([x], [y], seed=1)
    z0 = fe.depth_cov_z0
    assert z0 > 0 and z0 != 2.0
    dn, do = _block_pair(77, (640, 480), K_A, (517, 389), K_B)
    rng = np.random.default_rng(77)
    seen = _observe(fe, dn, K_A, do, K_B, TRANSFORMS["small"](rng) + TRANSFORMS["big"](rng), "latched")
    assert seen.min() > 0
    _reinit(fe)


# ---- the gate in match_node_pairs -----------------------------------------------------------------------------------------

W, H = 640, 480


def _gate_depths(layout):
    """Depth maps (newer, older) built from one kind per 8 x 8 block of raster cells (16 x 16 pixels at cloud step 2), each
    block centred on one EMM sample, under a transform close to the identity:
      'good'  both 2.0 m                         -> a good sample in each direction
      'diff'  newer 3.0 m, older 2.0 m           -> occluded newer -> older, bad older -> newer
      'nan'   no depth                           -> counted in all_points only
      'occ'   newer 3.0 m, older 2.0 m but no depth on the sampled cell of the older node -> one occluded sample only"""
    dn = np.zeros((H, W), np.float32)
    do = np.zeros((H, W), np.float32)
    for (j, i), kind in np.ndenumerate(layout):
        ys, xs = slice(max(0, 16 * j - 8), 16 * j + 8), slice(max(0, 16 * i - 8), 16 * i + 8)
        if kind == "good":
            dn[ys, xs] = do[ys, xs] = 2.0
        elif kind in ("diff", "occ"):
            dn[ys, xs], do[ys, xs] = 3.0, 2.0
            if kind == "occ":
                do[16 * j, 16 * i] = 0.0
    return dn, do


def _layout(rng, counts):
    kinds = np.array(sum(([k] * n for k, n in counts.items()), []), object)
    assert len(kinds) <= 1200
    kinds = np.concatenate([kinds, np.array(["nan"] * (1200 - len(kinds)), object)])
    return rng.permutation(kinds).reshape(30, 40)


def _feature_pair(fe, rng, ids, T=None, M=150, scramble=False):
    """Two feature nodes whose M correspondences agree with T (newer -> older; identity by default), with 2-D keypoints for
    the refinement.  scramble: the older points are shuffled, so RANSAC finds no transformation."""
    from rgbdslam_v2_b200 import synth
    from rgbdslam_v2_b200._capi import KEYPOINT_DTYPE
    T = np.eye(4) if T is None else T
    p = np.stack([rng.uniform(-1.0, 1.0, M), rng.uniform(-0.7, 0.7, M), rng.uniform(1.2, 3.5, M)], 1)
    q = p @ T[:3, :3].T + T[:3, 3]
    if scramble:
        q = q[rng.permutation(M)] + rng.normal(0, 0.3, (M, 3))
    desc_e = rng.integers(0, 256, (M + 1, 32), dtype=np.uint8)
    desc_n = desc_e[:M].copy()
    for i in range(M):
        for bit in rng.permutation(256)[:3]:
            desc_n[i, bit // 8] ^= 1 << (bit % 8)
    xyz_n = np.c_[p, np.ones(M)].astype(np.float32)
    xyz_e = np.r_[np.c_[q, np.ones(M)], [[0, 0, 1, 1]]].astype(np.float32)
    K = synth._KREF
    kp = lambda x: (x[:, :2] / x[:, 2:3]) * [K[0, 0], K[1, 1]] + [K[0, 2], K[1, 2]]
    a = fe.node_from_features(ids[0], desc_n, xyz_n)
    b = fe.node_from_features(ids[1], desc_e, xyz_e)
    ka = np.zeros(M, KEYPOINT_DTYPE)
    ka["x"], ka["y"] = kp(xyz_n[:, :3].astype(np.float64)).T
    kb = np.zeros(M + 1, KEYPOINT_DTYPE)
    kb["x"], kb["y"] = kp(xyz_e[:, :3].astype(np.float64)).T
    fe.node_set_keypoints(a, ka)
    fe.node_set_keypoints(b, kb)
    return a, b


def _gate_batch(fe):
    """Pairs: 0 quality 0.75 / certainty 0.6, 1 certainty exactly 0.25, 2 certainty just above 0.25, 3 all occluded,
    4 RANSAC-rejected, 5-6 rendered frames under a real motion, 7 two cameras with different intrinsics and sizes."""
    poses, depth = _frames([0, 4, 8])
    rng = np.random.default_rng(12)
    scenes = [_layout(rng, dict(good=300, diff=200)), _layout(rng, dict(good=100, diff=300)),
              _layout(rng, dict(good=100, diff=299)), _layout(rng, dict(occ=1200)), _layout(rng, dict(good=600))]
    pairs, zs = [], []
    for k, lay in enumerate(scenes):
        a, b = _feature_pair(fe, rng, (2 * k + 1, 2 * k), scramble=(k == 4))
        dn, do = _gate_depths(lay)
        fe.node_set_depth(a, dn, K_A)
        fe.node_set_depth(b, do, K_A)
        pairs.append((a, b))
        zs.append((ee.cloud_z(dn), ee.cloud_z(do)))
    for k, (i, j) in enumerate(((1, 0), (2, 0))):
        T = np.linalg.inv(poses[j]) @ poses[i]
        a, b = _feature_pair(fe, rng, (20 + 2 * k + 1, 20 + 2 * k), T=T, M=200)
        fe.node_set_depth(a, depth[i], K_A)
        fe.node_set_depth(b, depth[j], K_A)
        pairs.append((a, b))
        zs.append((ee.cloud_z(depth[i]), ee.cloud_z(depth[j])))
    # 7: block scenes on two cameras with different intrinsics and frame sizes
    dn, do = _block_pair(71, (640, 480), K_A, (517, 389), K_B)
    a, b = _feature_pair(fe, rng, (41, 40), T=ee.rigid(rng, 1.0, [0.02, -0.01, 0.03]).astype(np.float64))
    fe.node_set_depth(a, dn, K_A)
    fe.node_set_depth(b, do, K_B)
    pairs.append((a, b))
    zs.append((ee.cloud_z(dn), ee.cloud_z(do)))
    return pairs, zs


def _run_gate(fe, pairs, thr, refine):
    _reinit(fe, observability_threshold=thr, g2o_transformation_refinement=refine)
    res, allm, inl = fe.match_node_pairs([a for a, _ in pairs], [b for _, b in pairs], seed=4)
    return res, allm, inl


EMM_FIELDS = ("inlier_points", "outlier_points", "occluded_points", "all_points")


def test_gate_is_exact(fe):
    pairs, zs = _gate_batch(fe)
    for refine in (0, 3):
        base, ballm, binl = _run_gate(fe, pairs, -0.6, refine)        # the model off: RANSAC (+ refinement) alone
        assert (base["id1"][:4] >= 0).all() and base["id1"][4] < 0 and (base["id1"][5:] >= 0).all(), base["id1"]
        res, allm, inl = _run_gate(fe, pairs, 0.3, refine)
        exp = []
        for i, (r, (zn, zo)) in enumerate(zip(res, zs)):
            got = np.array([r[f] for f in EMM_FIELDS])
            if base[i]["id1"] < 0:                                       # not judged: bytes as without the model
                assert r.tobytes() == base[i].tobytes(), i
                exp.append(None)
                continue
            Kn, Ko = (K_A, K_B) if i == 7 else (K_A, K_A)
            e = ee.pairwise(r["ransac_trafo"].reshape(4, 4).T, zn, Kn, zo, Ko, czc=ee.cov_const(0.01, 2.0))
            _assert_counts(got, e, ("gate", refine, i))
            exp.append(e["counts"])
            ok, q, c = ee.criterion(e["counts"], 0.3)
            assert (r["id1"] >= 0) == ok, (i, q, c)
            # every field but the ids (and the model's own counts) is the RANSAC result
            for f in PAIR_FIELDS:
                assert np.array_equal(r[f], base[i][f]), (i, f)
            assert (r["id1"], r["id2"]) == ((base[i]["id1"], base[i]["id2"]) if ok else (-1, -1)), i
            if i < 4:
                assert np.abs(r["ransac_trafo"].reshape(4, 4) - np.eye(4)).max() < 1e-4
            assert np.array_equal(inl[i, :r["n_inliers"]], binl[i, :r["n_inliers"]]), i
        assert list(exp[0]) == [600, 200, 200, 2400] and list(exp[1]) == [200, 300, 300, 2400], exp[:2]
        assert list(exp[2]) == [200, 299, 299, 2400] and list(exp[3]) == [0, 0, 1200, 2400], exp[2:4]
        assert res["id1"][1] < 0 and ee.criterion(exp[1], 0.3)[2] == 0.25          # certainty exactly 0.25: rejected
        assert res["id1"][2] >= 0                                                  # just above: accepted
        assert res["id1"][3] < 0 and np.isnan(ee.criterion(exp[3], 0.3)[1])        # all occluded, NaN quality: rejected
        assert (res["id1"][[0, 5, 6]] >= 0).all() and min(exp[7][:3]) > 0, exp[7]
        # the strict > on quality: the realised quality itself rejects, one ulp below accepts
        q = 600 / 800
        for thr, accepted in ((q, False), (np.nextafter(q, 0.0), True)):
            r2, _, _ = _run_gate(fe, pairs[:1], float(thr), refine)
            assert (r2[0]["id1"] >= 0) == accepted, (thr, r2[0])
            assert np.array_equal([r2[0][f] for f in EMM_FIELDS], exp[0])
    _reinit(fe)


PAIR_FIELDS = ("n_all_matches", "n_inliers", "rmse", "valid_iterations", "ransac_trafo", "info_scale", "used_identity")

