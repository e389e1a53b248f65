"""The environment measurement model on nodes that keep their organised cloud (RGBDSLAM_B200_KEEP_CLOUD) against the numpy
restatement (tests/emm_cloud_exact.py, `pairwise_cloud`):

- observation_likelihood: all four counts equal the restatement wherever no sample is loose, over XYZ and XYZRGB clouds,
  emm_skip_step 1 / 3 / 8, latched and per-point covariance, K4 given and all zero, odd sizes, different widths, planted
  non-finite, zero and negative points on both sides, and x / y moved away from the pixel-grid back-projection.
- match_node_pairs with the model on: exact counts under the returned transform, the gate (the realised quality rejects,
  one ulp below accepts), a rejected pair keeps every field but its ids, and the synchronous call, the pipelined _submit
  call and a batch that mixes depth-image pairs with kept-cloud pairs agree.
- a cloud back-projected in the depth path's float order gives the depth nodes' counts at cloud_creation_skip_step 1.
- KEEP_CLOUD leaves features and detector thresholds bit-identical; every rejection launches nothing.
"""
import ctypes as C

import numpy as np
import pytest

import cloud_oracle as co
import emm_cloud_exact as ec
import emm_exact as ee
import node_helpers as nh
from test_emm_cloud_exact_cpu import K_0, SCENES, plant

pytestmark = pytest.mark.gpu
LOOSE_SEEN = []


@pytest.fixture(scope="module", autouse=True)
def _report_loose():
    yield
    print(f"\nkept-cloud EMM comparisons: {len(LOOSE_SEEN)}, loose samples: {sum(LOOSE_SEEN)}")


@pytest.fixture(scope="module")
def fe(built):
    from rgbdslam_v2_b200 import Frontend
    f = Frontend(0, nh.params(0))
    yield f
    f.close()


def _assert_counts(got, exp, what):
    n_loose = int(exp["loose"].sum())
    LOOSE_SEEN.append(n_loose)
    if n_loose == 0:
        assert np.array_equal(np.asarray(got, np.int64), exp["counts"]), (what, got, exp["counts"])
    else:
        assert np.abs(np.asarray(got, np.int64) - exp["counts"]).max() <= n_loose, (what, got, exp["counts"], n_loose)


def _gray(cloud, seed):
    """a rendered visual cropped to the cloud's size (the visual only feeds the features, which the model does not read)"""
    h, w = cloud.shape[:2]
    return np.ascontiguousarray(nh.render([seed])[0][0][:h, :w])


def _kept(fe, det, cloud, K4, gray=None, seed=0):
    gray = _gray(cloud, seed) if gray is None else gray
    h, _ = fe.nodes_create(det, gray[None], np.ascontiguousarray(cloud[None]), None, None if K4 is None else np.float32(K4),
                           keep_cloud=True)
    return h[0]


def _czc(z0):
    return None if z0 is None else ee.cov_const(0.01, z0)


@pytest.mark.parametrize("scene", SCENES, ids=[s[0] for s in SCENES])
def test_observation_likelihood_is_exact(fe, scene):
    name, cn, Kn, co_, Ko, T, step, z0 = scene
    det = nh.make_detector(fe, 0, emm_skip_step=step, depth_cov_z0=-1.0 if z0 is None else z0)
    a = _kept(fe, det, cn, None if Kn == K_0 else Kn, seed=1)   # NULL K4 stands for all zero
    b = _kept(fe, det, co_, Ko, seed=2)
    rng = np.random.default_rng(len(name))
    for k, Tk in enumerate([T, ee.rigid(rng, 0.3, rng.normal(0, 0.01, 3)), ee.rigid(rng, 15.0, rng.normal(0, 0.2, 3))]):
        got = fe.observation_likelihood(a, b, Tk)
        _assert_counts(got, ec.pairwise_cloud(Tk, cn, Kn, co_, Ko, skip_step=step, czc=_czc(z0)), (name, k))
    nh.destroy(fe, [a, b])
    fe.detector_destroy(det)
    nh.reinit(fe, 0)


# ---- match_node_pairs ------------------------------------------------------------------------------------------------------

PAIR_FIELDS = ("n_all_matches", "n_inliers", "rmse", "valid_iterations", "ransac_trafo", "info_scale", "used_identity")
EMM_FIELDS = ("inlier_points", "outlier_points", "occluded_points", "all_points")
PAIRS = ((1, 0), (2, 0), (2, 1), (3, 2))


@pytest.fixture(scope="module")
def scene(fe):
    """Four rendered frames: kept-cloud nodes (XYZRGB clouds with planted special points), and depth-image nodes of the
    same frames."""
    gray, depth = nh.stack(nh.render([0, 3, 6, 9]))
    rng = np.random.default_rng(8)
    clouds = np.stack([plant(rng, co.cloud_from_depth(d, nh.K4()), 8, n_each=3) for d in depth])
    for i, c in enumerate(clouds):   # a block of each cloud pushed 30 % further along its rays: bad and occluded samples
        c[100:180, 60 + 40 * i:140 + 40 * i, :3] *= np.float32(1.3)
    det = nh.make_detector(fe, 0, observability_threshold=0.3)
    kept, _ = fe.nodes_create(det, gray, clouds, None, np.float32(nh.K4()), keep_cloud=True)
    det2 = nh.make_detector(fe, 0, observability_threshold=0.3)
    depth_nodes, _ = fe.nodes_create(det2, gray, depth, None, np.float32(nh.K4()))
    nh.reinit(fe, 0)
    yield dict(gray=gray, depth=depth, clouds=clouds, kept=kept, depth_nodes=depth_nodes)
    nh.destroy(fe, kept + depth_nodes)
    fe.detector_destroy(det)
    fe.detector_destroy(det2)


def _match(fe, nodes, pairs, thr, **kw):
    nh.reinit(fe, 0, observability_threshold=thr, **kw)
    return fe.match_node_pairs([nodes[i] for i, _ in pairs], [nodes[j] for _, j in pairs], seed=4)


def _restated(res, pairs, clouds=None, depth=None):
    out = []
    for r, (i, j) in zip(res, pairs):
        T = r["ransac_trafo"].reshape(4, 4).T
        if clouds is not None:
            out.append(ec.pairwise_cloud(T, clouds[i], nh.K4(), clouds[j], nh.K4(), czc=ee.cov_const(0.01, 2.0)))
        else:
            out.append(ee.pairwise(T, ee.cloud_z(depth[i]), nh.K4(), ee.cloud_z(depth[j]), nh.K4(), czc=ee.cov_const(0.01, 2.0)))
    return out


def _check_judged(res, base, exps, thr, what):
    judged = 0
    for k, (r, b, e) in enumerate(zip(res, base, exps)):
        if b["id1"] < 0:
            assert r.tobytes() == b.tobytes(), (what, k)
            continue
        judged += 1
        _assert_counts([r[f] for f in EMM_FIELDS], e, (what, k))
        ok = ee.criterion(e["counts"], thr)[0]
        assert (r["id1"] >= 0) == ok, (what, k)
        for f in PAIR_FIELDS:
            assert np.array_equal(r[f], b[f]), (what, k, f)
        assert (r["id1"], r["id2"]) == ((b["id1"], b["id2"]) if ok else (-1, -1)), (what, k)
    return judged


def test_match_pairs_counts_and_gate(fe, scene):
    kept, clouds = scene["kept"], scene["clouds"]
    base, _, _ = _match(fe, kept, PAIRS, -0.6)
    assert (base["id1"] >= 0).sum() >= 3, base["id1"]
    res, _, _ = _match(fe, kept, PAIRS, 0.3)
    exps = _restated(res, PAIRS, clouds=clouds)
    assert _check_judged(res, base, exps, 0.3, "thr 0.3") >= 3
    k = int(np.nonzero((base["id1"] >= 0) & (res["inlier_points"] > 0) & (res["outlier_points"] > 0))[0][0])
    g, b = int(res[k]["inlier_points"]), int(res[k]["outlier_points"])
    q = g / (g + b)
    for thr, accepted in ((q, False), (float(np.nextafter(q, 0.0)), True)):
        r2, _, _ = _match(fe, kept, PAIRS, thr)
        assert (r2[k]["id1"] >= 0) == accepted, (thr, r2[k])
        assert _check_judged(r2, base, _restated(r2, PAIRS, clouds=clouds), thr, ("gate", thr)) >= 3
    nh.reinit(fe, 0)


def test_sync_submit_and_mixed_batch_agree(fe, scene):
    kept, dn = scene["kept"], scene["depth_nodes"]
    sync, _, _ = _match(fe, kept, PAIRS, 0.3)
    out = fe._alloc_out(len(PAIRS), True)
    newer = np.array([kept[i] for i, _ in PAIRS], np.uint64)
    older = np.array([kept[j] for _, j in PAIRS], np.uint64)
    fe.submit_node_pairs(1, newer, older, out, seed=4)
    fe.wait_slot(1)
    assert out[0].tobytes() == sync.tobytes()
    # one batch: the kept-cloud pairs first, then the same frames as depth-image pairs
    l0 = fe.lib.rgbdslam_b200_launch_count()
    mixed, _, _ = fe.match_node_pairs([kept[i] for i, _ in PAIRS] + [dn[i] for i, _ in PAIRS],
                                      [kept[j] for _, j in PAIRS] + [dn[j] for _, j in PAIRS], seed=4)
    assert fe.lib.rgbdslam_b200_launch_count() > l0
    assert mixed[:len(PAIRS)].tobytes() == sync.tobytes()
    dres = mixed[len(PAIRS):]   # other RANSAC seeds at these positions: each is judged under its own transform
    for k, r in enumerate(dres):
        if r["all_points"] == 0:
            continue
        e = _restated([r], [PAIRS[k]], depth=scene["depth"])[0]
        _assert_counts([r[f] for f in EMM_FIELDS], e, ("mixed depth", k))
        assert (r["id1"] >= 0) == ee.criterion(e["counts"], 0.3)[0], k
    assert (dres["all_points"] > 0).sum() >= 2, dres["all_points"]
    nh.reinit(fe, 0)


def test_depth_order_cloud_equals_depth_nodes(fe, scene):
    """A cloud built in the depth path's float order ((u - cx) * z * float(1 / fx)) at cloud_creation_skip_step 1, minimum
    depth below every depth and scaling 1 gives the depth nodes' counts."""
    gray, depth = scene["gray"], scene["depth"]
    K = nh.K4()
    f32 = np.float32
    fxinv, fyinv = f32(1.0 / np.float64(f32(K[0]))), f32(1.0 / np.float64(f32(K[1])))
    det = nh.make_detector(fe, 0, cloud_creation_skip_step=1, minimum_depth=-1.0, depth_scaling_factor=1.0)
    kept, dnodes = [], []
    for i in (0, 1):
        z = depth[i].astype(f32)
        v, u = np.mgrid[0:z.shape[0], 0:z.shape[1]].astype(f32)
        c = np.zeros(z.shape + (4,), f32)
        c[..., 0] = ((u - f32(K[2])) * z) * fxinv
        c[..., 1] = ((v - f32(K[3])) * z) * fyinv
        c[..., 2] = z
        kept.append(_kept(fe, det, c, K, gray=gray[i]))
        from rgbdslam_v2_b200 import synth
        b = synth.make_pair(i + 1, 40)
        dnodes.append(fe.node_from_features(i, b["desc_newer"], b["xyz_newer"]))
        fe.node_set_depth(dnodes[-1], depth[i], K)
    rng = np.random.default_rng(9)
    for Tk in [np.eye(4, dtype=np.float32)] + [ee.rigid(rng, 1.0, rng.normal(0, 0.03, 3)) for _ in range(4)]:
        for skip in (8, 3):
            nh.reinit(fe, 0, cloud_creation_skip_step=1, minimum_depth=-1.0, emm_skip_step=skip)
            got = fe.observation_likelihood(kept[1], kept[0], Tk)
            assert np.array_equal(got, fe.observation_likelihood(dnodes[1], dnodes[0], Tk)), (skip, got)
            assert got[:3].sum() > 0
    nh.destroy(fe, kept + dnodes)
    fe.detector_destroy(det)
    nh.reinit(fe, 0)


def test_keep_cloud_leaves_features_and_thresholds(fe, scene):
    gray, clouds = scene["gray"], scene["clouds"]
    d1, d2 = nh.make_detector(fe, 0), fe.detector_create()
    a, na = fe.nodes_create(d1, gray, clouds, None, np.float32(nh.K4()))
    b, nb = fe.nodes_create(d2, gray, clouds, None, np.float32(nh.K4()), keep_cloud=True)
    assert np.array_equal(na, nb) and nh.same_nodes(nh.node_dump(fe, a), nh.node_dump(fe, b))
    assert np.array_equal(fe.detector_thresholds(d1), fe.detector_thresholds(d2))
    nh.destroy(fe, a + b)
    fe.detector_destroy(d1)
    fe.detector_destroy(d2)


def test_rejections_launch_nothing(fe, scene):
    from rgbdslam_v2_b200._capi import B200Error, CLOUD_XYZRGB, KEEP_CLOUD, _ptr
    gray, depth, clouds, kept, dn = scene["gray"], scene["depth"], scene["clouds"], scene["kept"], scene["depth_nodes"]
    H, W = gray.shape[1:]
    K4 = np.float32(nh.K4())
    handles = np.zeros(1, np.uint64)
    nf = np.zeros(1, np.int32)
    cloud = np.ascontiguousarray(clouds[:1])
    det = nh.make_detector(fe, 0)

    def expect(rc_want, word, fn):
        l0 = fe.lib.rgbdslam_b200_launch_count()
        rc = fn()
        assert fe.lib.rgbdslam_b200_launch_count() == l0
        assert rc == rc_want and word in fe.lib.rgbdslam_b200_last_error(), (rc, fe.lib.rgbdslam_b200_last_error())

    g1 = np.ascontiguousarray(gray[:1])
    expect(1, b"KEEP_CLOUD", lambda: fe.lib.rgbdslam_b200_nodes_create_ex(det, 1, _ptr(g1), _ptr(np.ascontiguousarray(depth[:1])), None,
                                                                           W, H, _ptr(K4), None, KEEP_CLOUD, _ptr(handles), _ptr(nf)))
    # the flag is refused before the communicator is looked at
    expect(1, b"KEEP_CLOUD", lambda: fe.lib.rgbdslam_b200_nodes_create_sharded(det, C.c_uint64(0), 1, _ptr(g1), _ptr(cloud), None, W, H,
                                                                                _ptr(K4), None, CLOUD_XYZRGB | KEEP_CLOUD, _ptr(handles),
                                                                                _ptr(nf)))
    nh.reinit(fe, 0, observability_threshold=0.3)
    expect(3, b"measurement model", lambda: fe.lib.rgbdslam_b200_nodes_create_ex(det, 1, _ptr(g1), _ptr(cloud), None, W, H, _ptr(K4),
                                                                                  None, CLOUD_XYZRGB, _ptr(handles), _ptr(nf)))
    for newer, older in (([kept[1]], [dn[0]]), ([dn[1], kept[1]], [dn[0], dn[0]])):   # the second pair of the batch mixes
        a, b = np.array(newer, np.uint64), np.array(older, np.uint64)
        res, allm, inl = fe._alloc_out(len(a), True)
        expect(3, b"KEEP_CLOUD", lambda: fe.lib.rgbdslam_b200_match_pairs(_ptr(a), _ptr(b), len(a), 4, 0, _ptr(res), _ptr(allm), _ptr(inl)))
    T = np.ascontiguousarray(np.eye(4, dtype=np.float32))
    counts = np.zeros(4, np.uint32)
    expect(3, b"KEEP_CLOUD", lambda: fe.lib.rgbdslam_b200_observation_likelihood(C.c_uint64(kept[1]), C.c_uint64(dn[0]), _ptr(T),
                                                                                  _ptr(counts)))
    with pytest.raises(B200Error, match="KEEP_CLOUD"):
        fe.node_set_depth(kept[0], depth[0], nh.K4())
    fe.detector_destroy(det)
    nh.reinit(fe, 0)
