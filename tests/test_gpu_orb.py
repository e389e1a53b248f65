"""GPU parity tests of the Node-constructor path (ORB detect / compute / back-projection) against OpenCV itself
(cv2) + the reference's glue restated in oracle/orb_oracle.py."""
import numpy as np
import pytest

import node_helpers as nh

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def fe(built):
    from rgbdslam_v2_b200 import Frontend
    from rgbdslam_v2_b200._capi import default_params
    p = default_params()
    p.depth_cov_z0 = 2.0
    p.max_keypoints = 600
    f = Frontend(0, p)
    yield f
    f.close()


@pytest.fixture(scope="module")
def frames():
    return nh.render((0, 1, 2, 9), 40)


def _canon(kp):
    return np.sort(kp, order=["octave", "y", "x"])


def test_orb_compute_bit_exact_vs_cv2(fe, frames):
    """extractor->compute(): identical keypoint filtering/ordering and bit-identical 256-bit descriptors."""
    import cv2
    from oracle import orb_oracle
    for gray, _ in frames[:2]:
        det = cv2.ORB_create(10000, 1.2, 8, 15, 0, 2, 0, 31, 20)
        kps = det.detect(gray, None)
        rng = np.random.default_rng(0)
        sel = rng.permutation(len(kps))[:1500]  # unordered input incl. all octaves and border cases
        arr = np.zeros(len(sel), orb_oracle.KP_DTYPE)
        for i, j in enumerate(sel):
            k = kps[j]
            arr[i] = (k.pt[0], k.pt[1], k.size, k.angle, k.response, k.octave, -1)
        okp, odesc = orb_oracle.orb_compute(gray, arr)
        gkp, gdesc = fe.orb_compute(gray, arr)
        assert len(gkp) == len(okp) and len(okp) > 1000
        assert gkp.tobytes() == okp.tobytes()
        assert np.array_equal(gdesc, odesc)
        assert set(np.unique(gkp["octave"])) == set(range(8))


def test_orb_compute_edge_cases(fe, frames):
    from oracle import orb_oracle
    gray = frames[0][0]
    arr = np.zeros(8, orb_oracle.KP_DTYPE)
    xs = [30.4, 30.5, 30.6, 608.4, 608.5, 608.6, 320.0, 320.0]
    ys = [100.0] * 6 + [30.5, 448.5]
    for i in range(8):
        arr[i] = (xs[i], ys[i], 31.0, 33.0 * i, 1.0, i % 8, -1)
    okp, odesc = orb_oracle.orb_compute(gray, arr)
    gkp, gdesc = fe.orb_compute(gray, arr)
    assert gkp.tobytes() == okp.tobytes() and np.array_equal(gdesc, odesc)
    e, d = fe.orb_compute(gray, arr[:0])
    assert len(e) == 0


def test_grid_detect_vs_cv2_over_a_sequence(fe, frames):
    """detector->detect() incl. the per-cell adaptive thresholds carried across frames."""
    from oracle import orb_oracle
    from rgbdslam_v2_b200._capi import B200Error
    nh.reinit(fe, max_keypoints=600)
    det = fe.detector_create()
    st = orb_oracle.DetectorState()
    for gray, depth in frames:
        mask = orb_oracle.depth_to_mask(depth)
        orec = orb_oracle.grid_detect(gray, mask, st, max_keypoints=600)
        okp = orb_oracle.records_to_array(orec)
        gkp = fe.orb_detect(det, gray, mask)
        assert len(gkp) == len(okp) and len(okp) > 300
        assert _canon(gkp).tobytes() == _canon(okp).tobytes()  # same set, every field bit-exact
        assert gkp.tobytes() == okp.tobytes()                  # and the documented canonical order
        assert np.allclose(fe.detector_thresholds(det)[:9], st.thresh[:9], rtol=0, atol=0)
    with pytest.raises(B200Error, match="score map"):  # scores stay on chip: there is no plane 2
        fe.orb_debug_plane(2, 0, 0)
    fe.detector_destroy(det)


def test_nodes_create_vs_oracle(fe, frames, oracle_mod):
    """Full Node constructor (node.cpp:101-240) for a batch of frames processed in order."""
    from oracle import orb_oracle
    nh.reinit(fe, max_keypoints=600)
    det = fe.detector_create()
    st = orb_oracle.DetectorState()
    gray = np.stack([f[0] for f in frames]); depth = np.stack([f[1] for f in frames])
    mask = np.stack([orb_oracle.depth_to_mask(f[1]) for f in frames])
    K4 = nh.K4()
    handles, nf = fe.nodes_create(det, gray, depth, mask, K4, ids=[10, 11, 12, 13])
    for i, h in enumerate(handles):
        okp, odesc, oxyz = orb_oracle.node_construct(frames[i][0], frames[i][1], mask[i], K4, st, max_keypoints=600)
        gkp = fe.node_keypoints(h)
        gdesc, gxyz = fe.node_download(h)
        assert nf[i] == len(okp) and 300 < len(okp) <= 600
        assert gkp.tobytes() == okp.tobytes()
        assert np.array_equal(gdesc, odesc)
        assert np.array_equal(gxyz, oxyz)
        assert not np.isnan(gxyz).any()
    # nodes built from images feed the matcher like nodes built from features
    res, allm, inl = fe.match_node_pairs([handles[1]], [handles[0]], seed=3)
    assert res[0]["id1"] == 10 and res[0]["id2"] == 11 and res[0]["n_inliers"] > 50
    fe.detector_destroy(det)


def test_no_mask_and_other_parameters(fe, frames):
    from oracle import orb_oracle
    nh.reinit(fe, max_keypoints=1000)
    det = fe.detector_create()
    st = orb_oracle.DetectorState()
    gray = frames[3][0]
    orec = orb_oracle.grid_detect(gray, None, st, max_keypoints=1000)
    gkp = fe.orb_detect(det, gray, None)
    assert gkp.tobytes() == orb_oracle.records_to_array(orec).tobytes()
    # a textureless frame: thresholds decay (x0.7, clamped at 2) exactly like the reference's adjuster
    flat = np.full_like(gray, 128)
    orec = orb_oracle.grid_detect(flat, None, st, max_keypoints=1000)
    gkp = fe.orb_detect(det, flat, None)
    assert len(gkp) == len(orec) == 0
    assert np.array_equal(fe.detector_thresholds(det)[:9], np.array(st.thresh[:9]))
    fe.detector_destroy(det)
    nh.reinit(fe, max_keypoints=600)


@pytest.fixture(scope="module")
def seq40():
    return nh.seq(40)


def test_nodes_create_pipeline_variants_identical(fe, seq40):
    """The chunked, double-buffered constructor (40 frames = 2 chunks) gives bit-identical nodes and detector thresholds
    (a) frame by frame, (b) from pinned host memory, (c) with the mask derived from depth on the device."""
    import torch
    gray, depth, mask = seq40
    K4 = nh.K4()
    nh.reinit(fe, max_keypoints=600)

    def run(fn):
        det = fe.detector_create()
        out = fn(det)
        thr = fe.detector_thresholds(det).copy()
        fe.detector_destroy(det)
        dump = nh.node_dump(fe, out)
        for h in out:
            fe.node_destroy(h)
        return dump, thr

    ref, thr_ref = run(lambda det: fe.nodes_create(det, gray, depth, mask, K4)[0])
    assert len(ref) == 40 and min(len(k) for k, _, _ in ref) > 300

    def one_by_one(det):
        hs = []
        for k in range(40):
            hs += fe.nodes_create(det, gray[k:k + 1], depth[k:k + 1], mask[k:k + 1], K4, ids=[k])[0]
        return hs
    a, thr_a = run(one_by_one)
    assert nh.same_nodes(ref, a) and np.array_equal(thr_ref, thr_a)

    pg, pd, pm = (torch.from_numpy(x).pin_memory() for x in (gray, depth, mask))
    b, thr_b = run(lambda det: fe.nodes_create(det, pg, pd, pm, K4)[0])
    assert nh.same_nodes(ref, b) and np.array_equal(thr_ref, thr_b)

    c, thr_c = run(lambda det: fe.nodes_create(det, gray, depth, None, K4, mask_from_depth=True)[0])
    assert nh.same_nodes(ref, c) and np.array_equal(thr_ref, thr_c)


def test_nodes_create_without_mask_and_small_batches(fe, seq40):
    """mask = NULL (no mask pyramid at all) equals an all-255 mask; nodes of one call share a slab and survive the others"""
    gray, depth, _ = seq40
    K4 = nh.K4()
    nh.reinit(fe, max_keypoints=600)
    det = fe.detector_create()
    h1, _ = fe.nodes_create(det, gray[:3], depth[:3], None, K4)
    fe.detector_destroy(det)
    det = fe.detector_create()
    h2, _ = fe.nodes_create(det, gray[:3], depth[:3], np.full_like(gray[:3], 255), K4)
    fe.detector_destroy(det)
    a, b = nh.node_dump(fe, h1), nh.node_dump(fe, h2)
    assert nh.same_nodes(a, b)
    fe.node_destroy(h1[0]); fe.node_destroy(h1[2])  # the slab stays alive for the remaining node
    k, d, x = fe.node_keypoints(h1[1]), *fe.node_download(h1[1])
    assert np.array_equal(k, b[1][0]) and np.array_equal(d, b[1][1])
    for h in [h1[1]] + h2:
        fe.node_destroy(h)


def test_nodes_create_sharded_single_rank_equals_plain(fe, seq40):
    """The two-pass frame-sharded constructor (histogram exchange, threshold replay over the whole sequence, feature
    all-gather) on a 1-rank NCCL communicator == the plain constructor: nodes and final detector thresholds."""
    gray, depth, mask = seq40
    K4 = nh.K4()
    nh.reinit(fe, max_keypoints=600)
    det = fe.detector_create()
    h1, n1 = fe.nodes_create(det, gray, depth, mask, K4)
    thr1 = fe.detector_thresholds(det).copy()
    fe.detector_destroy(det)
    comm = fe.comm_init(0, 1, fe.comm_unique_id())
    det = fe.detector_create()
    h2, n2 = fe.nodes_create_sharded(det, comm, 40, gray, depth, mask, K4)
    thr2 = fe.detector_thresholds(det).copy()
    fe.detector_destroy(det)
    assert np.array_equal(n1, n2) and np.array_equal(thr1, thr2)
    assert nh.same_nodes(nh.node_dump(fe, h1), nh.node_dump(fe, h2))
    # matching works on the gathered nodes
    res, _, _ = fe.match_node_pairs(h2[1:6], h2[0:5], seed=3, want_matches=False)
    ref, _, _ = fe.match_node_pairs(h1[1:6], h1[0:5], seed=3, want_matches=False)
    assert np.array_equal(res["n_inliers"], ref["n_inliers"]) and np.array_equal(res["ransac_trafo"], ref["ransac_trafo"])
    fe.comm_destroy(comm)
    for h in h1 + h2:
        fe.node_destroy(h)
