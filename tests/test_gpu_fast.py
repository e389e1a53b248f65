"""GPU parity tests of the FAST detector (params.feature_detector_type = FAST) in the Node-constructor path against
OpenCV itself (cv2.FastFeatureDetector) + the reference's glue restated in tests/fast_oracle.py."""
import ctypes as C

import numpy as np
import pytest

import node_helpers as nh

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def fe(built):
    from rgbdslam_v2_b200 import Frontend
    from rgbdslam_v2_b200._capi import DETECTOR_FAST
    f = Frontend(0, nh.params(DETECTOR_FAST))
    yield f
    f.close()


@pytest.fixture(scope="module")
def frames():
    return nh.render((0, 1, 2, 9), 40)


@pytest.fixture(scope="module")
def seq40():
    return nh.seq(40)


def test_fast_detect_vs_cv2_over_a_sequence(fe, frames):
    """detector->detect() with the FAST detector: keypoints bit-identical to cv2 + the grid / adjuster glue, in the
    documented order, and the per-cell thresholds equal after every frame."""
    import fast_oracle
    from oracle import orb_oracle
    from rgbdslam_v2_b200._capi import DETECTOR_FAST
    det = nh.make_detector(fe, DETECTOR_FAST)
    st = orb_oracle.DetectorState()
    for gray, depth in frames:
        mask = orb_oracle.depth_to_mask(depth)
        okp = orb_oracle.records_to_array(fast_oracle.grid_detect(gray, mask, st, max_keypoints=600))
        gkp = fe.orb_detect(det, gray, mask)
        assert len(gkp) == len(okp) and len(okp) > 300
        assert gkp.tobytes() == okp.tobytes()
        assert (gkp["size"] == 7).all() and (gkp["angle"] == -1).all() and (gkp["octave"] == 0).all()
        assert np.array_equal(fe.detector_thresholds(det)[:9], np.array(st.thresh[:9]))
    # the inspection hook reports the corner score as the response of the candidates that pass the final threshold
    cand, resp, thr = fe.orb_debug_candidates(0)
    ok = ~np.isnan(resp)
    assert ok.any() and np.array_equal(resp[ok], cand["score"][ok].astype(np.float32)) and (cand["score"][ok] >= thr).all()
    assert (cand["level"] == 0).all()
    fe.detector_destroy(det)


def test_fast_textureless_frame_and_no_mask(fe, frames):
    """No mask; then a textureless frame: thresholds decay (x0.7, clamped at 2) exactly like the reference's adjuster."""
    import fast_oracle
    from oracle import orb_oracle
    from rgbdslam_v2_b200._capi import DETECTOR_FAST
    det = nh.make_detector(fe, DETECTOR_FAST, max_keypoints=1000)
    st = orb_oracle.DetectorState()
    gray = frames[3][0]
    orec = fast_oracle.grid_detect(gray, None, st, max_keypoints=1000)
    assert fe.orb_detect(det, gray, None).tobytes() == orb_oracle.records_to_array(orec).tobytes()
    flat = np.full_like(gray, 128)
    for _ in range(2):
        orec = fast_oracle.grid_detect(flat, None, st, max_keypoints=1000)
        gkp = fe.orb_detect(det, flat, None)
        assert len(gkp) == len(orec) == 0
        assert np.array_equal(fe.detector_thresholds(det)[:9], np.array(st.thresh[:9]))
    fe.detector_destroy(det)


def test_fast_nodes_create_vs_oracle(fe, frames, oracle_mod):
    """Node::Node with the FAST detector: keypoints, descriptors and points bit-identical to the oracle; consecutive
    frames give a valid edge."""
    import fast_oracle
    from oracle import orb_oracle
    from rgbdslam_v2_b200._capi import DETECTOR_FAST
    det = nh.make_detector(fe, DETECTOR_FAST)
    st = orb_oracle.DetectorState()
    gray = np.stack([f[0] for f in frames]); depth = np.stack([f[1] for f in frames])
    mask = np.stack([orb_oracle.depth_to_mask(f[1]) for f in frames])
    K4 = nh.K4()
    handles, nf = fe.nodes_create(det, gray, depth, mask, K4, ids=[10, 11, 12, 13])
    for i, h in enumerate(handles):
        okp, odesc, oxyz = fast_oracle.node_construct(frames[i][0], frames[i][1], mask[i], K4, st, max_keypoints=600)
        gkp = fe.node_keypoints(h)
        gdesc, gxyz = fe.node_download(h)
        assert nf[i] == len(okp) and 300 < len(okp) <= 600
        assert gkp.tobytes() == okp.tobytes()
        assert np.array_equal(gdesc, odesc)
        assert np.array_equal(gxyz, oxyz)
        assert (gkp["angle"] == -1).all() and (gkp["size"] == 7).all()
    assert np.array_equal(fe.detector_thresholds(det)[:9], np.array(st.thresh[:9]))
    res, _, _ = fe.match_node_pairs([handles[1]], [handles[0]], seed=3)
    assert res[0]["id1"] == 10 and res[0]["id2"] == 11 and res[0]["n_inliers"] > 50
    fe.detector_destroy(det)
    nh.destroy(fe, handles)


def test_fast_nodes_create_pipeline_variants_identical(fe, seq40):
    """40 frames (2 chunks) == frame by frame == from pinned memory == mask derived from depth on the device."""
    import torch
    from rgbdslam_v2_b200._capi import DETECTOR_FAST
    gray, depth, mask = seq40
    K4 = nh.K4()

    def run(fn):
        det = nh.make_detector(fe, DETECTOR_FAST)
        out = fn(det)
        thr = fe.detector_thresholds(det).copy()
        fe.detector_destroy(det)
        dump = nh.node_dump(fe, out)
        nh.destroy(fe, out)
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


def test_fast_nodes_create_sharded_single_rank_equals_plain(fe, seq40):
    from rgbdslam_v2_b200._capi import DETECTOR_FAST
    gray, depth, mask = seq40
    K4 = nh.K4()
    det = nh.make_detector(fe, DETECTOR_FAST)
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
    fe.comm_destroy(comm)
    nh.destroy(fe, h1 + h2)


def test_orb_and_fast_detectors_interleaved(fe, seq40):
    """An ORB and a FAST detector used alternately in one process give what each gives alone: the handle decides."""
    from rgbdslam_v2_b200._capi import DETECTOR_FAST, DETECTOR_ORB
    gray, depth, mask = seq40
    K4 = nh.K4()
    alone = {}
    for t in (DETECTOR_ORB, DETECTOR_FAST):
        det = nh.make_detector(fe, t)
        hs = []
        for k in range(0, 12, 4):
            hs += fe.nodes_create(det, gray[k:k + 4], depth[k:k + 4], mask[k:k + 4], K4)[0]
        alone[t] = (nh.node_dump(fe, hs), fe.detector_thresholds(det).copy(), fe.orb_detect(det, gray[20], mask[20]))
        fe.detector_destroy(det)
        nh.destroy(fe, hs)
    d_orb = nh.make_detector(fe, DETECTOR_ORB)
    d_fast = nh.make_detector(fe, DETECTOR_FAST)  # the parameters now say FAST; the ORB handle stays ORB
    hs = {DETECTOR_ORB: [], DETECTOR_FAST: []}
    for k in range(0, 12, 4):
        for t, det in ((DETECTOR_FAST, d_fast), (DETECTOR_ORB, d_orb)):
            hs[t] += fe.nodes_create(det, gray[k:k + 4], depth[k:k + 4], mask[k:k + 4], K4)[0]
    thr = {t: fe.detector_thresholds(det).copy() for t, det in ((DETECTOR_ORB, d_orb), (DETECTOR_FAST, d_fast))}
    kp = {DETECTOR_ORB: fe.orb_detect(d_orb, gray[20], mask[20]), DETECTOR_FAST: fe.orb_detect(d_fast, gray[20], mask[20])}
    for t, det in ((DETECTOR_ORB, d_orb), (DETECTOR_FAST, d_fast)):
        assert nh.same_nodes(alone[t][0], nh.node_dump(fe, hs[t]))
        assert np.array_equal(alone[t][1], thr[t])  # thresholds after the node batches, before the detect call
        assert kp[t].tobytes() == alone[t][2].tobytes()
        fe.detector_destroy(det)
        nh.destroy(fe, hs[t])
    assert not nh.same_nodes(alone[DETECTOR_ORB][0], alone[DETECTOR_FAST][0])


def test_invalid_detector_type_rejected_by_init(fe):
    from rgbdslam_v2_b200._capi import DETECTOR_FAST
    nh.reinit(fe, DETECTOR_FAST)
    p = nh.params(7)
    assert fe.lib.rgbdslam_b200_init(0, C.byref(p)) == 1
    assert b"feature_detector_type" in fe.lib.rgbdslam_b200_last_error()
    assert fe.lib.rgbdslam_b200_get_params(C.byref(p)) == 0 and p.feature_detector_type == DETECTOR_FAST  # unchanged
