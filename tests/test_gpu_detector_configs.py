"""The Node constructor under the three detectors createDetector returns (features.cpp:101-112, DESIGN.md 4.5.7): the
adjuster without a grid (cv::ORB's quotas in its counts), the bare DetectorAdjuster (adjuster_max_iterations <= 0), and the
2x2 grid whose per-cell maximum reaches cv::ORB's smallest quota -- bit-identical to tests/detector_config_oracle.py."""
import numpy as np
import pytest

import detector_config_oracle as dco
import node_helpers as nh
from oracle import orb_oracle as oo

pytestmark = pytest.mark.gpu

N_SEQ = 6


@pytest.fixture(scope="module")
def fe(built):
    from rgbdslam_v2_b200 import Frontend
    f = Frontend(0, nh.params())
    yield f
    f.close()


@pytest.fixture(scope="module")
def seq():
    return nh.seq(N_SEQ)


def _check(fe, hs, gray, depth, mask, det, detector, K, grid, iters, st):
    K4 = nh.K4()
    for k, h in enumerate(hs):
        okp, odesc, oxyz = dco.node_construct(detector, gray[k], depth[k], mask[k], K4, st, K, grid, iters)
        gkp = fe.node_keypoints(h)
        gdesc, gxyz = fe.node_download(h)
        assert len(gkp) == len(okp) > 0, k
        assert gkp.tobytes() == okp.tobytes(), k
        assert np.array_equal(gdesc, odesc), k
        assert np.array_equal(gxyz.view(np.uint32), oxyz.view(np.uint32)), k
    assert np.array_equal(fe.detector_thresholds(det)[:max(grid, 1) ** 2], np.array(st.thresh[:max(grid, 1) ** 2]))


CONFIGS = [(grid, iters, K) for grid, iters in [(0, 5), (1, 20), (0, 0), (3, 0)] for K in (600, 1000, 2730)] + [(2, 5, 2000)]


@pytest.mark.parametrize("detector", [0, 1], ids=["ORB", "FAST"])
@pytest.mark.parametrize("grid,iters,K", CONFIGS, ids=[f"grid{g}_it{i}_K{k}" for g, i, k in CONFIGS])
def test_c4_sequence_vs_oracle(fe, seq, detector, grid, iters, K):
    gray, depth, mask = seq
    det = nh.make_detector(fe, detector, max_keypoints=K, detector_grid_resolution=grid, adjuster_max_iterations=iters)
    st = oo.DetectorState()
    hs, _ = fe.nodes_create(det, gray, depth, None, nh.K4(), mask_from_depth=True)
    _check(fe, hs, gray, depth, mask, det, detector, K, grid, iters, st)
    nh.destroy(fe, hs)
    fe.detector_destroy(det)
    nh.reinit(fe, 0)


@pytest.mark.parametrize("detector", [0, 1], ids=["ORB", "FAST"])
@pytest.mark.parametrize("hw,iters", [((480, 640), 5), ((480, 640), 0), ((1023, 1023), 5), ((1023, 1023), 0)])
def test_dense_textures_vs_oracle(fe, detector, hw, iters):
    """dense textures: whole-frame detectors that return more than 4096 keypoints (Regular) and bind every quota"""
    h, w = hw
    gray = nh.textured(h, w, 2, seed=5)
    depth = np.ones((2, h, w), np.float32)
    mask = np.full((2, h, w), 255, np.uint8)
    K = 2730
    det = nh.make_detector(fe, detector, max_keypoints=K, detector_grid_resolution=0, adjuster_max_iterations=iters)
    st = oo.DetectorState()
    hs, _ = fe.nodes_create(det, gray, depth, mask, (500.0, 500.0, w / 2, h / 2))
    K4 = (500.0, 500.0, w / 2, h / 2)
    for k, hd in enumerate(hs):
        okp, odesc, oxyz = dco.node_construct(detector, gray[k], depth[k], mask[k], K4, st, K, 0, iters)
        assert fe.node_keypoints(hd).tobytes() == okp.tobytes()
        gdesc, gxyz = fe.node_download(hd)
        assert np.array_equal(gdesc, odesc) and np.array_equal(gxyz.view(np.uint32), oxyz.view(np.uint32))
    if iters == 0:
        assert len(dco.detect(detector, gray[0], mask[0], oo.DetectorState(), K, 0, 0)) > 4096
    nh.destroy(fe, hs)
    fe.detector_destroy(det)
    nh.reinit(fe, 0)


@pytest.mark.parametrize("start", [20.0, 15.0])
def test_quotas_flip_the_adjusters_decision(fe, start):
    """dco.flip_image at K 2730: from 20 the count with quotas is accepted at 14 where the one without them is too many, from
    15 it is too few where the one without them is accepted.  The device follows the quota-aware oracle bit for bit, and
    the oracle without quotas ends on another threshold with other keypoints."""
    import cv2
    img = dco.flip_image()[None]
    depth = np.ones(img.shape, np.float32)
    K, K4 = 2730, (500.0, 500.0, 320.0, 240.0)
    det = nh.make_detector(fe, 0, max_keypoints=K, detector_grid_resolution=0, adjuster_max_iterations=5)
    thr = fe.detector_thresholds(det).copy()
    thr[0] = start
    fe.detector_thresholds(det, thr)
    st, unbound = oo.DetectorState(), oo.DetectorState()
    st.thresh[0] = unbound.thresh[0] = start
    hs, _ = fe.nodes_create(det, img, depth, None, K4)
    okp, odesc, oxyz = dco.node_construct(0, img[0], depth[0], None, K4, st, K, 0, 5)
    gkp = fe.node_keypoints(hs[0])
    gdesc, gxyz = fe.node_download(hs[0])
    assert gkp.tobytes() == okp.tobytes() and np.array_equal(gdesc, odesc)
    assert np.array_equal(gxyz.view(np.uint32), oxyz.view(np.uint32))
    assert fe.detector_thresholds(det)[0] == st.thresh[0]
    oo.cv2 = nh.UnboundOrb()
    try:
        ukp, _, _ = dco.node_construct(0, img[0], depth[0], None, K4, unbound, K, 0, 5)
    finally:
        oo.cv2 = cv2
    assert unbound.thresh[0] != st.thresh[0] and ukp.tobytes() != gkp.tobytes()
    nh.destroy(fe, hs)
    fe.detector_destroy(det)
    nh.reinit(fe, 0)


@pytest.mark.parametrize("detector", [0, 1], ids=["ORB", "FAST"])
@pytest.mark.parametrize("iters", [5, 0], ids=["Adjuster", "Regular"])
def test_min_depth_and_cloud_input_vs_oracle(fe, seq, monkeypatch, detector, iters):
    """use_feature_min_depth (tests/min_depth_oracle.py) and CLOUD_XYZRGB + MASK_FROM_CLOUD (tests/cloud_oracle.py) with the
    whole-frame detectors, K 1000 on C4 frames, where the plain detector finds more than 4096 keypoints: keypoints,
    descriptors, points and thresholds bit-identical"""
    import cloud_oracle as co
    import min_depth_oracle as md
    dco.install(monkeypatch)
    gray, depth, mask = seq
    K, K4, name = 1000, nh.K4(), nh.name(detector)
    kw = dict(max_keypoints=K, detector_grid_resolution=0, adjuster_max_iterations=iters)
    if iters == 0:
        assert len(dco.detect(detector, gray[0], mask[0], oo.DetectorState(), K, 0, 0)) > 4096

    def check(hs, det, construct):
        st = oo.DetectorState()
        for k, h in enumerate(hs):
            okp, odesc, oxyz = construct(k, st)
            gdesc, gxyz = fe.node_download(h)
            assert fe.node_keypoints(h).tobytes() == okp.tobytes(), k
            assert np.array_equal(gdesc, odesc) and np.array_equal(gxyz.view(np.uint32), oxyz.view(np.uint32)), k
        assert fe.detector_thresholds(det)[0] == st.thresh[0]
        nh.destroy(fe, hs)
        fe.detector_destroy(det)

    det = nh.make_detector(fe, detector, use_feature_min_depth=True, **kw)
    hs, _ = fe.nodes_create(det, gray, depth, mask, K4)
    check(hs, det, lambda k, st: md.node_construct(gray[k], depth[k], mask[k], K4, st, K, 0, iters, detector=name))
    cloud = np.stack([co.cloud_from_depth(d, K4, "XYZRGB") for d in depth])
    det = nh.make_detector(fe, detector, **kw)
    hs, _ = fe.nodes_create(det, gray, cloud, None, None, mask_from_cloud=True)
    check(hs, det, lambda k, st: co.node_construct(gray[k], cloud[k], co.cloud_mask(cloud[k][..., 2]), st, K, 0, iters, detector=name))
    nh.reinit(fe, 0)


@pytest.mark.parametrize("detector", [0, 1], ids=["ORB", "FAST"])
@pytest.mark.parametrize("iters", [5, 0])
def test_call_shapes_and_inputs_are_identical(fe, detector, iters):
    """70 frames in one call == one call per frame == pinned input == a 1-rank _sharded call == _resized at equal sizes;
    colour input == its grey; use_feature_min_depth and cloud input: one call == one call per frame"""
    import torch
    gray, depth, mask = nh.seq(70)
    K4 = nh.K4()
    kw = dict(max_keypoints=1000, detector_grid_resolution=0, adjuster_max_iterations=iters)

    def run(fn, **extra):
        nh.reinit(fe, detector, **kw, **extra)
        det = fe.detector_create()
        hs = fn(det)
        thr = fe.detector_thresholds(det).copy()
        fe.detector_destroy(det)
        dump = nh.node_dump(fe, hs)
        nh.destroy(fe, hs)
        return dump, thr

    def same(a, b):
        assert nh.same_nodes(a[0], b[0]) and np.array_equal(a[1], b[1])

    ref = run(lambda det: fe.nodes_create(det, gray, depth, mask, K4)[0])
    same(ref, run(lambda det: sum((fe.nodes_create(det, gray[k:k + 1], depth[k:k + 1], mask[k:k + 1], K4)[0] for k in range(70)), [])))
    pg, pd, pm = (torch.from_numpy(x).pin_memory() for x in (gray, depth, mask))
    same(ref, run(lambda det: fe.nodes_create(det, pg, pd, pm, K4)[0]))
    comm = fe.comm_init(0, 1, fe.comm_unique_id())
    same(ref, run(lambda det: fe.nodes_create_sharded(det, comm, 70, gray, depth, mask, K4)[0]))
    fe.comm_destroy(comm)
    same(ref, run(lambda det: fe.nodes_create_resized(det, gray, depth, mask, K4)[0]))
    rgb = np.repeat(gray[..., None], 3, axis=3)
    same(ref, run(lambda det: fe.nodes_create(det, rgb, depth, mask, K4)[0]))
    md = run(lambda det: fe.nodes_create(det, gray, depth, mask, K4)[0], use_feature_min_depth=True)
    same(md, run(lambda det: sum((fe.nodes_create(det, gray[k:k + 1], depth[k:k + 1], mask[k:k + 1], K4)[0] for k in range(70)), []),
                 use_feature_min_depth=True))
    import cloud_oracle
    cloud = np.stack([cloud_oracle.cloud_from_depth(d, K4, "XYZRGB") for d in depth[:8]])
    c1 = run(lambda det: fe.nodes_create(det, gray[:8], cloud, None, None, mask_from_cloud=True)[0])
    same(c1, run(lambda det: sum((fe.nodes_create(det, gray[k:k + 1], cloud[k:k + 1], None, None, mask_from_cloud=True)[0]
                                  for k in range(8)), [])))
    nh.reinit(fe, 0)


def test_orb_detect_of_a_whole_frame_detector(fe, seq):
    """orb_detect with the plain ORB detector at a set threshold returns the oracle's detector output and leaves the
    threshold; a detector output above 4096 keypoints fails loudly"""
    from rgbdslam_v2_b200._capi import B200Error
    gray, depth, mask = seq
    det = nh.make_detector(fe, 0, max_keypoints=1000, detector_grid_resolution=3, adjuster_max_iterations=0)
    thr = fe.detector_thresholds(det).copy()
    thr[0] = 60.0
    fe.detector_thresholds(det, thr)
    st = oo.DetectorState()
    st.thresh[0] = 60.0
    for k in range(3):
        kp = fe.orb_detect(det, gray[k], mask[k])
        rec = dco.detect(0, gray[k], mask[k], st, 1000, 3, 0)
        assert len(kp) == len(rec) > 0
        assert np.array_equal(kp["x"], np.array([r["x"] for r in rec], np.float32))
        assert np.array_equal(kp["y"], np.array([r["y"] for r in rec], np.float32))
        assert np.array_equal(kp["response"], np.array([r["response"] for r in rec], np.float32))
    assert fe.detector_thresholds(det)[0] == 60.0
    fe.detector_destroy(det)
    det = nh.make_detector(fe, 1, max_keypoints=1000, detector_grid_resolution=0, adjuster_max_iterations=0)
    tex = nh.textured(480, 640, 1, seed=5)[0]
    with pytest.raises(B200Error):
        fe.orb_detect(det, tex, None)
    fe.detector_destroy(det)
    nh.reinit(fe, 0)


def test_large_frames_with_whole_frame_detectors_launch_nothing(fe):
    from rgbdslam_v2_b200._capi import B200Error
    lib = fe.lib
    for kw in (dict(detector_grid_resolution=3, adjuster_max_iterations=0), dict(detector_grid_resolution=0, adjuster_max_iterations=5)):
        nh.reinit(fe, 0, **kw)
        det = fe.detector_create()
        g = np.zeros((1, 720, 1280), np.uint8)
        d = np.ones((1, 720, 1280), np.float32)
        l0 = lib.rgbdslam_b200_launch_count()
        with pytest.raises(B200Error):
            fe.nodes_create(det, g, d, None, (500.0, 500.0, 640.0, 360.0))
        assert lib.rgbdslam_b200_launch_count() == l0
        fe.detector_destroy(det)
    nh.reinit(fe, 0)
