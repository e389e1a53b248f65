"""GPU parity tests of use_feature_min_depth (parameter_server.cpp:90) in the Node-constructor path: each keypoint's depth is
the minimum of its neighbourhood (misc.cpp:774-791) in removeDepthless and projectTo3D, checked bit for bit against the
restatement in tests/min_depth_oracle.py on top of the cv2-based ORB and FAST detection oracles."""
import ctypes as C

import numpy as np
import pytest

import node_helpers as nh

pytestmark = pytest.mark.gpu

SCENARIOS = ["mask", "no_mask", "mask_from_depth", "depth_scaling", "blobs"]


@pytest.fixture(scope="module")
def fe(built):
    from rgbdslam_v2_b200 import Frontend
    from rgbdslam_v2_b200._capi import DETECTOR_ORB
    f = Frontend(0, nh.params(DETECTOR_ORB, use_feature_min_depth=1))
    yield f
    f.close()


def _plant_blobs(depth, seed):
    """zero and NaN blobs on the textured scene, some of them on the image borders"""
    d = depth.copy()
    H, W = d.shape
    rng = np.random.default_rng(seed)
    for k in range(60):
        y, x = int(rng.integers(0, H - 6)), int(rng.integers(0, W - 6))
        s = int(rng.integers(1, 6))
        d[y:y + s, x:x + s] = 0.0 if k % 2 == 0 else np.nan
    d[100:140, 0:4] = 0.0
    d[H - 3:H, 200:260] = 0.0
    d[300:350, W - 5:W] = np.nan
    d[0:2, 400:480] = np.nan
    d[0, 0] = -0.0
    return d


@pytest.fixture(scope="module")
def frames():
    gray, depth = nh.stack(nh.render((0, 1, 2, 3), 40))
    blobs = np.stack([_plant_blobs(d, k) for k, d in enumerate(depth)])
    return gray, depth, blobs


@pytest.fixture(scope="module")
def seq70():
    """70 frames: two chunks of the constructor's pipeline"""
    return nh.seq(70)


def _pointwise_z(depth, kp, scaling=1.0):
    """projectTo3D's depth without the option: depth(round(y), round(x)) * depth_scaling"""
    rx = np.floor(kp["x"] + np.float32(0.5)).astype(int)
    ry = np.floor(kp["y"] + np.float32(0.5)).astype(int)
    return (depth[ry, rx].astype(np.float64) * scaling).astype(np.float32)


@pytest.mark.parametrize("scenario", SCENARIOS)
@pytest.mark.parametrize("detector", [0, 1], ids=["ORB", "FAST"])
def test_min_depth_nodes_vs_oracle(fe, frames, scenario, detector):
    """Node::Node with use_feature_min_depth, frame by frame: keypoints, descriptors and points bit-identical to the oracle,
    thresholds equal after every frame; consecutive nodes give valid edges."""
    import min_depth_oracle as md
    from oracle import orb_oracle
    gray, depth, blobs = frames
    if scenario == "blobs":
        depth = blobs
    scaling = 1.25 if scenario == "depth_scaling" else 1.0
    det = nh.make_detector(fe, detector, use_feature_min_depth=1, depth_scaling_factor=scaling)
    st = orb_oracle.DetectorState()
    K4 = nh.K4()
    handles, on_nan, below = [], 0, 0
    for k in range(len(gray)):
        mask = None if scenario in ("no_mask", "blobs") else orb_oracle.depth_to_mask(depth[k])
        dev_mask = None if scenario == "mask_from_depth" else (None if mask is None else mask[None])
        hs, nf = fe.nodes_create(det, gray[k:k + 1], depth[k:k + 1], dev_mask, K4, ids=[k],
                                 mask_from_depth=scenario == "mask_from_depth")
        handles += hs
        okp, odesc, oxyz = md.node_construct(gray[k], depth[k], mask, K4, st, max_keypoints=600, depth_scaling=scaling,
                                             detector=nh.name(detector))
        gkp = fe.node_keypoints(hs[0])
        gdesc, gxyz = fe.node_download(hs[0])
        assert nf[0] == len(okp) and 300 < len(okp) <= 600
        assert gkp.tobytes() == okp.tobytes()
        assert np.array_equal(gdesc, odesc)
        assert np.array_equal(gxyz.view(np.uint32), oxyz.view(np.uint32))
        assert np.array_equal(fe.detector_thresholds(det)[:9], np.array(st.thresh[:9]))
        assert not np.isnan(gxyz).any() and (gxyz[:, 2] != 0).all()
        # the rule is not vacuous: never deeper than the pixel under the keypoint, often nearer
        zp = _pointwise_z(depth[k], gkp, scaling)
        fin = ~np.isnan(zp)
        assert (gxyz[fin, 2] <= zp[fin]).all()
        below += int((gxyz[fin, 2] < zp[fin]).sum())
        on_nan += int((~fin).sum())
    assert below > 100
    if scenario in ("no_mask", "blobs"):
        assert on_nan > 0  # keypoints on NaN pixels, which the pointwise rule drops
    res, _, _ = fe.match_node_pairs(handles[1:], handles[:-1], seed=3)
    assert (res["id1"] == np.arange(len(handles) - 1)).all() and (res["id2"] == np.arange(1, len(handles))).all()
    assert (res["n_inliers"] > 50).all()
    fe.detector_destroy(det)
    nh.destroy(fe, handles)


@pytest.mark.parametrize("detector", [0, 1], ids=["ORB", "FAST"])
def test_min_depth_pipeline_variants_identical(fe, seq70, detector):
    """70 frames (2 chunks) == frame by frame == from pinned memory == mask from depth == 1-rank sharded."""
    import torch
    gray, depth, mask = seq70
    K4 = nh.K4()
    n = len(gray)

    def run(fn):
        det = nh.make_detector(fe, detector, use_feature_min_depth=1)
        out = fn(det)
        thr = fe.detector_thresholds(det).copy()
        fe.detector_destroy(det)
        dump = nh.node_dump(fe, out)
        nh.destroy(fe, out)
        return dump, thr

    ref, thr_ref = run(lambda det: fe.nodes_create(det, gray, depth, mask, K4)[0])
    assert len(ref) == n and min(len(k) for k, _, _ in ref) > 300

    def one_by_one(det):
        hs = []
        for k in range(n):
            hs += fe.nodes_create(det, gray[k:k + 1], depth[k:k + 1], mask[k:k + 1], K4, ids=[k])[0]
        return hs
    a, thr_a = run(one_by_one)
    assert nh.same_nodes(ref, a) and np.array_equal(thr_ref, thr_a)
    pg, pd, pm = (torch.from_numpy(x).pin_memory() for x in (gray, depth, mask))
    b, thr_b = run(lambda det: fe.nodes_create(det, pg, pd, pm, K4)[0])
    assert nh.same_nodes(ref, b) and np.array_equal(thr_ref, thr_b)
    c, thr_c = run(lambda det: fe.nodes_create(det, gray, depth, None, K4, mask_from_depth=True)[0])
    assert nh.same_nodes(ref, c) and np.array_equal(thr_ref, thr_c)
    comm = fe.comm_init(0, 1, fe.comm_unique_id())
    d, thr_d = run(lambda det: fe.nodes_create_sharded(det, comm, n, gray, depth, mask, K4)[0])
    fe.comm_destroy(comm)
    assert nh.same_nodes(ref, d) and np.array_equal(thr_ref, thr_d)


@pytest.mark.parametrize("detector", [0, 1], ids=["ORB", "FAST"])
def test_flag_switches_between_calls(fe, seq70, detector):
    """The parameters current at each nodes_create call decide the rule: re-initialising with the flag off gives the
    pointwise nodes again, and alternating the flag between calls on one detector gives each rule's result."""
    gray, depth, mask = seq70
    K4 = nh.K4()
    chunks = [(k, k + 4) for k in range(0, 16, 4)]
    alone = {}
    for flag in (0, 1):
        det = nh.make_detector(fe, detector, use_feature_min_depth=flag)
        hs = []
        for a, b in chunks:
            hs += fe.nodes_create(det, gray[a:b], depth[a:b], mask[a:b], K4)[0]
        alone[flag] = nh.node_dump(fe, hs)
        fe.detector_destroy(det)
        nh.destroy(fe, hs)
    assert not nh.same_nodes(alone[0], alone[1])
    # the thresholds depend only on the detection, so one detector serves both rules
    det = nh.make_detector(fe, detector, use_feature_min_depth=0)
    got = []
    for i, (a, b) in enumerate(chunks):
        flag = i % 2
        nh.reinit(fe, detector, use_feature_min_depth=flag)
        hs = fe.nodes_create(det, gray[a:b], depth[a:b], mask[a:b], K4)[0]
        got += nh.node_dump(fe, hs)
        nh.destroy(fe, hs)
        assert nh.same_nodes(got[a:b], alone[flag][a:b])
    fe.detector_destroy(det)
    # flag off again: the pointwise nodes, and the launch count of the pointwise path
    det = nh.make_detector(fe, detector, use_feature_min_depth=0)
    l0 = fe.lib.rgbdslam_b200_launch_count()
    hs = fe.nodes_create(det, gray[:4], depth[:4], mask[:4], K4)[0]
    l_off = fe.lib.rgbdslam_b200_launch_count() - l0
    assert nh.same_nodes(nh.node_dump(fe, hs), alone[0][:4])
    nh.destroy(fe, hs)
    fe.detector_destroy(det)
    det = nh.make_detector(fe, detector, use_feature_min_depth=1)
    l0 = fe.lib.rgbdslam_b200_launch_count()
    hs = fe.nodes_create(det, gray[:4], depth[:4], mask[:4], K4)[0]
    assert fe.lib.rgbdslam_b200_launch_count() - l0 == l_off + 1  # k_min_depth
    nh.destroy(fe, hs)
    fe.detector_destroy(det)


def test_init_rejects_other_values(fe):
    from rgbdslam_v2_b200._capi import DETECTOR_ORB
    nh.reinit(fe, DETECTOR_ORB, use_feature_min_depth=1)
    p = nh.params(DETECTOR_ORB, use_feature_min_depth=2)
    assert fe.lib.rgbdslam_b200_init(0, C.byref(p)) == 1
    assert b"use_feature_min_depth" in fe.lib.rgbdslam_b200_last_error()
    p = nh.params(DETECTOR_ORB, use_feature_min_depth=1, allow_features_without_depth_=1)
    assert fe.lib.rgbdslam_b200_init(0, C.byref(p)) == 1
    assert fe.lib.rgbdslam_b200_get_params(C.byref(p)) == 0 and p.use_feature_min_depth == 1  # unchanged
