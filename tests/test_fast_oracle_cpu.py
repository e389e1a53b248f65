"""The FAST detector (feature_detector_type FAST) pinned against cv2 on rendered frames, without a GPU: what the device
restates -- the histogram identity, the 3 px border rule, the keypoint fields, ORB compute on FAST keypoints -- and the
parameter that selects it."""
import ctypes as C

import cv2
import numpy as np
import pytest

import fast_oracle
from oracle import orb_oracle


@pytest.fixture(scope="module")
def frames():
    from rgbdslam_v2_b200 import synth
    poses = synth.trajectory(40)
    return [synth.render_frame(poses[k], seed=k) for k in (0, 1, 9)]


def _cells(gray, mask, grid=3):
    H, W = gray.shape
    for (y0, y1, x0, x1) in orb_oracle._cells(W, H, grid):
        yield np.ascontiguousarray(gray[y0:y1, x0:x1]), np.ascontiguousarray(mask[y0:y1, x0:x1])


def _cv2_fast(img, mask, t):
    return {(int(k.pt[0]), int(k.pt[1])): k.response for k in cv2.FastFeatureDetector_create(t).detect(img, mask)}


def test_threshold_is_a_histogram_lookup_per_cell(frames):
    """FAST(t) == FAST(2) filtered to response >= t, per cell with its mask: count(t) is a lookup in the histogram of S."""
    cases = 0
    for gray, depth in frames:
        mask = orb_oracle.depth_to_mask(depth)
        for sub, sm in _cells(gray, mask):
            base = _cv2_fast(sub, sm, 2)
            assert len(base) > 100
            for t in (3, 7, 14, 20, 28, 40):
                assert _cv2_fast(sub, sm, t) == {p: r for p, r in base.items() if r >= t}
                cases += 1
    assert cases == 162


def test_threshold_free_scores_and_border_rule_equal_cv2(frames):
    """The device's rule -- S on [3, n-4], score 0 outside it in the NMS, mask after the NMS -- gives cv::FAST's keypoints
    and responses exactly, on every cell of rendered frames and on a crop."""
    for gray, depth in frames:
        mask = orb_oracle.depth_to_mask(depth)
        for sub, sm in _cells(gray, mask):
            for t in (2, 20):
                assert fast_oracle.fast_nms(sub, sm, t) == _cv2_fast(sub, sm, t)
    gray = frames[0][0]
    crop = np.ascontiguousarray(gray[80:280, 100:350])
    assert fast_oracle.fast_nms(crop, None, 2) == _cv2_fast(crop, None, 2)


def test_border_rule_differs_from_the_full_image(frames):
    """cv::FAST on a cell keeps corners on rows / columns 3 and n-4 that the full image suppresses (their outer
    neighbours read as score 0): the FAST path cannot reuse ORB's 15 px border, where the NMS sees real neighbours."""
    gray = frames[0][0]
    x0, y0, w, h = 100, 80, 250, 200
    full = _cv2_fast(gray, None, 2)
    crop = _cv2_fast(np.ascontiguousarray(gray[y0:y0 + h, x0:x0 + w]), None, 2)
    extra = [(x, y) for (x, y) in crop if (x + x0, y + y0) not in full]
    on_frame = [(x, y) for (x, y) in extra if x in (3, w - 4) or y in (3, h - 4)]
    assert len(on_frame) > 10
    xs = np.array([p[0] for p in crop]); ys = np.array([p[1] for p in crop])
    assert xs.min() >= 3 and xs.max() <= w - 4 and ys.min() >= 3 and ys.max() <= h - 4


def test_keypoint_fields(frames):
    """size 7, angle -1, octave 0, integer positions, response = the integer corner score S."""
    gray, depth = frames[1]
    mask = orb_oracle.depth_to_mask(depth)
    st = orb_oracle.DetectorState()
    rec = fast_oracle.grid_detect(gray, mask, st, max_keypoints=600)
    kp = orb_oracle.records_to_array(rec)
    assert 300 < len(kp) <= 900
    assert (kp["size"] == 7).all() and (kp["angle"] == -1).all() and (kp["octave"] == 0).all()
    assert (kp["x"] == np.round(kp["x"])).all() and (kp["y"] == np.round(kp["y"])).all()
    assert (kp["response"] == np.round(kp["response"])).all() and kp["response"].min() >= 2
    s = fast_oracle.threshold_free_scores(gray)  # the score does not depend on the cell (the pixel is >= 3 inside it)
    assert np.array_equal(kp["response"], s[kp["y"].astype(int), kp["x"].astype(int)].astype(np.float32))


def test_orb_compute_keeps_fast_angle(frames):
    """ORB compute on FAST keypoints: drops those within 31 px of the border and keeps angle -1 (no orientation).  The
    pattern is steered by -1 degree; on the 31 x 31 patch that rotation moves no rounded sample (|13 sin 1 deg| < 0.5), so
    the descriptors are those of angle 0."""
    gray = frames[0][0]
    kps = cv2.FastFeatureDetector_create(20).detect(gray)
    arr = np.zeros(len(kps), orb_oracle.KP_DTYPE)
    for i, k in enumerate(kps):
        arr[i] = (k.pt[0], k.pt[1], k.size, k.angle, k.response, k.octave, -1)
    out, desc = orb_oracle.orb_compute(gray, arr)
    H, W = gray.shape
    inside = (arr["x"] >= 31) & (arr["x"] < W - 31) & (arr["y"] >= 31) & (arr["y"] < H - 31)
    assert len(out) == inside.sum() and out.tobytes() == arr[inside].tobytes()
    assert (out["angle"] == -1).all()
    zero = arr[inside].copy(); zero["angle"] = 0
    _, desc0 = orb_oracle.orb_compute(gray, zero)
    assert np.array_equal(desc, desc0)


def test_detector_type_parameter(built):
    """feature_detector_type takes reserved_[0]: same struct size and offsets; default ORB; init rejects other values
    before it looks for a device."""
    from rgbdslam_v2_b200 import _capi
    P = _capi.Params
    assert C.sizeof(P) == 128
    assert P.feature_detector_type.offset == P.allow_features_without_depth_.offset + 1 == 126
    assert P.reserved_.offset == 127
    p = _capi.default_params()
    assert p.feature_detector_type == _capi.DETECTOR_ORB == 0 and _capi.DETECTOR_FAST == 1
    lib = _capi.load_library()
    for bad in (2, 3, 255):
        p.feature_detector_type = bad
        assert lib.rgbdslam_b200_init(0, C.byref(p)) == 1
        assert b"feature_detector_type" in lib.rgbdslam_b200_last_error()
