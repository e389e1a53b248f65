"""k_quota_counts' rule (DESIGN.md 4.5.7), restated in numpy from threshold-free candidates, against the count cv2's
cv::ORB(10000, ...) detect returns at every threshold the adjuster can reach; and the bare DetectorAdjuster of the oracle
against cv2 run directly."""
import numpy as np
import pytest

import detector_config_oracle as dco
import orb_quota_oracle as qo
from oracle import orb_oracle as oo


def _c4(k):
    from rgbdslam_v2_b200 import synth
    gray, depth = synth.render_frame(synth.trajectory(240)[k], seed=k)[:2]
    return gray, oo.depth_to_mask(depth)


def _texture(h, w, seed, sigma):
    import node_helpers as nh
    return nh.textured(h, w, 1, seed=seed, sigma=sigma)[0], None


def _tiled():
    """a 64 x 64 patch tiled over 320 x 320: every corner repeats, so Harris responses tie at every quota"""
    rng = np.random.default_rng(3)
    return np.tile((rng.random((64, 64)) * 255).astype(np.uint8), (5, 5)), None


CASES = {"c4_frame_0": lambda: _c4(0), "c4_frame_27": lambda: _c4(27), "texture_640x480": lambda: _texture(480, 640, 1, 2.0),
         "texture_fine": lambda: _texture(480, 640, 2, 1.0), "tiled_patch": _tiled, "flip_noise": lambda: (dco.flip_image(), None)}


@pytest.mark.parametrize("case", list(CASES))
def test_quota_counts_equal_cv2_at_every_threshold(case):
    img, mask = CASES[case]()
    table = dco.quota_counts(*dco.candidates(img, mask))
    got = [len(qo.detect(img, mask, t, 10000)) for t in range(2, 256)]
    assert table[2:].tolist() == got
    assert max(got) > qo.N_PER_LEVEL[0], "a quota must bind"


def test_tiled_patch_has_harris_ties_at_a_quota():
    img, mask = _tiled()
    _, stats = qo.quota_rule(img, mask, 2)
    assert any(h > 0 for _, _, h, _ in stats)


def _adjust(img, thresh, K, quotas):
    """the ungridded ORB adjuster on one frame from the given threshold: (final threshold, keypoints as (octave, x, y))"""
    import cv2

    import node_helpers as nh
    st = oo.DetectorState()
    st.thresh[0] = thresh
    if not quotas:
        oo.cv2 = nh.UnboundOrb()
    try:
        rec = oo.grid_detect(img, None, st, K, 1, 5)
    finally:
        oo.cv2 = cv2
    return st.thresh[0], sorted((r["octave"], float(r["x"]), float(r["y"])) for r in rec)


def test_quotas_flip_the_adjusters_decision():
    """K 2730 (min 2730, max 4095) on dco.flip_image: from 20 the adjuster reaches 14, where the count with quotas is
    accepted and the count without them is too many; from 15 the count with quotas is too few and the one without them is
    accepted.  The table k_quota_counts restates gives the quota-aware side of both decisions, the score histogram's suffix
    sum (the count without quotas) the other."""
    img = dco.flip_image()
    lev, score, harris = dco.candidates(img, None)
    table = dco.quota_counts(lev, score, harris)
    plain = [int((score >= t).sum()) for t in range(256)]
    K, mx = 2730, 4095
    assert table[20] < K and plain[20] < K
    assert K <= table[14] <= mx < plain[14]
    assert table[15] < K <= plain[15] <= mx
    for start in (20.0, 15.0):
        with_q, without_q = _adjust(img, start, K, True), _adjust(img, start, K, False)
        assert with_q[0] != without_q[0] and with_q[1] != without_q[1]
    assert _adjust(img, 20.0, K, True)[0] == 20.0 * 0.7 ** 1  # accepted at 14: the threshold stays
    assert _adjust(img, 20.0, K, False)[0] == 20.0 * 0.7 * 1.3


@pytest.mark.parametrize("detector", [0, 1], ids=["ORB", "FAST"])
def test_regular_detector_ignores_the_grid_and_the_counts(detector):
    """adjuster_max_iterations 0 with a 3x3 grid configured: the oracle's plain detector is one whole-frame detection at
    cell 0's threshold (not the grid adjuster's cells), returns more than the adjuster's maximum without adapting, and
    leaves every threshold as it was"""
    import cv2
    img, mask = _c4(13)
    st = oo.DetectorState()
    st.thresh[0] = 17.0
    rec = dco.detect(detector, img, mask, st, 1000, 3, 0)
    direct = (cv2.ORB_create(10000, 1.2, 8, 15, 0, 2, 0, 31, 17) if detector == 0 else cv2.FastFeatureDetector_create(17)).detect(img, mask)
    assert sorted((r["octave"], float(r["x"]), float(r["y"])) for r in rec) == \
        sorted((k.octave, float(np.float32(k.pt[0])), float(np.float32(k.pt[1]))) for k in direct)
    assert len(rec) > 1500 and {r["cell"] for r in rec} == {0}
    grid = dco.detect(detector, img, mask, oo.DetectorState(), 1000, 3, 5)
    assert len({r["cell"] for r in grid}) == 9 and len(grid) <= 1500
    assert st.thresh == [17.0] + [20.0] * 15
