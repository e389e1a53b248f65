"""cv::ORB's per-level quotas (feature_adjuster.cpp:94: cv::ORB::create(10000, 1.2, 8, 15, 0, 2, HARRIS_SCORE, 31, t)) as
k_cell_select applies them, restated in numpy and pinned to cv2 4.13.

Per level l, with n_l = [2172, 1810, 1508, 1257, 1047, 873, 727, 606]: the FAST corners at threshold t inside the 15 px
border and the mask, retainBest(2 n_l) by FAST score, then retainBest(n_l) by Harris response, where retainBest(n) keeps
every keypoint whose response is >= the n-th largest (all ties at the cut).  The restatement takes the candidates from cv2
itself with quotas too large to bind (nfeatures 10^6): their Harris responses (HARRIS_SCORE) and FAST scores (FAST_SCORE)."""
import numpy as np
import pytest

cv2 = pytest.importorskip("cv2")

from orb_quota_oracle import N_PER_LEVEL, cv2_quota, quota_rule  # noqa: E402


def _noise(shape, seed, sigma=1.0):
    rng = np.random.default_rng(seed)
    t = cv2.GaussianBlur(rng.random(shape).astype(np.float32), (0, 0), sigma)
    return (t * 1024 % 256).astype(np.uint8)


def test_quotas_bind_at_every_level_with_fast_score_ties():
    """A 1400 x 1100 cell (a 3x3 grid cell of a 4095 x 3200 frame) of dense texture: every level is above 2 n_l, so both cuts
    bind everywhere, and the integer FAST scores tie at the 2 n_l cut."""
    img = _noise((1100, 1400), 1)
    mine, stats = quota_rule(img, None, 20)
    assert mine == cv2_quota(img, None, 20)
    assert all(c > 2 * n for (c, _, _, _), n in zip(stats, N_PER_LEVEL))
    assert all(f > 0 for _, f, _, _ in stats)
    assert sum(k for *_, k in stats) == 10000


def test_harris_ties_at_the_quota_are_all_kept():
    """A tiled 24 x 24 patch: level-0 corners repeat with bit-identical Harris responses, so the n_0 cut falls inside a tie
    and cv2 keeps every tied keypoint (more than 2172 at level 0)."""
    rng = np.random.default_rng(3)
    patch = (cv2.GaussianBlur(rng.random((24, 24)).astype(np.float32), (0, 0), 0.8) * 1024 % 256).astype(np.uint8)
    img = np.ascontiguousarray(np.tile(patch, (46, 58)))  # 1104 x 1392
    for t in (10, 20):
        mine, stats = quota_rule(img, None, t)
        assert mine == cv2_quota(img, None, t)
        assert stats[0][2] > 0 and stats[0][3] > N_PER_LEVEL[0]


def test_quota_under_a_mask_and_a_level_below_its_quota():
    """The quota counts the keypoints the mask leaves: a mask that removes most of the cell keeps some levels above and some
    below their quota; and a smooth cell where no level reaches it returns every candidate."""
    img = _noise((1000, 1300), 5, 1.3)
    mask = np.zeros(img.shape, np.uint8)
    mask[100:300, 150:400] = 255
    mask[800:880, 1000:1100] = 1
    mine, stats = quota_rule(img, mask, 12)
    assert mine == cv2_quota(img, mask, 12)
    assert any(c > n for (c, _, _, _), n in zip(stats, N_PER_LEVEL)) and any(c <= n for (c, _, _, _), n in zip(stats, N_PER_LEVEL))
    smooth = cv2.GaussianBlur(img[:500, :600], (0, 0), 3.0)
    mine, stats = quota_rule(smooth, None, 20)
    assert mine == cv2_quota(smooth, None, 20) and all(c == k for c, _, _, k in stats)


def test_a_cell_of_a_640x480_frame_can_reach_a_binding_quota():
    """The largest 3x3 grid cell of a 640 x 480 frame (275 x 222 px) of dense texture at the adjuster's initial threshold 20:
    the candidate buffer (12288 per cell) holds every candidate the device stores -- each strict 3x3 maximum of the
    threshold-free FAST score with score >= 2 at least 15 px inside its level, at every level -- and levels 0 and 1 still have
    more than n_l corners at threshold 20, so cv2's Harris quotas bind in a frame the narrow kernels accept."""
    import orb_pyramid_oracle as po
    img = _noise((222, 275), 11, 1.0)
    mine, stats = quota_rule(img, None, 20)
    corners = sum(c for c, *_ in stats)
    stored = sum(len(d) for d in po.orb_candidates(po.pyramid(img), po.mask_pyramid(np.full(img.shape, 255, np.uint8))))
    assert mine == cv2_quota(img, None, 20)
    assert corners <= stored <= 12288
    assert all(stats[l][0] > N_PER_LEVEL[l] and stats[l][3] == N_PER_LEVEL[l] for l in (0, 1))
    assert len(mine) < corners
