"""cv::ORB's per-level quotas (feature_adjuster.cpp:94: cv::ORB::create(10000, 1.2, 8, 15, 0, 2, HARRIS_SCORE, 31, t)),
restated in numpy from cv2's own unculled candidates -- TEST INFRASTRUCTURE, shared by tests/test_orb_quota_cpu.py and
tests/test_gpu_large_frames.py.

Per level l: the FAST corners at threshold t inside the 15 px border and the mask, retainBest(2 n_l) by FAST score, then
retainBest(n_l) by Harris response, where retainBest(n) keeps every keypoint whose response is >= the n-th largest."""
import cv2
import numpy as np

N_PER_LEVEL = [2172, 1810, 1508, 1257, 1047, 873, 727, 606]
UNBOUND = 10 ** 6  # per-level quotas of 217 000 ... 60 600: above any cell's candidate count here


def detect(img, mask, t, nfeatures, score=cv2.ORB_HARRIS_SCORE):
    return cv2.ORB_create(nfeatures, 1.2, 8, 15, 0, 2, score, 31, t).detect(img, mask)


def key(k):
    return (k.octave, k.pt[0], k.pt[1])


def quota_rule(img, mask, t):
    """(the keypoints cv::ORB(10000) keeps as {(octave, x, y): response}, per level (candidates, FAST-cut ties, Harris-cut
    ties, kept)); a tie count is the number of keypoints kept beyond the quota because they equal the cut's response."""
    allk = detect(img, mask, t, UNBOUND)
    fast = {key(k): k.response for k in detect(img, mask, t, UNBOUND, cv2.ORB_FAST_SCORE)}
    assert len(fast) == len(allk) and all(key(k) in fast for k in allk)
    lev = np.array([k.octave for k in allk], np.int64)
    harris = np.array([k.response for k in allk], np.float32)
    score = np.array([fast[key(k)] for k in allk], np.float32)
    kept, stats = np.zeros(len(allk), bool), []
    for l, n in enumerate(N_PER_LEVEL):
        idx = np.nonzero(lev == l)[0]
        assert len(idx) < N_PER_LEVEL[l] * UNBOUND // 10000, "the unbound detection must not cut"
        fast_ties = harris_ties = 0
        if len(idx) > 2 * n:
            cut = np.sort(score[idx])[::-1][2 * n - 1]
            idx = idx[score[idx] >= cut]
            fast_ties = len(idx) - 2 * n
        if len(idx) > n:
            cut = np.sort(harris[idx])[::-1][n - 1]
            idx = idx[harris[idx] >= cut]
            harris_ties = len(idx) - n
        kept[idx] = True
        stats.append((int((lev == l).sum()), fast_ties, harris_ties, len(idx)))
    return {key(k): k.response for k, m in zip(allk, kept) if m}, stats


def cv2_quota(img, mask, t):
    return {key(k): k.response for k in detect(img, mask, t, 10000)}
