"""The three detectors createDetector returns (features.cpp:101-112) on cv2 -- TEST INFRASTRUCTURE, shared by
tests/test_orb_quota_counts_cpu.py and tests/test_gpu_detector_configs.py.

  adjuster_max_iterations > 0, grid > 1   adjustedGridWrapper: grid_detect of oracle/orb_oracle.py / tests/fast_oracle.py
  adjuster_max_iterations > 0, grid <= 1  adjusterWrapper(K, (int)(1.5 K)): the same recurrence on one whole-frame cell,
                                          no keepStrongest (grid_detect with grid 1)
  adjuster_max_iterations <= 0            the bare DetectorAdjuster: one detection of the whole frame at the persistent
                                          threshold (cell 0), which never changes, whatever the grid

quota_counts restates in numpy what k_quota_counts tabulates: the count cv::ORB(10000, ..., t).detect returns, for every t,
from threshold-free candidates."""
import ctypes as C

import cv2
import numpy as np

import fast_oracle
import orb_quota_oracle as qo
from oracle import orb_oracle as oo


# the grid adjusters of the two detectors, kept before install() substitutes the three-branch dispatch for them
_GRID = {0: oo.grid_detect, 1: fast_oracle.grid_detect}


def _cv_detect(detector, gray, mask, t):
    if detector == 0:
        return cv2.ORB_create(10000, 1.2, 8, 15, 0, 2, 0, 31, int(t)).detect(gray, mask)
    return cv2.FastFeatureDetector_create(int(t)).detect(gray, mask)


def detect(detector, gray, mask, state, max_keypoints, grid, max_iters):
    """== detector->detect(gray, keypoints, mask) for detector 0 (ORB) or 1 (FAST); records as orb_oracle.grid_detect's"""
    if max_iters <= 0:
        rec = oo._kp_records(_cv_detect(detector, gray, mask, state.thresh[0]), 0, 0, 0)
        rec.sort(key=lambda r: (-abs(float(r["response"])), r["octave"], r["ly"], r["lx"]))  # the canonical detector order
        return rec
    return _GRID[detector](gray, mask, state, max_keypoints, max(grid, 1), max_iters)


def install(monkeypatch):
    """make orb_oracle.grid_detect and fast_oracle.grid_detect take the reference's three branches, so that the oracles built
    on them (tests/min_depth_oracle.py, tests/cloud_oracle.py) construct nodes with whichever detector the parameters name"""
    monkeypatch.setattr(oo, "grid_detect", lambda g, m, st, K=600, grid=3, it=5: detect(0, g, m, st, K, grid, it))
    monkeypatch.setattr(fast_oracle, "grid_detect", lambda g, m, st, K=600, grid=3, it=5: detect(1, g, m, st, K, grid, it))


def flip_image():
    """640x480 uniform noise, 128 +- 20, on which cv::ORB's quotas change the ungridded adjuster's decision at K 2730
    (min 2730, max 4095): cv::ORB(10000, ..., t) returns 377 / 2885 / 2558 keypoints at t 20 / 14 / 15, without quotas
    377 / 4518 / 3127.  From 20 the adjuster steps to 14 and accepts there, where the count without quotas is too many;
    from 15 the count with quotas is too few, the one without them accepted."""
    rng = np.random.default_rng(0)
    rng.random((480, 640))
    return (128 + (rng.random((480, 640)) - 0.5) * 40).astype(np.uint8)


def node_construct(detector, gray, depth, mask, K4, state, max_keypoints, grid, max_iters):
    """== Node::Node (node.cpp:101-240) with the detector of (grid, max_iters): orb_oracle.node_construct's steps after
    detection.  Returns (keypoints [KP_DTYPE], descriptors [n,32], xyz1 [n,4])."""
    from oracle import oracle as co
    H, W = gray.shape
    rec = detect(detector, gray, mask, state, max_keypoints, grid, max_iters)
    xy = np.array([[r["x"], r["y"]] for r in rec], np.float32).reshape(-1, 2)
    keep = np.zeros(len(rec), np.uint8)
    dcont = np.ascontiguousarray(depth, np.float32)
    if len(rec):
        co.lib().oracle_remove_depthless(xy.ctypes.data_as(C.c_void_p), C.c_int(len(rec)), dcont.ctypes.data_as(C.c_void_p),
                                         C.c_int(W), C.c_int(H), keep.ctypes.data_as(C.c_void_p))
    rec = [r for r, k in zip(rec, keep) if k]
    rec.sort(key=lambda r: (-float(r["response"]), r["cell"], r["octave"], r["ly"], r["lx"]))  # retainBest, canonical ties
    rec = rec[:max_keypoints]
    kp2, desc = oo.orb_compute(gray, oo.records_to_array(rec))
    xy = np.ascontiguousarray(np.stack([kp2["x"], kp2["y"]], 1), np.float32)
    xyz = np.zeros((len(kp2), 4), np.float32)
    keep = np.zeros(len(kp2), np.uint8)
    fn = co.lib().oracle_project_to_3d
    fn.restype = C.c_int
    n = 0
    if len(kp2):
        n = fn(xy.ctypes.data_as(C.c_void_p), C.c_int(len(kp2)), dcont.ctypes.data_as(C.c_void_p), C.c_int(W), C.c_int(H),
               C.c_double(K4[0]), C.c_double(K4[1]), C.c_double(K4[2]), C.c_double(K4[3]), C.c_double(1.0),
               C.c_int(max_keypoints), xyz.ctypes.data_as(C.c_void_p), keep.ctypes.data_as(C.c_void_p))
    assert n == len(kp2)
    return kp2, desc, xyz


def candidates(img, mask):
    """every keypoint cv::ORB finds at threshold 2 without binding quotas: (level, FAST score, Harris response) arrays"""
    allk = qo.detect(img, mask, 2, qo.UNBOUND)
    fast = {qo.key(k): k.response for k in qo.detect(img, mask, 2, qo.UNBOUND, cv2.ORB_FAST_SCORE)}
    lev = np.array([k.octave for k in allk], np.int64)
    score = np.array([fast[qo.key(k)] for k in allk], np.int64)
    harris = np.array([k.response for k in allk], np.float32)
    return lev, score, harris


def quota_counts(lev, score, harris):
    """count(t), t = 0..255: sum over levels of q_l(t) with B_l(t) = {S >= max(t, s_l)}, s_l the 2 n_l-th largest score (0 if
    fewer); q_l = |B_l| when |B_l| <= n_l, else |{k in B_l: H_k >= the n_l-th largest H of B_l}|"""
    out = np.zeros(256, np.int64)
    for l, n in enumerate(qo.N_PER_LEVEL):
        s, h = score[lev == l], harris[lev == l]
        s_l = np.sort(s)[::-1][2 * n - 1] if len(s) >= 2 * n else 0
        for t in range(256):
            b = s >= max(t, s_l)
            if b.sum() <= n:
                out[t] += b.sum()
            else:
                cut = np.sort(h[b])[::-1][n - 1]
                out[t] += int((h[b] >= cut).sum())
    return out
