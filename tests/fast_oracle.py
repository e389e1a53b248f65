"""FAST-detector Node-constructor oracle built on OpenCV itself (cv2 4.13) -- TEST INFRASTRUCTURE, not product code.

createDetector("FAST") (features.cpp:63-113) is DetectorAdjuster("FAST", 20) -> cv::FastFeatureDetector::create(int(thresh))
(feature_adjuster.cpp:88-91: FAST-9/16, non-max suppression on) under the same VideoDynamicAdaptedFeatureDetector and
VideoGridAdaptedFeatureDetector wrappers as the ORB detector.  This module is the FAST counterpart of grid_detect /
node_construct in oracle/orb_oracle.py and reuses its helpers and canonical tie orders; the Node constructor steps after
detection are the same (removeDepthless, retainBest, ORB compute, projectTo3D).  Every keypoint is on octave 0, so ties
inside a cell fall back to (y, x).

threshold_free_scores / fast_nms restate, in numpy, what the device computes: the corner score S of every pixel cv::FAST
scores (the band [3, n-4]), 0 elsewhere, a strict 3x3 maximum, the mask applied after the NMS.
"""
from __future__ import annotations

import ctypes as C

import cv2
import numpy as np

from oracle import orb_oracle as oo

# the 16-pixel Bresenham circle of radius 3 in cv::FAST order
CIRCLE = [(0, 3), (1, 3), (2, 2), (3, 1), (3, 0), (3, -1), (2, -2), (1, -3), (0, -3), (-1, -3), (-2, -2), (-3, -1), (-3, 0),
          (-3, 1), (-2, 2), (-1, 3)]


def grid_detect(gray, mask, state: oo.DetectorState, max_keypoints=600, grid=3, max_iters=5):
    """== detector->detect(gray, keypoints, mask) for the adjusted grid FAST detector."""
    H, W = gray.shape
    ncells = grid * grid
    mn, mx = max_keypoints, int(max_keypoints * 1.5)
    if grid > 1:
        cmin = int(np.floor(np.float32(mn) / np.float32(ncells) + 0.5))
        cmax = int(np.floor(np.float32(mx) / np.float32(ncells) + 0.5))
        per_cell = mx // ncells
    else:
        cmin, cmax, per_cell = mn, mx, 10 ** 9
    out = []
    for c, (y0, y1, x0, x1) in enumerate(oo._cells(W, H, grid)):
        sub = np.ascontiguousarray(gray[y0:y1, x0:x1])
        smask = None if mask is None else np.ascontiguousarray(mask[y0:y1, x0:x1])
        it = max_iters
        checked = False
        th = state.thresh[c]
        while True:
            kps = cv2.FastFeatureDetector_create(int(th)).detect(sub, smask)
            found = len(kps)
            if found < cmin:
                th = max(th * 0.7, 2.0)
                if found == 0 and not checked:
                    checked = True
                    if smask is not None and not smask.any():
                        break
            elif found > cmax:
                th = min(th * 1.3, 10000.0)
                break
            else:
                break
            it -= 1
            if not (it > 0 and 2.0 < th < 10000.0):
                break
        state.thresh[c] = th
        rec = oo._kp_records(kps, c, x0, y0)
        rec.sort(key=lambda r: (-abs(float(r["response"])), r["octave"], r["ly"], r["lx"]))  # keepStrongest, canonical ties
        out += rec[:per_cell]
    return out


def node_construct(gray, depth, mask, K4, state: oo.DetectorState, max_keypoints=600, grid=3, max_iters=5, depth_scaling=1.0):
    """== Node::Node (node.cpp:101-240) with the FAST detector.  Returns (keypoints [KP_DTYPE], descriptors [n,32], xyz1 [n,4])."""
    from oracle import oracle as co
    H, W = gray.shape
    rec = grid_detect(gray, mask, state, max_keypoints, grid, max_iters)
    xy = np.array([[r["x"], r["y"]] for r in rec], np.float32).reshape(-1, 2)
    keep = np.zeros(len(rec), np.uint8)
    dcont = np.ascontiguousarray(depth, np.float32)
    if len(rec):
        co.lib().oracle_remove_depthless(xy.ctypes.data_as(C.c_void_p), C.c_int(len(rec)), dcont.ctypes.data_as(C.c_void_p),
                                         C.c_int(W), C.c_int(H), keep.ctypes.data_as(C.c_void_p))
    rec = [r for r, k in zip(rec, keep) if k]
    rec.sort(key=lambda r: (-float(r["response"]), r["cell"], r["octave"], r["ly"], r["lx"]))  # retainBest, canonical ties
    rec = rec[:max_keypoints]
    kp2, desc = oo.orb_compute(gray, oo.records_to_array(rec))  # border filter; angle -1 is kept (no orientation)
    xy = np.ascontiguousarray(np.stack([kp2["x"], kp2["y"]], 1), np.float32)
    xyz = np.zeros((len(kp2), 4), np.float32)
    keep = np.zeros(len(kp2), np.uint8)
    fn = co.lib().oracle_project_to_3d
    fn.restype = C.c_int
    n = 0
    if len(kp2):
        n = fn(xy.ctypes.data_as(C.c_void_p), C.c_int(len(kp2)), dcont.ctypes.data_as(C.c_void_p), C.c_int(W), C.c_int(H),
               C.c_double(K4[0]), C.c_double(K4[1]), C.c_double(K4[2]), C.c_double(K4[3]), C.c_double(depth_scaling),
               C.c_int(max_keypoints), xyz.ctypes.data_as(C.c_void_p), keep.ctypes.data_as(C.c_void_p))
    assert n == len(kp2), "projectTo3D dropped a keypoint after removeDepthless (node.cpp:217-218 would assert)"
    return kp2, desc, xyz


def threshold_free_scores(img: np.ndarray) -> np.ndarray:
    """S of every pixel in [3, n-4] x [3, n-4] (0 elsewhere): the largest t for which 9 contiguous circle pixels are all
    darker than v - t or all brighter than v + t, minus 1, clamped at 0 (== cv::FAST's cornerScore<16>)."""
    h, w = img.shape
    v = img[3:h - 3, 3:w - 3].astype(np.int16)
    ring = np.stack([img[3 + dy:h - 3 + dy, 3 + dx:w - 3 + dx] for dx, dy in CIRCLE]).astype(np.int16)
    ring = np.concatenate([ring, ring[:8]])
    arc_max = np.stack([ring[k:k + 9].max(0) for k in range(16)]).min(0)
    arc_min = np.stack([ring[k:k + 9].min(0) for k in range(16)]).max(0)
    s = np.zeros(img.shape, np.int16)
    s[3:h - 3, 3:w - 3] = np.maximum(np.maximum(v - arc_max, arc_min - v) - 1, 0)
    return s


def fast_nms(img: np.ndarray, mask: np.ndarray | None, t: int):
    """{(x, y): S} of the keypoints cv::FAST(t) + runByPixelsMask finds, from the threshold-free scores."""
    s = threshold_free_scores(img)
    h, w = s.shape
    p = np.pad(s, 1)
    c = p[1:h + 1, 1:w + 1]
    ok = c >= t
    for dy in (-1, 0, 1):
        for dx in (-1, 0, 1):
            if dy or dx:
                ok &= c > p[1 + dy:h + 1 + dy, 1 + dx:w + 1 + dx]
    if mask is not None:
        ok &= mask != 0
    ys, xs = np.nonzero(ok)
    return {(int(x), int(y)): int(s[y, x]) for y, x in zip(ys, xs)}
