"""use_feature_min_depth Node-constructor oracle -- TEST INFRASTRUCTURE, not product code.

With use_feature_min_depth (parameter_server.cpp:90) the Node constructor takes as a keypoint's depth the nearest point of
its neighbourhood, getMinDepthInNeighborhood(depth, kp.pt, kp.size) (misc.cpp:774-791), in removeDepthless (node.cpp:82-83)
and projectTo3D (:940-941).  This module restates that rule in numpy and builds Node::Node with it on top of the ORB and
FAST detection oracles (oracle/orb_oracle.py, tests/fast_oracle.py), with their canonical tie orders.

The rule (the reference's C++ arithmetic):
  radius = int((size - 1) / 2)                              float, truncated
  top = max(int(y - r), 0), left = max(int(x - r), 0)       float, truncated toward zero
  bot = min(int(y + r), rows), right = min(int(x + r), cols)
  Z = min over depth[top:bot, left:right]                   cv::minMaxLoc on the ROI cv::Mat(depth, Range, Range)
  Z == 0 (or -0) -> NaN                                     the reference's FIXME branch
NaN pixels are ignored and a window without a number gives NaN: what OpenCV 3.x's scalar minMaxIdx does (a NaN never
compares below the running minimum; nothing found reads as 0, which the reference turns into NaN).  cv2 4.13's vectorised
minMaxIdx is not used for windows with NaN: its answer there depends on the SIMD lane layout (DESIGN.md 4.5.2).
"""
from __future__ import annotations

import numpy as np

from oracle import orb_oracle as oo

NAN = np.float32("nan")


def radius(size) -> int:
    return int((np.float32(size) - np.float32(1)) / np.float32(2))


def window(depth: np.ndarray, x, y, size) -> np.ndarray:
    """The neighbourhood of the keypoint as a slice (a view) of the full frame, as cv::Mat(depth, Range, Range) is."""
    H, W = depth.shape
    r = np.float32(radius(size))
    top = max(int(np.float32(y) - r), 0)
    left = max(int(np.float32(x) - r), 0)
    bot = min(int(np.float32(y) + r), H)
    right = min(int(np.float32(x) + r), W)
    return depth[top:bot, left:right]


def min_depth(depth: np.ndarray, x, y, size) -> np.float32:
    """getMinDepthInNeighborhood(depth, (x, y), size) with NaN pixels ignored."""
    w = window(depth, x, y, size)
    v = w[~np.isnan(w)]
    if v.size == 0:
        return NAN
    m = np.float32(v.min())
    return NAN if m == 0 else m


def _inside(x, y, W, H) -> bool:
    return not (x >= W or x < 0 or y >= H or y < 0 or np.isnan(x) or np.isnan(y))


def node_construct(gray, depth, mask, K4, state: oo.DetectorState, max_keypoints=600, grid=3, max_iters=5, depth_scaling=1.0,
                   detector="ORB"):
    """== Node::Node (node.cpp:101-240) with use_feature_min_depth, for the ORB or the FAST detector.
    Returns (keypoints [KP_DTYPE], descriptors [n,32], xyz1 [n,4])."""
    import fast_oracle
    H, W = gray.shape
    depth = np.asarray(depth, np.float32)
    detect = {"ORB": oo.grid_detect, "FAST": fast_oracle.grid_detect}[detector]
    rec = detect(gray, mask, state, max_keypoints, grid, max_iters)
    # removeDepthless (node.cpp:67-97) with the neighbourhood depth
    rec = [r for r in rec if _inside(r["x"], r["y"], W, H) and not np.isnan(min_depth(depth, r["x"], r["y"], r["size"]))]
    rec.sort(key=lambda r: (-float(r["response"]), r["cell"], r["octave"], r["ly"], r["lx"]))  # retainBest, canonical ties
    rec = rec[:max_keypoints]
    kp2, desc = oo.orb_compute(gray, oo.records_to_array(rec))  # border filter + stable octave sort
    # second removeDepthless (the same rule on the same keypoints: a no-op) + projectTo3D (node.cpp:206-210, 900-965)
    fxinv, fyinv = np.float32(1.0 / K4[0]), np.float32(1.0 / K4[1])
    cx, cy = np.float32(K4[2]), np.float32(K4[3])
    xyz = np.zeros((len(kp2), 4), np.float32)
    for i, k in enumerate(kp2):
        x, y = np.float32(k["x"]), np.float32(k["y"])
        Z = min_depth(depth, x, y, k["size"])
        assert _inside(x, y, W, H) and not np.isnan(Z), "projectTo3D dropped a keypoint after removeDepthless"
        Z = np.float32(np.float64(Z) * np.float64(depth_scaling))
        xyz[i] = ((x - cx) * Z * fxinv, (y - cy) * Z * fyinv, Z, np.float32(1))
    assert len(kp2) <= max_keypoints
    return kp2, desc, xyz
