"""Point-cloud Node-constructor oracle -- TEST INFRASTRUCTURE, not product code.

Node(visual, detector, extractor, point_cloud, detection_mask) (node.cpp:252-369) is what the reference runs for registered
Kinect clouds, stereo cameras and PCD replay (openni_listener.cpp:536-594, 676-758).  Per frame:
  cvtColor(visual, gray, CV_RGB2GRAY) for a CV_8UC3 visual (:275-277)
  detector->detect(gray, kp, mask)            the ORB / FAST grid oracles (oracle/orb_oracle.py, tests/fast_oracle.py)
  projectTo3D(kp, pts, cloud) (:309, 855-898) detector order; drop a keypoint outside the image or whose cloud point at
                                              ((int)x, (int)y) has a NaN coordinate; point = (x, y, z, 1) as stored; stop at
                                              max_keypoints kept points.  maximum_depth = +inf (its default): never drops.
  extractor->compute(gray, kp, desc) (:312)   cv2 ORB: 31 px border filter + stable octave sort
The reference does not carry feature_locations_3d_ through compute(); the library does (decision recorded in DESIGN.md 4.5.3),
and so does this oracle: each keypoint enters compute() with class_id = its index, which cv2 keeps while it drops and
re-orders keypoints, and leaves with class_id = -1 as the library writes it.

Also restated here: calculateDepthMask (openni_listener.cpp:520-534) with x86-64's conversion of z * 50.0 to uchar, and
OpenCV 4's 15-bit RGB -> grey conversion.
"""
from __future__ import annotations

import cv2
import numpy as np

from oracle import orb_oracle as oo

POINT_FLOATS = {"XYZRGB": 8, "XYZ": 4}  # pcl::PointXYZRGB (32 B) / pcl::PointXYZ (16 B): x, y, z at floats 0, 1, 2


def rgb_to_gray(rgb: np.ndarray) -> np.ndarray:
    """cv::cvtColor(CV_RGB2GRAY) of cv2 4.13: (R * 9798 + G * 19235 + B * 3735 + 2^14) >> 15, channel 0 = R."""
    c = rgb.astype(np.uint32)
    return ((c[..., 0] * 9798 + c[..., 1] * 19235 + c[..., 2] * 3735 + (1 << 14)) >> 15).astype(np.uint8)


def cloud_mask(z: np.ndarray) -> np.ndarray:
    """calculateDepthMask: static_cast<uchar>(z * 50.0) as x86-64 emits it (cvttsd2si: truncate to int32, 0x80000000 when
    the result does not fit; keep the low byte), 0 for NaN."""
    v = np.asarray(z, np.float32).astype(np.float64) * 50.0
    fits = (v > -2147483649.0) & (v < 2147483648.0)  # False for NaN and +-inf
    iv = np.where(fits, np.trunc(np.where(fits, v, 0.0)), -2147483648.0).astype(np.int64)
    out = (iv & 0xFF).astype(np.uint8)
    out[np.isnan(np.asarray(z, np.float32))] = 0
    return out


def cloud_from_depth(depth: np.ndarray, K4, point_type: str = "XYZRGB", rgb: np.ndarray | None = None) -> np.ndarray:
    """An organised cloud [H, W, 8 | 4] float32 back-projected from a depth image (what a registered depth camera driver
    publishes); NaN depth gives an all-NaN point.  The colour float of PointXYZRGB is packed b, g, r, a; padding floats 0."""
    H, W = depth.shape
    fx, fy, cx, cy = (np.float32(k) for k in K4)
    v, u = np.mgrid[0:H, 0:W].astype(np.float32)
    z = depth.astype(np.float32)
    cl = np.zeros((H, W, POINT_FLOATS[point_type]), np.float32)
    cl[..., 0] = (u - cx) * z / fx
    cl[..., 1] = (v - cy) * z / fy
    cl[..., 2] = z
    cl[np.isnan(z), :3] = np.nan
    if point_type == "XYZRGB":
        bgra = np.zeros((H, W, 4), np.uint8)
        if rgb is not None:
            bgra[..., 0], bgra[..., 1], bgra[..., 2] = rgb[..., 2], rgb[..., 1], rgb[..., 0]
        bgra[..., 3] = 255
        cl[..., 4] = bgra.view(np.float32)[..., 0]
    return cl


def project_to_3d(rec, cloud: np.ndarray, max_keypoints: int):
    """projectTo3D(kp, pts, cloud) (node.cpp:855-898): (kept records, their points [n, 4])."""
    H, W = cloud.shape[:2]
    kept, pts = [], []
    for r in rec:
        x, y = np.float32(r["x"]), np.float32(r["y"])
        if x >= W or x < 0 or y >= H or y < 0 or np.isnan(x) or np.isnan(y):
            continue
        p = cloud[int(y), int(x)]
        if np.isnan(p[0]) or np.isnan(p[1]) or np.isnan(p[2]):  # p.z > maximum_depth (+inf) never holds
            continue
        kept.append(r)
        pts.append((p[0], p[1], p[2], np.float32(1)))
        if len(kept) >= max_keypoints:
            break
    return kept, np.array(pts, np.float32).reshape(-1, 4)


def compute_tracked(gray, rec):
    """cv2 ORB compute() on the records with class_id = input index: (keypoints [KP_DTYPE], descriptors, input index of each
    output keypoint)."""
    kps = [cv2.KeyPoint(float(r["x"]), float(r["y"]), float(r["size"]), float(r["angle"]), float(r["response"]), int(r["octave"]), i)
           for i, r in enumerate(rec)]
    kps2, desc = cv2.ORB_create().compute(gray, kps)
    out = np.zeros(len(kps2), oo.KP_DTYPE)
    src = np.zeros(len(kps2), np.int64)
    for i, k in enumerate(kps2):
        out[i] = (k.pt[0], k.pt[1], k.size, k.angle, k.response, k.octave, -1)
        src[i] = k.class_id
    if desc is None:
        desc = np.zeros((0, 32), np.uint8)
    return out, desc, src


def detect(gray, mask, state: oo.DetectorState, max_keypoints=600, grid=3, max_iters=5, detector="ORB"):
    import fast_oracle
    fn = {"ORB": oo.grid_detect, "FAST": fast_oracle.grid_detect}[detector]
    return fn(gray, mask, state, max_keypoints, grid, max_iters)


def node_construct(visual, cloud, mask, state: oo.DetectorState, max_keypoints=600, grid=3, max_iters=5, detector="ORB"):
    """== Node(visual, detector, extractor, point_cloud, detection_mask) with 3-D points kept with their keypoints.
    visual: [H, W] grey or [H, W, 3] colour; cloud: [H, W, 4 | 8] float32.  Returns (keypoints, descriptors [n,32], xyz1 [n,4])."""
    gray = rgb_to_gray(visual) if visual.ndim == 3 else visual
    rec = detect(gray, mask, state, max_keypoints, grid, max_iters, detector)
    kept, pts = project_to_3d(rec, cloud, max_keypoints)
    kp, desc, src = compute_tracked(gray, kept)
    return kp, desc, pts[src].reshape(-1, 4)
