"""ORB / Node-constructor oracle built on OpenCV itself (cv2 4.13) -- TEST INFRASTRUCTURE, not product code.

The reference delegates keypoint detection and description to OpenCV (feature_adjuster.cpp:94,121; features.cpp:117-119;
node.cpp:160,189,202), so cv2 IS the arithmetic the reference runs (SURVEY.md 8c treats cv2 as ground truth for a2/a4/a5;
the reference targeted OpenCV 3.x, parity with 4.13 is what can be pinned here).  This module restates only the
reference's own glue around it:
  grid_detect      VideoGridAdaptedFeatureDetector::detect (feature_adjuster.cpp:286-317) over
                   VideoDynamicAdaptedFeatureDetector::detect (:185-224) over DetectorAdjuster (:85-150)
  node_construct   Node::Node (node.cpp:101-240): detect -> removeDepthless -> retainBest -> compute -> projectTo3D
Where the reference's order is unspecified (std::nth_element in keepStrongest / retainBest) a canonical order is used,
the same one the CUDA path documents: inside a cell |response| descending then (level, y, x); node features by
(octave, response descending, cell, y, x).
"""
from __future__ import annotations

import ctypes as C

import cv2
import numpy as np

KP_DTYPE = np.dtype([("x", "<f4"), ("y", "<f4"), ("size", "<f4"), ("angle", "<f4"), ("response", "<f4"),
                     ("octave", "<i4"), ("class_id", "<i4")])


def layer_scale(level: int) -> np.float32:
    return np.float32(np.float64(np.float32(1.2)) ** level)


def level_side(n: int, level: int) -> int:
    """a pyramid level's side as cv::ORB sizes it: cvRound(n * (1.f / scale)) in float (orb.cpp detectAndCompute)"""
    return n if level == 0 else int(np.rint(np.float32(n) * (np.float32(1) / layer_scale(level))))


def depth_to_mask(depth: np.ndarray) -> np.ndarray:
    """depthToCV8UC1 (misc.cpp:414-418): depth.convertTo(mono8, CV_8UC1, 100, 0) = saturate_cast<uchar>(cvRound(d * 100)),
    NaN -> 0, negative -> 0.  cv2's Python API has no Mat::convertTo; convertScaleAbs is the same conversion of |d * 100|,
    so negative depths (which convertTo saturates to 0) are cleared afterwards."""
    m = cv2.convertScaleAbs(depth, alpha=100)
    m[depth < 0] = 0
    return m


class DetectorState:
    """The persistent per-cell thresholds of the adjusted grid detector (features.cpp:92: initial 20)."""

    def __init__(self, ncells=9):
        self.thresh = [20.0] * 16


def _cells(W, H, grid, edge=31):
    out = []
    for i in range(grid):
        for j in range(grid):
            if grid == 1:
                out.append((0, H, 0, W))
                continue
            y0 = max((i * H) // grid - edge, 0); y1 = min(H, ((i + 1) * H) // grid + edge)
            x0 = max((j * W) // grid - edge, 0); x1 = min(W, ((j + 1) * W) // grid + edge)
            out.append((y0, y1, x0, x1))
    return out


def _kp_records(kps, cell, x0, y0):
    rec = []
    for k in kps:
        sc = layer_scale(k.octave)
        lx = int(round(float(np.float32(k.pt[0]) / sc))); ly = int(round(float(np.float32(k.pt[1]) / sc)))
        assert np.float32(lx) * sc == np.float32(k.pt[0]) and np.float32(ly) * sc == np.float32(k.pt[1])
        rec.append(dict(x=np.float32(np.float32(k.pt[0]) + np.float32(x0)), y=np.float32(np.float32(k.pt[1]) + np.float32(y0)),
                        size=np.float32(k.size), angle=np.float32(k.angle), response=np.float32(k.response),
                        octave=int(k.octave), cell=cell, lx=lx, ly=ly))
    return rec


def grid_detect(gray, mask, state: DetectorState, max_keypoints=600, grid=3, max_iters=5):
    """== detector->detect(gray, keypoints, mask) for the adjusted grid ORB detector."""
    H, W = gray.shape
    ncells = grid * grid
    mn, mx = max_keypoints, int(max_keypoints * 1.5)
    if grid > 1:
        # gridmin = round(min / static_cast<float>(gridcells)), likewise gridmax (features.cpp:52-53): C round(), half away from 0
        cmin = int(np.floor(np.float32(mn) / np.float32(ncells) + 0.5))
        cmax = int(np.floor(np.float32(mx) / np.float32(ncells) + 0.5))
        per_cell = mx // ncells
    else:
        cmin, cmax, per_cell = mn, mx, 10 ** 9
    out = []
    for c, (y0, y1, x0, x1) in enumerate(_cells(W, H, grid)):
        sub = np.ascontiguousarray(gray[y0:y1, x0:x1])
        smask = None if mask is None else np.ascontiguousarray(mask[y0:y1, x0:x1])
        it = max_iters
        checked = False
        th = state.thresh[c]
        while True:
            det = cv2.ORB_create(10000, 1.2, 8, 15, 0, 2, 0, 31, int(th))
            kps = det.detect(sub, smask)
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
        rec = _kp_records(kps, c, x0, y0)
        rec.sort(key=lambda r: (-abs(float(r["response"])), r["octave"], r["ly"], r["lx"]))  # keepStrongest, canonical ties
        out += rec[:per_cell]
    return out


def records_to_array(rec):
    a = np.zeros(len(rec), KP_DTYPE)
    for i, r in enumerate(rec):
        a[i] = (r["x"], r["y"], r["size"], r["angle"], r["response"], r["octave"], -1)
    return a


def orb_compute(gray, kp_array):
    """== extractor->compute(gray, keypoints, descriptors) with cv2.ORB_create() defaults."""
    kps = [cv2.KeyPoint(float(k["x"]), float(k["y"]), float(k["size"]), float(k["angle"]), float(k["response"]), int(k["octave"]), -1)
           for k in kp_array]
    ext = cv2.ORB_create()
    kps2, desc = ext.compute(gray, kps)
    out = np.zeros(len(kps2), KP_DTYPE)
    for i, k in enumerate(kps2):
        out[i] = (k.pt[0], k.pt[1], k.size, k.angle, k.response, k.octave, -1)
    if desc is None:
        desc = np.zeros((0, 32), np.uint8)
    return out, desc


def node_construct(gray, depth, mask, K4, state: DetectorState, max_keypoints=600, grid=3, max_iters=5, depth_scaling=1.0):
    """== Node::Node (node.cpp:101-240).  Returns (keypoints [KP_DTYPE], descriptors [n,32], xyz1 [n,4])."""
    from . import oracle as co
    H, W = gray.shape
    rec = grid_detect(gray, mask, state, max_keypoints, grid, max_iters)
    # removeDepthless (node.cpp:67-97)
    xy = np.array([[r["x"], r["y"]] for r in rec], np.float32).reshape(-1, 2)
    keep = np.zeros(len(rec), np.uint8)
    dcont = np.ascontiguousarray(depth, np.float32)
    if len(rec):
        co.lib().oracle_remove_depthless(xy.ctypes.data_as(C.c_void_p), C.c_int(len(rec)), dcont.ctypes.data_as(C.c_void_p),
                                         C.c_int(W), C.c_int(H), keep.ctypes.data_as(C.c_void_p))
    rec = [r for r, k in zip(rec, keep) if k]
    # retainBest(max_keypoints) + resize (node.cpp:187-191): canonical order, cut at K
    rec.sort(key=lambda r: (-float(r["response"]), r["cell"], r["octave"], r["ly"], r["lx"]))
    rec = rec[:max_keypoints]
    # compute(): border filter + stable octave sort happen inside cv2
    kp = records_to_array(rec)
    cells = np.array([r["cell"] for r in rec])
    kp2, desc = orb_compute(gray, kp)
    # second removeDepthless (no-op) + projectTo3D (node.cpp:206-210)
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
