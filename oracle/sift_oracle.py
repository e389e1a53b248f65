"""Oracle of the float-descriptor (SIFT-128) branch -- TEST INFRASTRUCTURE, not product code.

  root_sift            squareroot_descriptor_space (node.cpp:1557-1571)
  knn2_exact           exact 2-NN by squared L2 (what cv::flann::Index::knnSearch returns, node.cpp:1573-1581, when the
                       kd-tree search is exhaustive).  The reference's FLANN kd-tree (4 trees, 16 checks) is approximate;
                       the CUDA path replaces it with an exact search, so the oracle is the exact 2-NN ("semantic superset",
                       SURVEY.md 8a-a10).  float64 arithmetic on the float32 RootSIFT rows.
  feature_matching     node.cpp:638-667: ratio = d1/d2 < nn_distance_ratio, first-come unique trainIdx, distance = ratio,
                       then keepStrongestMatches (node.cpp:674) + the sort of node.cpp:1127.
"""
from __future__ import annotations

import ctypes as C

import numpy as np

from . import oracle as co


def root_sift(desc: np.ndarray) -> np.ndarray:
    d = np.abs(np.asarray(desc, np.float32))
    s = d.sum(1, dtype=np.float32)
    out = d.copy()
    nz = s != 0
    out[nz] = np.sqrt(d[nz] / s[nz, None]).astype(np.float32)
    return out


def knn2_exact(q: np.ndarray, t: np.ndarray):
    q64, t64 = q.astype(np.float64), t.astype(np.float64)
    D = (q64 * q64).sum(1)[:, None] + (t64 * t64).sum(1)[None, :] - 2 * q64 @ t64.T
    D = np.maximum(D, 0)
    idx = np.argsort(D, axis=1, kind="stable")[:, :2]
    d = np.take_along_axis(D, idx, 1)
    return idx.astype(np.int32), d


def feature_matching(q_root, t_root, nn_ratio=0.95, max_matches=300):
    idx, d = knn2_exact(q_root, t_root)
    out = []
    seen = set()
    for i in range(len(q_root)):
        ratio = np.float32(np.float32(d[i, 0]) / np.float32(d[i, 1]))
        # `double max_dist_ratio_fac > float dist_ratio_fac` compares in double; NumPy would compare a Python float
        # with a float32 in float32 and reject fl32(0.95) = 0.949999988 against 0.95
        if float(nn_ratio) > float(ratio):
            t = int(idx[i, 0])
            if t in seen:
                continue
            seen.add(t)
            out.append((i, t, -1, ratio))
    m = np.array(out, dtype=co.DMATCH_DTYPE) if out else np.zeros(0, co.DMATCH_DTYPE)
    order = np.lexsort((m["queryIdx"], m["distance"]))
    return m[order][:max_matches]


def match_node_pair(params, desc_newer, xyz_newer, id_newer, desc_older, xyz_older, id_older, seed, pair, nn_ratio=0.95,
                    use_root_sift=True):
    qn = root_sift(desc_newer) if use_root_sift else np.asarray(desc_newer, np.float32)
    tn = root_sift(desc_older) if use_root_sift else np.asarray(desc_older, np.float32)
    m = np.ascontiguousarray(feature_matching(qn, tn, nn_ratio, params.max_matches))
    res = np.zeros(1, co.RESULT_DTYPE)
    inl = np.zeros(max(params.max_matches, 1), co.DMATCH_DTYPE)
    x1 = np.ascontiguousarray(xyz_newer, np.float32); x2 = np.ascontiguousarray(xyz_older, np.float32)
    co.lib().oracle_match_node_pair_from_matches(C.byref(params), co._p(x1), C.c_int(id_newer), co._p(x2), C.c_int(id_older),
                                                 co._p(m) if len(m) else None, C.c_int(len(m)), C.c_uint64(seed), C.c_uint64(pair),
                                                 co._p(res), co._p(inl))
    return res[0], m, inl[: res[0]["n_inliers"]]


# ---------------------------------------------------------------------------------------------------
# matcher_type == "SIFTGPU" (node.cpp:553-557): SiftMatchGPU as vendored under external/SiftGPU.  Restated from the
# CUDA sources (the library itself needs GL/GLEW and is not buildable here -> parity unpinned for this branch).

def siftgpu_quantise(desc: np.ndarray) -> np.ndarray:
    """SiftMatchCU::SetDescriptors(float) (SiftMatchCU.cpp:87-101): pub[i] = int(512 * d + 0.5) stored in an unsigned char
    (wraps mod 256).  `512 * d` is a float product, `+ 0.5` promotes to double, int() truncates."""
    d = np.asarray(desc, np.float32)
    v = ((np.float32(512.0) * d).astype(np.float64) + 0.5).astype(np.int64)
    return (v & 0xFF).astype(np.uint8)


def _siftgpu_dist(dot: np.ndarray) -> np.ndarray:
    """acos(min(dot * 2^-18, 1.0)) -- float product, double min / acos, stored to float (ProgramCU.cu:1739-1740)."""
    prod = (dot.astype(np.float32) * np.float32(0.000003814697265625)).astype(np.float64)
    return np.arccos(np.minimum(prod, 1.0)).astype(np.float32)


def siftgpu_row_match(dot: np.ndarray, distmax=0.9, ratiomax=0.9) -> np.ndarray:
    """RowMatch_Kernel (ProgramCU.cu:1689-1745): per row the largest dot product, the runner-up VALUE (duplicates of the
    maximum count) and the index of the maximum.  32 threads stride the row (strict >, so each thread keeps its first
    maximum), then a tree reduction where the lower thread wins ties: the winner among equal maxima is the column with the
    smallest (col % 32, col).  Only dots > 0 register (initial max 0, index -1)."""
    n1, n2 = dot.shape
    out = np.full(n1, -1, np.int32)
    if n2 == 0:
        return out
    cols = np.arange(n2)
    prio = (cols % 32) * 4096 + cols // 32
    for r in range(n1):
        v = dot[r].astype(np.int64)
        mx = int(v.max())
        if mx <= 0:
            continue
        cand = np.nonzero(v == mx)[0]
        j = int(cand[np.argmin(prio[cand])])
        rest = np.delete(v, j)
        nxt = max(int(rest.max()) if len(rest) else 0, 0)
        dist, distn = _siftgpu_dist(np.array([mx]))[0], _siftgpu_dist(np.array([nxt]))[0]
        if dist < np.float32(distmax) and dist < np.float32(distn * np.float32(ratiomax)):
            out[r] = j
    return out


def siftgpu_col_match(dot: np.ndarray, distmax=0.9, ratiomax=0.9) -> np.ndarray:
    """MultiplyDescriptor_Kernel's per-8-row partial results + ColMatch_Kernel (ProgramCU.cu:1463-1478, 1764-1784): per
    column the largest dot (lowest row wins ties: strict > inside a block, strict < across blocks), runner-up value."""
    n1, n2 = dot.shape
    out = np.full(n2, -1, np.int32)
    for c in range(n2):
        v = dot[:, c].astype(np.int64)
        mx = int(v.max()) if n1 else 0
        if mx <= 0:
            continue  # make_int3(0, -1, 0) survives
        j = int(np.argmax(v))
        rest = np.delete(v, j)
        nxt = max(int(rest.max()) if len(rest) else 0, 0)
        dist, distn = _siftgpu_dist(np.array([mx]))[0], _siftgpu_dist(np.array([nxt]))[0]
        if dist < np.float32(distmax) and dist < np.float32(distn * np.float32(ratiomax)):
            out[c] = j
    return out


def siftgpu_match(desc1: np.ndarray, desc2: np.ndarray, distmax=0.9, ratiomax=0.9):
    """SiftGPUWrapper::match (sift_gpu_wrapper.cpp:169-227) on GetSiftMatch(num1, buf, 0.9, 0.9) with mutual best match
    (SiftMatchCU.cpp:139-176).  Returns DMatch records (queryIdx, trainIdx, imgIdx -1, distance = float L2 of the float
    descriptors, accumulated in index order) in ascending query order, BEFORE keepStrongestMatches."""
    d1, d2 = np.asarray(desc1, np.float32), np.asarray(desc2, np.float32)
    if len(d1) == 0 or len(d2) == 0:
        return np.zeros(0, co.DMATCH_DTYPE)
    q1, q2 = siftgpu_quantise(d1).astype(np.float64), siftgpu_quantise(d2).astype(np.float64)
    dot = (q1 @ q2.T).astype(np.int64)  # every dot and partial sum is an integer below 128 * 255^2 < 2^53: exact
    rows, colsm = siftgpu_row_match(dot, distmax, ratiomax), siftgpu_col_match(dot, distmax, ratiomax)
    pairs = [(i, int(rows[i])) for i in range(len(d1)) if rows[i] >= 0 and colsm[rows[i]] == i]
    out = []
    counter = 0
    for i, j in pairs:
        if i == 0 or j == 0:
            counter += 1  # "opengl context problem" heuristic (:204-213)
        if counter > 0.5 * len(pairs):
            return np.zeros(0, co.DMATCH_DTYPE)
        s = np.float32(0)
        for a in (d1[i] - d2[j]):
            s = np.float32(s + np.float32(a * a))
        out.append((i, j, -1, np.sqrt(s, dtype=np.float32)))
    return np.array(out, dtype=co.DMATCH_DTYPE) if out else np.zeros(0, co.DMATCH_DTYPE)


def siftgpu_feature_matching(desc1, desc2, max_matches=300):
    """+ keepStrongestMatches (node.cpp:674) and the sort of node.cpp:1127 (ties: query index, the library's canonical order)."""
    m = siftgpu_match(desc1, desc2)
    order = np.lexsort((m["queryIdx"], m["distance"]))
    return m[order][:max_matches]
