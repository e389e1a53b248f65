"""Bit-exact restatement of the SIFT-128 ratio matcher's GPU stages (sift_l2.cu, hamming_tc.cu) -- test helper.

  root_sift_f32          RootSIFT of k_sift_prepare: per-lane (|x|+|y|)+(|z|+|w|), xor-butterfly 16..1, sqrt(fl32(v/s))
  bf16_rne / bf16_norms  __float2bfloat16_rn of the operand tiles and k_sift_prepare's |b|^2 of the rounded rows
  l2_f32                 k_l2_refine's squared L2: per-lane fma(dx,dx,dy*dy) + fma(dz,dz,dw*dw), then the butterfly
  candidates_bf16        the tensor-core candidate set (top 4 of 2 a.b - |b|^2 on the bf16 rows, ties -> lower column),
                         with a flag for rows where fp32 accumulation error cannot change that set
  knn2_from_candidates   k_l2_refine's 2-NN among the candidates (ties -> lower index, -1 slots skipped, 3e38 sentinel)
  select_ratio           k_select_sift: ratio test in double, first passing query owns a train row, (ratio, queryIdx)
                         order, max_matches cap

A lane l of the warp that handles a 128-float row holds elements 4l..4l+3.  NumPy and the standard library only.
"""
from __future__ import annotations

from fractions import Fraction

import numpy as np

SENTINEL = np.float32(3.0e38)  # k_l2_refine's "no neighbour" distance
_LANES = np.arange(32)


def _lanes(rows: np.ndarray):
    """(..., 128) -> the four (..., 32) per-lane components x, y, z, w."""
    return rows[..., 0::4], rows[..., 1::4], rows[..., 2::4], rows[..., 3::4]


def _butterfly(s: np.ndarray) -> np.ndarray:
    """s += __shfl_xor_sync(s, o) for o = 16, 8, 4, 2, 1 over the last axis (32 lanes); every lane ends equal."""
    for o in (16, 8, 4, 2, 1):
        s = s + s[..., _LANES ^ o]
    return s[..., 0]


def _round_f32(x: Fraction, lo: np.float32, hi: np.float32) -> np.float32:
    """Round-to-nearest-even of x, which lies between the adjacent float32 values lo and hi."""
    dl, dh = abs(x - Fraction(float(lo))), abs(Fraction(float(hi)) - x)
    if dl != dh:
        return lo if dl < dh else hi
    return lo if (int(np.array(lo, np.float32).view(np.uint32)) & 1) == 0 else hi


def fma32(a, b, c) -> np.ndarray:
    """fl32(a * b + c) with one rounding, like __fmaf_rn.  a * b is exact in float64 (48-bit product), so float64 rounds
    the sum once; rounding that again to float32 is only wrong when the float64 result sits exactly on a float32
    midpoint, and those elements are redone in exact rational arithmetic."""
    a, b, c = np.broadcast_arrays(np.asarray(a, np.float32), np.asarray(b, np.float32), np.asarray(c, np.float32))
    r64 = a.astype(np.float64) * b.astype(np.float64) + c.astype(np.float64)
    with np.errstate(over="ignore"):
        r32 = r64.astype(np.float32)
    back = r32.astype(np.float64)
    diff = r64 - back
    toward = np.nextafter(r32, np.where(diff > 0, np.float32(np.inf), np.float32(-np.inf))).astype(np.float64)
    mid = np.isfinite(r64) & (diff != 0) & (r64 == (back + toward) / 2)
    if mid.any():
        r32 = r32.copy()
        for i in zip(*np.nonzero(mid)):
            x = Fraction(float(a[i])) * Fraction(float(b[i])) + Fraction(float(c[i]))
            o = np.float32(toward[i])
            lo, hi = (r32[i], o) if o > r32[i] else (o, r32[i])
            r32[i] = _round_f32(x, lo, hi)
    return r32


def root_sift_f32(desc) -> np.ndarray:
    """k_sift_prepare with root_sift = 1 (squareroot_descriptor_space, node.cpp:1557-1571), bit for bit."""
    v = np.abs(np.asarray(desc, np.float32).reshape(-1, 128))
    x, y, z, w = _lanes(v)
    s = _butterfly((x + y) + (z + w))
    out = v.copy()
    nz = s != 0
    out[nz] = np.sqrt(v[nz] / s[nz, None])
    return out


def bf16_rne(x) -> np.ndarray:
    """__float2bfloat16_rn on the uint32 bits, returned widened back to float32 (low 16 bits zero).  NaN stays NaN."""
    x = np.asarray(x, np.float32)
    bits = x.view(np.uint32).astype(np.uint64)
    r = ((bits + 0x7FFF + ((bits >> 16) & 1)) >> 16) << 16
    nan = (bits & 0x7FFFFFFF) > 0x7F800000
    r = np.where(nan, ((bits >> 16) | 0x40) << 16, r)
    return r.astype(np.uint32).view(np.float32)


def bf16_norms(rows) -> np.ndarray:
    """k_sift_prepare's |b|^2 of the bf16-rounded rows: per lane fma(f0,f0,f1*f1) + fma(f2,f2,f3*f3), butterfly."""
    x, y, z, w = _lanes(bf16_rne(np.asarray(rows, np.float32).reshape(-1, 128)))
    return _butterfly(fma32(x, x, y * y) + fma32(z, z, w * w))


def l2_f32(a, b) -> np.ndarray:
    """k_l2_refine's squared L2 distance of row pairs (a[..., :] against b[..., :]), bit for bit."""
    d = np.asarray(a, np.float32) - np.asarray(b, np.float32)
    dx, dy, dz, dw = _lanes(d)
    return _butterfly(fma32(dx, dx, dy * dy) + fma32(dz, dz, dw * dw))


def candidates_bf16(q_root, t_root, depth: int = 4, chunk: int = 512):
    """The tensor-core candidates of every query row: the `depth` best train columns by (score descending, column
    ascending), -1 past the last train row, with score = 2 a.b - |b|^2 on the bf16-rounded rows (|b|^2 as bf16_norms
    computes it), evaluated in float64.

    The GPU accumulates a.b in fp32 on the tensor cores and rounds 2 acc - |b|^2 once (fmaf).  Each of the <= 128
    accumulation steps errs by at most 2^-23 of the running sum, bounded by sum_k |a_k b_k|, so a GPU score lies within
        e = 2 * 128 * 2^-23 * sum_k |a_k b_k| + |score| * 2^-23
    of the float64 score.  `safe[i]` is set when every top-4 score minus its e exceeds every other score plus its e:
    then the GPU's 4-candidate set of row i is the restated one whatever the accumulation order.  Rows with at most 4
    train columns are always safe.  With integer rows whose products and partial sums stay below 2^24 the GPU scores are
    exact, and the restated set is the GPU's on every row, ties included."""
    qb = bf16_rne(np.asarray(q_root, np.float32).reshape(-1, 128)).astype(np.float64)
    tb = bf16_rne(np.asarray(t_root, np.float32).reshape(-1, 128)).astype(np.float64)
    nq, nt = len(qb), len(tb)
    cand = np.full((nq, depth), -1, np.int32)
    safe = np.ones(nq, bool)
    if nt == 0 or nq == 0:
        return cand, safe
    nb = bf16_norms(tb.astype(np.float32)).astype(np.float64)
    k = min(depth, nt)
    for r0 in range(0, nq, chunk):
        a = qb[r0:r0 + chunk]
        score = 2.0 * (a @ tb.T) - nb[None, :]
        order = np.argsort(-score, axis=1, kind="stable")  # stable: equal scores keep the lower column first
        cand[r0:r0 + chunk, :k] = order[:, :k]
        if nt > 4:
            err = 2.0 * 128 * 2.0 ** -23 * (np.abs(a) @ np.abs(tb).T) + np.abs(score) * 2.0 ** -23
            s = np.take_along_axis(score, order, 1)
            e = np.take_along_axis(err, order, 1)
            safe[r0:r0 + chunk] = (s[:, :4] - e[:, :4]).min(1) > (s[:, 4:] + e[:, 4:]).max(1)
    return cand, safe


def knn2_from_candidates(q, t, cand4):
    """k_l2_refine: exact fp32 squared L2 to each candidate column, then the 2 best by (distance, index) in candidate
    order.  Returns idx (n, 2) int32 (-1 = none) and dist (n, 2) float32 (3e38 = none), as knn2_l2 does."""
    q = np.asarray(q, np.float32).reshape(-1, 128)
    t = np.asarray(t, np.float32).reshape(-1, 128)
    cand = np.asarray(cand4, np.int32).reshape(len(q), 4)
    n = len(q)
    valid = cand >= 0
    d = np.full((n, 4), SENTINEL, np.float32)
    if valid.any():
        rows, ks = np.nonzero(valid)
        d[rows, ks] = l2_f32(q[rows], t[cand[rows, ks]])
    b1 = np.full(n, -1, np.int32); b2 = np.full(n, -1, np.int32)
    d1 = np.full(n, SENTINEL, np.float32); d2 = np.full(n, SENTINEL, np.float32)
    for k in range(4):
        c, dk, v = cand[:, k], d[:, k], valid[:, k]
        first = v & ((dk < d1) | ((dk == d1) & (c < b1)))
        second = v & ~first & ((dk < d2) | ((dk == d2) & (c < b2)))
        b2 = np.where(first, b1, np.where(second, c, b2)); d2 = np.where(first, d1, np.where(second, dk, d2))
        b1 = np.where(first, c, b1); d1 = np.where(first, dk, d1)
    return np.stack([b1, b2], 1).astype(np.int32), np.stack([d1, d2], 1).astype(np.float32)


MATCH_DTYPE = np.dtype([("queryIdx", "<i4"), ("trainIdx", "<i4"), ("distance", "<f4")])


def select_ratio(knn, nn_ratio: float, max_matches: int) -> np.ndarray:
    """k_select_sift (node.cpp:638-667, 674, 1127) on a knn2 table (idx (n, 2), dist (n, 2)).  A query with both
    neighbours passes when nn_ratio > fl32(d1 / d2), compared in double as the reference's `double max_dist_ratio_fac`
    does; 0/0 is NaN and fails.  Among passing queries the lowest index owns its train row (later ones are dropped even
    with a better ratio); distance = the ratio; order (ratio, queryIdx); cut at max_matches."""
    idx, dist = knn
    idx = np.asarray(idx, np.int32).reshape(-1, 2)
    dist = np.asarray(dist, np.float32).reshape(-1, 2)
    with np.errstate(divide="ignore", invalid="ignore"):
        ratio = dist[:, 0] / dist[:, 1]
    ok = (idx[:, 0] >= 0) & (idx[:, 1] >= 0) & (float(nn_ratio) > ratio.astype(np.float64))
    q = np.nonzero(ok)[0]
    _, first = np.unique(idx[q, 0], return_index=True)  # q is ascending, so the first occurrence is the lowest query
    q = q[first]
    m = np.zeros(len(q), MATCH_DTYPE)
    m["queryIdx"], m["trainIdx"], m["distance"] = q, idx[q, 0], ratio[q]
    return m[np.lexsort((m["queryIdx"], m["distance"]))][:max_matches]


def threshold_rows():
    """Three integer query rows with squared distances (19, 20), (20, 21), (18, 19) to train rows (0, 1), (2, 3),
    (4, 5); every other train row is far away.  fl32(19 / 20) = fl32(0.95) sits exactly at the default threshold."""
    q = np.zeros((3, 128), np.float32)
    t = np.zeros((6, 128), np.float32)
    offs = [([3, 3, 1], [4, 2]), ([4, 2], [4, 2, 1]), ([3, 3], [3, 3, 1])]
    for k, (u, w) in enumerate(offs):
        q[k, 40 * k] = 200.0
        t[2 * k] = q[k]
        t[2 * k, 40 * k + 1:40 * k + 1 + len(u)] += u
        t[2 * k + 1] = q[k]
        t[2 * k + 1, 40 * k + 20:40 * k + 20 + len(w)] += w
    return q, t
