"""Diagnostic (GPU box): compare the GPU FAST/NMS candidates of one grid cell with the numpy restatement."""
import sys
from pathlib import Path
sys.path.insert(0, str(Path(__file__).resolve().parent.parent))
import numpy as np
from oracle import orb_oracle
from rgbdslam_v2_b200 import Frontend, synth
from rgbdslam_v2_b200._capi import default_params

CIRC = [(0, 3), (1, 3), (2, 2), (3, 1), (3, 0), (3, -1), (2, -2), (1, -3), (0, -3), (-1, -3), (-2, -2), (-3, -1), (-3, 0), (-3, 1), (-2, 2), (-1, 3)]


def resize_exact(src, dw, dh):
    sh, sw = src.shape
    def coeffs(dst_n, src_n):
        scale = src_n / dst_n
        d = np.arange(dst_n); f = (d + 0.5) * scale - 0.5
        i = np.floor(f).astype(np.int64); fr = f - i
        lo = i < 0; i[lo] = 0; fr[lo] = 0
        hi = i >= src_n - 1; i[hi] = src_n - 1; fr[hi] = 0
        c1 = np.round(fr * 256).astype(np.int64)
        return i, 256 - c1, c1
    ox, ax0, ax1 = coeffs(dw, sw); oy, ay0, ay1 = coeffs(dh, sh)
    s = src.astype(np.int64)
    x1 = np.minimum(ox + 1, sw - 1)
    Hh = s[:, ox] * ax0[None, :] + s[:, x1] * ax1[None, :]
    y1 = np.minimum(oy + 1, sh - 1)
    V = Hh[oy, :] * ay0[:, None] + Hh[y1, :] * ay1[:, None]
    return ((V + (1 << 15)) >> 16).astype(np.uint8)


def score_map(img):
    H, W = img.shape; I = img.astype(np.int32)
    S = np.zeros((H, W), np.int32)
    c = I[3:H - 3, 3:W - 3]
    d = np.stack([c - I[3 + dy:H - 3 + dy, 3 + dx:W - 3 + dx] for dx, dy in CIRC], 0)
    d2 = np.concatenate([d, d[:9]], 0)
    A = np.zeros_like(c)
    for k in range(16):
        arc = d2[k:k + 9]
        A = np.maximum(A, np.maximum(arc.min(0), (-arc).min(0)))
    S[3:H - 3, 3:W - 3] = np.maximum(A - 1, 0)
    return S


p = default_params(); p.depth_cov_z0 = 2.0; p.max_keypoints = 600
fe = Frontend(0, p)
poses = synth.trajectory(40)
det = fe.detector_create()
gray, depth = synth.render_frame(poses[0], seed=0)
gkp = fe.orb_detect(det, gray, None)
cells = orb_oracle._cells(640, 480, 3)
for cell in (0, 4):
    y0, y1, x0, x1 = cells[cell]
    sub = np.ascontiguousarray(gray[y0:y1, x0:x1])
    for l in (0, 1):
        gi = fe.orb_debug_plane(0, cell, l); gm = fe.orb_debug_plane(1, cell, l)
        ref = sub if l == 0 else resize_exact(sub, gi.shape[1], gi.shape[0])
        print(f"cell {cell} level {l}: img shape {gi.shape} equal {np.array_equal(gi, ref)} ndiff {(gi != ref).sum() if gi.shape == ref.shape else -1}; mask all255 {(gm == 255).all()}")
    cand, resp, thr = fe.orb_debug_candidates(cell)
    y0, y1, x0, x1 = cells[cell]
    sub = np.ascontiguousarray(gray[y0:y1, x0:x1])
    print(f"cell {cell} rect {cells[cell]} gpu candidates {len(cand)} thr {thr} survivors {(~np.isnan(resp)).sum()}")
    lv = sub
    for l in range(8):
        if l > 0:
            sc = orb_oracle.layer_scale(l)
            w = int(np.rint(np.float32(sub.shape[1]) / sc)); h = int(np.rint(np.float32(sub.shape[0]) / sc))
            lv = resize_exact(lv, w, h)
        S = score_map(lv)
        H, W = lv.shape
        P = np.pad(S, 1)
        nb = np.stack([P[1 + dy:1 + dy + H, 1 + dx:1 + dx + W] for dy in (-1, 0, 1) for dx in (-1, 0, 1) if (dx, dy) != (0, 0)], 0).max(0)
        keep = (S >= 2) & (S > nb)
        keep[:15] = False; keep[-15:] = False; keep[:, :15] = False; keep[:, -15:] = False
        ys, xs = np.nonzero(keep)
        ref = set(zip(xs.tolist(), ys.tolist(), S[ys, xs].tolist()))
        g = cand[cand["level"] == l]
        got = set(zip(g["x"].tolist(), g["y"].tolist(), g["score"].tolist()))
        print(f"  level {l} size {W}x{H}: numpy {len(ref)} gpu {len(got)} common {len(ref & got)}; only numpy {sorted(ref - got)[:4]} only gpu {sorted(got - ref)[:4]}")
