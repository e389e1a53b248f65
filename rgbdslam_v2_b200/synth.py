"""Seeded synthetic inputs for the frame-pair hot path (numpy only; shared by tests and bench.py).

Feature-level generator: what ``Node`` holds after construction (node.h:167-174) -- ORB descriptors
(N x 32 B) and back-projected points (N x (x,y,z,1), camera frame, metres) -- for a pair of frames that
see an overlapping set of scene points under a small rigid motion, with descriptor bit noise, depth
noise and non-overlapping (outlier) features.  Pinhole model = the reference defaults
fx=fy=525, cx=319.5, cy=239.5 (graph_manager.cpp:189-192), 640x480.
"""
from __future__ import annotations

import numpy as np

FX = FY = 525.0
CX, CY = 319.5, 239.5
W, H = 640, 480


def random_rigid(rng: np.random.Generator, max_trans: float, max_rot_deg: float) -> np.ndarray:
    axis = rng.normal(size=3)
    axis /= np.linalg.norm(axis)
    ang = np.deg2rad(rng.uniform(0.2, 1.0) * max_rot_deg)
    K = np.array([[0, -axis[2], axis[1]], [axis[2], 0, -axis[0]], [-axis[1], axis[0], 0]])
    R = np.eye(3) + np.sin(ang) * K + (1 - np.cos(ang)) * (K @ K)
    t = rng.normal(size=3)
    t *= rng.uniform(0.2, 1.0) * max_trans / np.linalg.norm(t)
    T = np.eye(4)
    T[:3, :3] = R
    T[:3, 3] = t
    return T


def _random_points(rng, n):
    u = rng.uniform(31, W - 31, n)
    v = rng.uniform(31, H - 31, n)
    z = rng.uniform(0.8, 4.0, n)
    return np.stack([(u - CX) * z / FX, (v - CY) * z / FY, z], 1)


def make_pair(seed: int, n_kp: int = 1000, overlap: float | None = None, max_trans: float = 0.05,
              max_rot_deg: float = 2.0, depth_noise: float = 0.0015):
    """One frame pair.  Returns dict with desc_newer/xyz_newer/desc_older/xyz_older and T_true
    (maps newer-frame points into the older frame, the direction of MatchingResult::ransac_trafo)."""
    rng = np.random.default_rng(seed)
    if overlap is None:
        overlap = rng.uniform(0.08, 0.8)
    n_common = int(round(overlap * n_kp))
    T = random_rigid(rng, max_trans, max_rot_deg)  # newer -> older
    # older frame
    p_old = _random_points(rng, n_kp)
    d_old = rng.integers(0, 256, size=(n_kp, 32), dtype=np.uint8)
    # common points, seen from the newer frame: p_new = T^-1 p_old
    Tinv = np.linalg.inv(T)
    common_idx = rng.permutation(n_kp)[:n_common]
    p_new_common = p_old[common_idx] @ Tinv[:3, :3].T + Tinv[:3, 3]
    # descriptor bit noise: per-feature flip probability in [0.02, 0.2]
    flip_p = rng.uniform(0.02, 0.2, n_common)
    flips = rng.random((n_common, 256)) < flip_p[:, None]
    d_new_common = d_old[common_idx] ^ np.packbits(flips, axis=1, bitorder="little")
    # unrelated features
    n_rest = n_kp - n_common
    p_new_rest = _random_points(rng, n_rest)
    d_new_rest = rng.integers(0, 256, size=(n_rest, 32), dtype=np.uint8)
    p_new = np.concatenate([p_new_common, p_new_rest])
    d_new = np.concatenate([d_new_common, d_new_rest])
    perm = rng.permutation(n_kp)
    p_new, d_new = p_new[perm], d_new[perm]
    # sensor noise: sigma_z = depth_noise * z^2 along the ray (both frames)
    for p in (p_old, p_new):
        z = p[:, 2].copy()
        zn = z + rng.normal(size=len(z)) * depth_noise * z * z
        p *= (zn / z)[:, None]
    to4 = lambda p: np.concatenate([p, np.ones((len(p), 1))], 1).astype(np.float32)
    return dict(desc_newer=np.ascontiguousarray(d_new), xyz_newer=to4(p_new), desc_older=np.ascontiguousarray(d_old),
                xyz_older=to4(p_old), T_true=T, n_common=n_common)


def sift_like(rng: np.random.Generator, n: int, kind: str = "sift") -> np.ndarray:
    """128-d float descriptors with SIFT-like statistics.  'sift': non-negative, gamma-distributed magnitudes, values 0..255 (what
    cv::SIFT emits; Node applies RootSIFT); 'siftgpu': unit L2 norm, clipped at 0.2 and renormalised (SiftGPU's output)."""
    if kind == "sift":
        return np.minimum(rng.gamma(0.6, 30.0, size=(n, 128)), 255.0).astype(np.float32)
    d = rng.gamma(0.6, 1.0, size=(n, 128)).astype(np.float32)
    d /= np.linalg.norm(d, axis=1, keepdims=True)
    d = np.minimum(d, 0.2)
    return (d / np.linalg.norm(d, axis=1, keepdims=True)).astype(np.float32)


def make_pair_sift(seed: int, n_kp: int = 2000, overlap: float = 0.5, kind: str = "sift", **kw):
    """make_pair with 128-d float descriptors (BASELINE config C3): same geometry / noise model, the common features of the
    newer frame carry noisy copies of the older frame's descriptors."""
    p = make_pair(seed, n_kp, overlap=overlap, **kw)
    rng = np.random.default_rng(seed + 7919)
    # correspondences of the binary generator: a common feature's descriptor is a few-bit-flip copy of its older twin
    d_old = sift_like(rng, n_kp, kind)
    d_new = sift_like(rng, n_kp, kind)
    bits_o = np.unpackbits(p["desc_older"], axis=1)
    bits_n = np.unpackbits(p["desc_newer"], axis=1)
    # exact nearest older row for each newer row (256-bit Hamming, blockwise matmul on +-1 vectors)
    so = bits_o.astype(np.float32) * 2 - 1
    sn = bits_n.astype(np.float32) * 2 - 1
    dots = sn @ so.T
    nn = dots.argmax(1)
    common = dots[np.arange(n_kp), nn] > 256 - 2 * 70  # hd < 70: flipped copies have hd ~ 256 * [0.02, 0.2]
    noise = rng.normal(0, 5.0 if kind == "sift" else 0.01, (int(common.sum()), 128)).astype(np.float32)
    d_new[common] = np.abs(d_old[nn[common]] + noise)
    return dict(desc_newer=d_new, xyz_newer=p["xyz_newer"], desc_older=d_old, xyz_older=p["xyz_older"], T_true=p["T_true"],
                n_common=int(common.sum()))


def make_batch(npairs: int, n_kp: int = 1000, seed0: int = 0, **kw):
    """Concatenated host buffers for match_pairs_host / the oracle batch driver."""
    pairs = [make_pair(seed0 + i, n_kp, **kw) for i in range(npairs)]
    cat = lambda k: np.ascontiguousarray(np.concatenate([p[k] for p in pairs]))
    return dict(
        desc_newer=cat("desc_newer"), xyz_newer=cat("xyz_newer"), desc_older=cat("desc_older"), xyz_older=cat("xyz_older"),
        n_newer=np.full(npairs, n_kp, np.int32), n_older=np.full(npairs, n_kp, np.int32),
        id_newer=np.arange(npairs, dtype=np.int32) + 1, id_older=np.arange(npairs, dtype=np.int32),
        T_true=np.stack([p["T_true"] for p in pairs]), n_common=np.array([p["n_common"] for p in pairs]),
        pairs=pairs)


# ---------------------------------------------------------------------------------------------------
# Pose graph (BASELINE config C5 / SURVEY 8d): poses on a smooth closed trajectory, odometry + loop edges.

def _quat_mul(a, b):  # (x y z w)
    ax, ay, az, aw = a[..., 0], a[..., 1], a[..., 2], a[..., 3]
    bx, by, bz, bw = b[..., 0], b[..., 1], b[..., 2], b[..., 3]
    return np.stack([aw * bx + ax * bw + ay * bz - az * by, aw * by - ax * bz + ay * bw + az * bx,
                     aw * bz + ax * by - ay * bx + az * bw, aw * bw - ax * bx - ay * by - az * bz], -1)


def _quat_conj(q):
    return q * np.array([-1, -1, -1, 1.0])


def _quat_rot(q, v):
    qv = np.concatenate([v, np.zeros(v.shape[:-1] + (1,))], -1)
    return _quat_mul(_quat_mul(q, qv), _quat_conj(q))[..., :3]


def pose_compose(a, b):  # a * b, 7-vectors (t, q)
    return np.concatenate([a[..., :3] + _quat_rot(a[..., 3:], b[..., :3]), _quat_mul(a[..., 3:], b[..., 3:])], -1)


def pose_inverse(a):
    qc = _quat_conj(a[..., 3:])
    return np.concatenate([-_quat_rot(qc, a[..., :3]), qc], -1)


def make_pose_graph(nv: int = 5000, ne: int = 30000, seed: int = 0, laps: float = 2.5, trans_noise: float = 0.01,
                    rot_noise_deg: float = 0.5, outlier_frac: float = 0.0):
    """Returns dict(gt [nv,7], init [nv,7], ij [ne,2], meas [ne,7], info [ne,36], fixed [nv]).
    Edges: nv-1 odometry edges (i, i+1) + loop/neighbour edges between poses that are close on the trajectory
    (different laps or small index distance).  measurement = GT relative pose (+) noise; information =
    I * n_inl/rmse^2 with n_inl ~ U[20,300], rmse ~ U[0.5,2] (the edge weights node.cpp:1335 produces).
    init = odometry chain (vertex estimate = v1 * T, graph_manager.cpp:858); vertex 0 fixed (pose_relative_to=first)."""
    rng = np.random.default_rng(seed)
    s = np.linspace(0, 2 * np.pi * laps, nv)
    pos = np.stack([3 * np.cos(s), 2 * np.sin(2 * s) * 0.5 + 2 * np.sin(s), 0.3 * np.sin(3 * s)], 1)
    yaw = s + np.pi / 2
    q = np.stack([np.zeros(nv), np.zeros(nv), np.sin(yaw / 2), np.cos(yaw / 2)], 1)
    tilt = 0.1 * np.sin(5 * s)
    qt = np.stack([np.sin(tilt / 2), np.zeros(nv), np.zeros(nv), np.cos(tilt / 2)], 1)
    gt = np.concatenate([pos, _quat_mul(q, qt)], 1)
    period = int(round(nv / laps))
    ii = [np.arange(nv - 1)]
    jj = [np.arange(1, nv)]
    n_extra = ne - (nv - 1)
    a = rng.integers(0, nv, size=4 * n_extra)
    kind = rng.random(4 * n_extra)
    lap_jump = rng.integers(1, int(np.ceil(laps)) + 1, size=4 * n_extra) * period
    near = rng.integers(2, 12, size=4 * n_extra)
    wob = rng.integers(-15, 16, size=4 * n_extra)
    b = np.where(kind < 0.5, a + near, a + lap_jump + wob)
    ok = (b < nv) & (b > a)
    a, b = a[ok][:n_extra], b[ok][:n_extra]
    assert len(a) == n_extra, "not enough loop candidates"
    ii.append(a); jj.append(b)
    ij = np.stack([np.concatenate(ii), np.concatenate(jj)], 1).astype(np.int32)
    rel = pose_compose(pose_inverse(gt[ij[:, 0]]), gt[ij[:, 1]])
    # noise (+): right-multiply a small random transform
    ax = rng.normal(size=(ne, 3)); ax /= np.linalg.norm(ax, axis=1, keepdims=True)
    ang = np.deg2rad(rot_noise_deg) * rng.normal(size=ne)
    dq = np.concatenate([ax * np.sin(ang / 2)[:, None], np.cos(ang / 2)[:, None]], 1)
    dt = rng.normal(size=(ne, 3)) * trans_noise
    n_out = int(outlier_frac * n_extra)
    if n_out:
        idx = (nv - 1) + rng.permutation(n_extra)[:n_out]
        dt[idx] += rng.normal(size=(n_out, 3)) * 1.0
    meas = pose_compose(rel, np.concatenate([dt, dq], 1))
    n_inl = rng.uniform(20, 300, ne); rmse = rng.uniform(0.5, 2.0, ne)
    info = np.zeros((ne, 36)); info[:, ::7] = (n_inl / rmse ** 2)[:, None]
    init = np.zeros((nv, 7)); init[0] = gt[0]
    for k in range(nv - 1):
        init[k + 1] = pose_compose(init[k], meas[k])
    fixed = np.zeros(nv, np.uint8); fixed[0] = 1
    return dict(gt=gt, init=init, ij=ij, meas=np.ascontiguousarray(meas), info=info, fixed=fixed)


def ate_align(est_xyz: np.ndarray, gt_xyz: np.ndarray):
    """Horn alignment without scale -- port of align(model, data), rgbd_benchmark/evaluate_ate_module.pyx:35-55
    (model = estimated positions, data = ground truth, both [n,3] here).  Returns (rot [3,3], trans [3]).
    Pinned to the reference's own function by tests/golden/ate_align.npz."""
    model, data = np.asarray(est_xyz, np.float64).T, np.asarray(gt_xyz, np.float64).T
    mz = model - model.mean(1, keepdims=True)
    dz = data - data.mean(1, keepdims=True)
    Wm = np.zeros((3, 3))
    for c in range(model.shape[1]):  # :41-42, same summation order
        Wm += np.outer(mz[:, c], dz[:, c])
    U, d, Vh = np.linalg.svd(Wm.T)
    S = np.eye(3)
    if np.linalg.det(U) * np.linalg.det(Vh) < 0:
        S[2, 2] = -1
    rot = U @ S @ Vh
    trans = data.mean(1) - rot @ model.mean(1)
    return rot, trans


def ate_rmse(est_xyz: np.ndarray, gt_xyz: np.ndarray) -> float:
    """Absolute trajectory error: align (above), then the RMSE of the translational error
    (evaluate_ate_module.pyx:50-53,197)."""
    rot, trans = ate_align(est_xyz, gt_xyz)
    err = rot @ np.asarray(est_xyz, np.float64).T + trans[:, None] - np.asarray(gt_xyz, np.float64).T
    te = np.sqrt((err * err).sum(0))
    return float(np.sqrt(np.dot(te, te) / len(te)))


# ---------------------------------------------------------------------------------------------------
# Rendered RGB-D frames (SURVEY 8d): a textured box room seen by a pinhole camera (cv2 only used for remap/blur).

_TEX = {}


def _texture(seed: int, size: int = 1024) -> np.ndarray:
    """Band-limited noise + random rectangles: FAST fires thousands of times per frame."""
    key = (seed, size)
    if key not in _TEX:
        import cv2
        rng = np.random.default_rng(seed)
        t = rng.random((size, size)).astype(np.float32)
        t = cv2.GaussianBlur(t, (0, 0), 1.6)
        t = (t - t.min()) / (t.max() - t.min())
        img = (t * 255).astype(np.float32)
        for _ in range(size // 3):
            x, y = rng.integers(0, size - 8, 2)
            w, h = rng.integers(6, 70, 2)
            img[y:y + h, x:x + w] += rng.integers(-90, 90)
        _TEX[key] = np.clip(img, 0, 255).astype(np.uint8)
    return _TEX[key]


def intrinsics(w: int = W, h: int = H):
    """(fx, fy, cx, cy) of a w x h rendering: the 640x480 camera's field of view at w x h pixels"""
    return FX * w / W, FY * h / H, (w - 1) / 2, (h - 1) / 2


def render_frame(pose_wc: np.ndarray, tex_seed: int = 7, nan_frac: float = 0.03, seed: int = 0, depth_noise: float = 0.0,
                 shape: tuple[int, int] = (H, W)):
    """pose_wc: 4x4 camera-to-world.  Scene: back wall z=4, floor y=1.3, left wall x=-3, right wall x=3 (world frame).
    Returns gray u8 [h,w], depth f32 [h,w] (metres, NaN holes) for shape (h, w), camera intrinsics(w, h)."""
    import cv2
    rng = np.random.default_rng(seed)
    H, W = shape
    fx, fy, cx, cy = intrinsics(W, H)
    v, u = np.mgrid[0:H, 0:W].astype(np.float64)
    rays_c = np.stack([(u - cx) / fx, (v - cy) / fy, np.ones_like(u)], -1)
    R, t = pose_wc[:3, :3], pose_wc[:3, 3]
    rays_w = rays_c @ R.T
    planes = [((0, 0, 1.0), 4.0, 0), ((0, 1.0, 0), 1.3, 1), ((-1.0, 0, 0), 3.0, 2), ((1.0, 0, 0), 3.0, 3)]  # n.x = d
    best = np.full((H, W), np.inf)
    tu = np.zeros((H, W)); tv = np.zeros((H, W)); tid = np.zeros((H, W), int)
    for n, d, pid in planes:
        n = np.array(n)
        denom = rays_w @ n
        lam = (d - t @ n) / np.where(np.abs(denom) < 1e-9, 1e-9, denom)
        ok = (lam > 0.3) & (lam < best)
        P = t + rays_w * lam[..., None]
        if pid == 0: a, b = P[..., 0], P[..., 1]
        elif pid == 1: a, b = P[..., 0], P[..., 2]
        else: a, b = P[..., 2], P[..., 1]
        best = np.where(ok, lam, best); tu = np.where(ok, a, tu); tv = np.where(ok, b, tv); tid = np.where(ok, pid, tid)
    tex = _texture(tex_seed)
    S = tex.shape[0]
    mapx = ((tu * 110.0 + 37.0 * tid + 4000.0) % (S - 1)).astype(np.float32)
    mapy = ((tv * 110.0 + 91.0 * tid + 4000.0) % (S - 1)).astype(np.float32)
    gray = cv2.remap(tex, mapx, mapy, cv2.INTER_LINEAR)
    depth = best.astype(np.float32)  # rays_c has z = 1 -> lambda is the camera-frame depth
    depth[~np.isfinite(depth)] = np.nan
    if depth_noise > 0:
        depth = (depth + rng.normal(size=depth.shape) * depth_noise * depth * depth).astype(np.float32)
    holes = rng.random(((H + 7) // 8, (W + 7) // 8)) < nan_frac
    depth[np.kron(holes, np.ones((8, 8), bool))[:H, :W]] = np.nan
    depth[rng.random(depth.shape) < nan_frac / 3] = np.nan
    return np.ascontiguousarray(gray), np.ascontiguousarray(depth)


def render_frames_torch(poses_wc: np.ndarray, device, first_index: int = 0, tex_seed: int = 7, nan_frac: float = 0.03,
                        chunk: int = 32):
    """The scene of render_frame, rendered for many frames on a CUDA device with torch (data generation for the sequence
    bench: 2000 frames take minutes in numpy).  Same geometry and texture; bilinear texture lookup and the NaN-hole pattern
    come from torch, so the pixels are NOT bit-identical to render_frame -- every consumer (CUDA path, CPU oracle) must use
    the same arrays.  The hole pattern of frame k is seeded by first_index + k, i.e. independent of how a sequence is
    sharded over ranks.  Returns (gray u8 [n,H,W], depth f32 [n,H,W]) torch tensors on `device`."""
    import torch
    n = len(poses_wc)
    dev = torch.device(device)
    tex = torch.from_numpy(_texture(tex_seed).astype(np.float32)).to(dev)
    S = tex.shape[0]
    v, u = torch.meshgrid(torch.arange(H, device=dev, dtype=torch.float64), torch.arange(W, device=dev, dtype=torch.float64),
                          indexing="ij")
    rays_c = torch.stack([(u - CX) / FX, (v - CY) / FY, torch.ones_like(u)], -1)  # [H,W,3]
    planes = [((0, 0, 1.0), 4.0, 0), ((0, 1.0, 0), 1.3, 1), ((-1.0, 0, 0), 3.0, 2), ((1.0, 0, 0), 3.0, 3)]
    grays, depths = [], []
    for c0 in range(0, n, chunk):
        P = torch.from_numpy(np.asarray(poses_wc[c0:c0 + chunk], np.float64)).to(dev)  # [b,4,4]
        b = P.shape[0]
        R, t = P[:, :3, :3], P[:, :3, 3]
        rays_w = torch.einsum("hwk,bjk->bhwj", rays_c, R)  # rays_c @ R^T
        best = torch.full((b, H, W), float("inf"), device=dev, dtype=torch.float64)
        tu = torch.zeros_like(best); tv = torch.zeros_like(best); tid = torch.zeros_like(best)
        for nrm, d, pid in planes:
            nv = torch.tensor(nrm, device=dev, dtype=torch.float64)
            denom = rays_w @ nv
            denom = torch.where(denom.abs() < 1e-9, torch.full_like(denom, 1e-9), denom)
            lam = (d - t @ nv)[:, None, None] / denom
            ok = (lam > 0.3) & (lam < best)
            Pw = t[:, None, None, :] + rays_w * lam[..., None]
            if pid == 0: a, bb = Pw[..., 0], Pw[..., 1]
            elif pid == 1: a, bb = Pw[..., 0], Pw[..., 2]
            else: a, bb = Pw[..., 2], Pw[..., 1]
            best = torch.where(ok, lam, best); tu = torch.where(ok, a, tu); tv = torch.where(ok, bb, tv)
            tid = torch.where(ok, torch.full_like(tid, float(pid)), tid)
        mapx = torch.remainder(tu * 110.0 + 37.0 * tid + 4000.0, S - 1)
        mapy = torch.remainder(tv * 110.0 + 91.0 * tid + 4000.0, S - 1)
        x0 = mapx.floor().long().clamp_(0, S - 2); y0 = mapy.floor().long().clamp_(0, S - 2)
        fx = (mapx - x0).float(); fy = (mapy - y0).float()
        t00 = tex[y0, x0]; t01 = tex[y0, x0 + 1]; t10 = tex[y0 + 1, x0]; t11 = tex[y0 + 1, x0 + 1]
        g = (t00 * (1 - fx) + t01 * fx) * (1 - fy) + (t10 * (1 - fx) + t11 * fx) * fy
        gray = g.round().clamp_(0, 255).to(torch.uint8)
        depth = best.float()
        depth[~torch.isfinite(depth)] = float("nan")
        for k in range(b):
            gen = torch.Generator(device=dev)
            gen.manual_seed(1000003 * (first_index + c0 + k) + 17)
            holes = torch.rand((H // 8, W // 8), device=dev, generator=gen) < nan_frac
            holes = holes.repeat_interleave(8, 0).repeat_interleave(8, 1)
            speck = torch.rand((H, W), device=dev, generator=gen) < nan_frac / 3
            depth[k][holes | speck] = float("nan")
        grays.append(gray); depths.append(depth)
    return torch.cat(grays), torch.cat(depths)


def trajectory(n: int, seed: int = 0) -> np.ndarray:
    """Smooth camera-to-world poses [n,4,4]: Lissajous translation + yaw/pitch sweep that revisits places."""
    s = np.linspace(0, 2 * np.pi, n, endpoint=False)
    out = np.zeros((n, 4, 4))
    for k, a in enumerate(s):
        yaw = 0.45 * np.sin(a); pitch = 0.12 * np.sin(2 * a + 0.3)
        Ry = np.array([[np.cos(yaw), 0, np.sin(yaw)], [0, 1, 0], [-np.sin(yaw), 0, np.cos(yaw)]])
        Rx = np.array([[1, 0, 0], [0, np.cos(pitch), -np.sin(pitch)], [0, np.sin(pitch), np.cos(pitch)]])
        out[k, :3, :3] = Ry @ Rx
        out[k, :3, 3] = [0.9 * np.sin(a), 0.25 * np.sin(2 * a), 0.6 * np.cos(a) - 0.2]
        out[k, 3, 3] = 1
    return out


# ---- two views of a point set with pixel observations (pairwise g2o refinement tests) --------------------------------
_KREF = np.array([[521.0, 0, 319.5], [0, 521.0, 239.5], [0, 0, 1]])  # the camera hard-coded in transformation_estimation.cpp:56


def _rodrigues(axis, ang):
    axis = np.asarray(axis, float) / np.linalg.norm(axis)
    x, y, z = axis
    Kx = np.array([[0, -z, y], [z, 0, -x], [-y, x, 0]])
    return np.eye(3) + np.sin(ang) * Kx + (1 - np.cos(ang)) * Kx @ Kx


def make_refine_scene(rng, n, noise_px=0.3, noise_z=0.002, angle=0.08, trans=(0.10, -0.03, 0.05)):
    """Points seen by the newer camera (world frame) and by the earlier camera at pose X1 (world-from-earlier)."""
    X1 = np.eye(4); X1[:3, :3] = _rodrigues([0.2, 1.0, 0.1], angle); X1[:3, 3] = trans
    pw = np.stack([rng.uniform(-1.2, 1.2, n), rng.uniform(-0.9, 0.9, n), rng.uniform(1.0, 4.0, n)], 1)
    pe = (np.linalg.inv(X1) @ np.c_[pw, np.ones(n)].T).T[:, :3]

    def observe(p):
        uv = (_KREF @ p.T).T
        uv = uv[:, :2] / uv[:, 2:3] + rng.normal(0, noise_px, (len(p), 2))
        z = p[:, 2] + rng.normal(0, noise_z, len(p))
        xyz = np.c_[(uv[:, 0] - _KREF[0, 2]) * z / _KREF[0, 0], (uv[:, 1] - _KREF[1, 2]) * z / _KREF[1, 1], z, np.ones(len(p))]
        return uv.astype(np.float32), xyz.astype(np.float32)

    kp_n, xyz_n = observe(pw)
    kp_e, xyz_e = observe(pe)
    return X1, kp_n, xyz_n, kp_e, xyz_e




# ------------------------------------------------------------------------------------------------
# landmark bundle adjustment problems (landmark.cpp:97-187: cameras, 3-D landmarks, (u, v, depth) observations)
def landmark_information(depths: np.ndarray, sigma_depth: float = 0.01, static_first: bool = False) -> np.ndarray:
    """point_information_matrix (misc2.h:37-47) per observation: diag(1, 1, 1 / depth_covariance(d)), depth_covariance =
    (sigma_depth d^2)^2 (misc2.h:20-35).  static_first=True reproduces the reference's function-local statics: the covariance
    of the FIRST depth ever passed is reused for every later call."""
    d = np.asarray(depths, np.float64)
    ref = np.full_like(d, d.flat[0]) if (static_first and d.size) else d
    w = np.ones((d.size, 3))
    w[:, 2] = 1.0 / (sigma_depth * ref.reshape(-1) ** 2) ** 2
    return w


def make_ba_problem(n_cams: int = 6, n_points: int = 60, seed: int = 0, pix_noise: float = 0.3, depth_sigma: float = 0.002,
                    pose_noise: float = 0.03, rot_noise_deg: float = 1.5, K4=(525.0, 525.0, 319.5, 239.5), with_edges: bool = True,
                    edge_noise: float = 0.01):
    """Cameras on a short arc looking at a point cloud; every point is observed by every camera that sees it inside 640x480.
    Returns a dict with ground truth, perturbed initial poses, landmarks initialised from their FIRST observation through the
    initial pose of that camera (updateLandmarkInGraph, landmark.cpp:100-121), observations and odometry-like pose edges."""
    rng = np.random.default_rng(seed)
    fx, fy, cx, cy = K4
    gt = np.zeros((n_cams, 7))
    step_ang, step_x = min(0.08, 0.6 / n_cams), min(0.15, 1.2 / n_cams)  # the whole arc keeps the cloud in view
    for c in range(n_cams):
        ang = step_ang * c
        q = np.array([0.0, np.sin(ang / 2), 0.0, np.cos(ang / 2)])
        gt[c, :3] = [step_x * c, 0.02 * np.sin(c), 0.2 * step_x * c]
        gt[c, 3:] = q
    pts = np.stack([rng.uniform(-1.2, 1.8, n_points), rng.uniform(-0.9, 0.9, n_points), rng.uniform(1.5, 4.0, n_points)], 1)
    oc, op, uvd = [], [], []
    for c in range(n_cams):
        R = _quat_to_rot(gt[c, 3:])
        pc = (pts - gt[c, :3]) @ R  # R^T (p - t)
        u = fx * pc[:, 0] / pc[:, 2] + cx
        v = fy * pc[:, 1] / pc[:, 2] + cy
        ok = (pc[:, 2] > 0.4) & (u > 0) & (u < 639) & (v > 0) & (v < 479)
        for p in np.nonzero(ok)[0]:
            oc.append(c); op.append(p)
            uvd.append([u[p] + rng.normal(0, pix_noise), v[p] + rng.normal(0, pix_noise), pc[p, 2] + rng.normal(0, depth_sigma)])
    oc, op, uvd = np.array(oc, np.int32), np.array(op, np.int32), np.array(uvd)
    seen = np.zeros(n_points, bool); seen[op] = True
    remap = -np.ones(n_points, np.int64); remap[seen] = np.arange(seen.sum())
    pts = pts[seen]; op = remap[op].astype(np.int32)
    init = gt.copy()
    for c in range(1, n_cams):
        d = np.concatenate([rng.normal(0, pose_noise, 3), np.deg2rad(rot_noise_deg) / 2 * rng.normal(0, 1, 3)])
        init[c] = pose_compose(gt[c], np.concatenate([d[:3], d[3:], [np.sqrt(max(0.0, 1 - d[3:] @ d[3:]))]]))
    p0 = np.zeros_like(pts)
    first = {}
    for o in range(len(oc)):
        first.setdefault(int(op[o]), o)
    for p, o in first.items():
        c = oc[o]
        x = (uvd[o, 0] - cx) / fx * uvd[o, 2]; y = (uvd[o, 1] - cy) / fy * uvd[o, 2]
        p0[p] = init[c, :3] + _quat_to_rot(init[c, 3:]) @ np.array([x, y, uvd[o, 2]])
    fixed = np.zeros(n_cams, np.uint8); fixed[0] = 1
    out = dict(gt_poses=gt, gt_points=pts, poses=init, points=p0, fixed=fixed, obs_cam=oc, obs_point=op, obs_uvd=uvd,
               obs_info3=landmark_information(uvd[:, 2], sigma_depth=max(depth_sigma, 0.002) / 4.0), K4=np.array(K4, np.float64))
    if with_edges:
        ij, meas, info = [], [], []
        for c in range(n_cams - 1):
            rel = pose_compose(pose_inverse(gt[c]), gt[c + 1])
            d = np.concatenate([rng.normal(0, edge_noise, 3), rng.normal(0, edge_noise / 2, 3)])
            rel = pose_compose(rel, np.concatenate([d, [np.sqrt(1 - d[3:] @ d[3:])]]))
            ij.append([c, c + 1]); meas.append(rel); info.append((np.eye(6) * 400.0).reshape(-1))
        out.update(ij=np.array(ij, np.int32), meas=np.array(meas), info=np.array(info))
    return out


def _quat_to_rot(q):
    x, y, z, w = q / np.linalg.norm(q)
    return np.array([[1 - 2 * (y * y + z * z), 2 * (x * y - z * w), 2 * (x * z + y * w)],
                     [2 * (x * y + z * w), 1 - 2 * (x * x + z * z), 2 * (y * z - x * w)],
                     [2 * (x * z - y * w), 2 * (y * z + x * w), 1 - 2 * (x * x + y * y)]])
