"""One pass over every kernel family that has a SURVEY section-8 row (ORB node constructor, SIFT matchers, pose graph,
landmark bundle adjustment, EMM, pairwise refinement) -- one run to time or profile them together.

  python tools/run_families.py [orb] [sift] [posegraph] [landmark] [emm] [refine]      (default: all)
Prints CUDA-event / wall times per family as one JSON line (NOT a bench value when run under ncu)."""
import json
import sys
import time
from pathlib import Path

sys.path.insert(0, str(Path(__file__).resolve().parent.parent))
import numpy as np

from rgbdslam_v2_b200 import Frontend, synth
from rgbdslam_v2_b200._capi import default_params

which = set(sys.argv[1:]) or {"orb", "sift", "posegraph", "landmark", "emm", "refine"}
out = {}
K4 = (synth.FX, synth.FY, synth.CX, synth.CY)


def frames(n):
    from oracle import orb_oracle  # only depth_to_mask (cv2.convertScaleAbs), data preparation
    poses = synth.trajectory(240)[:n]
    fr = [synth.render_frame(poses[k], seed=k) for k in range(n)]
    gray = np.stack([f[0] for f in fr]); depth = np.stack([f[1] for f in fr])
    mask = np.stack([orb_oracle.depth_to_mask(d) for d in depth])
    return gray, depth, mask


if "orb" in which:
    import os
    import torch
    n = int(os.environ.get("RB200_ORB_FRAMES", "64"))
    reps = int(os.environ.get("RB200_ORB_REPS", "4"))
    gray, depth, mask = frames(min(n, 64))
    if n > 64:  # tile the rendered frames (timing only)
        k = (n + 63) // 64
        gray, depth, mask = (np.concatenate([x] * k)[:n] for x in (gray, depth, mask))
    p = default_params(); p.depth_cov_z0 = 2.0; p.max_keypoints = 1000
    fe = Frontend(0, p)
    res = {}
    pin = [torch.from_numpy(x).pin_memory() for x in (gray, depth, mask)]
    for name, args, kw in (("pageable_mask", (gray, depth, mask), {}), ("pinned_mask", tuple(pin), {}),
                           ("pinned_mask_from_depth", (pin[0], pin[1], None), {"mask_from_depth": True})):
        det = fe.detector_create()
        ts = []
        for it in range(reps):
            t0 = time.perf_counter()
            h, nf = fe.nodes_create(det, *args, K4, **kw)
            ts.append(time.perf_counter() - t0)
            for x in h:
                fe.node_destroy(x)
        fe.detector_destroy(det)
        res[name] = n / min(ts[1:]) if len(ts) > 1 else n / ts[0]
    out["orb"] = {"frames": n, "frames_per_s": res, "mean_features": float(np.mean(nf))}
    fe.close()

if "sift" in which:
    rng = np.random.default_rng(0)
    p = default_params(); p.depth_cov_z0 = 2.0
    fe = Frontend(0, p)
    npairs, nk = 32, 2000
    for matcher in (0, 1):
        fe.set_sift_matcher(matcher)
        hs = []
        for k in range(npairs + 1):
            d = np.abs(rng.normal(size=(nk, 128))).astype(np.float32)
            d /= np.linalg.norm(d, axis=1, keepdims=True)
            if matcher == 1:
                d = np.minimum(d, 0.2); d /= np.linalg.norm(d, axis=1, keepdims=True)
            xyz = np.concatenate([rng.uniform(-1, 1, (nk, 2)), rng.uniform(1, 4, (nk, 1)), np.ones((nk, 1))], 1).astype(np.float32)
            hs.append(fe.node_from_sift(k, d, xyz))
        for it in range(3):
            t0 = time.perf_counter()
            fe.match_node_pairs(hs[1:], hs[:-1], seed=1, want_matches=False)
            dt = time.perf_counter() - t0
        out[f"sift_matcher{matcher}"] = {"pairs": npairs, "kp": nk, "pairs_per_s": npairs / dt, "stages": fe.stage_times(0)}
    fe.close()

if "posegraph" in which:
    p = default_params(); p.depth_cov_z0 = 2.0
    fe = Frontend(0, p)
    g = synth.make_pose_graph(5000, 30000, seed=0)
    for it in range(2):
        t0 = time.perf_counter()
        x, chi2, lm, cg = fe.optimize_graph(g["init"], g["fixed"], g["ij"], g["meas"], g["info"], stop=0.01)
        dt = time.perf_counter() - t0
    out["posegraph"] = {"seconds": dt, "lm": lm, "pcg": cg, "chi2": chi2}
    fe.close()

if "landmark" in which:
    p = default_params(); p.depth_cov_z0 = 2.0
    fe = Frontend(0, p)
    d = synth.make_ba_problem(n_cams=60, n_points=6000, seed=11, edge_noise=0.02)
    for it in range(2):
        t0 = time.perf_counter()
        x, pts, c0, c1, lm, cg = fe.landmark_ba(d["poses"], d["fixed"], d["points"], d["obs_cam"], d["obs_point"], d["obs_uvd"], d["obs_info3"],
                                                d["K4"], ij=d["ij"], meas=d["meas"], info=d["info"], iterations=6)
        dt = time.perf_counter() - t0
    err = float(np.linalg.norm(x[:, :3] - d["gt_poses"][:, :3], axis=1).max())
    out["landmark_ba"] = {"cams": len(x), "points": len(pts), "observations": int(len(d["obs_cam"])), "seconds": dt, "lm": lm, "pcg": cg,
                          "chi2_before": c0, "chi2_after": c1, "max_cam_error_m": err}
    fe.close()

if "emm" in which or "refine" in which:
    gray, depth, mask = frames(12)
    for name, setp in (("emm", lambda p: setattr(p, "observability_threshold", 0.5)),
                       ("refine", lambda p: setattr(p, "g2o_transformation_refinement", 5))):
        if name not in which:
            continue
        p = default_params(); p.depth_cov_z0 = 2.0; p.max_keypoints = 600
        setp(p)
        fe = Frontend(0, p)
        det = fe.detector_create()
        h, nf = fe.nodes_create(det, gray, depth, mask, K4)
        newer = [h[k] for k in range(1, 12) for d in (1, 2, 3) if k - d >= 0]
        older = [h[k - d] for k in range(1, 12) for d in (1, 2, 3) if k - d >= 0]
        for it in range(3):
            t0 = time.perf_counter()
            res, _, _ = fe.match_node_pairs(newer, older, seed=3, want_matches=False)
            dt = time.perf_counter() - t0
        out[name] = {"pairs": len(newer), "seconds": dt, "valid": int((res["id1"] >= 0).sum())}
        fe.close()

print(json.dumps(out))
