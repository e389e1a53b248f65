"""Node constructor with the ORB and the FAST detector (params.feature_detector_type) on the same rendered 640x480 frames.

1. rgbdslam_b200_nodes_create_ex with MASK_FROM_DEPTH from pinned host memory, both detector types alternated --rounds
   times; host clock around the call, which returns after the device work has finished (it downloads the feature counts).
2. The C4 sequence (bench.py: --frames frames, 3 sequential + 4 window + 4 random candidate pairs per frame) with nodes of
   each detector type through matching, graph construction, the pose-graph solve and ATE against the rendering ground truth.

--min-depth: every detector type also with params.use_feature_min_depth (keypoint depth = the nearest point of its
neighbourhood), alternated with the pointwise rule in step 1 and run through step 2 as well ("ORB+min_depth", ...).

--cloud: instead, the ORB detector with other inputs, alternated --rounds times in step 1: the depth-image constructor with
grey and with colour visuals (MASK_FROM_DEPTH, pinned), the point-cloud constructor with organised PointXYZRGB clouds
(MASK_FROM_CLOUD) from pinned and from pageable memory (--cloud-frames frames per call: a 640x480 XYZRGB cloud is 9.8 MB);
the host-to-device bytes per frame of each; the new kernels' device times from torch.profiler in a separate pass; and step 2
with cloud nodes against depth-image nodes (cloud nodes built --cloud-chunk frames per call, one detector: the same nodes as
one call).

--raw: instead, the ORB detector on the listener's raw inputs against the converted ones, alternated --rounds times in
step 1 from pinned and from pageable memory: grey + float metres, grey + 16-bit millimetres (DEPTH_U16), colour + float
metres and Bayer + 16-bit millimetres (VISUAL_BAYER_GR | DEPTH_U16), all with MASK_FROM_DEPTH; the host-to-device bytes per
frame of each; the device time of the conversion kernels from torch.profiler in a separate pass; the host time per frame of
the conversions a caller no longer makes (cv2 / numpy, one thread); and step 2 with 16-bit nodes against float nodes
(millimetre quantisation and the 0.51 m mask change the results).

Prints one JSON object, with the card name and power limit read in the same run.
Usage: python tools/run_nodes.py [--min-depth | --cloud | --raw]
"""
import argparse
import ctypes as C
import json
import re
import subprocess
import sys
import time
from pathlib import Path

sys.path.insert(0, str(Path(__file__).resolve().parent.parent))
import numpy as np  # noqa: E402


def card() -> dict:
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                       text=True)
    name, power, clk = (x.strip() for x in q.stdout.splitlines()[0].split(","))
    return {"name": name, "power_limit": power, "max_sm_clock": clk}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--timing-frames", type=int, default=512)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--frames", type=int, default=2000, help="C4 sequence length")
    ap.add_argument("--keypoints", type=int, default=1000)
    ap.add_argument("--min-depth", action="store_true", help="also with use_feature_min_depth, alternated with the pointwise rule")
    ap.add_argument("--cloud", action="store_true", help="colour and point-cloud input (ORB detector) instead of the detector types")
    ap.add_argument("--cloud-frames", type=int, default=256)
    ap.add_argument("--cloud-chunk", type=int, default=128)
    ap.add_argument("--raw", action="store_true", help="16-bit depth and Bayer input (ORB detector) instead of the detector types")
    args = ap.parse_args()
    if args.cloud:
        return main_cloud(args)
    if args.raw:
        return main_raw(args)

    import torch
    from rgbdslam_v2_b200 import Frontend, pipeline, synth
    from rgbdslam_v2_b200._capi import DETECTOR_FAST, DETECTOR_ORB, PAIR_RESULT_DTYPE, default_params, graph_from_pairs
    if not torch.cuda.is_available():
        raise SystemExit("run_nodes.py measures on the GPU; no CUDA device found")
    dev = torch.device("cuda", 0)
    K4 = (synth.FX, synth.FY, synth.CX, synth.CY)
    seed = 11
    types = {DETECTOR_ORB: "ORB", DETECTOR_FAST: "FAST"}
    configs = [(t, m) for t in types for m in ((0, 1) if args.min_depth else (0,))]  # (detector type, use_feature_min_depth)
    names = {(t, m): types[t] + ("+min_depth" if m else "") for t, m in configs}

    def params(cfg):
        p = default_params(); p.depth_cov_z0 = 2.0; p.max_keypoints = args.keypoints
        p.feature_detector_type, p.use_feature_min_depth = cfg
        return p

    fe = Frontend(0, params(configs[0]))

    def use(cfg):
        p = params(cfg)
        fe.params = p
        fe._check(fe.lib.rgbdslam_b200_init(0, C.byref(p)))

    n = max(args.frames, args.timing_frames)
    poses = synth.trajectory(n)
    g_d, d_d = synth.render_frames_torch(poses, dev)
    gray = torch.empty(g_d.shape, dtype=torch.uint8).pin_memory(); gray.copy_(g_d)
    depth = torch.empty(d_d.shape, dtype=torch.float32).pin_memory(); depth.copy_(d_d)
    del g_d, d_d
    torch.cuda.synchronize()
    out = {"card": card(), "image": "640x480", "max_keypoints": args.keypoints}

    # ---- 1. the Node constructor alone, configurations alternated
    nt = args.timing_frames
    timing = {names[c]: [] for c in configs}
    feats = {}
    for r in range(args.rounds + 1):  # round 0 warms up every configuration (allocations, first launches)
        for t in configs:
            use(t)
            det = fe.detector_create()
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            hs, nf = fe.nodes_create(det, gray[:nt], depth[:nt], None, K4, mask_from_depth=True)
            dt = time.perf_counter() - t0
            fe.detector_destroy(det)
            for h in hs:
                fe.node_destroy(h)
            if r:
                timing[names[t]].append(nt / dt)
            feats[names[t]] = float(np.mean(nf))
    out["nodes_create_frames_per_s"] = {k: {"runs": [round(v, 1) for v in vs], "min": round(min(vs), 1), "max": round(max(vs), 1)}
                                        for k, vs in timing.items()}
    out["nodes_create_mean_features"] = feats
    out["nodes_create_frames"] = nt

    # ---- 2. the C4 sequence with nodes of each detector type
    nf_ = args.frames
    pairs = np.array(pipeline.candidate_pairs(nf_, seed=seed), np.int64)
    gt = np.stack([pipeline.mat_to_pose7(np.linalg.inv(poses[0]) @ P) for P in poses[:nf_]])
    fe.posegraph_reserve(nf_, 12 * nf_)

    def sequence(t, nf):
        """frames [0, nf) with detector type t -> nodes, pair results, graph, trajectory; stage seconds"""
        pp = pairs[pairs[:, 0] < nf]
        use(t)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        det = fe.detector_create()
        hs, nfeat = fe.nodes_create(det, gray[:nf], depth[:nf], None, K4, ids=np.arange(nf, dtype=np.int32), mask_from_depth=True)
        t1 = time.perf_counter()
        res = np.zeros(len(pp), PAIR_RESULT_DTYPE); res["id1"] = -1; res["id2"] = -1
        pipeline.match_pairs_pipelined(fe, hs, pp, seed=seed, first_pair_index=0, out=res)
        t2 = time.perf_counter()
        graph = graph_from_pairs(pp, res, nf)
        traj, chi2, lm, cg = fe.optimize_graph(graph["init"], graph["fixed"], graph["ij"], graph["meas"], graph["info"], stop=0.01)
        t3 = time.perf_counter()
        fe.detector_destroy(det)
        for h in hs:
            fe.node_destroy(h)
        return nfeat, res, graph, traj, chi2, lm, (t0, t1, t2, t3)

    c4 = {}
    for t in configs[::-1]:
        sequence(t, min(nf_, 96))  # warm-up of every stage (allocations, first launches), as bench.py does
        nfeat, res, graph, traj, chi2, lm, (t0, t1, t2, t3) = sequence(t, nf_)
        c4[names[t]] = {"frames": nf_, "pairs": int(len(pairs)), "valid_edges": int(graph["n_valid_edges"]),
                        "mean_features": float(np.mean(nfeat)), "mean_inliers_valid": float(res["n_inliers"][res["id1"] >= 0].mean()),
                        "lm_iterations": lm, "chi2": chi2, "ate_vs_gt_m": synth.ate_rmse(traj[:, :3], gt[:, :3]),
                        "seconds": {"nodes": t1 - t0, "match": t2 - t1, "graph_and_solve": t3 - t2, "total": t3 - t0}}
    out["c4"] = c4
    fe.close()
    print(json.dumps(out))


def main_cloud(args):
    import torch
    from torch.profiler import ProfilerActivity, profile

    from rgbdslam_v2_b200 import Frontend, pipeline, synth
    from rgbdslam_v2_b200._capi import DETECTOR_ORB, PAIR_RESULT_DTYPE, default_params, graph_from_pairs
    if not torch.cuda.is_available():
        raise SystemExit("run_nodes.py measures on the GPU; no CUDA device found")
    dev = torch.device("cuda", 0)
    K4 = (synth.FX, synth.FY, synth.CX, synth.CY)
    seed = 11
    p = default_params(); p.depth_cov_z0 = 2.0; p.max_keypoints = args.keypoints; p.feature_detector_type = DETECTOR_ORB
    fe = Frontend(0, p)

    n = max(args.frames, args.timing_frames, args.cloud_frames)
    poses = synth.trajectory(n)
    g_d, d_d = synth.render_frames_torch(poses, dev)
    H, W = g_d.shape[1:]
    v, u = torch.meshgrid(torch.arange(H, device=dev, dtype=torch.float32), torch.arange(W, device=dev, dtype=torch.float32),
                          indexing="ij")

    def cloud_of(d):  # organised PointXYZRGB clouds [n, H, W, 8] of depth frames (a registered depth camera's output)
        c = torch.zeros(d.shape + (8,), dtype=torch.float32, device=dev)
        c[..., 0] = (u - K4[2]) * d / K4[0]
        c[..., 1] = (v - K4[3]) * d / K4[1]
        c[..., 2] = d
        return c

    def pinned(t):
        h = torch.empty(t.shape, dtype=t.dtype).pin_memory()
        h.copy_(t)
        return h

    gray = pinned(g_d)
    depth = pinned(d_d)
    nt, nc = args.timing_frames, args.cloud_frames
    rgb = pinned(torch.stack([g_d[:nt], g_d[:nt].roll(3, -1), g_d[:nt].roll(5, -2)], -1))
    cloud_pin = pinned(cloud_of(d_d[:nc]))
    cloud_pag = cloud_pin.numpy().copy()
    del g_d
    torch.cuda.synchronize()
    px = H * W
    out = {"card": card(), "image": f"{W}x{H}", "max_keypoints": args.keypoints, "detector": "ORB"}
    # name: (visual, depth or cloud, frames, keyword, host->device bytes per frame)
    configs = {
        "depth_gray_pinned": (gray, depth, nt, {"mask_from_depth": True}, px + 4 * px),
        "depth_rgb_pinned": (rgb, depth, nt, {"mask_from_depth": True}, 3 * px + 4 * px),
        "cloud_xyzrgb_pinned": (gray, cloud_pin, nc, {"mask_from_cloud": True}, px + 32 * px),
        "cloud_xyzrgb_pageable": (gray.numpy(), cloud_pag, nc, {"mask_from_cloud": True}, px + 32 * px),
    }

    def call(cfg, frames=None):
        vis, dep, m, kw, _ = configs[cfg]
        m = frames or m
        det = fe.detector_create()
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        hs, nf = fe.nodes_create(det, vis[:m], dep[:m], None, None if "mask_from_cloud" in kw else K4, **kw)
        dt = time.perf_counter() - t0
        fe.detector_destroy(det)
        for h in hs:
            fe.node_destroy(h)
        return m / dt, float(np.mean(nf))

    # ---- 1. the constructor alone, inputs alternated
    timing = {c: [] for c in configs}
    feats = {}
    for r in range(args.rounds + 1):  # round 0 warms up every configuration
        for c in configs:
            fps, feats[c] = call(c)
            if r:
                timing[c].append(fps)
    out["nodes_create_frames_per_s"] = {k: {"frames": configs[k][2], "runs": [round(x, 1) for x in vs], "min": round(min(vs), 1),
                                            "max": round(max(vs), 1)} for k, vs in timing.items()}
    out["nodes_create_mean_features"] = feats
    out["h2d_bytes_per_frame"] = {k: c[4] for k, c in configs.items()}

    # ---- the kernels' device time per frame (torch.profiler, separate pass: tracing slows the host)
    kernels = ("k_rgb_to_gray", "k_cloud_mask", "k_frame_finalize", "k_frame_emit")
    prof_frames = min(64, nt, nc)
    ktimes = {}
    for c in ("depth_rgb_pinned", "cloud_xyzrgb_pinned"):
        call(c, prof_frames)
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            call(c, prof_frames)
        tot = {}
        for e in prof.events():
            if e.device_type.name != "CUDA":
                continue
            # keyed on the template-id: one row per instantiation (point source, detector)
            m = re.search(r"rb200::((k_\w+)(<[^>]*>)?)", e.name)
            if m and m.group(2) in kernels:
                tot[m.group(1)] = tot.get(m.group(1), 0.0) + e.device_time
        allk = sum(e.device_time for e in prof.events() if e.device_type.name == "CUDA" and "rb200::k_" in e.name)
        ktimes[c] = {k: round(t / prof_frames, 2) for k, t in sorted(tot.items())}
        ktimes[c]["all_library_kernels"] = round(allk / prof_frames, 2)
    out["kernel_us_per_frame"] = ktimes

    # ---- 2. the C4 sequence with cloud nodes against depth-image nodes
    nf_ = args.frames
    pairs = np.array(pipeline.candidate_pairs(nf_, seed=seed), np.int64)
    gt = np.stack([pipeline.mat_to_pose7(np.linalg.inv(poses[0]) @ P) for P in poses[:nf_]])
    fe.posegraph_reserve(nf_, 12 * nf_)
    stage = torch.empty((args.cloud_chunk, H, W, 8), dtype=torch.float32).pin_memory()

    def sequence(kind, nf):
        pp = pairs[pairs[:, 0] < nf]
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        det = fe.detector_create()
        if kind == "depth":
            hs, nfeat = fe.nodes_create(det, gray[:nf], depth[:nf], None, K4, ids=np.arange(nf, dtype=np.int32), mask_from_depth=True)
        else:
            hs, nfeat = [], []
            for a in range(0, nf, args.cloud_chunk):
                b = min(a + args.cloud_chunk, nf)
                stage[:b - a].copy_(cloud_of(d_d[a:b]))
                h, f = fe.nodes_create(det, gray[a:b], stage[:b - a], None, None, ids=np.arange(a, b, dtype=np.int32),
                                       mask_from_cloud=True)
                hs += h
                nfeat += list(f)
        t1 = time.perf_counter()
        res = np.zeros(len(pp), PAIR_RESULT_DTYPE); res["id1"] = -1; res["id2"] = -1
        pipeline.match_pairs_pipelined(fe, hs, pp, seed=seed, first_pair_index=0, out=res)
        graph = graph_from_pairs(pp, res, nf)
        traj, chi2, lm, cg = fe.optimize_graph(graph["init"], graph["fixed"], graph["ij"], graph["meas"], graph["info"], stop=0.01)
        t2 = time.perf_counter()
        fe.detector_destroy(det)
        for h in hs:
            fe.node_destroy(h)
        return nfeat, res, graph, traj, chi2, lm, t2 - t0

    c4 = {}
    for kind in ("cloud", "depth"):
        sequence(kind, min(nf_, 96))
        nfeat, res, graph, traj, chi2, lm, secs = sequence(kind, nf_)
        c4[kind] = {"frames": nf_, "pairs": int(len(pairs)), "valid_edges": int(graph["n_valid_edges"]),
                    "mean_features": float(np.mean(nfeat)), "mean_inliers_valid": float(res["n_inliers"][res["id1"] >= 0].mean()),
                    "lm_iterations": lm, "chi2": chi2, "ate_vs_gt_m": synth.ate_rmse(traj[:, :3], gt[:, :3]), "seconds": secs}
    out["c4"] = c4
    fe.close()
    print(json.dumps(out))


def main_raw(args):
    import cv2
    import torch
    from torch.profiler import ProfilerActivity, profile

    from rgbdslam_v2_b200 import Frontend, pipeline, synth
    from rgbdslam_v2_b200._capi import DETECTOR_ORB, PAIR_RESULT_DTYPE, default_params, graph_from_pairs
    if not torch.cuda.is_available():
        raise SystemExit("run_nodes.py measures on the GPU; no CUDA device found")
    dev = torch.device("cuda", 0)
    K4 = (synth.FX, synth.FY, synth.CX, synth.CY)
    seed = 11
    p = default_params(); p.depth_cov_z0 = 2.0; p.max_keypoints = args.keypoints; p.feature_detector_type = DETECTOR_ORB
    fe = Frontend(0, p)

    n = max(args.frames, args.timing_frames)
    poses = synth.trajectory(n)
    g_d, d_d = synth.render_frames_torch(poses, dev)
    H, W = g_d.shape[1:]

    def pinned(t):
        h = torch.empty(t.shape, dtype=t.dtype).pin_memory()
        h.copy_(t)
        return h

    # what a 16UC1 sensor sends: millimetres, 0 where there is no depth
    mm = d_d * 1000.0
    ok = torch.isfinite(mm) & (mm > 0) & (mm < 65535.5)
    depth_mm = pinned(torch.where(ok, mm.nan_to_num(0.0).round(), torch.zeros_like(mm)).to(torch.int32).cpu().to(torch.uint16))
    del mm, ok
    nt = args.timing_frames
    rgb_d = torch.stack([g_d[:nt], g_d[:nt].roll(3, -1), g_d[:nt].roll(5, -2)], -1)
    yy, xx = torch.meshgrid(torch.arange(H, device=dev), torch.arange(W, device=dev), indexing="ij")
    ch = torch.where(yy % 2 == 0, torch.where(xx % 2 == 0, 1, 2), torch.where(xx % 2 == 0, 0, 1))  # G B / R G
    bayer = pinned(torch.gather(rgb_d, 3, ch.expand(nt, H, W).unsqueeze(-1)).squeeze(-1).contiguous())
    rgb = pinned(rgb_d)
    gray = pinned(g_d)
    depth = pinned(d_d)
    del g_d, rgb_d
    torch.cuda.synchronize()
    px = H * W
    out = {"card": card(), "image": f"{W}x{H}", "max_keypoints": args.keypoints, "detector": "ORB", "mask": "MASK_FROM_DEPTH"}
    # name: (visual, depth, keyword, host->device bytes per frame)
    base = {"gray_float": (gray, depth, {}, px + 4 * px), "gray_u16": (gray, depth_mm, {}, px + 2 * px),
            "rgb_float": (rgb, depth, {}, 3 * px + 4 * px), "bayer_u16": (bayer, depth_mm, {"bayer": True}, px + 2 * px)}
    configs = {}
    for k, (v, d, kw, b) in base.items():
        configs[k + "_pinned"] = (v[:nt], d[:nt], kw, b)
    for k, (v, d, kw, b) in base.items():
        configs[k + "_pageable"] = (v[:nt].numpy().copy(), d[:nt].numpy().copy(), kw, b)

    def call(cfg, frames=None):
        vis, dep, kw, _ = configs[cfg]
        m = frames or nt
        det = fe.detector_create()
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        hs, nf = fe.nodes_create(det, vis[:m], dep[:m], None, K4, mask_from_depth=True, **kw)
        dt = time.perf_counter() - t0
        fe.detector_destroy(det)
        for h in hs:
            fe.node_destroy(h)
        return m / dt, float(np.mean(nf))

    # ---- 1. the constructor alone, inputs alternated
    timing = {c: [] for c in configs}
    feats = {}
    for r in range(args.rounds + 1):  # round 0 warms up every configuration
        for c in configs:
            fps, feats[c] = call(c)
            if r:
                timing[c].append(fps)
    out["nodes_create_frames"] = nt
    out["nodes_create_frames_per_s"] = {k: {"runs": [round(x, 1) for x in vs], "min": round(min(vs), 1), "max": round(max(vs), 1)}
                                        for k, vs in timing.items()}
    out["nodes_create_mean_features"] = feats
    out["h2d_bytes_per_frame"] = {k: c[3] for k, c in base.items()}

    # ---- the conversion kernels' device time per frame (torch.profiler, separate pass)
    kernels = ("k_depth_gather", "k_bayer_gr_to_gray", "k_rgb_to_gray")
    prof_frames = min(64, nt)
    ktimes = {}
    for c in ("bayer_u16_pinned", "rgb_float_pinned"):
        call(c, prof_frames)
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            call(c, prof_frames)
        tot = {}
        for e in prof.events():
            m = re.search(r"rb200::(k_\w+)", e.name)
            if e.device_type.name == "CUDA" and m and m.group(1) in kernels:
                tot[m.group(1)] = tot.get(m.group(1), 0.0) + e.device_time
        allk = sum(e.device_time for e in prof.events() if e.device_type.name == "CUDA" and "rb200::k_" in e.name)
        ktimes[c] = {k: round(t / prof_frames, 3) for k, t in sorted(tot.items())}
        ktimes[c]["all_library_kernels"] = round(allk / prof_frames, 2)
    out["kernel_us_per_frame"] = ktimes

    # ---- the host conversions a caller no longer makes, per frame (one thread)
    cv2.setNumThreads(1)
    hb, hd = bayer[:64].numpy(), depth_mm[:64].numpy()

    def per_frame_us(fn):
        for f in range(4):
            fn(f)
        t0 = time.perf_counter()
        for f in range(len(hb)):
            fn(f)
        return round((time.perf_counter() - t0) / len(hb) * 1e6, 1)
    out["host_us_per_frame"] = {
        "cv2_cvtColor_BayerGR2RGB": per_frame_us(lambda f: cv2.cvtColor(hb[f], cv2.COLOR_BayerGR2RGB)),
        "numpy_depth_u16_to_float": per_frame_us(lambda f: hd[f].astype(np.float32) * np.float32(0.001)),
        "cv2_convertScaleAbs_u16_mask": per_frame_us(lambda f: cv2.convertScaleAbs(hd[f], alpha=0.05, beta=-25)),
    }

    # ---- 2. the C4 sequence with 16-bit nodes against float nodes
    nf_ = args.frames
    pairs = np.array(pipeline.candidate_pairs(nf_, seed=seed), np.int64)
    gt = np.stack([pipeline.mat_to_pose7(np.linalg.inv(poses[0]) @ P) for P in poses[:nf_]])
    fe.posegraph_reserve(nf_, 12 * nf_)

    def sequence(dep, nf):
        pp = pairs[pairs[:, 0] < nf]
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        det = fe.detector_create()
        hs, nfeat = fe.nodes_create(det, gray[:nf], dep[:nf], None, K4, ids=np.arange(nf, dtype=np.int32), mask_from_depth=True)
        res = np.zeros(len(pp), PAIR_RESULT_DTYPE); res["id1"] = -1; res["id2"] = -1
        pipeline.match_pairs_pipelined(fe, hs, pp, seed=seed, first_pair_index=0, out=res)
        graph = graph_from_pairs(pp, res, nf)
        traj, chi2, lm, cg = fe.optimize_graph(graph["init"], graph["fixed"], graph["ij"], graph["meas"], graph["info"], stop=0.01)
        t1 = time.perf_counter()
        zeros = 0
        for h in hs[:64]:
            zeros += int((fe.node_download(h)[1][:, 2] == 0).sum())
        fe.detector_destroy(det)
        for h in hs:
            fe.node_destroy(h)
        return nfeat, res, graph, traj, chi2, lm, t1 - t0, zeros

    c4 = {}
    for kind, dep in (("u16", depth_mm), ("float", depth)):
        sequence(dep, min(nf_, 96))
        nfeat, res, graph, traj, chi2, lm, secs, zeros = sequence(dep, nf_)
        c4[kind] = {"frames": nf_, "pairs": int(len(pairs)), "valid_edges": int(graph["n_valid_edges"]),
                    "mean_features": float(np.mean(nfeat)), "mean_inliers_valid": float(res["n_inliers"][res["id1"] >= 0].mean()),
                    "lm_iterations": lm, "chi2": chi2, "ate_vs_gt_m": synth.ate_rmse(traj[:, :3], gt[:, :3]), "seconds": secs,
                    "z0_points_first_64_nodes": zeros}
    out["c4"] = c4
    fe.close()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
