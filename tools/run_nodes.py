"""Node constructor with the ORB and the FAST detector (params.feature_detector_type) on the same rendered 640x480 frames.

1. rgbdslam_b200_nodes_create_ex with MASK_FROM_DEPTH from pinned host memory, both detector types alternated --rounds
   times; host clock around the call, which returns after the device work has finished (it downloads the feature counts).
2. The C4 sequence (bench.py: --frames frames, 3 sequential + 4 window + 4 random candidate pairs per frame) with nodes of
   each detector type through matching, graph construction, the pose-graph solve and ATE against the rendering ground truth.

--min-depth: every detector type also with params.use_feature_min_depth (keypoint depth = the nearest point of its
neighbourhood), alternated with the pointwise rule in step 1 and run through step 2 as well ("ORB+min_depth", ...).

Prints one JSON object, with the card name and power limit read in the same run.  Usage: python tools/run_nodes.py [--min-depth]
"""
import argparse
import ctypes as C
import json
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
    args = ap.parse_args()

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


if __name__ == "__main__":
    main()
