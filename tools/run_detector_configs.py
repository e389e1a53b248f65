"""Node-constructor throughput and the reference's detector experiment under the three detectors createDetector returns
(DESIGN.md 4.5.7): Grid (3x3 adjuster), Adjuster (ungridded adjuster) and Regular (adjuster_max_iterations 0), ORB and FAST.

Throughput: 640x480 rendered C4 frames at max_keypoints 1000, mask from depth, from pinned buffers.  --distinct frames of the
240-pose trajectory are rendered and cycled to --frames frames.  Each configuration is one call over all frames with a fresh
detector, timed with a host clock around the work, which ends in a device synchronisation; --rounds rounds alternate the
configurations, and the best and the worst round of each are reported.

Experiment (the reference's test/experiments.sh compares its detectors by the edges they give and the trajectory): the
--c4-frames-frame C4 sequence of bench.py (torch-rendered frames, the same candidate pairs and seed, max_keypoints 1000,
ORB) through nodes_create, the pipelined pair matcher, the host graph and the pose-graph solve, per configuration: valid
edges, mean features and the ATE against the rendering's ground truth.

Prints one JSON object, with the card name and power limit read in the same run.
Usage: python tools/run_detector_configs.py [--frames 600] [--distinct 60] [--rounds 5] [--c4-frames 2000]
"""
import argparse
import json
import subprocess
import sys
import time
from pathlib import Path

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))
sys.path.insert(0, str(ROOT / "tests"))
import numpy as np  # noqa: E402

CONFIGS = {"Grid": dict(detector_grid_resolution=3, adjuster_max_iterations=5),
           "Adjuster": dict(detector_grid_resolution=0, adjuster_max_iterations=5),
           "Regular": dict(detector_grid_resolution=0, adjuster_max_iterations=0)}


def card() -> dict:
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                       text=True)
    name, power, clk = (x.strip() for x in q.stdout.splitlines()[0].split(","))
    return {"name": name, "power_limit": power, "max_sm_clock": clk}


_C4 = {}


def c4_experiment(fe, n_frames, kw, seed=11):
    """bench.py's C4 chain with the ORB detector of kw: valid edges, mean features and ATE against the ground truth"""
    import torch

    import node_helpers as nh
    from rgbdslam_v2_b200 import pipeline, synth
    from rgbdslam_v2_b200._capi import PAIR_RESULT_DTYPE, graph_from_pairs
    poses = synth.trajectory(n_frames)
    if n_frames not in _C4:  # rendered once for the three configurations
        g, d = synth.render_frames_torch(poses, torch.device("cuda", 0))
        _C4[n_frames] = g.cpu().pin_memory(), d.cpu().pin_memory()
        del g, d
    gray, depth = _C4[n_frames]
    pairs = np.array(pipeline.candidate_pairs(n_frames, seed=seed), np.int64)
    gt = np.stack([pipeline.mat_to_pose7(np.linalg.inv(poses[0]) @ P) for P in poses])
    nh.reinit(fe, 0, max_keypoints=1000, **kw)
    fe.posegraph_reserve(n_frames, 12 * n_frames)
    det = fe.detector_create()
    handles, nfeat = fe.nodes_create(det, gray, depth, None, nh.K4(), ids=np.arange(n_frames, dtype=np.int32), mask_from_depth=True)
    res = np.zeros(len(pairs), PAIR_RESULT_DTYPE)
    res["id1"] = -1
    res["id2"] = -1
    pipeline.match_pairs_pipelined(fe, handles, pairs, seed=seed, out=res)
    graph = graph_from_pairs(pairs, res, n_frames)
    traj, chi2, lm, cg = fe.optimize_graph(graph["init"], graph["fixed"], graph["ij"], graph["meas"], graph["info"], stop=0.01)
    fe.detector_destroy(det)
    nh.destroy(fe, handles)
    return {"pairs": int(len(pairs)), "valid_edges": int(graph["n_valid_edges"]), "mean_features": round(float(np.mean(nfeat)), 1),
            "ate_vs_gt_m": synth.ate_rmse(traj[:, :3], gt[:, :3])}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=600)
    ap.add_argument("--distinct", type=int, default=60)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--c4-frames", type=int, default=2000)
    args = ap.parse_args()
    import torch

    import node_helpers as nh
    from rgbdslam_v2_b200 import Frontend
    gray, depth, _ = nh.seq(args.distinct)
    idx = np.arange(args.frames) % args.distinct
    pg, pd = torch.from_numpy(gray[idx]).pin_memory(), torch.from_numpy(depth[idx]).pin_memory()
    fe = Frontend(0, nh.params())
    rates = {}
    for _ in range(args.rounds):
        for det_type in (0, 1):
            for name, kw in CONFIGS.items():
                nh.reinit(fe, det_type, max_keypoints=1000, **kw)
                det = fe.detector_create()
                t0 = time.perf_counter()
                hs, nf = fe.nodes_create(det, pg, pd, None, nh.K4(), mask_from_depth=True)
                dt = time.perf_counter() - t0
                fe.detector_destroy(det)
                nh.destroy(fe, hs)
                rates.setdefault(f"{nh.name(det_type)}_{name}", []).append((args.frames / dt, float(np.mean(nf))))
    best = {k: {"frames_per_s_best": round(max(r for r, _ in v), 1), "frames_per_s_worst": round(min(r for r, _ in v), 1),
                "mean_features": round(v[0][1], 1)} for k, v in rates.items()}
    c4 = {name: c4_experiment(fe, args.c4_frames, kw) for name, kw in CONFIGS.items()} if args.c4_frames else {}
    fe.close()
    print(json.dumps({"card": card(), "frames": args.frames, "rounds": args.rounds, "max_keypoints": 1000, "size": "640x480",
                      "configs": best, "c4_orb": c4}))


if __name__ == "__main__":
    main()
