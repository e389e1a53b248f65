"""The ICP fallback of matchNodePair (rgbdslam_b200_icp_align) on the C4 sequence: --frames rendered 640x480 frames, grey
visuals, float depth, STORE_CLOUD, cloud_creation_skip_step 2, max_cloud_size 10000, each raw and voxel-reduced (0.02).

For each kind of cloud:
1. online: one adjacent pair (k -> k + 1, older onto newer) per call, as matchNodePair meets it once per new node: wall time
   per call (host clock, each call ends in a device synchronise), --online-calls calls after a warm-up;
2. batch: --batch adjacent pairs in one call: wall time, best of --rounds after a warm-up;
3. the device time per kernel of one batch call (torch.profiler, a pass of its own);
4. a host baseline: the float64 ICP of tests/test_icp_exact_cpu.py (scipy cKDTree, numpy SVD; a restatement with the same
   rules, not PCL) on --host-pairs pairs of the filtered clouds, projected to the batch.

Prints one JSON object, with the card name, power limit and maximum SM clock read in the same run.
Usage: python tools/run_icp.py [--frames 1001] [--batch 1000] [--online-calls 200] [--rounds 3] [--host-pairs 10]
"""
import argparse
import json
import re
import statistics
import sys
import time
from pathlib import Path

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))
sys.path.insert(0, str(ROOT / "tests"))
sys.path.insert(0, str(ROOT / "tools"))
import numpy as np  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=1001)
    ap.add_argument("--batch", type=int, default=1000)
    ap.add_argument("--online-calls", type=int, default=200)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--host-pairs", type=int, default=10)
    args = ap.parse_args()

    import torch
    from torch.profiler import ProfilerActivity, profile

    import icp_exact as ix
    import map_cloud_exact as mx
    from run_map import card
    from test_icp_exact_cpu import icp64
    from rgbdslam_v2_b200 import Frontend, synth
    from rgbdslam_v2_b200._capi import default_params
    if not torch.cuda.is_available():
        raise SystemExit("run_icp.py measures on the GPU; no CUDA device found")
    dev = torch.device("cuda", 0)
    out = {"card": card(), "frames": args.frames, "skip_step": 2, "max_cloud_size": 10000}
    K4 = (synth.FX, synth.FY, synth.CX, synth.CY)
    poses = synth.trajectory(args.frames)
    g_d, d_d = synth.render_frames_torch(poses, dev)
    gray = torch.empty(g_d.shape, dtype=torch.uint8).pin_memory()
    gray.copy_(g_d)
    depth = torch.empty(d_d.shape, dtype=torch.float32).pin_memory()
    depth.copy_(d_d)
    del g_d, d_d
    torch.cuda.synchronize()
    torch.cuda.empty_cache()
    n = gray.shape[0]
    nb = min(args.batch, n - 1)

    p = default_params()
    p.depth_cov_z0 = 2.0
    p.cloud_creation_skip_step = 2
    fe = Frontend(0, p)
    det = fe.detector_create()
    hs, _ = fe.nodes_create(det, gray, depth, None, K4, store_cloud=True)
    fe.detector_destroy(det)
    hp = min(args.host_pairs, n - 1)
    g_np, d_np = gray[:hp + 1].numpy(), depth[:hp + 1].numpy()
    pcs = [mx.create_cloud(d_np[k], g_np[k], K4, 2, p.depth_scaling_factor, p.minimum_depth) for k in range(hp + 1)]
    for kind in ("raw", "voxel_0.02"):
        res = {}
        if kind != "raw":
            fe.reduce_clouds(hs, 0.02)
            import voxel_exact as vx
            pcs = [vx.reduce_cloud(pc, 0.02) for pc in pcs]
        src, tgt = hs[:-1], hs[1:]
        fe.icp_align(src[:8], tgt[:8])  # warm-up
        walls = []
        for k in range(min(args.online_calls, n - 1)):
            t0 = time.perf_counter()
            fe.icp_align([src[k]], [tgt[k]])
            walls.append(time.perf_counter() - t0)
        res["online_ms_per_call"] = {"median": round(statistics.median(walls) * 1e3, 3), "min": round(min(walls) * 1e3, 3),
                                     "max": round(max(walls) * 1e3, 3), "calls": len(walls)}
        fe.icp_align(src[:nb], tgt[:nb])  # warm-up at the batch's size
        walls = []
        for _ in range(args.rounds):
            t0 = time.perf_counter()
            r = fe.icp_align(src[:nb], tgt[:nb])
            walls.append(time.perf_counter() - t0)
        res["batch"] = {"pairs": nb, "wall_s": [round(w, 4) for w in walls], "wall_s_best": round(min(walls), 4),
                        "pairs_per_s": round(nb / min(walls), 1)}
        res["iterations"] = {str(int(v)): int((r["iterations"] == v).sum()) for v in np.unique(r["iterations"])}
        res["criteria"] = {str(int(v)): int((r["criterion"] == v).sum()) for v in np.unique(r["criterion"])}
        res["mean_points"] = {"source": round(float(r["n_source"].mean()), 1), "correspondences": round(float(r["n_correspondences"].mean()), 1)}
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            fe.icp_align(src[:nb], tgt[:nb])
            fe.synchronize()
        kern = {}
        for e in prof.events():
            mm = re.search(r"rb200::(k_icp_\w+)", e.name) if e.device_type.name == "CUDA" else None
            if mm:
                kern[mm.group(1)] = kern.get(mm.group(1), 0.0) + e.device_time
        res["batch_device_kernel_ms"] = {k: round(v / 1e3, 3) for k, v in sorted(kern.items())}
        res["batch_device_kernel_ms_total"] = round(sum(kern.values()) / 1e3, 3)
        # the float64 host restatement (not PCL) on the first pairs, and the device's agreement with the float32 one
        clouds = [ix.filter_cloud(pc, 10000) for pc in pcs]
        t0 = time.perf_counter()
        ref = [icp64(clouds[k], clouds[k + 1], margin=None) for k in range(hp)]
        host = time.perf_counter() - t0
        got = fe.icp_align(src[:hp], tgt[:hp])
        dev_T = [g["T"].reshape(4, 4).T.astype(np.float64) for g in got]
        res["host_float64_restatement"] = {
            "pairs": hp, "s_per_pair": round(host / hp, 4), "projected_s_batch": round(host / hp * nb, 1),
            "max_abs_T_difference_to_device": float(max(np.abs(a["T"] - b).max() for a, b in zip(ref, dev_T)))}
        res["speedup_batch_vs_host_projected"] = round(host / hp * nb / min(walls), 1)
        out[kind] = res
    fe.close()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
