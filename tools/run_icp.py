"""The ICP fallback of matchNodePair (rgbdslam_b200_icp_align_ex) on the C4 sequence: --frames rendered 640x480 frames, grey
visuals, float depth, STORE_CLOUD, cloud_creation_skip_step 2, max_cloud_size 10000, each raw and voxel-reduced (0.02), for
icp_method "icp", "icp_nl" or both (--method), on the same pairs in one run.

For each method and kind of cloud:
1. online: one adjacent pair (k -> k + 1, older onto newer) per call, as matchNodePair meets it once per new node: wall time
   per call (host clock, each call ends in a device synchronise), --online-calls calls after a warm-up;
2. batch: --batch adjacent pairs in one call: wall time, best of --rounds after a warm-up;
3. the device time per kernel of one batch call (torch.profiler, a pass of its own);
4. a host baseline: the float64 ICP of tests/test_icp_exact_cpu.py (scipy cKDTree, numpy SVD; a restatement with the same
   rules, not PCL) on --host-pairs pairs of the filtered clouds, projected to the batch (icp only);
5. icp_nl only: the LM iterations (Jacobians) and function evaluations per ICP iteration, from the float32 restatement of
   tests/icp_nl_exact.py (equal to the device bit for bit) on --lm-pairs pairs.
And for each method, on the raw clouds: max |T - M| of frames 0->1, 20->21, 50->51, 100->101 against the true motion M of the
trajectory, beside the identity's.

Prints one JSON object, with the card name, power limit and maximum SM clock read in the same run.
Usage: python tools/run_icp.py [--method icp|icp_nl|both] [--frames 1001] [--batch 1000] [--online-calls 200] [--rounds 3]
                                [--host-pairs 10] [--lm-pairs 4]
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
    ap.add_argument("--lm-pairs", type=int, default=4)
    ap.add_argument("--method", choices=("icp", "icp_nl", "both"), default="icp")
    args = ap.parse_args()

    import torch
    from torch.profiler import ProfilerActivity, profile

    import icp_exact as ix
    import icp_nl_exact as nx
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
    hq = max(hp, min(args.lm_pairs, n - 1))
    g_np, d_np = gray[:hq + 1].numpy(), depth[:hq + 1].numpy()
    pcs = [mx.create_cloud(d_np[k], g_np[k], K4, 2, p.depth_scaling_factor, p.minimum_depth) for k in range(hq + 1)]
    methods = ("icp", "icp_nl") if args.method == "both" else (args.method,)
    # max |T - M| against the true motion (older camera frame -> newer), beside the identity's
    truth = {}
    for k in (0, 20, 50, 100):
        if k + 1 < n:
            M = np.linalg.inv(poses[k + 1]) @ poses[k]
            for method in methods:
                T = fe.icp_align([hs[k]], [hs[k + 1]], method=method)[0]["T"].reshape(4, 4).T.astype(np.float64)
                truth.setdefault(method, {})[f"{k}->{k + 1}"] = round(float(np.abs(T - M).max()), 4)
            truth.setdefault("identity", {})[f"{k}->{k + 1}"] = round(float(np.abs(np.eye(4) - M).max()), 4)
    out["max_abs_T_minus_true_motion"] = truth
    for kind in ("raw", "voxel_0.02"):
        if kind != "raw":
            import voxel_exact as vx
            fe.reduce_clouds(hs, 0.02)
            pcs = [vx.reduce_cloud(pc, 0.02) for pc in pcs]
        for method in methods:
            out.setdefault(method, {})[kind] = measure(fe, hs, pcs, method, args, n, nb, hp, ix, nx)
    fe.close()
    print(json.dumps(out))


def measure(fe, hs, pcs, method, args, n, nb, hp, ix, nx):
    from torch.profiler import ProfilerActivity, profile
    from test_icp_exact_cpu import icp64
    res = {}
    src, tgt = hs[:-1], hs[1:]
    fe.icp_align(src[:8], tgt[:8], method=method)  # warm-up
    walls = []
    for k in range(min(args.online_calls, n - 1)):
        t0 = time.perf_counter()
        fe.icp_align([src[k]], [tgt[k]], method=method)
        walls.append(time.perf_counter() - t0)
    res["online_ms_per_call"] = {"median": round(statistics.median(walls) * 1e3, 3), "min": round(min(walls) * 1e3, 3),
                                 "max": round(max(walls) * 1e3, 3), "calls": len(walls)}
    fe.icp_align(src[:nb], tgt[:nb], method=method)  # warm-up at the batch's size
    walls = []
    for _ in range(args.rounds):
        t0 = time.perf_counter()
        r = fe.icp_align(src[:nb], tgt[:nb], method=method)
        walls.append(time.perf_counter() - t0)
    res["batch"] = {"pairs": nb, "wall_s": [round(w, 4) for w in walls], "wall_s_best": round(min(walls), 4),
                    "pairs_per_s": round(nb / min(walls), 1)}
    res["iterations"] = {str(int(v)): int((r["iterations"] == v).sum()) for v in np.unique(r["iterations"])}
    res["criteria"] = {str(int(v)): int((r["criterion"] == v).sum()) for v in np.unique(r["criterion"])}
    res["mean_points"] = {"source": round(float(r["n_source"].mean()), 1), "correspondences": round(float(r["n_correspondences"].mean()), 1)}
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fe.icp_align(src[:nb], tgt[:nb], method=method)
        fe.synchronize()
    kern = {}
    for e in prof.events():
        # k_icp_filter, k_icp_cells and the align kernel of the method's estimator: k_icp_align<IcpSvd> or <IcpLm>
        mm = re.search(r"rb200::(k_icp_\w+(?:<rb200::\w+>)?)", e.name) if e.device_type.name == "CUDA" else None
        if mm:
            k = mm.group(1).replace("rb200::", "")
            kern[k] = kern.get(k, 0.0) + e.device_time
    res["batch_device_kernel_ms"] = {k: round(v / 1e3, 3) for k, v in sorted(kern.items())}
    res["batch_device_kernel_ms_total"] = round(sum(kern.values()) / 1e3, 3)
    clouds = [ix.filter_cloud(pc, 10000) for pc in pcs]
    if method == "icp":  # the float64 host restatement (not PCL) on the first pairs, and the device's agreement with it
        t0 = time.perf_counter()
        ref = [icp64(clouds[k], clouds[k + 1], margin=None) for k in range(hp)]
        host = time.perf_counter() - t0
        got = fe.icp_align(src[:hp], tgt[:hp])
        dev_T = [g["T"].reshape(4, 4).T.astype(np.float64) for g in got]
        res["host_float64_restatement"] = {
            "pairs": hp, "s_per_pair": round(host / hp, 4), "projected_s_batch": round(host / hp * nb, 1),
            "max_abs_T_difference_to_device": float(max(np.abs(a["T"] - b).max() for a, b in zip(ref, dev_T)))}
        res["speedup_batch_vs_host_projected"] = round(host / hp * nb / min(walls), 1)
    else:  # the LM's work per ICP iteration, from the float32 restatement (equal to the device), and that they agree
        lp = min(args.lm_pairs, len(clouds) - 1)
        t0 = time.perf_counter()
        ref = [nx.align_points(clouds[k], clouds[k + 1]) for k in range(lp)]
        host = time.perf_counter() - t0
        got = fe.icp_align(src[:lp], tgt[:lp], method=method)
        lm = [x for e in ref for x in e["lm"]]
        res["lm_per_icp_iteration"] = {
            "pairs": lp, "icp_iterations": [e["iterations"] for e in ref], "lm_iterations": [x[2] for x in lm],
            "function_evaluations": [x[1] for x in lm], "status": [x[0] for x in lm],
            "restatement_s_per_pair": round(host / max(lp, 1), 2),
            "device_equals_restatement": bool(all(np.array_equal(g["T"], e["T"].T.ravel()) and g["iterations"] == e["iterations"]
                                                  for g, e in zip(got, ref)))}
    return res


if __name__ == "__main__":
    main()
