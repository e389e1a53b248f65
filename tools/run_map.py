"""The stored colour clouds (RGBDSLAM_B200_STORE_CLOUD) and the registered map (rgbdslam_b200_render_cloud) on the C4 sequence:
--frames rendered 640x480 frames, max_keypoints --keypoints, grey visuals, float depth, MASK_FROM_DEPTH, pinned input.

1. nodes_create_ex frames/s of the whole sequence in one call, without and with STORE_CLOUD, alternated --rounds times (host
   clock around the call, which returns after the device work has finished).
2. The device time per frame of k_store_depth_cloud (torch.profiler, separate pass) and the device bytes per node.
3. render_cloud of the whole map (every node, its ground-truth pose through saveAllCloudsToFile's cam2rgb composition) into a
   pinned host buffer: wall time (best of --rounds), the device time of the map kernels and of the device-to-host copies
   (torch.profiler, separate pass), the bytes copied and GB/s against the copy bound -- a plain pinned device-to-host copy of
   the same number of bytes, measured in the same run.
4. The host baseline: the numpy restatement (tests/map_cloud_exact.py, one thread) of createXYZRGBPointCloud and
   transformAndAppendPointCloud on the first --host-nodes nodes, checked against the device records, projected to the
   whole sequence.

Prints one JSON object, with the card name and power limit read in the same run.
Usage: python tools/run_map.py [--frames 2000] [--rounds 3]
"""
import argparse
import json
import re
import subprocess
import sys
import time
from pathlib import Path

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))
sys.path.insert(0, str(ROOT / "tests"))
import numpy as np  # noqa: E402


def card() -> dict:
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                       text=True)
    name, power, clk = (x.strip() for x in q.stdout.splitlines()[0].split(","))
    return {"name": name, "power_limit": power, "max_sm_clock": clk}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=2000)
    ap.add_argument("--keypoints", type=int, default=1000)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--profile-frames", type=int, default=256)
    ap.add_argument("--host-nodes", type=int, default=100)
    args = ap.parse_args()

    import torch
    from torch.profiler import ProfilerActivity, profile

    import map_cloud_exact as mx
    from rgbdslam_v2_b200 import Frontend, synth
    from rgbdslam_v2_b200._capi import default_params
    if not torch.cuda.is_available():
        raise SystemExit("run_map.py measures on the GPU; no CUDA device found")
    dev = torch.device("cuda", 0)
    out = {"card": card(), "frames": args.frames, "keypoints": args.keypoints}
    K4 = (synth.FX, synth.FY, synth.CX, synth.CY)
    poses = synth.trajectory(args.frames)
    g_d, d_d = synth.render_frames_torch(poses, dev)
    gray = torch.empty(g_d.shape, dtype=torch.uint8).pin_memory()
    gray.copy_(g_d)
    depth = torch.empty(d_d.shape, dtype=torch.float32).pin_memory()
    depth.copy_(d_d)
    del g_d, d_d
    torch.cuda.synchronize()
    n, H, W = gray.shape

    p = default_params()
    p.depth_cov_z0 = 2.0
    p.max_keypoints = args.keypoints
    fe = Frontend(0, p)

    def create(m, store):
        det = fe.detector_create()
        t0 = time.perf_counter()
        hs, _ = fe.nodes_create(det, gray[:m], depth[:m], None, K4, mask_from_depth=True, store_cloud=store)
        dt = time.perf_counter() - t0
        fe.detector_destroy(det)
        return hs, dt

    # ---- 1. Node constructor with and without stored clouds, alternated
    for store in (False, True):  # warm-up: module load, buffers
        hs, _ = create(min(64, n), store)
        for h in hs:
            fe.node_destroy(h)
    fps = {"plain": [], "store_cloud": []}
    keep = None
    for r in range(args.rounds):
        for store in (False, True):
            hs, dt = create(n, store)
            fps["store_cloud" if store else "plain"].append(round(n / dt, 1))
            if store and r == args.rounds - 1:
                keep = hs
            else:
                for h in hs:
                    fe.node_destroy(h)
    out["nodes_create_fps"] = fps
    out["nodes_create_fps_best"] = {k: max(v) for k, v in fps.items()}

    # ---- 2. the store kernel's device time per frame, device bytes per node
    m = min(args.profile_frames, n)
    hs, _ = create(m, True)
    for h in hs:
        fe.node_destroy(h)
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        hs, _ = create(m, True)
    for h in hs:
        fe.node_destroy(h)
    ks = sum(e.device_time for e in prof.events() if e.device_type.name == "CUDA" and "k_store_depth_cloud" in e.name)
    out["k_store_depth_cloud_us_per_frame"] = round(ks / m, 3)
    step = p.cloud_creation_skip_step
    cw, ch = W // step, H // step
    out["cloud_bytes_per_node"] = (cw * ch * 8 + 255) // 256 * 256
    out["cloud_points_per_node"] = cw * ch

    # ---- 3. the whole map
    T = np.stack([mx.world2cam(P) for P in poses])
    npts = fe.render_cloud(keep, T, count_only=True)
    buf = torch.empty(npts * 32, dtype=torch.uint8).pin_memory()
    fe.render_cloud(keep, T, out=buf)  # warm-up
    walls = []
    for _ in range(args.rounds):
        t0 = time.perf_counter()
        fe.render_cloud(keep, T, out=buf)
        walls.append(time.perf_counter() - t0)
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fe.render_cloud(keep, T, out=buf)
    kern, copy = {}, 0.0
    for e in prof.events():
        if e.device_type.name != "CUDA":
            continue
        mm = re.search(r"rb200::(k_map_\w+)", e.name)
        if mm:
            kern[mm.group(1)] = kern.get(mm.group(1), 0.0) + e.device_time
        elif "Memcpy DtoH" in e.name or "DtoH" in e.name:
            copy += e.device_time
    # the copy bound: one pinned device-to-host copy of the same bytes
    src = torch.empty(npts * 32, dtype=torch.uint8, device=dev)
    buf.copy_(src, non_blocking=True)
    torch.cuda.synchronize()
    cb = []
    for _ in range(args.rounds):
        t0 = time.perf_counter()
        buf.copy_(src, non_blocking=True)
        torch.cuda.synchronize()
        cb.append(time.perf_counter() - t0)
    del src
    nbytes = npts * 32
    out["render"] = {
        "nodes": len(keep), "points": int(npts), "bytes_to_host": int(nbytes), "wall_s": [round(w, 4) for w in walls],
        "wall_s_best": round(min(walls), 4), "gb_per_s": round(nbytes / min(walls) / 1e9, 2),
        "copy_bound_s": round(min(cb), 4), "copy_bound_gb_per_s": round(nbytes / min(cb) / 1e9, 2),
        "share_of_copy_bound": round(min(cb) / min(walls), 3),
        "device_kernel_ms": {k: round(v / 1e3, 2) for k, v in sorted(kern.items())}, "device_copy_ms": round(copy / 1e3, 2),
    }

    # ---- 4. host baseline: the numpy restatement on one thread, checked against the device records
    hn = min(args.host_nodes, n)
    g_np, d_np = gray[:hn].numpy(), depth[:hn].numpy()
    t0 = time.perf_counter()
    pcs = [mx.create_cloud(d_np[k], g_np[k], K4, step, p.depth_scaling_factor, p.minimum_depth) for k in range(hn)]
    ref = mx.render(pcs, T[:hn])
    host = time.perf_counter() - t0
    got, _ = fe.render_cloud(keep[:hn], T[:hn])
    out["host_restatement"] = {"nodes": hn, "s": round(host, 3), "s_per_node": round(host / hn, 5),
                               "projected_s_all_nodes": round(host / hn * n, 1), "equal_to_device": bool(
                                   np.array_equal(got.view(np.uint8), ref.view(np.uint8)))}
    out["speedup_vs_host_projected"] = round(host / hn * n / min(walls), 1)
    for h in keep:
        fe.node_destroy(h)
    fe.close()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
