"""The voxel filter of the stored clouds (rgbdslam_b200_reduce_clouds) on the C4 sequence: --frames rendered 640x480 frames,
grey visuals, float depth, MASK_FROM_DEPTH, STORE_CLOUD, cloud_creation_skip_step 2, pinned input.

For every leaf size of --leaves (the nodes are built anew each time: the filter replaces their clouds):
1. reduce_clouds of all nodes in one call: wall time with a final synchronise (host clock, --rounds repetitions after a
   warm-up), the points before / after, and the device memory in use (cudaMemGetInfo) before / after.
2. The device time per kernel of one such call (torch.profiler, a pass of its own).
3. render_cloud of the reduced map into a pinned host buffer against render_cloud of the raw map, in the same run: wall time
   (best of --rounds) and bytes.
4. The host baseline: the numpy restatement (tests/voxel_exact.py, one thread) on the first --host-nodes nodes, its records
   compared with the device's, projected to the whole sequence.

Prints one JSON object, with the card name, power limit and maximum SM clock read in the same run.
Usage: python tools/run_voxel.py [--frames 2000] [--rounds 3] [--leaves 0.01,0.02,0.05]
"""
import argparse
import json
import re
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
    ap.add_argument("--frames", type=int, default=2000)
    ap.add_argument("--keypoints", type=int, default=1000)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--host-nodes", type=int, default=100)
    ap.add_argument("--leaves", default="0.01,0.02,0.05")
    args = ap.parse_args()

    import torch
    from torch.profiler import ProfilerActivity, profile

    import map_cloud_exact as mx
    import voxel_exact as vx
    from run_map import card
    from rgbdslam_v2_b200 import Frontend, synth
    from rgbdslam_v2_b200._capi import default_params
    if not torch.cuda.is_available():
        raise SystemExit("run_voxel.py measures on the GPU; no CUDA device found")
    dev = torch.device("cuda", 0)
    out = {"card": card(), "frames": args.frames}
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

    p = default_params()
    p.depth_cov_z0 = 2.0
    p.max_keypoints = args.keypoints
    fe = Frontend(0, p)

    def create():
        det = fe.detector_create()
        hs, _ = fe.nodes_create(det, gray, depth, None, K4, mask_from_depth=True, store_cloud=True)
        fe.detector_destroy(det)
        return hs

    def destroy(hs):
        for h in hs:
            fe.node_destroy(h)

    def used():
        fe.synchronize()
        free, total = torch.cuda.mem_get_info()
        return total - free

    def render_walls(hs, buf):
        fe.render_cloud(hs, T, out=buf)  # warm-up
        walls = []
        for _ in range(args.rounds):
            t0 = time.perf_counter()
            fe.render_cloud(hs, T, out=buf)
            walls.append(time.perf_counter() - t0)
        return walls

    T = np.stack([mx.world2cam(P) for P in poses])
    hs = create()
    raw_points = fe.render_cloud(hs, T, count_only=True)
    buf = torch.empty(raw_points * 32, dtype=torch.uint8).pin_memory()
    walls = render_walls(hs, buf)
    out["render_raw"] = {"points": int(raw_points), "bytes_to_host": int(raw_points) * 32, "wall_s": [round(w, 4) for w in walls],
                         "wall_s_best": round(min(walls), 4)}
    destroy(hs)

    hn = min(args.host_nodes, n)
    g_np, d_np = gray[:hn].numpy(), depth[:hn].numpy()
    pcs = [mx.create_cloud(d_np[k], g_np[k], K4, p.cloud_creation_skip_step, p.depth_scaling_factor, p.minimum_depth)
           for k in range(hn)]
    out["leaves"] = {}
    for leaf in (float(x) for x in args.leaves.split(",")):
        res = {}
        walls = []
        for r in range(args.rounds + 1):  # round 0 warms up
            hs = create()
            before = used()
            stored_points = sum(int(np.prod(fe.node_cloud(h).shape)) for h in hs[:1]) * len(hs)
            fe.synchronize()
            t0 = time.perf_counter()
            counts = fe.reduce_clouds(hs, leaf)
            fe.synchronize()
            dt = time.perf_counter() - t0
            after = used()
            if r > 0:
                walls.append(dt)
            if r < args.rounds:
                destroy(hs)
        res["reduce_wall_s"] = [round(w, 4) for w in walls]
        res["reduce_wall_s_best"] = round(min(walls), 4)
        res["points_before"] = int(stored_points)
        res["points_after"] = int(counts.sum())
        res["nodes_left_alone"] = int((counts < 0).sum())
        res["device_bytes_in_use_before"] = int(before)
        res["device_bytes_in_use_after"] = int(after)
        # the reduced map against the raw one
        rp = fe.render_cloud(hs, T, count_only=True)
        walls = render_walls(hs, buf)
        res["render_reduced"] = {"points": int(rp), "bytes_to_host": int(rp) * 32, "wall_s": [round(w, 4) for w in walls],
                                 "wall_s_best": round(min(walls), 4)}
        # host baseline on the first nodes, compared with the device's records
        t0 = time.perf_counter()
        ref = [vx.reduce_cloud(pc, leaf) for pc in pcs]
        host = time.perf_counter() - t0
        equal = all(np.array_equal(fe.node_cloud(h).view(np.uint8), mx.organised(e).view(np.uint8)) for h, e in zip(hs[:hn], ref))
        res["host_restatement"] = {"nodes": hn, "s": round(host, 3), "s_per_node": round(host / hn, 5),
                                   "projected_s_all_nodes": round(host / hn * n, 1), "equal_to_device": bool(equal)}
        res["speedup_vs_host_projected"] = round(host / hn * n / min(res["reduce_wall_s"]), 1)
        destroy(hs)
        # per-kernel device time, a pass of its own
        hs = create()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            fe.reduce_clouds(hs, leaf)
            fe.synchronize()
        kern = {}
        for e in prof.events():
            mm = re.search(r"rb200::(k_(?:vox|map)_\w+)", e.name) if e.device_type.name == "CUDA" else None
            if mm:
                kern[mm.group(1)] = kern.get(mm.group(1), 0.0) + e.device_time
        res["device_kernel_ms"] = {k: round(v / 1e3, 2) for k, v in sorted(kern.items())}
        res["device_kernel_ms_total"] = round(sum(kern.values()) / 1e3, 2)
        destroy(hs)
        out["leaves"][str(leaf)] = res
    fe.close()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
