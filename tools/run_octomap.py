"""The colour OctoMap (include/rgbdslam_b200/octomap.h) on the C4 sequence: --frames rendered 640x480 colour frames with
STORE_CLOUD at cloud_creation_skip_step 2 (76 800 rays per node), each node under octomap_pose of its ground-truth pose,
resolution 0.05 and the reference's other defaults.

1. Insert rate: one octomap_insert of every node into an empty map (host clock; the call returns after the device work),
   best of --rounds, as nodes/s and rays/s (both measured).  cells_per_s_extrapolated is not measured: it takes the ray and
   occupied cells per node that the oracle counts on the --host-nodes prefix as every node's count.
2. The device time per kernel of one insert of --profile-nodes nodes, and of one write (torch.profiler, separate pass).
3. Write: octomap_write of the whole map (wall, best of --rounds), its size and node / leaf counts.
4. The host baseline: the C oracle (tests/octomap_oracle.c, one thread) on the first --host-nodes nodes, its bytes checked
   against the device's for the same nodes, projected to the whole sequence.

Prints one JSON object, with the card name and power limit read in the same run.
Usage: python tools/run_octomap.py [--frames 300] [--rounds 3]
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
    ap.add_argument("--frames", type=int, default=300)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--profile-nodes", type=int, default=32)
    ap.add_argument("--host-nodes", type=int, default=3)
    args = ap.parse_args()

    import torch
    from torch.profiler import ProfilerActivity, profile

    import octomap_exact as ox
    from rgbdslam_v2_b200 import Frontend, synth
    from rgbdslam_v2_b200._capi import default_params, octomap_pose
    if not torch.cuda.is_available():
        raise SystemExit("run_octomap.py measures on the GPU; no CUDA device found")
    dev = torch.device("cuda", 0)
    out = {"card": card(), "frames": args.frames}
    K4 = (synth.FX, synth.FY, synth.CX, synth.CY)
    poses = synth.trajectory(args.frames)
    g_d, d_d = synth.render_frames_torch(poses, dev)
    gray = g_d.cpu().numpy()
    depth = d_d.cpu().numpy()
    del g_d, d_d
    colour = np.ascontiguousarray(np.stack([gray, np.roll(gray, 3, axis=-1), np.roll(gray, 5, axis=-2)], -1))
    n, H, W = gray.shape
    p = default_params()
    p.depth_cov_z0 = 2.0
    fe = Frontend(0, p)
    det = fe.detector_create()
    hs = []
    for k0 in range(0, n, 64):
        h, _ = fe.nodes_create(det, colour[k0:k0 + 64], depth[k0:k0 + 64], None, K4, store_cloud=True)
        hs += list(h)
    fe.detector_destroy(det)
    T = np.stack([octomap_pose(P) for P in poses])
    step = p.cloud_creation_skip_step
    rays = ((W + step - 1) // step) * ((H + step - 1) // step)
    out["rays_per_node"] = rays

    def insert(m):
        om = fe.octomap_create()
        t0 = time.perf_counter()
        fe.octomap_insert(om, hs[:m], T[:m])
        return om, time.perf_counter() - t0

    om, _ = insert(min(8, n))  # warm-up: module load, buffers
    fe.octomap_destroy(om)
    walls = []
    for _ in range(args.rounds):
        om, dt = insert(n)
        walls.append(dt)
        if len(walls) < args.rounds:
            fe.octomap_destroy(om)

    # ---- 3. the write
    size = len(fe.octomap_write(om))  # warm-up
    ww = []
    for _ in range(args.rounds):
        t0 = time.perf_counter()
        fe.octomap_write(om)
        ww.append(time.perf_counter() - t0)
    nodes, leaves = fe.octomap_stats(om)
    fe.octomap_destroy(om)

    # ---- 4. the oracle on a prefix
    hn = min(args.host_nodes, n)
    m = ox.Oracle()
    cells = 0
    t0 = time.perf_counter()
    for k in range(hn):
        r = fe.node_cloud(hs[k]).reshape(-1)
        cells += m.insert_cloud(dict(x=r["x"], y=r["y"], z=r["z"], rgb=r["rgb"]), T[k])
    ref = m.write()
    host = time.perf_counter() - t0
    om, _ = insert(hn)
    equal = fe.octomap_write(om) == ref
    fe.octomap_destroy(om)
    cells_per_node = cells / hn
    best = min(walls)
    out["insert"] = {"nodes": n, "wall_s": [round(w, 4) for w in walls], "wall_s_best": round(best, 4),
                     "nodes_per_s": round(n / best, 1), "rays_per_s": round(n * rays / best, 1),
                     "cells_per_node_prefix": round(cells_per_node),
                     "cells_per_s_extrapolated": round(cells_per_node * n / best, 1)}
    out["write"] = {"bytes": size, "tree_nodes": nodes, "leaves": leaves, "wall_s": [round(w, 4) for w in ww],
                    "wall_s_best": round(min(ww), 4)}
    out["host_oracle"] = {"nodes": hn, "s": round(host, 3), "s_per_node": round(host / hn, 3),
                          "projected_s_all_nodes": round(host / hn * n, 1), "equal_to_device": bool(equal)}
    out["speedup_vs_host_projected"] = round(host / hn * n / best, 1)

    # ---- 2. device time per kernel (separate pass)
    pn = min(args.profile_nodes, n)
    om, _ = insert(pn)
    fe.octomap_destroy(om)
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        om, _ = insert(pn)
        fe.octomap_write(om)
    fe.octomap_destroy(om)
    kern = {}
    for e in prof.events():
        if e.device_type.name != "CUDA":
            continue
        mm = re.search(r"rb200::(k_(?:oct|map)_\w+)", e.name)
        if mm:
            kern[mm.group(1)] = kern.get(mm.group(1), 0.0) + e.device_time
    out["profile"] = {"nodes": pn, "device_kernel_ms": {k: round(v / 1e3, 3) for k, v in sorted(kern.items())},
                      "device_kernel_ms_total": round(sum(kern.values()) / 1e3, 3)}
    for h in hs:
        fe.node_destroy(h)
    fe.close()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
