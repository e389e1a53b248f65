"""The occupancy filter and online creation of the colour OctoMap on the C4 sequence: --frames rendered 640x480 colour frames
with STORE_CLOUD at cloud_creation_skip_step 2 (76 800 points per node), each node under octomap_pose of its ground-truth pose,
resolution 0.05.

1. Filter: octomap_filter_clouds of every node (sensor pose cloud_sensor_pose of its pose) after one insert of them all,
   on fresh nodes each round; device time from CUDA events around the call (it returns after the device work), best of
   --rounds, and the points kept.  The default threshold 3e4 keeps part of each cloud (0.9, the reference's default, drops
   nearly every point at a 5 cm resolution, DESIGN.md 4.15).  The first call on a map also builds its occupancy table on the host (reported apart).
2. The C oracle's filter (tests/octomap_filter_oracle.c, one thread) on the first --host-nodes nodes against a map of those nodes,
   checked against the device's on the same map.
3. Online creation: one single-node octomap_insert into a growing map after each node; the time per node (host clock
   around the synchronous call), mean and last.

Prints one JSON object, with the card name and power limit read in the same run.
Usage: python tools/run_octomap_filter.py [--frames 300] [--rounds 3] [--threshold 3e4]
"""
import argparse
import json
import sys
import time
from pathlib import Path

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))
sys.path.insert(0, str(ROOT / "tests"))
sys.path.insert(0, str(ROOT / "tools"))
import numpy as np  # noqa: E402
from run_octomap import card  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=300)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--host-nodes", type=int, default=3)
    ap.add_argument("--threshold", type=float, default=3e4)
    args = ap.parse_args()

    import torch

    import octomap_filter_exact as fx
    from rgbdslam_v2_b200 import Frontend, synth
    from rgbdslam_v2_b200._capi import cloud_sensor_pose, default_params, octomap_pose
    if not torch.cuda.is_available():
        raise SystemExit("run_octomap_filter.py measures on the GPU; no CUDA device found")
    dev = torch.device("cuda", 0)
    out = {"card": card(), "frames": args.frames, "threshold": args.threshold}
    K4 = (synth.FX, synth.FY, synth.CX, synth.CY)
    poses = synth.trajectory(args.frames)
    g_d, d_d = synth.render_frames_torch(poses, dev)
    gray, depth = g_d.cpu().numpy(), d_d.cpu().numpy()
    del g_d, d_d
    colour = np.ascontiguousarray(np.stack([gray, np.roll(gray, 3, axis=-1), np.roll(gray, 5, axis=-2)], -1))
    n = gray.shape[0]
    p = default_params()
    p.depth_cov_z0 = 2.0
    fe = Frontend(0, p)
    det = fe.detector_create()

    def make_nodes():
        hs = []
        for k0 in range(0, n, 64):
            h, _ = fe.nodes_create(det, colour[k0:k0 + 64], depth[k0:k0 + 64], None, K4, store_cloud=True)
            hs += list(h)
        return hs

    T = np.stack([octomap_pose(P) for P in poses])
    S = np.stack([np.concatenate(cloud_sensor_pose(P)) for P in poses]).astype(np.float32)
    ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)

    # ---- 1. the filter
    hs = make_nodes()
    om = fe.octomap_create()
    fe.octomap_insert(om, hs, T)
    fe.octomap_filter_clouds(om, hs[:2], S[:2], args.threshold)  # warm-up: module load, buffers, the occupancy table
    for h in hs:
        fe.node_destroy(h)
    t_first, dev_ms, kept = None, [], None
    for r in range(args.rounds + 1):
        hs = make_nodes()
        if r == 0:  # a fresh map: the first call builds its occupancy table
            fe.octomap_destroy(om)
            om = fe.octomap_create()
            fe.octomap_insert(om, hs, T)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        ev0.record()
        counts = fe.octomap_filter_clouds(om, hs, S, args.threshold)
        ev1.record()
        ev1.synchronize()
        if r == 0:
            t_first = time.perf_counter() - t0
        else:
            dev_ms.append(ev0.elapsed_time(ev1))
        kept = int(counts.sum())
        for h in hs:
            fe.node_destroy(h)
    points = n * 76800
    out["filter"] = {"nodes": n, "points": points, "kept": kept, "event_ms": [round(x, 3) for x in dev_ms],
                     "event_ms_best": round(min(dev_ms), 3), "points_per_s": round(points / (min(dev_ms) / 1e3), 1),
                     "first_call_with_occupancy_table_s": round(t_first, 4)}
    _, leaves = fe.octomap_stats(om)
    out["filter"]["leaves"] = leaves

    print("filter done", flush=True)
    # ---- 2. the oracle on a prefix
    # (a map of the prefix only: the oracle's insert takes seconds per node)
    hn = min(args.host_nodes, n)
    fe.octomap_destroy(om)
    hs = make_nodes()
    om = fe.octomap_create()
    fe.octomap_insert(om, hs[:hn], T[:hn])
    m = fx.FilterOracle()
    recs = [fe.node_cloud(h).reshape(-1) for h in hs[:hn]]
    for r, t in zip(recs, T):
        m.insert_cloud(dict(x=r["x"], y=r["y"], z=r["z"], rgb=r["rgb"]), t)
    t0 = time.perf_counter()
    keeps = [m.occupancy_filter(np.stack([r["x"], r["y"], r["z"]], 1), s[:4], s[4:], args.threshold) for r, s in zip(recs, S)]
    host = time.perf_counter() - t0
    fe.octomap_filter_clouds(om, hs[:hn], S[:hn], args.threshold)
    equal = all(fe.node_cloud(h).reshape(-1).tobytes() == r[k].tobytes() for h, r, k in zip(hs, recs, keeps))
    print("host oracle done", flush=True)
    out["host_oracle"] = {"nodes": hn, "s_per_node": round(host / hn, 4), "equal_to_device": bool(equal),
                          "speedup_vs_device_per_node": round(host / hn / (min(dev_ms) / 1e3 / n), 1)}
    for h in hs:
        fe.node_destroy(h)
    fe.octomap_destroy(om)

    # ---- 3. online creation: one single-node insert after each node
    hs = make_nodes()
    om = fe.octomap_create()
    fe.octomap_insert(om, hs[:1], T[:1])  # warm-up
    fe.octomap_clear(om)
    per = []
    for k in range(n):
        t0 = time.perf_counter()
        fe.octomap_insert(om, hs[k:k + 1], T[k:k + 1])
        per.append(time.perf_counter() - t0)
    out["online"] = {"nodes": n, "s_per_node_mean": round(float(np.mean(per)), 5), "s_per_node_last": round(per[-1], 5),
                     "s_total": round(float(np.sum(per)), 3)}
    fe.octomap_destroy(om)
    for h in hs:
        fe.node_destroy(h)
    fe.detector_destroy(det)
    fe.close()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
