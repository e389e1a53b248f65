"""The Node constructor on 1280x1024 colour frames with 640x480 16-bit depth (an Xtion / Kinect v1 in SXGA mode), MASK_FROM_DEPTH,
from pinned buffers -- the depth resized on the device (nodes_create_resized) against what a caller does without it: a host
cv2.resize(INTER_NEAREST) of every frame's depth into a pinned full-size buffer, then nodes_create_ex on the 1280x1024 16-bit
depth.

--distinct frames are rendered by synth.render_frame (visual at 1280x1024, depth at 640x480, same pose) and cycled to --frames
frames.  Each arm is one call over all frames with a fresh detector, timed with a host clock around the work, which ends in a
device synchronisation; --rounds rounds alternate the two arms, the best of each is reported.  Both arms must build the same
nodes.  A separate pass under torch.profiler gives the device time per frame of the resize kernel (k_depth_gather).

Prints one JSON object with frames/s, depth bytes uploaded per frame, and the card name and power limit read in the same run.
Usage: python tools/run_depth_resize.py [--frames 300] [--distinct 24] [--rounds 3]
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

W, H, DW, DH = 1280, 1024, 640, 480


def card() -> dict:
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                       text=True)
    name, power, clk = (x.strip() for x in q.stdout.splitlines()[0].split(","))
    return {"name": name, "power_limit": power, "max_sm_clock": clk}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=300)
    ap.add_argument("--distinct", type=int, default=24)
    ap.add_argument("--rounds", type=int, default=3)
    args = ap.parse_args()

    import cv2
    import torch
    from torch.profiler import ProfilerActivity, profile

    import node_helpers as nh
    import raw_input_oracle as ro
    from rgbdslam_v2_b200 import Frontend, synth
    if not torch.cuda.is_available():
        raise SystemExit("run_depth_resize.py measures on the GPU; no CUDA device found")
    n = args.frames
    poses = synth.trajectory(240)
    vis, dep = [], []
    for k in range(args.distinct):
        g = synth.render_frame(poses[k], seed=k, shape=(H, W))[0]
        vis.append(np.stack([g, np.roll(g, 3, axis=-1), np.roll(g, 5, axis=-2)], -1))
        dep.append(ro.to_millimetres(synth.render_frame(poses[k], seed=k, shape=(DH, DW))[1]))
    idx = np.arange(n) % args.distinct
    colour = torch.from_numpy(np.stack(vis)[idx]).pin_memory()
    depth = torch.from_numpy(np.stack(dep)[idx]).pin_memory()
    big = torch.empty((n, H, W), dtype=torch.uint16).pin_memory()  # the host arm's upload buffer
    big_np, depth_np = big.numpy(), depth.numpy()
    K4 = synth.intrinsics(W, H)
    fe = Frontend(0, nh.params(0))

    def run(arm):
        """(seconds, feature counts, detector thresholds) of one call over all frames"""
        det = fe.detector_create()
        fe.synchronize()
        t0 = time.perf_counter()
        if arm == "device":
            hs, nf = fe.nodes_create_resized(det, colour, depth, None, K4, mask_from_depth=True)
        else:
            for k in range(n):
                big_np[k] = cv2.resize(depth_np[k], (W, H), interpolation=cv2.INTER_NEAREST)
            hs, nf = fe.nodes_create(det, colour, big, None, K4, mask_from_depth=True)
        fe.synchronize()
        dt = time.perf_counter() - t0
        thr = fe.detector_thresholds(det).copy()
        fe.detector_destroy(det)
        nh.destroy(fe, hs)
        return dt, nf.copy(), thr

    arms = ("device", "host")
    ref = {a: run(a) for a in arms}  # warm-up: buffers, tables, module load
    assert np.array_equal(ref["device"][1], ref["host"][1]) and np.array_equal(ref["device"][2], ref["host"][2])
    times = {a: [] for a in arms}
    for _ in range(args.rounds):
        for a in arms:
            dt, nf, thr = run(a)
            assert np.array_equal(nf, ref[a][1]) and np.array_equal(thr, ref[a][2])
            times[a].append(dt)

    det = fe.detector_create()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        hs, _ = fe.nodes_create_resized(det, colour, depth, None, K4, mask_from_depth=True)
        fe.synchronize()
    gather_us = sum(e.device_time for e in prof.events() if e.device_type.name == "CUDA" and "k_depth_gather" in e.name)
    fe.detector_destroy(det)
    nh.destroy(fe, hs)
    fe.close()

    out = {"card": card(), "frames": n, "distinct_frames": args.distinct, "visual": f"{W}x{H} colour",
           "depth": f"{DW}x{DH} u16", "rounds": args.rounds,
           "seconds": {a: times[a] for a in arms},
           "frames_per_s": {a: n / min(times[a]) for a in arms},
           "depth_bytes_uploaded_per_frame": {"device": DW * DH * 2, "host": W * H * 2},
           "k_depth_gather_us_per_frame": gather_us / n,
           "features_per_frame": float(ref["device"][1].mean())}
    out["speedup"] = out["frames_per_s"]["device"] / out["frames_per_s"]["host"]
    print(json.dumps(out, indent=1))


if __name__ == "__main__":
    main()
