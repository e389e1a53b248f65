"""Node constructor throughput at RGB-D sensor sizes next to 640x480: rgbdslam_b200_nodes_create_ex frames/s and the device
time of every library kernel per frame.

Rendered frames (synth.render_frame at each size: the 640x480 camera's field of view, max_keypoints scaled with the area
from 1000 at 640x480, capped at 2700 so that 1.5 K fits the 4096-keypoint frame buffer), ORB detector, 3x3 grid, mask from
depth, pinned input, --frames frames per call (the same for every size; a 1920x1080 call runs in chunks of 9 frames).
1. Host clock around each call, which returns after the device work has finished (it downloads the feature counts).  Per
   size: one untimed call (a new frame size re-prepares the geometry and reallocates the work buffers), then --rounds
   timed calls at that size, so the timed calls include no allocation.
2. torch.profiler with CUDA activities in a separate pass (tracing slows the host): device time per frame of each kernel
   (one row per template instantiation) and of all library kernels.
Prints one JSON object, with the card name and power limit read in the same run.
Usage: python tools/run_large_frames.py [--frames 64] [--rounds 3]
"""
import argparse
import ctypes as C
import json
import re
import sys
import time
from pathlib import Path

sys.path.insert(0, str(Path(__file__).resolve().parent.parent))
sys.path.insert(0, str(Path(__file__).resolve().parent))
import numpy as np  # noqa: E402
from run_nodes import card  # noqa: E402

SIZES = [(480, 640), (720, 1280), (1080, 1920)]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=64)
    ap.add_argument("--rounds", type=int, default=3)
    args = ap.parse_args()
    import torch
    from torch.profiler import ProfilerActivity, profile

    from rgbdslam_v2_b200 import Frontend, synth
    from rgbdslam_v2_b200._capi import default_params
    if not torch.cuda.is_available():
        raise SystemExit("no GPU: this script measures on the device only")
    poses = synth.trajectory(240)
    fe = Frontend(0, default_params())
    out = {"card": card(), "frames_per_call": args.frames, "sizes": {}}
    inputs = {}
    for h, w in SIZES:
        fr = [synth.render_frame(poses[k % 240], seed=k, shape=(h, w)) for k in range(args.frames)]
        g = torch.from_numpy(np.stack([f[0] for f in fr])).pin_memory()
        d = torch.from_numpy(np.stack([f[1] for f in fr])).pin_memory()
        K = int(min(2700, round(1000 * h * w / (640 * 480))))
        inputs[(h, w)] = (g, d, synth.intrinsics(w, h), K)

    def call(size, n=None):
        g, d, K4, K = inputs[size]
        p = default_params()
        p.max_keypoints = K
        fe.params = p
        fe._check(fe.lib.rgbdslam_b200_init(0, C.byref(p)))
        det = fe.detector_create()
        n = n or len(g)
        t0 = time.perf_counter()
        hs, nf = fe.nodes_create(det, g[:n], d[:n], None, K4, mask_from_depth=True)
        dt = time.perf_counter() - t0
        fe.detector_destroy(det)
        for hh in hs:
            fe.node_destroy(hh)
        return dt, float(np.mean(nf)), K

    for s in SIZES:
        call(s)  # warm-up at this size: geometry, buffers, module load
        rates = []
        for _ in range(args.rounds):
            dt, feats, K = call(s)
            rates.append(args.frames / dt)
        out["sizes"][f"{s[1]}x{s[0]}"] = dict(max_keypoints=K, features_per_node=round(feats, 1),
                                              frames_per_s=[round(r, 1) for r in rates])

    for s in SIZES:
        n = min(args.frames, 32)
        call(s, n)
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            call(s, n)
        tot = {}
        for e in prof.events():
            if e.device_type.name != "CUDA":
                continue
            m = re.search(r"rb200::((k_\w+)(<[^>]*>)?)", e.name)
            if m:
                tot[m.group(1)] = tot.get(m.group(1), 0.0) + e.device_time
        per = {k: round(t / n, 2) for k, t in sorted(tot.items(), key=lambda kv: -kv[1])}
        per["all_library_kernels"] = round(sum(tot.values()) / n, 2)
        out["sizes"][f"{s[1]}x{s[0]}"]["kernel_us_per_frame"] = per
    fe.close()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
