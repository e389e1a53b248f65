"""Where the C2 step's match-selection and RANSAC time goes (the bench's headline workload: 256 pairs x 1000 ORB keypoints,
node handles resident, bench.make_workload for ranks 0-4).

  python tools/run_ransac.py [--steps 20] [--out DIR] [--dump DIR]

Prints the card, its power limit and maximum SM clock, then one JSON line per part:
  * "sync" / "pipelined": device time per step of every library kernel from torch.profiler (CUDA activities), over --steps
    synchronous steps in one profiled region and over --steps steps pipelined over 5 slots (as bench.py's `value`) in
    another.  The two launches of ransac_hyp_kernel are told apart by their grid (phase 1 has one CTA per pair).
  * "phases": pairs per step that the first RANSAC phase finishes, and phase-2 CTAs launched against CTAs that do work
    (for --hyps-per-cta hypotheses per CTA).
    The index the sequential loop visits after hypotheses [0, 4) is replayed on the host from the library's own results
    with ransac_iterations = 1 .. 4: the first hypothesis that becomes the best with > 50 % inliers jumps the loop by
    10 (and 10 more above 75 %) and ends it above 80 %.
--dump DIR saves the results and match lists of the five batch sets, and of the same sets with max_matches 512,
ransac_iterations 1000, a latched depth covariance (depth_cov_z0 = 0) and the per-point covariance (depth_cov_z0 < 0).
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile
from pathlib import Path

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))
import numpy as np  # noqa: E402

import bench  # noqa: E402
from rgbdslam_v2_b200 import Frontend  # noqa: E402
from rgbdslam_v2_b200._capi import default_params, PAIR_RESULT_DTYPE, DMATCH_DTYPE  # noqa: E402

DEPTH = 5
KPHASE1 = 4  # phase-1 hypotheses (csrc/frontend_kernels.cu)


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                       capture_output=True, text=True)
    return q.stdout.strip()


class Sets:
    """The five C2 batch sets on one Frontend, as bench.py builds them."""

    def __init__(self, **prm_kw):
        prm = default_params()
        prm.depth_cov_z0 = 2.0
        for k, v in prm_kw.items():
            setattr(prm, k, v)
        self.prm = prm
        self.fe = Frontend(0, prm)
        self.sets = []
        for j in range(DEPTH):
            b = bench.make_workload(j)
            newer = np.array([self.fe.node_from_features(int(b["id_newer"][i]), p["desc_newer"], p["xyz_newer"])
                              for i, p in enumerate(b["pairs"])], np.uint64)
            older = np.array([self.fe.node_from_features(int(b["id_older"][i]), p["desc_older"], p["xyz_older"])
                              for i, p in enumerate(b["pairs"])], np.uint64)
            self.sets.append(dict(first=j * bench.PAIRS_PER_GPU, newer=newer, older=older,
                                  res=np.zeros(bench.PAIRS_PER_GPU, PAIR_RESULT_DTYPE)))

    def sync_step(self, k, want_matches=False):
        st = self.sets[k % DEPTH]
        return self.fe.match_node_pairs(st["newer"], st["older"], seed=bench.SEED, first_pair_index=st["first"],
                                        want_matches=want_matches)

    def pipelined(self, K):
        def submit(k):
            st = self.sets[k % DEPTH]
            self.fe.submit_node_pairs(1 + k % DEPTH, st["newer"], st["older"], (st["res"], None, None), seed=bench.SEED,
                                      first_pair_index=st["first"])
        for k in range(K):
            if k >= DEPTH:
                self.fe.wait_slot(1 + (k - DEPTH) % DEPTH)
            submit(k)
        for k in range(max(0, K - DEPTH), K):
            self.fe.wait_slot(1 + k % DEPTH)

    def close(self):
        self.fe.close()


def kernel_name(ev):
    n, grid = ev["name"], ev.get("args", {}).get("grid", [0, 0, 0])
    if "ransac_hyp_kernel" in n:
        return f"ransac_hyp_kernel phase {1 if grid[0] == 1 else 2}"
    return n.split("(")[0].replace("void ", "").replace("rb200::", "")


def profile(run, steps, out_dir):
    import torch
    from torch.profiler import profile as tprofile, ProfilerActivity
    with tprofile(activities=[ProfilerActivity.CUDA]) as prof:
        run()
        torch.cuda.synchronize()
    path = Path(out_dir) / f"trace_{os.getpid()}.pt.trace.json"
    prof.export_chrome_trace(str(path))
    evs = json.loads(path.read_text())["traceEvents"]
    path.unlink()
    tot = {}
    for ev in evs:
        if ev.get("cat") == "kernel":
            k = kernel_name(ev)
            tot[k] = tot.get(k, 0.0) + ev["dur"] * 1e-3
    return {k: round(v / steps, 5) for k, v in sorted(tot.items(), key=lambda kv: -kv[1])}


def phase_counts(min_matches, hyps_per_cta, H=200):
    """Phase-1 outcome per pair replayed from results with ransac_iterations = 1 .. 4 (see the module docstring)."""
    runs = []
    for h in range(1, KPHASE1 + 1):
        s = Sets(ransac_iterations=h, max_keypoints=bench.N_KP)
        runs.append([s.sync_step(j, want_matches=False)[0].copy() for j in range(DEPTH)])
        s.close()
    done = cta_launched = cta_work = 0
    ncta = -(-(H - KPHASE1) // hyps_per_cta)
    for j in range(DEPTH):
        for p in range(bench.PAIRS_PER_GPU):
            M = int(runs[-1][j]["n_all_matches"][p])
            if not (M > min_matches and M >= 4):
                cta_launched += ncta
                continue
            nxt = KPHASE1
            for h in range(KPHASE1):
                r = runs[h][j][p]
                if r["used_identity"] or int(r["valid_iterations"]) == 0:
                    continue
                cnt = int(r["n_inliers"])
                if cnt > 0.5 * M:  # the first best above 50 %: hypothesis h jumped (best models only grow in count)
                    nxt = h + 1 + 10 + (10 if cnt > 0.75 * M else 0)
                    if cnt > 0.8 * M:
                        nxt = H
                    break
            done += nxt >= H
            cta_launched += ncta
            cta_work += sum(1 for bx in range(ncta) if nxt < KPHASE1 + (bx + 1) * hyps_per_cta and nxt < H)
    return {"pairs_per_step": bench.PAIRS_PER_GPU, "finished_in_phase1_per_step": done / DEPTH,
            "phase2_ctas_launched_per_step": cta_launched / DEPTH, "phase2_ctas_with_work_per_step": cta_work / DEPTH}


def dump(out_dir):
    variants = {"default": {}, "max_matches512": {"max_matches": 512}, "iterations1000": {"ransac_iterations": 1000},
                "z0_latched": {"depth_cov_z0": 0.0}, "cov_per_point": {"depth_cov_z0": -1.0}}
    d = Path(out_dir)
    d.mkdir(parents=True, exist_ok=True)
    for name, kw in variants.items():
        s = Sets(max_keypoints=bench.N_KP, **kw)
        for j in range(DEPTH):
            res, allm, inl = s.sync_step(j, want_matches=True)
            np.save(d / f"{name}_set{j}_res.npy", res.view(np.uint8))
            np.save(d / f"{name}_set{j}_all.npy", allm.view(np.uint8))
            # inlier lists are compacted: only the first n_inliers entries of a row are written
            n = res["n_inliers"]
            np.save(d / f"{name}_set{j}_inl.npy",
                    np.concatenate([inl[p, :max(int(n[p]), 0)] for p in range(len(n))]).view(np.uint8))
        s.close()
    print(json.dumps({"dumped": str(d), "variants": list(variants)}))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--out", help="directory for the profiler's temporary trace (default: a temporary directory)")
    ap.add_argument("--dump", metavar="DIR")
    ap.add_argument("--no-profile", action="store_true")
    ap.add_argument("--hyps-per-cta", type=int, default=32,
                    help="hypotheses per phase-2 CTA of the library measured (kRansacHyps; 8 before the blocked kernel)")
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("run_ransac.py: no CUDA device")
    print(json.dumps({"card": card()}))
    if args.dump:
        dump(args.dump)
    if args.no_profile:
        return
    tmp = args.out or tempfile.mkdtemp()
    s = Sets(max_keypoints=bench.N_KP)
    for k in range(2 * DEPTH):  # warm every set and slot
        s.sync_step(k)
    s.pipelined(2 * DEPTH)
    torch.cuda.synchronize()
    K = args.steps

    def sync_run():
        for k in range(K):
            s.sync_step(k)
    print(json.dumps({"part": "sync", "steps": K, "device_ms_per_step": profile(sync_run, K, tmp)}))
    print(json.dumps({"part": "pipelined", "steps": K, "device_ms_per_step": profile(lambda: s.pipelined(K), K, tmp)}))
    min_matches = s.prm.min_matches
    s.close()
    print(json.dumps({"part": "phases", **phase_counts(min_matches, args.hyps_per_cta)}))


if __name__ == "__main__":
    main()
