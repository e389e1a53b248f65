"""A few synchronous passes of the C2 workload (256 pairs x 1000 ORB keypoints, resident nodes): per-launch Hamming kernel times."""
import sys
from pathlib import Path
sys.path.insert(0, str(Path(__file__).resolve().parent.parent))
import numpy as np
from rgbdslam_v2_b200 import Frontend, synth
from rgbdslam_v2_b200._capi import default_params, PAIR_RESULT_DTYPE
n = int(sys.argv[1]) if len(sys.argv) > 1 else 4
prm = default_params(); prm.depth_cov_z0 = 2.0; prm.max_keypoints = 1000
fe = Frontend(0, prm)
import os
if os.environ.get("RB200_HAMMING_PATH"):
    fe.set_hamming_path(int(os.environ["RB200_HAMMING_PATH"]))
b = synth.make_batch(256, 1000, seed0=1234)
newer = np.array([fe.node_from_features(int(b["id_newer"][k]), q["desc_newer"], q["xyz_newer"]) for k, q in enumerate(b["pairs"])], np.uint64)
older = np.array([fe.node_from_features(int(b["id_older"][k]), q["desc_older"], q["xyz_older"]) for k, q in enumerate(b["pairs"])], np.uint64)
r = np.zeros(256, PAIR_RESULT_DTYPE)
ham = []
for k in range(n):
    fe.match_node_pairs(newer, older, seed=1, out=(r, None, None))
    ham.append(fe.stage_times(0)["hamming"] * 1e3)
print("hamming us per call:", " ".join(f"{x:.1f}" for x in ham), "| median %.1f min %.1f" % (float(np.median(ham[1:])), min(ham)))
print("valid", int((r["id1"] >= 0).sum()), "stages", fe.stage_times(0))
