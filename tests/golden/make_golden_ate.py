"""Generates tests/golden/ate_align.npz by running the REFERENCE's own align()
(<reference tree>/rgbd_benchmark/evaluate_ate_module.pyx:35-55, extracted by line range and executed under Python 3 --
the one substitution is numpy.linalg.linalg.svd -> numpy.linalg.svd, a module path numpy 2 no longer has) together with
the RMSE expression of :197 (`numpy.sqrt(numpy.dot(trans_error,trans_error) / len(trans_error))`).
Usage: python tests/golden/make_golden_ate.py <reference tree>; the .npz is committed, so the test needs no reference tree."""
import sys
from pathlib import Path

import numpy
import numpy as np

REF = Path(sys.argv[1]) / "rgbd_benchmark" / "evaluate_ate_module.pyx"
lines = REF.read_text().splitlines()
start = next(i for i, l in enumerate(lines) if l.startswith("def align(model,data):"))
end = next(i for i in range(start + 1, len(lines)) if lines[i].startswith("def "))
src = "\n".join(lines[start:end]).replace("numpy.linalg.linalg.svd", "numpy.linalg.svd")
assert "U*S*Vh" in src and "numpy.outer" in src, "unexpected reference text"
ns = {"numpy": numpy}
exec(compile(src, str(REF), "exec"), ns)
align = ns["align"]

rng = np.random.default_rng(20260923)
cases = {}
for name, n, noise, reflect in [("small", 12, 0.01, False), ("traj", 400, 0.03, False), ("planar", 50, 0.002, False),
                                ("mirror", 30, 0.05, True)]:
    gt = rng.normal(size=(3, n)) * np.array([[2.0], [1.0], [0.3 if name != "planar" else 0.0]])
    ang = rng.uniform(-1, 1, 3)
    cx, cy, cz = np.cos(ang); sx, sy, sz = np.sin(ang)
    R = (np.array([[cz, -sz, 0], [sz, cz, 0], [0, 0, 1]]) @ np.array([[cy, 0, sy], [0, 1, 0], [-sy, 0, cy]])
         @ np.array([[1, 0, 0], [0, cx, -sx], [0, sx, cx]]))
    est = R.T @ (gt - rng.normal(size=(3, 1))) + rng.normal(size=(3, n)) * noise
    if reflect:
        est[2] *= -1  # the det(U) det(Vh) < 0 branch
    rot, trans, trans_error = align(numpy.matrix(est), numpy.matrix(gt))  # align(second_xyz, first_xyz), :193
    rmse = numpy.sqrt(numpy.dot(trans_error, trans_error) / len(trans_error))
    cases[f"{name}_est"], cases[f"{name}_gt"] = est.T.copy(), gt.T.copy()
    cases[f"{name}_rot"], cases[f"{name}_trans"] = np.asarray(rot), np.asarray(trans).ravel()
    cases[f"{name}_rmse"] = np.float64(rmse)
np.savez_compressed(Path(__file__).parent / "ate_align.npz", **cases)
print({k: (v.shape if hasattr(v, "shape") else v) for k, v in cases.items() if k.endswith("rmse") or k.endswith("rot")})
