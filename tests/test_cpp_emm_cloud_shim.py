"""The C++ shim's point-cloud Node with the environment measurement model on (tests/cpp/test_emm_cloud_shim.cpp): CPU:
compile + link + 'no CPU fallback' exit path; GPU: matchNodePair reports the counts of the restatement
(tests/emm_cloud_exact.py) under the transform it returns, and accepts exactly the pairs the criterion accepts."""
import subprocess
from pathlib import Path

import numpy as np
import pytest

ROOT = Path(__file__).resolve().parent.parent


def _compile(tmp_path):
    exe = tmp_path / "test_emm_cloud_shim"
    libdir = ROOT / "rgbdslam_v2_b200"
    subprocess.run(["g++", "-std=c++17", "-O2", "-Wall", f"-I{ROOT / 'include'}", str(ROOT / "tests/cpp/test_emm_cloud_shim.cpp"),
                    "-o", str(exe), f"-L{libdir}", "-lrgbdslam_b200", f"-Wl,-rpath,{libdir}"], check=True)
    return exe


def _input(tmp_path):
    """three rendered frames as grey images and PointXYZRGB clouds, a block of each cloud pushed 30 % further along its
    rays (bad and occluded samples)"""
    import cloud_oracle as co
    import node_helpers as nh
    gray, depth = nh.stack(nh.render([0, 3, 6]))
    clouds = np.stack([co.cloud_from_depth(d, nh.K4()) for d in depth])
    for i, c in enumerate(clouds):
        c[100:180, 60 + 40 * i:140 + 40 * i, :3] *= np.float32(1.3)
    F, H, W = gray.shape
    path = tmp_path / "frames.bin"
    with open(path, "wb") as f:
        f.write(np.array([W, H, F], np.int32).tobytes())
        f.write(np.array(nh.K4(), np.float32).tobytes())
        f.write(np.ascontiguousarray(gray, np.uint8).tobytes())
        f.write(np.ascontiguousarray(clouds, np.float32).tobytes())
    return path, clouds, nh.K4()


def test_emm_cloud_shim_compiles_and_refuses_cpu(built, tmp_path):
    import torch
    exe = _compile(tmp_path)
    r = subprocess.run([str(exe), str(tmp_path / "absent.bin")], capture_output=True, text=True)
    if not torch.cuda.is_available():
        assert r.returncode == 77 and "init failed" in r.stdout


@pytest.mark.gpu
def test_emm_cloud_shim_reports_restated_counts(built, tmp_path):
    import emm_cloud_exact as ec
    import emm_exact as ee
    exe = _compile(tmp_path)
    path, clouds, K = _input(tmp_path)
    r = subprocess.run([str(exe), str(path)], capture_output=True, text=True)
    assert r.returncode == 0, r.stdout + r.stderr
    assert "EMM CLOUD SHIM OK" in r.stdout
    rows = [l.split()[1:] for l in r.stdout.splitlines() if l.startswith("PAIR ")]
    assert len(rows) == 3
    judged = 0
    for row in rows:
        i, j, id1 = (int(x) for x in row[:3])
        got = np.array([int(x) for x in row[3:7]], np.int64)
        if got[3] == 0:   # RANSAC found no transformation: the model does not judge the pair
            assert id1 == -1 and not got.any(), row
            continue
        judged += 1
        T = np.array([float(x) for x in row[7:]], np.float32).reshape(4, 4).T
        exp = ec.pairwise_cloud(T, clouds[i], K, clouds[j], K, czc=ee.cov_const(0.01, 2.0))
        assert exp["loose"].sum() == 0
        assert np.array_equal(got, exp["counts"]), (i, j, got, exp["counts"])
        assert (id1 == j) == ee.criterion(exp["counts"], 0.3)[0], (i, j, id1)
    assert judged >= 2, rows
