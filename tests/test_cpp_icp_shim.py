"""The C++ shim's ICP fallback (tests/cpp/test_icp_shim.cpp): CPU: compile + link + 'no CPU fallback' exit path; GPU: with
RANSAC made to fail, the adjacent pair takes the ICP edge in the reference's direction with a zero information matrix, the
non-adjacent pair and the pair with too few matches stay invalid, max_connections is honoured in order, the online
GraphManager over 30 frames optimises to finite poses, and with Node::pcl_icp() off the results are those of the RANSAC path;
with Node::icp_method() = "icp_nl" the ICP edge equals rgbdslam_b200_icp_align_ex(..., ICP_NL), and "gicp" or an unknown
name gives the "icp" edge."""
import subprocess
from pathlib import Path

import numpy as np
import pytest

ROOT = Path(__file__).resolve().parent.parent


def _compile(tmp_path):
    exe = tmp_path / "test_icp_shim"
    libdir = ROOT / "rgbdslam_v2_b200"
    subprocess.run(["g++", "-std=c++17", "-O2", "-Wall", f"-I{ROOT / 'include'}", str(ROOT / "tests/cpp/test_icp_shim.cpp"),
                    "-o", str(exe), f"-L{libdir}", "-lrgbdslam_b200", f"-Wl,-rpath,{libdir}"], check=True)
    return exe


def test_icp_shim_compiles_and_refuses_cpu(built, tmp_path):
    import torch
    exe = _compile(tmp_path)
    r = subprocess.run([str(exe), str(tmp_path / "absent.bin")], capture_output=True, text=True)
    if not torch.cuda.is_available():
        assert r.returncode == 77 and "init failed" in r.stdout


@pytest.mark.gpu
def test_icp_fallback_through_the_shim(built, tmp_path):
    import node_helpers as nh
    exe = _compile(tmp_path)
    gray, depth = nh.stack(nh.render(range(30)))
    F, H, W = gray.shape
    path = tmp_path / "frames.bin"
    with open(path, "wb") as f:
        f.write(np.array([W, H, F], np.int32).tobytes())
        f.write(np.ascontiguousarray(gray, np.uint8).tobytes())
        f.write(np.ascontiguousarray(depth, np.float32).tobytes())
    r = subprocess.run([str(exe), str(path)], capture_output=True, text=True)
    assert r.returncode == 0 and "ICP SHIM OK" in r.stdout, r.stdout + r.stderr
