"""icp_method through the C++ shim (tests/cpp/test_icp_nl_shim.cpp): CPU: compile + link + 'no CPU fallback' exit path; GPU:
with Node::icp_method() = "icp_nl" the ICP edge equals rgbdslam_b200_icp_align_ex(..., ICP_NL), and "gicp" or an unknown name
gives the "icp" edge."""
import subprocess
from pathlib import Path

import numpy as np
import pytest

ROOT = Path(__file__).resolve().parent.parent


def _compile(tmp_path):
    exe = tmp_path / "test_icp_nl_shim"
    libdir = ROOT / "rgbdslam_v2_b200"
    subprocess.run(["g++", "-std=c++17", "-O2", "-Wall", f"-I{ROOT / 'include'}", str(ROOT / "tests/cpp/test_icp_nl_shim.cpp"),
                    "-o", str(exe), f"-L{libdir}", "-lrgbdslam_b200", f"-Wl,-rpath,{libdir}"], check=True)
    return exe


def test_icp_nl_shim_compiles_and_refuses_cpu(built, tmp_path):
    import torch
    exe = _compile(tmp_path)
    r = subprocess.run([str(exe), str(tmp_path / "absent.bin")], capture_output=True, text=True)
    if not torch.cuda.is_available():
        assert r.returncode == 77 and "init failed" in r.stdout


@pytest.mark.gpu
def test_icp_method_through_the_shim(built, tmp_path):
    import node_helpers as nh
    exe = _compile(tmp_path)
    gray, depth = nh.stack(nh.render(range(2)))
    F, H, W = gray.shape
    path = tmp_path / "frames.bin"
    with open(path, "wb") as f:
        f.write(np.array([W, H, F], np.int32).tobytes())
        f.write(np.ascontiguousarray(gray, np.uint8).tobytes())
        f.write(np.ascontiguousarray(depth, np.float32).tobytes())
    r = subprocess.run([str(exe), str(path)], capture_output=True, text=True)
    assert r.returncode == 0 and "ICP_NL SHIM OK" in r.stdout, r.stdout + r.stderr
