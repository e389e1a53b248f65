"""The C++ shim's listenerNode on depth images of another size than the visual (tests/cpp/test_resize_shim.cpp): CPU: compile
+ link + 'no CPU fallback' exit path; GPU: run it."""
import subprocess
from pathlib import Path

import pytest

ROOT = Path(__file__).resolve().parent.parent


def _compile(tmp_path):
    exe = tmp_path / "test_resize_shim"
    libdir = ROOT / "rgbdslam_v2_b200"
    subprocess.run(["g++", "-std=c++17", "-O2", "-Wall", f"-I{ROOT / 'include'}", str(ROOT / "tests/cpp/test_resize_shim.cpp"),
                    "-o", str(exe), f"-L{libdir}", "-lrgbdslam_b200", f"-Wl,-rpath,{libdir}"], check=True)
    return exe


def test_resize_shim_compiles_and_refuses_cpu(built, tmp_path):
    import torch
    exe = _compile(tmp_path)
    r = subprocess.run([str(exe)], capture_output=True, text=True)
    if not torch.cuda.is_available():
        assert r.returncode == 77 and "init failed" in r.stdout


@pytest.mark.gpu
def test_resize_shim_runs_on_gpu(built, tmp_path):
    exe = _compile(tmp_path)
    r = subprocess.run([str(exe)], capture_output=True, text=True)
    assert r.returncode == 0, r.stdout + r.stderr
    assert "RESIZE SHIM OK" in r.stdout
    assert r.stdout.count("equal") == 2, r.stdout
