"""The C++ shim (include/rgbdslam_b200/node.hpp) keeps the reference-shaped call sites compiling:
CPU: compile + link + 'no CPU fallback' exit path; GPU: run it."""
import subprocess
from pathlib import Path

import pytest

ROOT = Path(__file__).resolve().parent.parent


def _compile(tmp_path, name="test_shim"):
    exe = tmp_path / name
    libdir = ROOT / "rgbdslam_v2_b200"
    subprocess.run(["g++", "-std=c++17", "-O2", "-Wall", f"-I{ROOT / 'include'}", str(ROOT / f"tests/cpp/{name}.cpp"), "-o", str(exe),
                    f"-L{libdir}", "-lrgbdslam_b200", f"-Wl,-rpath,{libdir}"], check=True)
    return exe


def test_shim_compiles_and_refuses_cpu(built, tmp_path):
    import torch
    exe = _compile(tmp_path)
    r = subprocess.run([str(exe)], capture_output=True, text=True)
    if not torch.cuda.is_available():
        assert r.returncode == 77 and "no CPU fallback" in r.stdout


@pytest.mark.gpu
def test_shim_runs_on_gpu(built, tmp_path):
    exe = _compile(tmp_path)
    r = subprocess.run([str(exe)], capture_output=True, text=True)
    assert r.returncode == 0, r.stdout + r.stderr
    assert "SHIM OK" in r.stdout


def test_graph_manager_shim_compiles_and_refuses_cpu(built, tmp_path):
    """include/rgbdslam_b200/graph_manager.hpp: addNode / nodeComparisons / optimizeGraph / pruneEdgesWithErrorAbove call sites"""
    import torch
    exe = _compile(tmp_path, "test_graph_manager")
    r = subprocess.run([str(exe)], capture_output=True, text=True)
    if not torch.cuda.is_available():
        assert r.returncode == 77 and "no CPU fallback" in r.stdout


@pytest.mark.gpu
def test_graph_manager_shim_runs_on_gpu(built, tmp_path):
    exe = _compile(tmp_path, "test_graph_manager")
    r = subprocess.run([str(exe)], capture_output=True, text=True)
    assert r.returncode == 0, r.stdout + r.stderr
    assert "GRAPH MANAGER SHIM OK" in r.stdout


def test_graph_manager_trace_compiles_and_refuses_cpu(built, tmp_path):
    """tests/cpp/test_graph_manager_trace.cpp, the shim's trace for tests/test_gpu_graph_manager_parity.py"""
    import numpy as np
    import torch
    exe = _compile(tmp_path, "test_graph_manager_trace")
    frames, params = tmp_path / "frames.bin", tmp_path / "params.bin"
    with open(frames, "wb") as f:  # one 8 x 8 frame
        np.array([1, 8, 8], np.int64).tofile(f)
        np.array([8.0, 8.0, 3.5, 3.5, 0.0], np.float64).tofile(f)
        np.zeros(64, np.uint8).tofile(f); np.ones(64, np.float32).tofile(f); np.zeros(64, np.uint8).tofile(f)
    np.array([0, 2.0, 600], np.float64).tofile(params)
    r = subprocess.run([str(exe), str(frames), str(params), str(tmp_path / "out.bin")], capture_output=True, text=True)
    if not torch.cuda.is_available():
        assert r.returncode == 77 and "no CPU fallback" in r.stdout
