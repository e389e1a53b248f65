"""The C++ shim's voxel filter (tests/cpp/test_voxel_shim.cpp): CPU: compile + link + 'no CPU fallback' exit path; GPU: the
online GraphManager over 30 frames, reducePointClouds(), then saveAllClouds: the PCD holds exactly the render_cloud records of
the reduced nodes and is smaller than the map saved before; Node::reducePointCloud with an invalid size changes nothing."""
import subprocess
from pathlib import Path

import numpy as np
import pytest

ROOT = Path(__file__).resolve().parent.parent


def _compile(tmp_path):
    exe = tmp_path / "test_voxel_shim"
    libdir = ROOT / "rgbdslam_v2_b200"
    subprocess.run(["g++", "-std=c++17", "-O2", "-Wall", f"-I{ROOT / 'include'}", str(ROOT / "tests/cpp/test_voxel_shim.cpp"),
                    "-o", str(exe), f"-L{libdir}", "-lrgbdslam_b200", f"-Wl,-rpath,{libdir}"], check=True)
    return exe


def test_voxel_shim_compiles_and_refuses_cpu(built, tmp_path):
    import torch
    exe = _compile(tmp_path)
    r = subprocess.run([str(exe), str(tmp_path / "absent.bin"), str(tmp_path / "m"), str(tmp_path / "r.bin")], capture_output=True,
                       text=True)
    if not torch.cuda.is_available():
        assert r.returncode == 77 and "init failed" in r.stdout


def _read_pcd(path):
    head, body = Path(path).read_bytes().split(b"DATA binary\n", 1)
    fields = dict(l.split(" ", 1) for l in head.decode().splitlines() if not l.startswith("#"))
    return fields, np.frombuffer(body, np.float32).reshape(-1, 4)


@pytest.mark.gpu
def test_reduce_point_clouds_then_save_all_clouds(built, tmp_path):
    import map_cloud_exact as mx
    import node_helpers as nh
    exe = _compile(tmp_path)
    gray, depth = nh.stack(nh.render(range(30)))
    F, H, W = gray.shape
    path = tmp_path / "frames.bin"
    with open(path, "wb") as f:
        f.write(np.array([W, H, F], np.int32).tobytes())
        f.write(np.ascontiguousarray(gray, np.uint8).tobytes())
        f.write(np.ascontiguousarray(depth, np.float32).tobytes())
    r = subprocess.run([str(exe), str(path), str(tmp_path / "map"), str(tmp_path / "render.bin")], capture_output=True, text=True)
    assert r.returncode == 0 and "VOXEL SHIM OK" in r.stdout, r.stdout + r.stderr
    assert r.stderr.count("invalid voxelfilter_size") == 3
    _, raw = _read_pcd(tmp_path / "map_raw.pcd")
    fields, pts = _read_pcd(tmp_path / "map_reduced.pcd")
    rec = np.fromfile(tmp_path / "render.bin", mx.POINT32)
    assert int(fields["POINTS"]) == len(pts) == len(rec) and 0 < len(pts) < len(raw) // 4
    assert np.array_equal(pts[:, :3].view(np.uint32), np.stack([rec["x"], rec["y"], rec["z"]], 1).view(np.uint32))
    assert np.array_equal(pts[:, 3].view(np.uint32), rec["rgb"])
    assert np.isfinite(pts[:, :3]).all()  # centroids of finite points only
