"""The C++ shim's map path (tests/cpp/test_map_shim.cpp): CPU: compile + link + 'no CPU fallback' exit path; GPU:
GraphManager::saveAllClouds writes a binary PCD that parses to exactly the render_cloud records of the valid nodes, whose
transforms agree with the restated double composition of saveAllCloudsToFile (tests/map_cloud_exact.py)."""
import subprocess
from pathlib import Path

import numpy as np
import pytest

ROOT = Path(__file__).resolve().parent.parent


def _compile(tmp_path):
    exe = tmp_path / "test_map_shim"
    libdir = ROOT / "rgbdslam_v2_b200"
    subprocess.run(["g++", "-std=c++17", "-O2", "-Wall", f"-I{ROOT / 'include'}", str(ROOT / "tests/cpp/test_map_shim.cpp"),
                    "-o", str(exe), f"-L{libdir}", "-lrgbdslam_b200", f"-Wl,-rpath,{libdir}"], check=True)
    return exe


def test_map_shim_compiles_and_refuses_cpu(built, tmp_path):
    import torch
    exe = _compile(tmp_path)
    r = subprocess.run([str(exe), str(tmp_path / "absent.bin"), str(tmp_path / "m.pcd"), str(tmp_path / "r.bin")],
                       capture_output=True, text=True)
    if not torch.cuda.is_available():
        assert r.returncode == 77 and "init failed" in r.stdout


def read_pcd(path):
    """header fields and the (n, 4) float32 / uint32 body of a binary PCD"""
    raw = Path(path).read_bytes()
    head, body = raw.split(b"DATA binary\n", 1)
    fields = dict(l.split(" ", 1) for l in head.decode().splitlines() if not l.startswith("#"))
    return fields, np.frombuffer(body, np.float32).reshape(-1, 4)


@pytest.mark.gpu
def test_save_all_clouds_writes_the_rendered_map(built, tmp_path):
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
    assert r.returncode == 0 and "MAP SHIM OK" in r.stdout, r.stdout + r.stderr
    fields, pts = read_pcd(tmp_path / "map.pcd")  # ".pcd" appended
    assert fields["FIELDS"] == "x y z rgb" and fields["SIZE"] == "4 4 4 4" and fields["TYPE"] == "F F F F"
    rec = np.fromfile(tmp_path / "render.bin", mx.POINT32)
    assert fields["WIDTH"] == "1" and int(fields["HEIGHT"]) == int(fields["POINTS"]) == len(pts) == len(rec) > 0
    assert np.array_equal(pts[:, :3].view(np.uint32), np.stack([rec["x"], rec["y"], rec["z"]], 1).view(np.uint32))
    assert np.array_equal(pts[:, 3].view(np.uint32), rec["rgb"])
    nodes = [l.split()[1:] for l in r.stdout.splitlines() if l.startswith("NODE ")]
    assert len(nodes) >= F // 2
    for row in nodes:
        e = np.array([float(x) for x in row[2:9]])
        T = np.array([float(x) for x in row[9:]]).reshape(3, 4)
        from scipy.spatial.transform import Rotation
        P = np.eye(4)
        P[:3, :3] = Rotation.from_quat(e[3:]).as_matrix()
        P[:3, 3] = e[:3]
        exp = mx.world2cam(P)
        # the float matrices the map uses are within one float ulp of the restated composition
        assert np.all(np.abs(T.astype(np.float32).view(np.int32).astype(np.int64) - exp.astype(np.float32).view(np.int32)) <= 1), row
