"""The C++ shim's online OctoMap and occupancy filter (tests/cpp/test_octomap_online_shim.cpp).  CPU: it compiles, links and
refuses without a GPU.  GPU: with octomap_online_creation, saveOctomap writes the bytes of the oracle (tests/octomap_oracle.c)
replaying one single-node insert per optimisation -- the newest node under the pose it held --; with
octomap_clear_raycasted_clouds every rendered node is left without a cloud; occupancyFilterClouds leaves every node's cloud
equal to the oracle's filter (tests/octomap_filter_oracle.c) under the sensor pose the node recorded, PCL's default for nodes updateCloudOrigin never saw."""
import subprocess
from pathlib import Path

import numpy as np
import pytest

ROOT = Path(__file__).resolve().parent.parent
IDENTITY7 = np.array([0, 0, 0, 1, 0, 0, 0], np.float32)


def _compile(tmp_path):
    exe = tmp_path / "test_octomap_online_shim"
    libdir = ROOT / "rgbdslam_v2_b200"
    subprocess.run(["g++", "-std=c++17", "-O2", "-Wall", f"-I{ROOT / 'include'}", str(ROOT / "tests/cpp/test_octomap_online_shim.cpp"),
                    "-o", str(exe), f"-L{libdir}", "-lrgbdslam_b200", f"-Wl,-rpath,{libdir}"], check=True)
    return exe


def test_online_shim_compiles_and_refuses_cpu(built, tmp_path):
    import torch
    exe = _compile(tmp_path)
    r = subprocess.run([str(exe), str(tmp_path / "absent.bin"), str(tmp_path)], capture_output=True, text=True)
    if not torch.cuda.is_available():
        assert r.returncode == 77 and "init failed" in r.stdout


def _hex(words):
    return np.array([int(h, 16) for h in words], np.uint32).view(np.float32)


def _run(exe, tmp_path, clear):
    import node_helpers as nh
    gray, depth = nh.stack(nh.render(range(16)))
    F, H, W = gray.shape
    path = tmp_path / "frames.bin"
    with open(path, "wb") as f:
        f.write(np.array([W, H, F], np.int32).tobytes())
        f.write(np.ascontiguousarray(gray, np.uint8).tobytes())
        f.write(np.ascontiguousarray(depth, np.float32).tobytes())
    out = tmp_path / ("clear" if clear else "keep")
    out.mkdir()
    if clear:
        (out / "clear").write_text("")
    r = subprocess.run([str(exe), str(path), str(out)], capture_output=True, text=True)
    assert r.returncode == 0 and "ONLINE SHIM OK" in r.stdout, r.stdout + r.stderr
    lines = [l.split() for l in r.stdout.splitlines()]
    renders = []  # (node id, float 3 x 4) of every insert, in order
    for l in lines:
        if l[0] == "ADDED" and l[2] == "1" and l[4] == "1" and l[5] == "1" and len(l) == 18:
            renders.append((int(l[3]), _hex(l[6:18]).reshape(3, 4)))
    sensor = {int(l[1]): _hex(l[2:9]) for l in lines if l[0] == "SENSOR"}
    cloud = {int(l[1]): int(l[2]) for l in lines if l[0] == "CLOUD"}
    return out, renders, sensor, cloud


@pytest.mark.gpu
def test_online_creation_and_occupancy_filter_equal_the_oracle(built, tmp_path):
    import map_cloud_exact as mx
    import octomap_exact as ox
    import octomap_filter_exact as fx
    exe = _compile(tmp_path)
    out, renders, sensor, cloud = _run(exe, tmp_path, clear=False)
    assert len(renders) >= 4 and len({i for i, _ in renders}) >= 4
    m = fx.FilterOracle()
    clouds = {i: np.fromfile(out / f"before_{i}.bin", mx.POINT32) for i in sensor}
    for i, T in renders:
        rec = clouds[i]
        m.insert_cloud(dict(x=rec["x"], y=rec["y"], z=rec["z"], rgb=rec["rgb"]), T)
    data = (out / "online.ot").read_bytes()
    assert data == m.write() and ox.parse(data)[0] > 1000
    rendered = {i for i, _ in renders}
    mixed = 0
    for i, rec in clouds.items():
        s = sensor[i]
        if i not in rendered:
            assert s.tobytes() == IDENTITY7.tobytes()
        keep = m.occupancy_filter(np.stack([rec["x"], rec["y"], rec["z"]], 1), s[:4], s[4:], 3e4)
        after = np.fromfile(out / f"after_{i}.bin", mx.POINT32)
        assert cloud[i] == 1 and after.tobytes() == rec[keep].tobytes(), i
        mixed += 0 < keep.sum() < len(keep)
    assert mixed >= 2

    out, renders, sensor, cloud = _run(exe, tmp_path, clear=True)
    rendered = {i for i, _ in renders}
    assert rendered and all(cloud[i] == 0 for i in rendered)
    assert all(cloud[i] == 1 for i in cloud if i not in rendered)
