"""The C++ shim's per-node exports (tests/cpp/test_export_shim.cpp).  CPU: it compiles, links and refuses without a GPU.  GPU:
over 30 rendered frames, saveIndividualClouds writes for every node with a valid estimate and a non-empty cloud a PCD that
parses to the node's cloud -- as stored, then transformed once and twice with transform_individual_clouds, equal to the
restatement of tests/cloud_export_exact.py -- with the pinned WIDTH / HEIGHT / VIEWPOINT, and the restated pose text; the
nodes it skips have no files; the pose becomes the node's cloud sensor pose; saveAllFeatures writes the bytes cv2.FileStorage
writes of the restated locations and the nodes' descriptors."""
import subprocess
from pathlib import Path

import numpy as np
import pytest

ROOT = Path(__file__).resolve().parent.parent


def _compile(tmp_path):
    exe = tmp_path / "test_export_shim"
    libdir = ROOT / "rgbdslam_v2_b200"
    subprocess.run(["g++", "-std=c++17", "-O2", "-Wall", f"-I{ROOT / 'include'}", str(ROOT / "tests/cpp/test_export_shim.cpp"),
                    "-o", str(exe), f"-L{libdir}", "-lrgbdslam_b200", f"-Wl,-rpath,{libdir}"], check=True)
    return exe


def test_export_shim_compiles_and_refuses_cpu(built, tmp_path):
    import torch
    exe = _compile(tmp_path)
    r = subprocess.run([str(exe), str(tmp_path / "absent.bin"), str(tmp_path)], capture_output=True, text=True)
    if not torch.cuda.is_available():
        assert r.returncode == 77 and "init failed" in r.stdout


def _read_pcd(path):
    raw = Path(path).read_bytes()
    head, body = raw.split(b"DATA binary\n", 1)
    fields = dict(l.split(" ", 1) for l in head.decode().splitlines() if not l.startswith("#"))
    return fields, np.frombuffer(body, np.float32).reshape(-1, 4)


def _hex(words):
    return np.array([int(h, 16) for h in words], np.uint32).view(np.float32)


@pytest.mark.gpu
def test_individual_clouds_and_features_equal_the_restatement(built, tmp_path):
    import cloud_export_exact as ex
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
    out = tmp_path / "out"
    out.mkdir()
    r = subprocess.run([str(exe), str(path), str(out)], capture_output=True, text=True)
    assert r.returncode == 0 and "EXPORT SHIM OK" in r.stdout, r.stdout + r.stderr
    lines = [l.split() for l in r.stdout.splitlines() if l.strip()]
    nodes = {}
    for l in lines:
        if l[0] == "NODE":
            v = np.array([float(x) for x in l[4:]]).reshape(-1, 3, 4)
            nodes[int(l[1])] = dict(valid=l[2] == "1", est=l[3] == "1", iso=v[0] if len(v) else None, tf=v[1] if len(v) else None,
                                    map=v[2] if len(v) else None)
    cloud = {int(l[1]): (int(l[2]), int(l[3])) for l in lines if l[0] == "CLOUD"}
    sensor = {(l[1], int(l[2])): _hex(l[3:10]) for l in lines if l[0] == "SENSOR"}
    saved = {l[1]: int(l[2]) for l in lines if l[0] == "SAVED"}
    cleared = [int(l[1]) for l in lines if l[0] == "CLEARED"]
    assert sorted(nodes) == list(range(len(nodes))) and len(nodes) >= F // 2 and len(cleared) == 1
    written = [i for i, n in nodes.items() if n["valid"] and n["est"] and i in cloud and cloud[i][0] * cloud[i][1] > 0]
    assert cleared[0] not in written and not nodes[1]["valid"] and len(written) >= 5, r.stdout
    assert saved["plain"] == saved["xf1"] == saved["xf2"] == len(written)
    for i in nodes:
        for name in ("plain", "xf1", "xf2"):
            for ext in ("pcd", "txt"):
                assert (out / f"{name}_{i:04d}.{ext}").exists() == (i in written), (i, name, ext)
    for i in written:
        w, h = cloud[i]
        rec = np.fromfile(out / f"before_{i}.bin", mx.POINT32)
        pc = ex.from_records(rec, w, h)
        steps = {"plain": pc, "xf1": ex.transform_cloud(pc, nodes[i]["iso"])}
        steps["xf2"] = ex.transform_cloud(steps["xf1"], nodes[i]["iso"])
        for name, exp in steps.items():
            q, o = ex.sensor_pose(None if name != "plain" else nodes[i]["tf"])
            fields, pts = _read_pcd(out / f"{name}_{i:04d}.pcd")
            assert fields["FIELDS"] == "x y z rgb" and fields["WIDTH"] == str(w) and fields["HEIGHT"] == str(h)
            assert fields["POINTS"] == str(w * h) and fields["VIEWPOINT"] == ex.viewpoint(q, o), (i, name, fields)
            body = np.stack([exp["x"].view(np.uint32), exp["y"].view(np.uint32), exp["z"].view(np.uint32), exp["rgb"]], 1)
            assert np.array_equal(pts.view(np.uint32), body), (i, name)
            assert (out / f"{name}_{i:04d}.txt").read_text() == ex.pose_text(q, o), (i, name)
            assert sensor[(name, i)].tobytes() == np.concatenate([q, o]).astype(np.float32).tobytes(), (i, name)
            if name != "plain":
                after = np.fromfile(out / f"{name}_{i}.bin", mx.POINT32)
                assert np.array_equal(after.view(np.uint8), mx.organised(exp).reshape(-1).view(np.uint8)), (i, name)
        assert (out / f"xf1_{i:04d}.txt").read_text() == "-1 0 0 0 0 -1 0 0 0 0 1 0 0 0 0 1\n"
    # a node skipped by saveIndividualClouds keeps PCL's default sensor pose and, if it has a cloud, its cloud
    for i in set(nodes) - set(written):
        assert sensor[("xf2", i)].tobytes() == np.array([0, 0, 0, 1, 0, 0, 0], np.float32).tobytes()
        if i in cloud:
            assert (out / f"xf2_{i}.bin").read_bytes() == (out / f"before_{i}.bin").read_bytes()
    # saveAllFeatures
    locs, desc = [], []
    for i in sorted(nodes):
        raw = (out / f"features_{i}.bin").read_bytes()
        n = int(np.frombuffer(raw[:4], np.int32)[0])
        xyz = np.frombuffer(raw[4:4 + 16 * n], np.float32).reshape(n, 4)[:, :3]
        desc.append(np.frombuffer(raw[4 + 16 * n:], np.uint8).reshape(n, 32))
        if nodes[i]["valid"]:
            locs.append(ex.feature_locations(nodes[i]["map"], xyz))
    locs = np.concatenate(locs)
    assert saved["features"] == len(locs) > 0
    exp = ex.cv2_features_yaml(tmp_path / "cv2.yml", locs, np.concatenate(desc))
    assert (out / "features.yml").read_bytes() == exp
