"""The C++ shim's OctoMap path (tests/cpp/test_octomap_shim.cpp).  CPU: it compiles and links, refuses without a GPU, and its
octomapPose equals rgbdslam_v2_b200._capi.octomap_pose bit for bit -- two restatements of the pose chain, native float /
double arithmetic against numpy scalars.  GPU: GraphManager::saveOctomap writes the oracle's bytes (tests/octomap_oracle.c)
for the selected nodes, at every autosave and at the end, keeps the map without octomap_clear_after_save and empties it
with it, and octomap_clear_raycasted_clouds leaves the rendered nodes without clouds."""
import subprocess
from pathlib import Path

import numpy as np
import pytest

from rgbdslam_v2_b200._capi import octomap_pose

ROOT = Path(__file__).resolve().parent.parent


def _compile(tmp_path):
    exe = tmp_path / "test_octomap_shim"
    libdir = ROOT / "rgbdslam_v2_b200"
    subprocess.run(["g++", "-std=c++17", "-O2", "-Wall", f"-I{ROOT / 'include'}", str(ROOT / "tests/cpp/test_octomap_shim.cpp"),
                    "-o", str(exe), f"-L{libdir}", "-lrgbdslam_b200", f"-Wl,-rpath,{libdir}"], check=True)
    return exe


def test_octomap_shim_compiles_and_refuses_cpu(built, tmp_path):
    import torch
    exe = _compile(tmp_path)
    r = subprocess.run([str(exe), str(tmp_path / "absent.bin"), str(tmp_path)], capture_output=True, text=True)
    if not torch.cuda.is_available():
        assert r.returncode == 77 and "init failed" in r.stdout


def _pose_cases():
    from scipy.spatial.transform import Rotation
    import test_octomap_oracle_cpu as tc
    rng = np.random.default_rng(7)
    Rs = list(Rotation.random(3000, random_state=11).as_matrix())
    for axis in ([1, 0, 0], [0, 1, 0], [0, 0, 1], [1, 1, 0], [1, 1, 1], [1, -1, 0]):  # near and at 180 degrees, equal diagonals
        for deg in (180.0, 179.9999, 179.99, 120.0, 240.0, 90.0):
            Rs.append(Rotation.from_rotvec(np.radians(deg) * np.asarray(axis, float) / np.linalg.norm(axis)).as_matrix())
    Rs += [np.array(v[0]) for v in tc.DIVERGING.values()]
    Rs += [np.diag(d).astype(float) for d in ([1, -1, -1], [-1, 1, -1], [-1, -1, 1])]
    return [(R, rng.uniform(-5, 5, 3)) for R in Rs]


def test_shim_pose_chain_equals_the_python_restatement(built, tmp_path):
    exe = _compile(tmp_path)
    cases = _pose_cases()
    text = "\n".join(" ".join(repr(float(v)) for v in list(R.ravel()) + list(t)) for R, t in cases) + "\n"
    r = subprocess.run([str(exe), "pose"], input=text, capture_output=True, text=True, check=True)
    got = [[int(h, 16) for h in line.split()] for line in r.stdout.splitlines()]
    assert len(got) == len(cases)
    for (R, t), g in zip(cases, got):
        T = np.eye(4)
        T[:3, :3], T[:3, 3] = R, t
        assert g == [int(v) for v in octomap_pose(T).ravel().view(np.uint32)], R


@pytest.mark.gpu
def test_save_octomap_writes_the_oracle_bytes(built, tmp_path):
    import map_cloud_exact as mx
    import node_helpers as nh
    import octomap_exact as ox
    exe = _compile(tmp_path)
    gray, depth = nh.stack(nh.render(range(24)))
    F, H, W = gray.shape
    path = tmp_path / "frames.bin"
    with open(path, "wb") as f:
        f.write(np.array([W, H, F], np.int32).tobytes())
        f.write(np.ascontiguousarray(gray, np.uint8).tobytes())
        f.write(np.ascontiguousarray(depth, np.float32).tobytes())
    r = subprocess.run([str(exe), str(path), str(tmp_path)], capture_output=True, text=True)
    assert r.returncode == 0 and "OCTOMAP SHIM OK" in r.stdout, r.stdout + r.stderr
    rows = [l.split()[1:] for l in r.stdout.splitlines() if l.startswith("NODE ")]
    sel = [row for row in rows if row[1] == "1"]
    assert len(sel) >= F // 2
    m = ox.Oracle()
    autosaves = []
    for k, row in enumerate(sel):
        R = np.array([float(x) for x in row[2:11]]).reshape(3, 3)
        t = np.array([float(x) for x in row[11:14]])
        Tbits = np.array([int(h, 16) for h in row[14:26]], np.uint32)
        P = np.eye(4)
        P[:3, :3], P[:3, 3] = R, t
        assert np.array_equal(Tbits, octomap_pose(P).ravel().view(np.uint32))
        rec = np.fromfile(tmp_path / f"cloud_{row[0]}.bin", mx.POINT32)
        m.insert_cloud(dict(x=rec["x"], y=rec["y"], z=rec["z"], rgb=rec["rgb"]), Tbits.view(np.float32).reshape(3, 4))
        if (k + 1) % 3 == 0:
            autosaves.append(m.write())
    final = m.write()
    writes = {l.split()[1]: int(l.split()[2]) for l in r.stdout.splitlines() if l.startswith("WRITES ")}
    assert writes == {"a": len(autosaves) + 1, "b": len(autosaves) + 1}
    for run in ("a", "b"):
        for k, exp in enumerate(autosaves):
            assert (tmp_path / f"{run}_{k + 1}.ot").read_bytes() == exp, (run, k)
        assert (tmp_path / f"{run}_{len(autosaves) + 1}.ot").read_bytes() == final == (tmp_path / f"{run}.ot").read_bytes()
    assert ox.parse(final)[0] > 1000
    assert (tmp_path / "a_again.ot").read_bytes() == final  # no clear_after_save: the map stays
    assert (tmp_path / "b_after.ot").read_bytes() == ox.Oracle().write()  # clear_after_save: an empty map
    cleared = {l.split()[1]: int(l.split()[2]) for l in r.stdout.splitlines() if l.startswith("CLEARED ")}
    assert all(cleared[row[0]] == 1 for row in sel)
