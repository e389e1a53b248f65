"""The numpy restatement of the voxel filter (tests/voxel_exact.py) against its C oracle (tests/voxel_oracle.c), bit for bit,
on the inputs where the rule's decisions show; the PTX check that the centroid kernel keeps the uncontracted float sums; and
the export of the entry point."""
import re
import shutil
import subprocess
from pathlib import Path

import numpy as np
import pytest

import map_cloud_exact as mx
import voxel_exact as vx

ROOT = Path(__file__).resolve().parent.parent
F32 = np.float32


def _pc(xyz, rgb=None):
    xyz = np.asarray(xyz, F32).reshape(-1, 3)
    rgb = np.arange(len(xyz), dtype=np.uint32) * 2654435761 & 0xFFFFFF if rgb is None else np.asarray(rgb, np.uint32)
    return dict(x=xyz[:, 0].copy(), y=xyz[:, 1].copy(), z=xyz[:, 2].copy(), rgb=rgb, w16=rgb.copy(), w=len(rgb), h=1)


def _same(a, b):
    if a is None or b is None:
        return a is None and b is None
    return all(a[k].shape == b[k].shape and np.array_equal(a[k].view(np.uint32), b[k].view(np.uint32)) for k in ("x", "y", "z", "rgb"))


def _both(pc, vfs):
    got, exp = vx.reduce_cloud(pc, vfs), vx.oracle_reduce_cloud(pc, vfs)
    assert _same(got, exp), vfs
    return got


def rendered_cloud(k, step=4):
    """the stored cloud of rendered frame k (NaN holes included) with a colour visual"""
    import node_helpers as nh
    gray, depth = nh.render([k])[0]
    vis = np.stack([gray, np.roll(gray, 3, axis=-1), np.roll(gray, 5, axis=-2)], -1)
    return mx.create_cloud(depth, vis, nh.K4(), step, 1.0, 0.1)


@pytest.mark.parametrize("vfs", [0.01, 0.05, 0.2, 1.03])
def test_rendered_depth_clouds(vfs):
    for k in (0, 7):
        pc = rendered_cloud(k)
        out = _both(pc, vfs)
        n_finite = int(np.isfinite(pc["z"]).sum())
        assert 0 < out["w"] <= n_finite < len(pc["z"]) and out["h"] == 1
        if vfs >= 0.05:
            assert out["w"] < n_finite // 2
        # every centroid lies inside the bounds of the cloud, and the voxel indices ascend: z-major, then y, then x
        fin, inv, min_b, div_b = vx.grid(pc, vfs)
        ijk = [np.floor(out[c] * inv).astype(np.int64) - min_b[a] for a, c in enumerate("xyz")]
        idx = ijk[0] + div_b[0] * (ijk[1] + div_b[1] * ijk[2])
        assert (np.diff(idx) >= 0).all()


def test_non_finite_points_take_no_part():
    rng = np.random.default_rng(1)
    xyz = rng.uniform(-2, 2, (4000, 3)).astype(F32)
    clean = _both(_pc(xyz), 0.25)
    # 300 points with one NaN / +inf / -inf coordinate between the clean points, which keep their order
    slots = np.ones(4300, bool)
    slots[rng.choice(4300, 300, replace=False)] = False
    all_xyz = np.zeros((4300, 3), F32)
    all_rgb = np.full(4300, 0xFFFFFF, np.uint32)
    all_xyz[slots], all_rgb[slots] = xyz, _pc(xyz)["rgb"]
    bad = xyz[:300].copy()
    for j, v in enumerate((np.nan, np.inf, -np.inf)):
        bad[j * 100:(j + 1) * 100, j] = v
    all_xyz[~slots] = bad
    assert _same(_both(_pc(all_xyz, all_rgb), 0.25), clean)


def test_negative_coordinates_floor_and_faces():
    """floor, not truncation, below zero; a point exactly on a voxel face belongs to the voxel above"""
    xyz = [[-0.75, 0.0, 0.0], [-0.25, 0.0, 0.0], [0.25, 0.0, 0.0], [0.5, 0.0, 0.0], [-0.5, 0.0, 0.0], [-1.0, 0.0, 0.0], [0.0, 0.0, 0.0]]
    out = _both(_pc(xyz), 0.5)
    # voxels [-1, -0.5), [-0.5, 0), [0, 0.5), [0.5, 1)
    assert out["w"] == 4
    assert np.array_equal(out["x"], np.array([(-0.75 - 1.0) / 2, (-0.25 - 0.5) / 2, (0.25 + 0.0) / 2, 0.5], F32))
    rng = np.random.default_rng(2)
    grid_pts = rng.integers(-40, 40, (5000, 3)).astype(F32) * F32(0.125)  # exact multiples of the leaf: all on faces
    out = _both(_pc(grid_pts), 0.125)
    assert out["w"] == len(np.unique(grid_pts, axis=0))


def test_single_point_no_point_and_one_voxel():
    one = _both(_pc([[0.3, -0.2, 1.5]], [0x123456]), 0.05)
    assert one["w"] == 1 and one["rgb"][0] == 0x123456 and np.array_equal(one["x"], np.array([0.3], F32))
    none = _both(_pc([[np.nan, 0, 0], [0, np.inf, 0], [1, 1, -np.inf]]), 0.05)
    assert none["w"] == 0 and none["h"] == 1
    assert _both(_pc(np.zeros((0, 3))), 0.05)["w"] == 0
    rng = np.random.default_rng(3)
    xyz = rng.uniform(0.01, 0.99, (30000, 3)).astype(F32)
    every = _both(_pc(xyz), 1.0)
    assert every["w"] == 1
    seq = F32(0)
    for v in xyz[:, 0]:
        seq = seq + v
    assert every["x"][0] == seq * (F32(1) / F32(30000))  # the sum runs point after point


def test_colour_sum_beyond_2_to_24():
    """70000 points of colour 255 in one voxel: the float sum passes 2^24 = 16777216 and stays exact (multiples of 255 are not
    all representable beyond it, so the sequential order matters)"""
    n = 70000
    rng = np.random.default_rng(4)
    xyz = rng.uniform(0.1, 0.9, (n, 3)).astype(F32)
    rgb = rng.integers(250, 256, n).astype(np.uint32) * 0x010101
    out = _both(_pc(xyz, rgb), 1.0)
    assert out["w"] == 1 and 250 * n > 2**24
    assert 250 <= (out["rgb"][0] & 255) <= 255


def test_leaf_too_small_leaves_the_cloud():
    rng = np.random.default_rng(5)
    xyz = rng.uniform(-1, 1, (2000, 3)).astype(F32)
    assert _both(_pc(xyz), 0.01)["w"] > 1000
    far = np.concatenate([xyz, [[3000.0, 2500.0, 900.0]]]).astype(F32)  # 300001 x 250001 x ~ 90000 cells of 0.01
    assert _both(_pc(far), 0.01) is None
    assert _both(_pc(far), 2.0)["w"] > 1
    # 1291^3 > INT32_MAX > 1290^3: the decision sits on the product
    edge = np.array([[0, 0, 0], [1289.5, 1289.5, 1289.5]], F32)
    assert _both(_pc(edge), 1.0)["w"] == 2
    assert _both(_pc(edge + F32(1.0) * np.array([[0], [1]], F32)), 1.0) is None


@pytest.mark.parametrize("n", [3, 7, 49])
def test_mean_multiplies_by_the_reciprocal(n):
    """sums whose product with the float reciprocal of n differs from their quotient by n"""
    rng = np.random.default_rng(n)
    found = 0
    for _ in range(200):
        xyz = rng.uniform(0.05, 0.95, (n, 3)).astype(F32)
        out = _both(_pc(xyz), 1.0)
        s = np.zeros(3, F32)
        for p in xyz:
            s = s + p
        mul, div = s * (F32(1) / F32(n)), s / F32(n)
        assert np.array_equal(np.array([out["x"][0], out["y"][0], out["z"][0]], F32).view(np.uint32), mul.view(np.uint32))
        found += int((mul.view(np.uint32) != div.view(np.uint32)).sum())
    assert found > 10


def test_colour_mean_is_truncated():
    # (255 * 199 + 254) / 200 = 254.995 -> 254; (3 * 1 + 0) / 4 = 0.75 -> 0
    xyz = np.full((200, 3), 0.5, F32)
    rgb = np.full(200, 0xFF00FF, np.uint32)
    rgb[17] = 0xFE00FE
    out = _both(_pc(xyz, rgb), 1.0)
    assert out["rgb"][0] == 0xFE00FE
    out = _both(_pc(xyz[:4], [0x010000, 0x010100, 0x010000, 0x000000]), 1.0)
    assert out["rgb"][0] == 0


# ---- the device side -----------------------------------------------------------------------------------------------------

def _nvcc():
    for c in (shutil.which("nvcc"), "/usr/local/cuda/bin/nvcc"):
        if c and Path(c).exists():
            return c
    return None


@pytest.mark.skipif(_nvcc() is None, reason="nvcc not available")
def test_voxel_ptx_has_no_contracted_fma(tmp_path):
    from rgbdslam_v2_b200.build import NVCC_FLAGS
    flags = [f for f in NVCC_FLAGS if f not in ("-shared", "-ldl", "-Xcompiler", "-fPIC")]
    out = tmp_path / "voxel.ptx"
    subprocess.run([_nvcc(), *flags, "-ptx", "-o", str(out), str(ROOT / "rgbdslam_v2_b200" / "csrc" / "voxel.cu")], check=True,
                   capture_output=True)
    kernels = {m.group(1): m.group(0) for m in re.finditer(r"\.entry\s+(\S*k_vox_\S*)\(.*?\n}\n", out.read_text(), re.S)}
    assert len(kernels) == 9, sorted(kernels)
    for name, body in kernels.items():
        assert "fma.rn" not in body, name
    cen = [b for n, b in kernels.items() if "k_vox_centroids" in n][0]
    assert cen.count("add.rn.f32") >= 6 and cen.count("mul.rn.f32") >= 6 and cen.count("div.rn.f32") == 1


def test_reduce_clouds_is_declared_and_exported(built):
    from rgbdslam_v2_b200 import _capi
    lib = _capi.load_library()
    txt = re.sub(r"/\*.*?\*/", "", (ROOT / "include" / "rgbdslam_b200" / "voxel.h").read_text(), flags=re.S)
    assert re.findall(r"\b(rgbdslam_b200_[a-z0-9_]+)\s*\(", txt) == ["rgbdslam_b200_reduce_clouds"]
    assert lib.rgbdslam_b200_reduce_clouds.argtypes
    assert '#include "voxel.h"' in (ROOT / "include" / "rgbdslam_b200" / "node.hpp").read_text()


def test_reduce_clouds_before_init(built):
    import torch
    if torch.cuda.is_available():
        pytest.skip("GPU present: the library may already be initialised in this process")
    from rgbdslam_v2_b200 import _capi
    lib = _capi.load_library()
    assert lib.rgbdslam_b200_reduce_clouds(0, None, 0.05, None) == 3  # ERR_STATE: no CPU fallback
