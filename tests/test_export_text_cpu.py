"""CPU tests of the per-node exports' text and host logic: include/rgbdslam_b200/export_text.hpp (compiled with g++, without the
library) writes the YAML cv2.FileStorage writes of the same calls and std::ostream's float text; the restatements of
tests/cloud_export_exact.py keep the reference's quirks; the transform kernel's PTX is uncontracted; the C entry point exists
and refuses without an initialised library."""
import ctypes as C
import re
import shutil
import subprocess
from pathlib import Path

import numpy as np
import pytest

import cloud_export_exact as ex
import map_cloud_exact as mx

ROOT = Path(__file__).resolve().parent.parent
F32 = np.float32


@pytest.fixture(scope="module")
def exe(tmp_path_factory):
    out = tmp_path_factory.mktemp("export_text") / "test_export_text"
    subprocess.run(["g++", "-std=c++17", "-O2", "-Wall", f"-I{ROOT / 'include'}", str(ROOT / "tests/cpp/test_export_text.cpp"), "-o",
                    str(out)], check=True)
    return out


SPECIAL = np.array([np.nan, np.inf, -np.inf, 0.0, -0.0, 0.1, 2 ** 31 - 1, 2 ** 31, -2 ** 31, 1e16, 1e20, -1e20, 1e-40, -1e-45, 3.0, -2.5,
                    123456789.0, 1.5e-5, 2 ** 24 + 2, -7.0, 0.5, 65504.0, 3.4028235e38], F32)


def _yaml(exe, tmp_path, locs, desc):
    spec = tmp_path / "spec.bin"
    locs = np.ascontiguousarray(locs, F32).reshape(-1, 3)
    desc = np.ascontiguousarray(desc, np.uint8).reshape(-1, 32)
    spec.write_bytes(np.int32(len(locs)).tobytes() + locs.tobytes() + np.int32(len(desc)).tobytes() + desc.tobytes())
    out = tmp_path / "ours.yml"
    subprocess.run([str(exe), "yaml", str(spec), str(out)], check=True)
    return out.read_bytes(), ex.cv2_features_yaml(tmp_path / "cv2.yml", locs, desc)


@pytest.mark.parametrize("rows", [0, 1, 37])
def test_yaml_equals_cv2_filestorage(exe, tmp_path, rows):
    rng = np.random.default_rng(rows)
    locs = np.concatenate([SPECIAL, rng.permutation(SPECIAL), (rng.standard_normal(3 * rows) * 10.0 ** rng.integers(-8, 9, 3 * rows))])
    locs = locs[: len(locs) // 3 * 3].astype(F32)
    desc = rng.integers(0, 256, (rows, 32)).astype(np.uint8)
    ours, theirs = _yaml(exe, tmp_path, locs, desc)
    assert ours == theirs
    assert b".Nan" in ours and b"-.Inf" in ours and b"0.10000000149011612" in ours and b"2147483648" in ours and b"1e+20" not in ours


def test_yaml_of_nothing_and_of_long_rows_equals_cv2(exe, tmp_path):
    ours, theirs = _yaml(exe, tmp_path, np.zeros((0, 3)), np.zeros((0, 32)))
    assert ours == theirs and b"Feature_Locations:\n   []\n" in ours
    # three 23-character values: the flow map wraps as FileStorage does past column 71
    big = np.full((4, 3), -1.0000000200408773e+20, F32)
    big[1] = [-9.9999461011147596e-41, -1.2345678e-30, -3.3333333e-33]
    ours, theirs = _yaml(exe, tmp_path, big, np.full((2, 32), 255))
    assert ours == theirs and b",\n       z:" in ours


def test_double_text_matches_cv2_for_exact_doubles(exe, tmp_path):
    """1e20 is not a float: 1e20f forwarded as a double prints all 17 digits, as cv2 does"""
    ours, _ = _yaml(exe, tmp_path, np.array([[1e20, 2 ** 31, -0.0]], F32), np.zeros((0, 32)))
    assert b"{ x:1.0000000200408773e+20, y:2147483648, z:0. }" in ours


def test_ostream_floats_equal_percent_g(exe, tmp_path):
    rng = np.random.default_rng(3)
    vals = np.concatenate([SPECIAL[~np.isnan(SPECIAL)], (rng.standard_normal(400) * 10.0 ** rng.integers(-12, 12, 400)),
                           np.array([1e-5, 1e-4, 123456.5, 1234567.0, 999999.5, -0.0], F32)]).astype(F32)
    spec = tmp_path / "g.bin"
    spec.write_bytes(np.int32(len(vals)).tobytes() + vals.tobytes())
    got = subprocess.run([str(exe), "g", str(spec)], check=True, capture_output=True, text=True).stdout.splitlines()
    assert got == ["%g" % v for v in vals]


def test_restated_pose_text_keeps_the_reference_quirks():
    q, o = ex.sensor_pose(None)
    assert ex.pose_text(q, o) == "-1 0 0 0 0 -1 0 0 0 0 1 0 0 0 0 1\n"
    assert ex.viewpoint(q, o) == "0 0 0 0 0 0 1"
    # the identity estimate: eigenTransf2TF is the identity, and base2points.inverse() turns the origin's zeros to -0
    I = np.concatenate([np.eye(3), np.zeros((3, 1))], 1)
    W = ex.world_to_points(I)
    assert np.array_equal(W, I) and np.signbit(ex.tf_inverse(I)[:, 3]).all()
    q, o = ex.sensor_pose(I)
    assert ex.pose_text(q, o) == "1 0 0 0 0 1 0 0 0 0 1 0 0 0 0 1\n" and ex.viewpoint(q, o) == "0 0 0 1 0 0 0"
    # a half turn about x: the rotation's exact zeros pass through the identity products
    M = np.array([[1.0, 0, 0, 0.5], [0, -1.0, 0, -0.25], [0, 0, -1.0, 2.0]])
    q, o = ex.sensor_pose(M)
    assert np.array_equal(q, [1, 0, 0, 0]) and ex.pose_text(q, o).startswith("1 0 0 0.5 0 -1 0 -0.25 0 0 -1 2 ")


def test_restated_transform_leaves_non_finite_points():
    x = np.array([1.0, np.nan, 2.0, np.inf, 0.5], F32)
    y = np.array([2.0, 0.0, -np.inf, 1.0, 0.25], F32)
    z = np.array([3.0, 1.0, 1.0, 1.0, np.nan], F32)
    pc = dict(x=x, y=y, z=z, rgb=np.arange(5, dtype=np.uint32), w16=np.arange(5, dtype=np.uint32), w=5, h=1)
    T = np.array([[0.0, -1.0, 0.0, 1.0], [1.0, 0.0, 0.0, 2.0], [0.0, 0.0, 1.0, 3.0]])
    out = ex.transform_cloud(pc, T)
    assert out["x"][0] == -1.0 and out["y"][0] == 3.0 and out["z"][0] == 6.0
    for k in "xyz":
        assert np.array_equal(out[k][1:].view(np.uint32), pc[k][1:].view(np.uint32))
    # an +inf point is left by transformPointCloud, and transformed by transformAndAppendPointCloud (the map)
    assert out["x"][3] == np.inf and out["y"][3] == 1.0
    assert np.isnan(mx.render([pc], [T], preserve=True)["x"][3])  # 0 * inf


def test_restated_feature_locations_propagate_inf():
    T = np.array([[0.0, 0.0, 1.0, 0.0], [-1.0, 0.0, 0.0, -0.04], [0.0, -1.0, 0.0, 0.0]])
    got = ex.feature_locations(T, [[1.0, 2.0, 3.0], [0.0, 0.0, np.inf]])
    assert np.array_equal(got[0], np.array([3.0, F32(-1.0) + F32(-0.04), -2.0], F32)) and np.isinf(got[1]).any()


def _nvcc():
    for c in (shutil.which("nvcc"), "/usr/local/cuda/bin/nvcc"):
        if c and Path(c).exists():
            return c
    return None


@pytest.mark.skipif(_nvcc() is None, reason="nvcc not available")
def test_transform_kernel_ptx_has_no_fma(tmp_path):
    from rgbdslam_v2_b200.build import NVCC_FLAGS
    flags = [f for f in NVCC_FLAGS if f not in ("-shared", "-ldl", "-Xcompiler", "-fPIC")]
    out = tmp_path / "map.ptx"
    subprocess.run([_nvcc(), *flags, "-ptx", "-o", str(out), str(ROOT / "rgbdslam_v2_b200" / "csrc" / "map.cu")], check=True,
                   capture_output=True)
    m = re.search(r"\.entry\s+\S*k_transform_clouds\S*\(.*?\n}\n", out.read_text(), re.S)
    assert m
    body = m.group(0)
    assert "fma" not in body
    assert body.count("mul.rn.f32") >= 9 and body.count("add.rn.f32") >= 9  # the chain is there, rounded step by step


def test_transform_entry_point_is_declared_exported_and_refuses_before_init(built):
    import torch
    from rgbdslam_v2_b200 import _capi
    txt = re.sub(r"/\*.*?\*/", "", (ROOT / "include" / "rgbdslam_b200" / "cloud_transform.h").read_text(), flags=re.S)
    assert re.findall(r"\b(rgbdslam_b200_[a-z0-9_]+)\s*\(", txt) == ["rgbdslam_b200_transform_clouds"]
    assert '#include "cloud_transform.h"' in (ROOT / "include" / "rgbdslam_b200" / "node.hpp").read_text()
    lib = _capi.load_library()
    assert lib.rgbdslam_b200_transform_clouds.argtypes
    if torch.cuda.is_available():
        pytest.skip("GPU present: the library may already be initialised in this process")
    assert lib.rgbdslam_b200_set_hamming_path(7) == 1
    sentinel = lib.rgbdslam_b200_last_error()
    assert lib.rgbdslam_b200_transform_clouds(0, None, None) == 3
    assert lib.rgbdslam_b200_last_error() not in (b"", sentinel)
    lib.rgbdslam_b200_set_hamming_path(1)
