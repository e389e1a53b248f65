"""The numpy restatement of the colour clouds and the map (tests/map_cloud_exact.py) against its C oracle
(tests/map_cloud_oracle.c), bit for bit, and the PTX check that the map kernels keep the reference's uncontracted float chain."""
import re
import shutil
import subprocess
from pathlib import Path

import numpy as np
import pytest

import map_cloud_exact as mx

ROOT = Path(__file__).resolve().parent.parent
K = (525.0, 521.5, 319.5, 239.25)


def frame(rng, w=160, h=120, planted=(0.5, 2.0)):
    """random depths in [0.05, 9) m with NaN, +-inf, 0, negative and planted exact values, and a colour visual"""
    d = rng.uniform(0.05, 9.0, (h, w)).astype(np.float32)
    for v in (np.nan, np.inf, -np.inf, 0.0, -1.0, *planted):
        ys, xs = rng.integers(0, h, 40), rng.integers(0, w, 40)
        d[ys, xs] = v
        d[ys // 4 * 4, xs // 4 * 4] = v  # on every skip step's grid
    d[::4, ::4][rng.random((h // 4, w // 4)) < 0.05] = np.nan  # holes on every skip-step grid
    return d, rng.integers(0, 256, (h, w, 3)).astype(np.uint8)


def _bits(a):
    return a.view(np.uint8)


@pytest.mark.parametrize("step", [1, 2, 4])
@pytest.mark.parametrize("scaling", [1.0, 1.03, 0.001])
@pytest.mark.parametrize("bgr", [True, False])
@pytest.mark.parametrize("grey", [False, True])
@pytest.mark.parametrize("point_bytes", [32, 16])
def test_create_cloud_equals_the_oracle(step, scaling, bgr, grey, point_bytes):
    rng = np.random.default_rng(step * 100 + int(scaling * 1000) % 97)
    d, rgb = frame(rng)
    vis = rgb[..., 0].copy() if grey else rgb
    # minimum_depth equal to a planted depth (times the scaling, as the comparison sees it)
    min_depth = float(np.float32(np.float64(2.0) * scaling))
    got = mx.organised(mx.create_cloud(d, vis, K, step, scaling, min_depth, bgr), point_bytes)
    exp = mx.oracle_create_cloud(d, vis, K, step, scaling, min_depth, bgr, point_bytes)
    assert np.array_equal(_bits(got), _bits(exp))
    z = got["z"].ravel()
    assert np.isnan(z).sum() > 0 and (z == np.float32(min_depth)).sum() > 0


def _clouds(rng, n=3):
    return [mx.create_cloud(*frame(rng), K, 2, 1.0, 0.1, True) for _ in range(n)]


def _transforms(rng, n):
    from scipy.spatial.transform import Rotation
    out = []
    for _ in range(n):
        R = Rotation.from_rotvec(rng.normal(0, 0.6, 3)).as_matrix()
        out.append(np.concatenate([R, rng.normal(0, 2.0, (3, 1))], 1))
    return np.array(out)


@pytest.mark.parametrize("preserve", [False, True])
@pytest.mark.parametrize("maximum_depth", [3.5, np.inf, -1.0, 0.0])
def test_render_equals_the_oracle(preserve, maximum_depth):
    rng = np.random.default_rng(7)
    pcs = _clouds(rng)
    T = _transforms(rng, len(pcs))
    got = mx.render(pcs, T, maximum_depth, preserve, 32)
    exp = mx.oracle_render([mx.organised(pc) for pc in pcs], T, maximum_depth, preserve)
    assert np.array_equal(_bits(got), _bits(exp))
    n_all = sum(len(pc["x"]) for pc in pcs)
    if preserve:
        assert len(got) == n_all
    else:
        assert 0 < len(got) < n_all if maximum_depth != 0.0 else len(got) == 0
    # +-inf depths are not NaN: they are transformed (and only a finite maximum_depth drops them)
    if maximum_depth == np.inf and not preserve:
        assert np.isinf(got["x"]).any() or np.isnan(got["x"]).any()


def test_world2cam_is_a_rigid_transform():
    """the restated composition keeps a rotation (det 1, orthonormal) and cam2rgb maps the optical z axis to the ROS x axis"""
    from scipy.spatial.transform import Rotation
    P = np.eye(4)
    P[:3, :3] = Rotation.from_rotvec([0.3, -0.2, 0.5]).as_matrix()
    P[:3, 3] = [1.0, 2.0, -0.5]
    W = mx.world2cam(P)
    assert abs(np.linalg.det(W[:, :3]) - 1) < 1e-12 and np.allclose(W[:, :3] @ W[:, :3].T, np.eye(3), atol=1e-12)
    C0 = mx.world2cam(np.eye(4))
    assert np.allclose(C0[:, :3] @ [0, 0, 1], [1, 0, 0], atol=2e-3) and np.allclose(C0[:, 3], [0, -0.04, 0])


# ---- the map kernels keep the float chain uncontracted ------------------------------------------------------------------

def _nvcc():
    for c in (shutil.which("nvcc"), "/usr/local/cuda/bin/nvcc"):
        if c and Path(c).exists():
            return c
    return None


def _kernel_ops(ptx: str):
    """fma / mul / add counts (f32 and f64) of every kernel of map.cu"""
    out = {}
    for m in re.finditer(r"\.entry\s+(\S*k_(?:store|map)_\S*)\(.*?\n}\n", ptx, re.S):
        body = m.group(0)
        out[m.group(1)] = tuple(body.count(op) for op in ("fma.rn.f32", "fma.rn.f64", "mul.rn.f32", "add.rn.f32", "mul.rn.f64"))
    return out


@pytest.mark.skipif(_nvcc() is None, reason="nvcc not available")
def test_map_ptx_has_no_contracted_fma(tmp_path):
    from rgbdslam_v2_b200.build import NVCC_FLAGS
    flags = [f for f in NVCC_FLAGS if f not in ("-shared", "-ldl", "-Xcompiler", "-fPIC")]
    src = ROOT / "rgbdslam_v2_b200" / "csrc" / "map.cu"
    counts = []
    for extra in ([], ["--fmad=false"]):
        out = tmp_path / f"map{len(extra)}.ptx"
        subprocess.run([_nvcc(), *flags, *extra, "-ptx", "-o", str(out), str(src)], check=True, capture_output=True)
        counts.append(_kernel_ops(out.read_text()))
    assert len(counts[0]) == 5, counts[0]
    assert counts[0] == counts[1], counts
    for name, c in counts[0].items():
        assert c[0] == 0 and c[1] == 0, (name, c)
    scatter = [c for n, c in counts[0].items() if "k_map_scatter" in n][0]
    assert scatter[2] >= 15 and scatter[3] >= 11, scatter  # the point chain is there, as separate roundings
