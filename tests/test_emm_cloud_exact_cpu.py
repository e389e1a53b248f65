"""The numpy restatement of the environment measurement model on kept point clouds (tests/emm_cloud_exact.py,
`pairwise_cloud`) against its C oracle (tests/emm_cloud_oracle.c), count for count, and the PTX check that both
instantiations of the EMM kernels keep the reference's uncontracted float chain."""
import re
import shutil
import subprocess
from pathlib import Path

import numpy as np
import pytest

import emm_cloud_exact as ec
import emm_exact as ee

ROOT = Path(__file__).resolve().parent.parent
K_A = (525.0, 525.0, 319.5, 239.5)
K_B = (481.2, 479.7, 305.25, 251.5)
K_S = (300.0, 301.0, 175.5, 173.25)
K_0 = (0.0, 0.0, 0.0, 0.0)
SPECIALS = ("nan-z", "nan-x", "+inf-z", "-inf-z", "zero-z", "neg-z")


def make_cloud(rng, w, h, K, stride, perturb=0.02):
    """An organised cloud (h, w, stride) float32 of a block scene seen by K: x / y scaled by 1 + N(0, perturb) away from the
    pixel-grid back-projection, no-depth pixels NaN in all three coordinates (as PCL marks them); stride 8 carries colour
    bits in channel 4."""
    d = ee.block_scene(rng, w, h, K)
    fx, fy, cx, cy = K
    u, v = np.meshgrid(np.arange(w, dtype=np.float32), np.arange(h, dtype=np.float32))
    c = np.zeros((h, w, stride), np.float32)
    c[..., 0] = (u - cx) * d / fx * (1 + rng.normal(0, perturb, d.shape))
    c[..., 1] = (v - cy) * d / fy * (1 + rng.normal(0, perturb, d.shape))
    c[..., 2] = d
    c[np.isnan(d), :3] = np.nan
    if stride == 8:
        c[..., 4] = rng.integers(0, 1 << 24, d.shape).astype(np.uint32).view(np.float32)
    return c


def plant(rng, c, step, n_each=6):
    """Plant each special point kind n_each times on the sample grid of `step` (and as often off it)."""
    h, w = c.shape[:2]
    for kind in SPECIALS:
        for on_grid in (True, False):
            ys = rng.integers(0, (h - 1) // step + 1, n_each) * step if on_grid else rng.integers(0, h, n_each)
            xs = rng.integers(0, (w - 1) // step + 1, n_each) * step if on_grid else rng.integers(0, w, n_each)
            p = c[ys, xs]
            p[:, :3] = [0.3, -0.2, 2.0] if kind != "zero-z" else [0.0, 0.0, 0.0]
            if kind == "nan-z":
                p[:, 2] = np.nan
            elif kind == "nan-x":
                p[:, 0] = np.nan
            elif kind == "+inf-z":
                p[:, 2] = np.inf
            elif kind == "-inf-z":
                p[:, 2] = -np.inf
            elif kind == "neg-z":
                p[:, 2] = -1.5
            c[ys, xs] = p
    return c


def scenes():
    """(name, newer cloud, newerK, older cloud, olderK, T newer -> older, skip step, z0 or None for per-point)"""
    rng = np.random.default_rng(41)
    out = []
    T_small = ee.rigid(rng, 1.5, [0.03, -0.02, 0.04])
    T_big = ee.rigid(rng, 20.0, [0.3, 0.1, -0.2])
    for stride in (4, 8):
        a = make_cloud(rng, 640, 480, K_A, stride)
        b = make_cloud(rng, 640, 480, K_B, stride)
        for step in (1, 3, 8):
            an, bn = plant(rng, a.copy(), step), plant(rng, b.copy(), step)
            for z0 in (2.0, None):
                out.append((f"xyz{stride}/step{step}/z0-{z0}", an, K_A, bn, K_B, T_small, step, z0))
        out.append((f"xyz{stride}/big", a, K_A, b, K_A, T_big, 8, 2.0))
        out.append((f"xyz{stride}/K0", plant(rng, a.copy(), 8), K_0, plant(rng, b.copy(), 8), K_0, T_small, 8, 2.0))
        out.append((f"xyz{stride}/K0-per-point", plant(rng, a.copy(), 3), K_0, b, K_0, T_small, 3, None))
    # odd sizes (large enough for the Node constructor's grid); the same width with different heights; different widths
    # (both directions skipped)
    o1 = plant(rng, make_cloud(rng, 351, 347, K_S, 8), 3)
    o2 = plant(rng, make_cloud(rng, 351, 341, K_S, 8), 3)
    o3 = make_cloud(rng, 353, 347, K_S, 8)
    out.append(("odd/same-width", o1, K_S, o2, K_S, T_small, 3, 2.0))
    out.append(("odd/same-width-per-point", o2, K_S, o1, K_S, T_small, 1, None))
    out.append(("odd/other-width", o1, K_S, o3, K_S, T_small, 3, 2.0))
    return out


SCENES = scenes()


def _oracle(T, cn, Kn, co, Ko, step, z0):
    return ec.oracle_pairwise_cloud(T, cn, Kn, co, Ko, step, z0=z0)


def _restated(T, cn, Kn, co, Ko, step, z0):
    return ec.pairwise_cloud(T, cn, Kn, co, Ko, skip_step=step, czc=None if z0 is None else ee.cov_const(0.01, z0))


@pytest.mark.parametrize("scene", SCENES, ids=[s[0] for s in SCENES])
def test_cloud_restatement_equals_the_oracle(scene):
    name, cn, Kn, co, Ko, T, step, z0 = scene
    exp = _oracle(T, cn, Kn, co, Ko, step, z0)
    got = _restated(T, cn, Kn, co, Ko, step, z0)
    assert got["loose"].sum() == 0, name
    assert np.array_equal(got["counts"], exp), (name, got["counts"], exp)
    if name == "odd/other-width":
        assert list(exp) == [0, 0, 0, 0]
    elif name.endswith("K0"):
        assert exp[3] > 0 and exp[:3].sum() > 0, exp   # everything lands on pixel (0, 0)
    else:
        assert min(exp[:3]) > 0, (name, exp)           # good, bad and occluded samples all occur


def _single_point_clouds(kind, w=7, h=5):
    """A newer cloud whose only finite-ish point (sampled at (2, 2)) is of `kind`, an older cloud at 2 m everywhere."""
    cn = np.full((h, w, 4), np.nan, np.float32)
    p = {"nan-x": [np.nan, 0.1, 2.0], "+inf-z": [0.1, 0.1, np.inf], "inf-x-inf-z": [np.inf, 0.1, np.inf]}[kind]
    cn[2, 2, :3] = p
    co = np.zeros((h, w, 4), np.float32)
    co[..., 2] = 2.0
    return cn, co


@pytest.mark.parametrize("z0", [2.0, None])
def test_non_finite_points_as_the_reference_treats_them(z0):
    """A +inf z is kept untransformed and judged at (round(cx), round(cy)): bad with per-point covariance (NaN cdf
    argument), occluded with the latched one.  A NaN x with a finite z, and inf / inf, convert to INT_MIN and are skipped."""
    K = (100.0, 100.0, 3.4, 2.2)
    T = ee.rigid(np.random.default_rng(3), 2.0, [0.01, 0.02, 0.03])
    for kind, counts in (("+inf-z", [0, 1, 0] if z0 is None else [0, 0, 1]), ("nan-x", [0, 0, 0]), ("inf-x-inf-z", [0, 0, 0])):
        cn, co = _single_point_clouds(kind)
        got = ec.direction_cloud(T, cn, co, K, skip_step=1, czc=None if z0 is None else ee.cov_const(0.01, z0))
        assert list(got["counts"]) == counts + [35], (kind, got["counts"])
        exp = _oracle(T, cn, K, co, K, 1, z0)
        assert np.array_equal(ec.pairwise_cloud(T, cn, K, co, K, skip_step=1,
                                                czc=None if z0 is None else ee.cov_const(0.01, z0))["counts"], exp), kind


def test_stored_points_are_not_the_grid_back_projection():
    """Recomputing x / y from the pixel grid gives other counts on these clouds: the comparison above would catch it."""
    name, cn, Kn, co, Ko, T, step, z0 = SCENES[0]
    grid = cn.copy()
    fx, fy, cx, cy = Kn
    u, v = np.meshgrid(np.arange(cn.shape[1], dtype=np.float32), np.arange(cn.shape[0], dtype=np.float32))
    grid[..., 0] = (u - cx) * grid[..., 2] / fx
    grid[..., 1] = (v - cy) * grid[..., 2] / fy
    assert not np.array_equal(_oracle(T, grid, Kn, co, Ko, step, z0), _oracle(T, cn, Kn, co, Ko, step, z0))


# ---- both instantiations of the kernels keep the float chain uncontracted -------------------------------------------------

def _nvcc():
    for c in (shutil.which("nvcc"), "/usr/local/cuda/bin/nvcc"):
        if c and Path(c).exists():
            return c
    return None


def _fma_counts(ptx: str):
    """fma.rn.f32 / fma.rn.f64 counts of every instantiation of the two EMM kernels"""
    out = {}
    for m in re.finditer(r"\.entry\s+(\S*(?:k_emm_pairs|k_emm_single)\S*)\(.*?\n}\n", ptx, re.S):
        out[m.group(1)] = (m.group(0).count("fma.rn.f32"), m.group(0).count("fma.rn.f64"))
    return out


@pytest.mark.skipif(_nvcc() is None, reason="nvcc not available")
def test_emm_ptx_instantiations_have_no_contracted_fma(tmp_path):
    from rgbdslam_v2_b200.build import NVCC_FLAGS
    flags = [f for f in NVCC_FLAGS if f not in ("-shared", "-ldl", "-Xcompiler", "-fPIC")]
    src = ROOT / "rgbdslam_v2_b200" / "csrc" / "emm.cu"
    counts = []
    for extra in ([], ["--fmad=false"]):
        out = tmp_path / f"emm{len(extra)}.ptx"
        subprocess.run([_nvcc(), *flags, *extra, "-ptx", "-o", str(out), str(src)], check=True, capture_output=True)
        counts.append(_fma_counts(out.read_text()))
    assert len(counts[0]) == 4, counts[0]   # k_emm_pairs and k_emm_single, depth and kept-cloud sources
    assert counts[0] == counts[1], counts
