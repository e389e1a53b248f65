"""The numpy restatement of the environment measurement model (tests/emm_exact.py) against the C oracle
(oracle/emm_oracle.c), and a PTX check that csrc/emm.cu keeps the reference's uncontracted float chain."""
import re
import shutil
import subprocess
from pathlib import Path

import numpy as np
import pytest

import emm_exact as ee

ROOT = Path(__file__).resolve().parent.parent
K_A = (525.0, 525.0, 319.5, 239.5)
K_B = (481.2, 479.7, 305.25, 251.5)


def scenes():
    """(name, newer depth, newerK, older depth, olderK, T newer -> older, config) across frame sizes, intrinsics, steps,
    scalings, minimum depths, covariance regimes and transforms that put points behind the camera or off the raster."""
    rng = np.random.default_rng(31)
    out = []
    d_a = ee.block_scene(rng, 640, 480, K_A)
    d_b = ee.block_scene(rng, 517, 389, K_B)
    d_c = ee.block_scene(rng, 333, 250, (300.0, 301.0, 166.0, 124.5))
    T_small = ee.rigid(rng, 1.5, [0.03, -0.02, 0.04])
    T_big = ee.rigid(rng, 25.0, [0.4, 0.1, -0.3])
    T_back = np.diag([-1.0, 1.0, -1.0, 1.0]).astype(np.float32)  # rotated 180 deg about y: everything behind the camera
    T_back[:3, 3] = [0.0, 0.0, 1.5]                               # ... except what the translation brings back
    T_off = ee.rigid(rng, 0.5, [2.5, 0.0, 0.0])                   # most points leave the raster
    cfg = dict(cloud_step=2, skip_step=8, scaling=1.0, min_depth=0.1, z0=2.0)
    for T, tn in ((T_small, "small"), (T_big, "big"), (T_back, "behind"), (T_off, "off-raster")):
        out.append((f"same-K/{tn}", d_a, K_A, d_a, K_A, T, cfg))
        out.append((f"other-K/{tn}", d_a, K_A, d_b, K_B, T, cfg))
        out.append((f"other-K-rev/{tn}", d_b, K_B, d_c, (300.0, 301.0, 166.0, 124.5), T, cfg))
    for steps in ((3, 5), (1, 7), (4, 3)):
        out.append((f"steps{steps}", d_b, K_B, d_a, K_A, T_small, dict(cfg, cloud_step=steps[0], skip_step=steps[1])))
    out.append(("scaling", (d_a * 1000).astype(np.float32), K_A, (d_b * 1000).astype(np.float32), K_B, T_small,
                dict(cfg, scaling=0.001)))
    out.append(("min-depth", d_a, K_A, d_b, K_B, T_small, dict(cfg, min_depth=1.7)))
    out.append(("per-point", d_a, K_A, d_b, K_B, T_small, dict(cfg, z0=None)))
    out.append(("per-point/steps", d_b, K_B, d_c, (300.0, 301.0, 166.0, 124.5), T_big, dict(cfg, z0=None, cloud_step=3,
                                                                                                skip_step=5)))
    out.append(("latched-z0", d_a, K_A, d_b, K_B, T_small, dict(cfg, z0=float(np.float32(3.1379)))))
    return out


SCENES = scenes()


def _oracle_counts(oracle_mod, T, dn, Kn, do, Ko, cfg):
    prm = oracle_mod.make_params(depth_cov_z0=cfg["z0"] if cfg["z0"] is not None else -1.0)
    zn = oracle_mod.create_cloud_z(dn, cfg["cloud_step"], cfg["scaling"], cfg["min_depth"])
    zo = oracle_mod.create_cloud_z(do, cfg["cloud_step"], cfg["scaling"], cfg["min_depth"])
    return zn, zo, oracle_mod.pairwise_observation(prm, T, zn, Kn, zo, Ko, cfg["cloud_step"], cfg["skip_step"])


@pytest.mark.parametrize("scene", SCENES, ids=[s[0] for s in SCENES])
def test_restatement_equals_the_oracle(oracle_mod, scene):
    name, dn, Kn, do, Ko, T, cfg = scene
    zn, zo, exp = _oracle_counts(oracle_mod, T, dn, Kn, do, Ko, cfg)
    assert np.array_equal(zn, ee.cloud_z(dn, cfg["cloud_step"], cfg["scaling"], cfg["min_depth"]), equal_nan=True)
    assert np.array_equal(zo, ee.cloud_z(do, cfg["cloud_step"], cfg["scaling"], cfg["min_depth"]), equal_nan=True)
    czc = None if cfg["z0"] is None else ee.cov_const(0.01, cfg["z0"])
    got = ee.pairwise(T, zn, Kn, zo, Ko, cloud_step=cfg["cloud_step"], skip_step=cfg["skip_step"], czc=czc)
    assert got["loose"].sum() == 0, name
    assert np.array_equal(got["counts"], exp.astype(np.int64)), (name, got["counts"], exp)
    if name.startswith("same-K/small") or name.startswith("steps"):
        assert min(got["counts"][:3]) > 0, (name, got["counts"])   # every category is reached
    if "behind" in name or "off-raster" in name:
        assert got["counts"][:3].sum() < 0.5 * got["counts"][3], (name, got["counts"])


def test_restatement_reaches_projection_boundaries(oracle_mod):
    """Shift a scene by sub-cell translations so that samples land on both sides of many floor(x + 0.5) boundaries: the
    restatement's float chain stays count for count with the oracle's."""
    rng = np.random.default_rng(5)
    d = ee.block_scene(rng, 640, 480, K_A, holes=0.0)
    cfg = dict(cloud_step=2, skip_step=8, scaling=1.0, min_depth=0.1, z0=2.0)
    for dx in np.linspace(0.0, 0.01, 9):
        T = ee.rigid(rng, 0.2, [dx, 0.5 * dx, 0.0])
        zn, zo, exp = _oracle_counts(oracle_mod, T, d, K_A, d, K_A, cfg)
        got = ee.pairwise(T, zn, K_A, zo, K_A, czc=ee.cov_const(0.01, 2.0))
        assert np.array_equal(got["counts"], exp.astype(np.int64)), (dx, got["counts"], exp)


# ---- the kernels keep the float chain uncontracted ------------------------------------------------------------------------

def _nvcc():
    for c in (shutil.which("nvcc"), "/usr/local/cuda/bin/nvcc"):
        if c and Path(c).exists():
            return c
    return None


def _fma_counts(ptx: str):
    """fma.rn.f32 / fma.rn.f64 counts per entry point of the two EMM kernels"""
    out = {}
    for name in ("k_emm_pairs", "k_emm_single"):
        m = re.search(r"\.entry\s+\S*" + name + r"\S*\(.*?\n}\n", ptx, re.S)
        assert m, name
        body = m.group(0)
        out[name] = (body.count("fma.rn.f32"), body.count("fma.rn.f64"))
    return out


@pytest.mark.skipif(_nvcc() is None, reason="nvcc not available")
def test_emm_ptx_has_no_contracted_fma(tmp_path):
    """nvcc contracts a * b + c into an FMA unless told otherwise; the reference's float transform, projection and cofactor
    inverse round every product.  The EMM kernels compiled with the default --fmad=true must therefore contain exactly the
    FMAs of a --fmad=false build (the ones erf and the float64 division use on purpose)."""
    from rgbdslam_v2_b200.build import NVCC_FLAGS
    flags = [f for f in NVCC_FLAGS if f not in ("-shared", "-ldl", "-Xcompiler", "-fPIC")]
    src = ROOT / "rgbdslam_v2_b200" / "csrc" / "emm.cu"
    counts = []
    for extra in ([], ["--fmad=false"]):
        out = tmp_path / f"emm{len(extra)}.ptx"
        subprocess.run([_nvcc(), *flags, *extra, "-ptx", "-o", str(out), str(src)], check=True, capture_output=True)
        counts.append(_fma_counts(out.read_text()))
    assert counts[0] == counts[1], counts
