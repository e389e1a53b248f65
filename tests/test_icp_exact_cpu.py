"""The ICP restatement (tests/icp_exact.py): filterCloud's index walk against a literal transcription of icp.cpp:20-45, the
float32 ICP against an independent float64 ICP (cKDTree, np.linalg.svd Umeyama, the same stopping rules) on inputs whose
decisions are margin-certified, every stopping criterion on planted clouds, ties, non-finite points and reflections; and the
C ABI of rgbdslam_b200_icp_align as far as it can be checked without a GPU."""
import ctypes as C
import re
import shutil
import subprocess
from pathlib import Path

import numpy as np
import pytest
from scipy.spatial import cKDTree

import icp_exact as ix

F32 = np.float32
ROOT = Path(__file__).resolve().parent.parent


def _filter_literal(z, desired):
    """icp.cpp:20-45 as written: non-NaN indices, float step, float loop, (unsigned) index"""
    non_nan = [i for i in range(len(z)) if not np.isnan(z[i])]
    step = F32(F32(len(non_nan)) / F32(desired))
    step = F32(1.0) if step < 1.0 else step
    out = []
    i = F32(0.0)
    while i < F32(len(non_nan)):
        out.append(non_nan[int(i)])
        i = F32(i + step)
    return np.asarray(out, np.int64)


@pytest.mark.parametrize("n", [0, 1, 2, 3, 7, 640, 9999, 10000, 10001, 10002, 19999, 20001, 33333, 76800, 99991, 307200])
@pytest.mark.parametrize("desired", [1, 3, 10000, 400000])
def test_filter_walk_equals_the_literal_transcription(n, desired):
    rng = np.random.default_rng(n + desired)
    z = rng.uniform(0.5, 4.0, n).astype(F32)
    z[rng.random(n) < 0.1] = np.nan
    z[rng.random(n) < 0.01] = np.inf  # kept: only NaN is dropped
    if n > 20000 and desired == 1:  # the literal loop in Python is slow; the walk of desired 1 keeps index 0 or 0 and 1
        z = z[:20000]
    got = ix.filter_indices(z, desired)
    assert np.array_equal(got, _filter_literal(z, desired))
    m = int((~np.isnan(z)).sum())
    assert len(got) <= max(m, 0) and (m <= desired or len(got) in (desired, desired + 1) or len(got) > desired)


def test_filter_walk_can_keep_one_more_than_desired():
    extra = [(n, d) for d in (3, 7, 10000) for n in range(d + 1, 3 * d + 40, 1 if d < 100 else 97)
             if len(ix.filter_indices(np.zeros(n, F32), d)) == d + 1]
    assert extra, "no size keeps desired + 1 points"
    for n, d in extra[:5]:
        assert len(_filter_literal(np.zeros(n, F32), d)) == d + 1


# ---- an independent float64 ICP --------------------------------------------------------------------------------------------

def icp64(src, tgt, margin=1e-4):
    """float64 ICP with the same rules; asserts that every decision it takes is at least `margin` (metres) away from the
    threshold and from a tie, so that float32 arithmetic cannot take another one (margin None: no certification)"""
    src = src.astype(np.float64)
    tgt = tgt.astype(np.float64)
    tf = np.isfinite(tgt).all(0)
    tree = cKDTree(tgt[:, tf].T)
    tj = np.flatnonzero(tf)
    ws = src.copy()
    final = np.eye(4)
    prev, it, corr = np.finfo(np.float64).max, 0, []
    while True:
        fin = np.isfinite(ws).all(0)
        dd, k = tree.query(ws[:, fin].T, k=2)
        near = dd[:, 0]
        assert margin is None or (np.all(np.abs(near - 0.05) > margin) and np.all((dd[:, 1] - near > margin) | (near > 0.05)))
        j = np.full(ws.shape[1], -1)
        j[fin] = np.where(near <= 0.05, tj[k[:, 0]], -1)
        corr.append(j)
        ok = j >= 0
        n = int(ok.sum())
        if n < 3:
            return dict(criterion=0, iterations=it, corr=corr, T=np.eye(4))
        a, b = ws[:, ok], tgt[:, j[ok]]
        am, bm = a.mean(1, keepdims=True), b.mean(1, keepdims=True)
        U, _, Vt = np.linalg.svd((b - bm) @ (a - am).T / n)
        S = np.eye(3)
        if np.linalg.det(U) * np.linalg.det(Vt) < 0:
            S[2, 2] = -1
        R = U @ S @ Vt
        T = np.eye(4)
        T[:3, :3], T[:3, 3] = R, (bm - R @ am)[:, 0]
        ws = np.where(np.isfinite(ws).all(0), R @ ws + T[:3, 3:], ws)
        final = T @ final
        it += 1
        mse = float(np.sum(np.sum((a - b) ** 2, 0)) / n)
        tr = float(np.sqrt(T[:3, 3] @ T[:3, 3]))
        ang = float(np.arccos(np.clip(0.5 * (np.trace(R) - 1), -1.0, 1.0)))
        if it >= 50:
            c = 1
        elif tr <= 1e-4 and ang < 1.4e-4:
            c = 2
        elif abs(mse - prev) < 1e-12:
            c = 3
        elif abs(mse - prev) / prev < 1:
            c = 4
        else:
            # going on must be certain: in float the rotation rule holds whenever the trace rounds to 3 (below about 3e-4
            # rad, or above that through the rounding of R), so the translation or the angle must rule it out clearly
            assert margin is None or tr > 1.2e-4 or ang > 5e-4
            prev = mse
            continue
        return dict(criterion=c, iterations=it, corr=corr, T=final)


def _rot(axis, ang):
    a = np.asarray(axis, float) / np.linalg.norm(axis)
    K = np.array([[0, -a[2], a[1]], [a[2], 0, -a[0]], [-a[1], a[0], 0]])
    return np.eye(3) + np.sin(ang) * K + (1 - np.cos(ang)) * K @ K


def _scene(seed, n_side=10, outliers=20):
    """a jittered 0.2 m grid (nearest neighbours unique by far) and the same points moved by up to 1 cm / 0.6 degrees with
    1 mm noise, and outliers further than 0.1 m from every target"""
    rng = np.random.default_rng(seed)
    g = np.stack(np.meshgrid(np.arange(n_side), np.arange(n_side), np.arange(4)), -1).reshape(-1, 3) * 0.2
    tgt = (g + rng.uniform(-0.02, 0.02, g.shape)).T
    R = _rot(rng.normal(size=3), rng.uniform(0.002, 0.01))
    src = R @ tgt + rng.uniform(-0.01, 0.01, (3, 1)) + rng.normal(0, 0.001, tgt.shape)
    out = g[rng.choice(len(g), outliers, replace=False)].T + 0.1
    src = np.concatenate([src, out], 1)[:, rng.permutation(src.shape[1] + outliers)]
    return src.astype(F32), tgt.astype(F32)


@pytest.mark.parametrize("seed", range(8))
def test_restatement_agrees_with_a_float64_icp(seed):
    src, tgt = _scene(seed)
    r32 = ix.align_points(src, tgt)
    r64 = icp64(src, tgt)
    # both stop at the same iteration; whether the transform rule or the relative MSE rule stops them is not certain in float
    assert r32["criterion"] == r64["criterion"] or {r32["criterion"], r64["criterion"]} <= {2, 4}
    assert r32["iterations"] == r64["iterations"] >= 2
    assert len(r32["corr"]) == len(r64["corr"]) and all(np.array_equal(a, b) for a, b in zip(r32["corr"], r64["corr"]))
    assert np.abs(r32["T"].astype(np.float64) - r64["T"]).max() < 1e-5


def test_stopping_criteria_on_planted_clouds():
    src, tgt = _scene(2)
    assert ix.align_points(src, tgt)["criterion"] == 4
    far = (tgt + F32(0.5)).astype(F32)  # more than 5 cm from every target: no correspondence
    r = ix.align_points(far, tgt)
    assert (r["criterion"], r["converged"], r["iterations"], r["n_correspondences"]) == (0, 0, 0, 0)
    assert np.array_equal(r["T"], np.eye(4, dtype=F32)) and r["mse"] == 0.0
    assert ix.align_points(src[:, :2], tgt)["criterion"] == 0  # two points cannot make three correspondences
    # identical clouds: T_inc is the identity up to rounding
    r = ix.align_points(tgt, tgt)
    assert (r["criterion"], r["iterations"], r["mse"]) == (2, 1, 0.0) and np.abs(r["T"] - np.eye(4)).max() < 1e-6
    # identical clouds 10 km away: T_inc's rounding leaves a translation above 1e-4 m, the MSE stays 0
    rng = np.random.default_rng(1)
    p = (rng.uniform(-0.3, 0.3, (3, 40)) + 1e4).astype(F32)
    r = ix.align_points(p, p)
    assert (r["criterion"], r["iterations"]) == (3, 2)
    # the iteration limit: the restatement's limit lowered, since PCL 1.7's relative rule normally stops at iteration 2
    for k in (1, 2):
        r = ix.align_points(src, tgt, max_iterations=k)
        assert (r["criterion"], r["iterations"], r["converged"]) == (1, k, 1)
    r1, r50 = ix.align_points(src, tgt, max_iterations=1), ix.align_points(src, tgt)
    assert np.array_equal(r1["corr"][0], r50["corr"][0])


def tie_clouds():
    """four source points, each exactly equidistant (dyadic coordinates) from two targets 1/32 m apart along x; the lower
    index of each pair comes first in pairs 2 and 4 and second in pairs 1 and 3"""
    h = 1.0 / 64
    tx = [2 * h, 0.0, 0.5, 0.5 + 2 * h, 2 * h, 0.0, 1.0, 1.0 + 2 * h]
    tgt = np.array([tx, [0.0, 0.0, 0.0, 0.0, 0.5, 0.5, 1.0, 1.0], [1.0] * 8], F32)
    src = np.array([[h, 0.5 + h, h, 1.0 + h], [0.0, 0.0, 0.5, 1.0], [1.0] * 4], F32)
    return src, tgt


def test_ties_go_to_the_lowest_target_index():
    src, tgt = tie_clouds()
    idx, dist = ix.nearest(src, tgt)
    assert list(idx) == [0, 2, 4, 6] and np.all(dist == F32(1.0 / 64) ** 2)
    r = ix.align_points(src, tgt)
    assert list(r["corr"][0]) == [0, 2, 4, 6]


def test_non_finite_points_take_no_part():
    src, tgt = _scene(3)
    src2, tgt2 = src.copy(), tgt.copy()
    src2[0, 5] = np.inf
    src2[1, 9] = np.nan
    src2[2, 11] = -np.inf
    tgt2 = np.concatenate([tgt2, np.array([[np.nan, np.inf, 0.0], [0.0, 0.0, -np.inf], [1.0, 1.0, np.inf]], F32)], 1)
    r = ix.align_points(src2, tgt2)
    assert r["n_source"] == src.shape[1] and r["n_target"] == tgt.shape[1] + 3
    for k in (5, 9, 11):
        assert all(c[k] == -1 for c in r["corr"])
    assert all(np.all(c < tgt.shape[1]) for c in r["corr"])
    # the finite points' decisions equal those of the clouds without the non-finite points
    keep = np.setdiff1d(np.arange(src.shape[1]), [5, 9, 11])
    r0 = ix.align_points(src[:, keep], tgt)
    assert r["criterion"] == r0["criterion"] and np.array_equal(r["corr"][0][keep], r0["corr"][0])


def test_reflection_correlations_take_the_proper_rotation():
    # sigma of mirrored point sets has det < 0: S_3 = -1 keeps R a rotation
    rng = np.random.default_rng(5)
    a = rng.normal(size=(3, 30)).astype(F32)
    b = (np.diag([1.0, 1.0, -1.0]) @ a).astype(F32)
    T = ix.umeyama(a, b, np.ones(30, bool))
    R = T[:3, :3].astype(np.float64)
    assert abs(np.linalg.det(R) - 1.0) < 1e-5 and np.abs(R.T @ R - np.eye(3)).max() < 1e-5
    U, s, V = ix.svd3(np.asarray([[F32(x) for x in row] for row in (b @ a.T / 30)], F32))
    assert s[0] >= s[1] >= s[2] >= 0


def test_svd_reconstructs_its_input():
    rng = np.random.default_rng(7)
    for _ in range(50):
        A = rng.normal(size=(3, 3)).astype(F32)
        U, s, V = ix.svd3(A)
        Uf, Vf = np.array(U, np.float64), np.array(V, np.float64)
        assert np.abs(Uf @ np.diag(np.array(s, np.float64)) @ Vf.T - A).max() < 1e-5
        assert np.abs(Uf.T @ Uf - np.eye(3)).max() < 1e-5 and np.abs(Vf.T @ Vf - np.eye(3)).max() < 1e-5
        assert list(s) == sorted(s, reverse=True)


# ---- C ABI --------------------------------------------------------------------------------------------------------------------

def test_icp_result_layout_matches_the_header():
    from rgbdslam_v2_b200 import _capi
    txt = (ROOT / "include" / "rgbdslam_b200" / "icp.h").read_text()
    body = re.search(r"typedef struct rgbdslam_b200_icp_result \{(.*?)\}", txt, re.S).group(1)
    body = re.sub(r"/\*.*?\*/", "", body, flags=re.S)
    names = [n for line in body.split(";") for n in re.findall(r"(\w+)(?:\[\d+\])?\s*(?:,|$)", line.strip())]
    assert names == [f[0] for f in _capi.IcpResult._fields_] == list(_capi.ICP_RESULT_DTYPE.names)
    for f in _capi.IcpResult._fields_:
        assert getattr(_capi.IcpResult, f[0]).offset == _capi.ICP_RESULT_DTYPE.fields[f[0]][1]
    assert C.sizeof(_capi.IcpResult) == 96


def test_icp_align_is_exported_and_refuses_before_init(built):
    from rgbdslam_v2_b200._capi import ICP_RESULT_DTYPE, load_library
    lib = load_library()
    assert hasattr(lib, "rgbdslam_b200_icp_align")
    import torch
    if torch.cuda.is_available():
        pytest.skip("GPU present: the library may already be initialised in this process")
    out = np.zeros(1, ICP_RESULT_DTYPE)
    h = np.zeros(1, np.uint64)
    assert lib.rgbdslam_b200_icp_align(1, h.ctypes.data, h.ctypes.data, 10000, out.ctypes.data) == 3  # ERR_STATE
    assert b"init" in lib.rgbdslam_b200_last_error()


def _nvcc():
    for c in (shutil.which("nvcc"), "/usr/local/cuda/bin/nvcc"):
        if c and Path(c).exists():
            return c
    return None


PTX_OPS = ("fma.rn.f32", "fma.rn.f64", "mul.rn.f32", "add.rn.f32", "sub.rn.f32", "div.rn.f32", "sqrt.rn.f32", "mul.rn.f64",
           "add.rn.f64", "sub.rn.f64", "div.rn.f64")


def _kernel_ops(ptx):
    """{kernel: op counts} of the k_icp_* entries; the align kernel is named by its estimator, as align<IcpSvd>"""
    out = {}
    for m in re.finditer(r"\.entry\s+(\S*k_icp_\S*)\(.*?\n}\n", ptx, re.S):
        k = re.search(r"k_icp_(filter|cells|align)(?:INS_\d+(\w+?)EE)?", m.group(1))
        out[k.group(1) + (f"<{k.group(2)}>" if k.group(2) else "")] = tuple(m.group(0).count(op) for op in PTX_OPS)
    return out


@pytest.mark.skipif(_nvcc() is None, reason="nvcc not available")
def test_icp_ptx_has_no_contracted_or_approximate_operations(tmp_path):
    """both ICP sources: every k_icp_* entry has no fma, the same operations under --fmad=false, and no approximate
    operation; the entries are filterCloud, the cells and one align kernel per estimator"""
    from rgbdslam_v2_b200.build import NVCC_FLAGS
    flags = [f for f in NVCC_FLAGS if f not in ("-shared", "-ldl", "-Xcompiler", "-fPIC")]
    entries = {"icp.cu": {"filter", "cells", "align<IcpSvd>"}, "icp_nl.cu": {"align<IcpLm>"}}
    for name, expected in entries.items():
        src = ROOT / "rgbdslam_v2_b200" / "csrc" / name
        counts, texts = [], []
        for extra in ([], ["--fmad=false"]):
            out = tmp_path / f"{name}{len(extra)}.ptx"
            subprocess.run([_nvcc(), *flags, *extra, "-ptx", "-o", str(out), str(src)], check=True, capture_output=True)
            texts.append(out.read_text())
            counts.append(_kernel_ops(texts[-1]))
        assert set(counts[0]) == expected and len(re.findall(r"\.entry", texts[0])) == len(expected), (name, counts[0])
        assert counts[0] == counts[1], (name, counts)
        assert all(c[0] == c[1] == 0 for c in counts[0].values()), (name, counts[0])
        assert not re.search(r"\b(rcp|rsqrt|sqrt\.approx|div\.approx|div\.full|ex2|lg2)\b", texts[0]), name
