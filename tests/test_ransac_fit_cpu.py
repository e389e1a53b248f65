"""CPU tests of the RANSAC rigid fit's restatements (tests/ransac_exact.py): the float64 weighted Kabsch `kabsch_f64`, the
case families `fit_cases` at the fit's conditioning edges, and the error bound `fit_bound`, which the float32 emulation of
the kernel's fit (`fit_f32`) must meet with 8x headroom on every family.  tests/test_gpu_ransac_fit.py holds the kernel
itself to the same bound."""
import numpy as np
import pytest

import ransac_exact as rx

CASES = rx.fit_cases()
FAMILIES = sorted({c["family"] for c in CASES})
HEADROOM = 8.0


def test_kabsch_f64_direction_on_a_planted_pair(oracle_mod):
    """kabsch_f64(frm, to) maps from (query / newer side) onto to (train / older side), as get_transform_from_matches and
    the returned ransac_trafo do."""
    rng = np.random.default_rng(5)
    P = rx.frustum_points(rng, 30, 1.0, 3.0)
    T = np.eye(4)
    T[:3, :3] = rx.rot_axis(rx.OBLIQUE, 25.0)
    T[:3, 3] = [0.3, -0.2, 0.4]
    frm, to = rx.to4(P), rx.to4(P @ T[:3, :3].T + T[:3, 3])
    R, t, s, d = rx.kabsch_f64(frm, to)
    assert np.abs(R - T[:3, :3]).max() < 1e-6 and np.abs(t - T[:3, 3]).max() < 1e-6 and d == 1
    m = np.zeros(len(P), oracle_mod.DMATCH_DTYPE)
    m["queryIdx"] = m["trainIdx"] = np.arange(len(P))
    To = oracle_mod.get_transform_from_matches(frm, to, m)
    assert np.abs(To[:3, :3] - R).max() < 5e-5 and np.abs(To[:3, 3] - t).max() < 5e-5


def test_kabsch_f64_skips_nan_depth_rows():
    rng = np.random.default_rng(6)
    P = rx.frustum_points(rng, 12, 1.0, 3.0)
    frm, to = rx.to4(P), rx.to4(P @ rx.rot_axis((0, 1, 0), 10.0).T + 0.1)
    ref = rx.kabsch_f64(frm[3:], to[3:])
    frm[0, 2] = np.nan
    to[1, 2] = np.nan
    frm[2, 2] = to[2, 2] = np.nan
    got = rx.kabsch_f64(frm, to)
    assert np.array_equal(got[0], ref[0]) and np.array_equal(got[1], ref[1])
    sub = rx.kabsch_f64(frm, to, np.arange(6))
    assert np.array_equal(sub[0], rx.kabsch_f64(frm[3:6], to[3:6])[0])


def test_fit_bound_constant():
    """K = 2 (ceil(M/32) + 5 + 118) + 60: fixed by the operation counts of the module docstring, not fitted."""
    assert rx.fit_K(4) == 2 * (1 + 5 + 118) + 60
    assert rx.fit_K(32) == rx.fit_K(4) and rx.fit_K(33) == rx.fit_K(4) + 2 and rx.fit_K(512) == 2 * (16 + 5 + 118) + 60


def test_fit_cases_are_built_as_intended():
    by = {}
    for c in CASES:
        by.setdefault(c["family"], []).append(c)
        assert np.nanmin(c["to"][:, 2]) >= 0.3 and np.nanmin(c["frm"][:, 2]) >= 0.3, c["name"]
    assert set(by) == {"trivial", "rotation", "coplanar", "reflection", "collinear", "isotropic", "scale", "weights", "nan", "M"}
    for c in by["coplanar"]:  # rank 2 on the from side: s3 is rounding
        _, _, s, _ = rx.kabsch_f64(c["frm"], c["to"])
        assert s[2] < 1e-6 * s[0], c["name"]
    assert any(c["name"].endswith("180-M4") for c in by["coplanar"]) and any("normal" in c["name"] for c in by["coplanar"])
    for c in by["reflection"]:
        assert rx.kabsch_f64(c["frm"], c["to"])[3] == -1, c["name"]
    for c in by["collinear"]:
        spread = float(c["name"].split("-")[0][5:])
        _, _, s, _ = rx.kabsch_f64(c["frm"], c["to"])
        assert s[1] < spread * s[0], c["name"]
    for c in by["isotropic"]:
        _, _, s, _ = rx.kabsch_f64(c["frm"], c["to"])
        if c["name"].startswith("square"):
            assert s[1] > 0.999 * s[0] and s[2] < 1e-9 * s[0], c["name"]
        else:
            assert s[2] > 0.75 * s[0], c["name"]
    sizes = {c["name"].split("-")[0] for c in by["scale"]}
    assert {"0.0001m", "0.0003m", "0.001m", "0.01m", "10m", "2cm"} <= sizes
    for c in by["weights"]:
        for x in (c["frm"], c["to"]):
            assert x[:, 2].min() < 0.35 and x[:, 2].max() > 14.0, c["name"]
    assert {c["name"] for c in by["nan"]} == {"nan-from", "nan-to", "nan-both"}
    assert sorted(c["M"] for c in by["M"]) == [4, 5, 31, 32, 33, 63, 64, 65, 300, 320, 321, 512]


@pytest.mark.parametrize("family", FAMILIES)
def test_fit_f32_inside_the_bound(family):
    """The float32 emulation of the kernel's fit over every finite row of each case sits at least 8x inside the bound: the
    bound has headroom over the arithmetic it describes, so a kernel outside it computes something else."""
    for c in (c for c in CASES if c["family"] == family):
        ref = rx.fit_bound(c["frm"], c["to"])
        R, t, ok = rx.fit_f32(c["frm"], c["to"], np.arange(c["M"]))
        assert ok, c["name"]
        eR, et, shape = rx.fit_errors(R, t, ref)
        assert eR * HEADROOM <= ref["rot"], (c["name"], eR, ref["rot"])
        assert et * HEADROOM <= ref["trans"], (c["name"], et, ref["trans"])
        assert shape * HEADROOM <= rx.SHAPE_TOL, (c["name"], shape)


def test_fit_f32_sees_a_short_sweep_cap():
    """The bound is not vacuous for the Jacobi: cut to 2 sweeps, the emulated fit leaves it on a well-conditioned case."""
    worst = 0.0
    for c in CASES:
        if c["family"] != "rotation":
            continue
        ref = rx.fit_bound(c["frm"], c["to"])
        R, t, ok = rx.fit_f32(c["frm"], c["to"], np.arange(c["M"]), sweeps=2)
        worst = max(worst, rx.fit_errors(R, t, ref)[0] / ref["rot"])
    assert worst > 1.0, worst
