"""The pose-graph solve (`csrc/posegraph.cu`) one LM iteration at a time against the C oracle's trace
(`oracle.posegraph_lm_trace`, the float64 LM + block-Jacobi PCG of `oracle/posegraph_oracle.c`), on both PCG kernels
(`pg_pcg_kernel`, `RB200_PG_RESIDENT=0`, and `pg_pcg_resident_kernel`, `=1`) at the shapes where their indexing changes: fewer
vertices than CTAs, one and two vertices per CTA, 16 / 17 / 79 / 80 vertices per CTA (80 x SM count is the last graph the
resident kernel takes; one more vertex and the host must pick the general kernel), a CTA whose incidences end just below, at
and just above the 568 it stages in shared memory, hubs whose incidences spill to global memory, fixed vertices at CTA edges,
Huber-active and duplicate edges, and an ill-conditioned chain whose LM rejects trials.

Every LM iteration starts from the oracle's poses (`stop=1` runs exactly one iteration on both sides, with fresh lambda and
`_residual`), so differences do not compound.  Per iteration:

- PCG counts.  The GPU's `cg_iters` equals the oracle's total over the iteration's trials when every stop is certified (and
  the total is at most EXACT_PCG; longer solves within LONG_PCG_REL of it, see there): the
  r'M^-1 r sequence of every trial stays more than 1e-6 relative above the tolerance (max(1e-6, _residual)) until the stop, and
  at the stop it is more than 1e-6 relative below it (or the stop is the iteration cap).  The LM decisions must be certified
  too (|rho| > 1e-6 and the trial chi2 more than 1e-9 relative from the current one, as in the landmark BA's exact test), else
  the trial count itself may differ.  Uncertified iterations are counted and reported; they must be a small minority.
- Step.  Both PCGs run the same recurrence to the same stopping index on the same system (the GPU's `q = A s + beta q` form is
  the textbook `q = A d` in exact arithmetic).  Each iterate lies within |dx_pcg - dx_direct| of the direct solution of
  (H + lambda I) dx = b up to its own rounding, so the two iterates lie within 2 |dx_pcg - dx_direct| of each other; the
  residual the stop admits and two summation orders (CSR order on the device, edge order in the oracle) at most double that,
  and a final factor 2 covers the Krylov sequences drifting apart by rounding over hundreds of iterations: 8 |dx_pcg -
  dx_direct| (max norm).  1e-12 |dx| is the rounding of the recurrences themselves when the PCG error is below it.  Near the
  optimum b is a small difference of large sums and its rounding decides how far two evaluations of the step may lie apart:
  every entry of b and H is a sum of at most n terms (the vertex's incidences) with a few roundings each, so another order
  moves it by at most (n + 8) eps sum|terms|; with H positive semi-definite (a sum of J'wWJ, w > 0) the smallest eigenvalue of
  H + lambda I is at least lambda, so the step moves by at most |(n + 8) eps (babs + |A| |dx|)|_2 / lambda.  That floor is
  added as it is.  A step difference bc (max norm) moves t + R dt and q * (v, sqrt(1 - |v|^2)) by at most 2 bc, plus a few ulps
  of the poses: the pose bound of the landmark BA's exact test.  The same bound holds between the two kernels.
- Fixed vertices are bit-identical to the input.
- chi2.  `graph_chi2` of the GPU poses equals the oracle's chi2 of the same poses to 1e-12 relative, plus the rounding of
  the residuals near zero (chi2_floor).
"""
import functools

import numpy as np
import pytest
import scipy.sparse.linalg as spla

from oracle import oracle as co
from rgbdslam_v2_b200 import _capi, synth

pytestmark = pytest.mark.gpu

EPS = np.finfo(np.float64).eps
CERT_BAND = 1e-6
RHO_BAND = 1e-6
CHI2_BAND = 1e-9
CAP_MAX = (200 * 1024 - 128) // 360  # incidences a CTA of the resident kernel stages in shared memory (posegraph.cu): 568
RES_VPC = 80                         # vertices per CTA of the resident kernel: 16 warps x 5 groups of 6 lanes
# Past a few hundred iterations two float64 PCGs in different summation orders lose the exact stopping index even where the
# oracle's r'M^-1 r sequence is certified: their sequences drift apart by more than 1e-6 relative.  Measured on an H100 SXM
# (700 W): off by 1-5 iterations in 300-550 on the well-conditioned graphs, where every iteration of at most 200 PCG steps
# matched exactly.  On the chain with weights over twelve decades the stopping index is decided by rounding (18 in 280, 4 in
# 101, 13 in 83): its PCG counts are not compared, its steps, chi2 and fixed vertices are.
EXACT_PCG = 200
LONG_PCG_REL = 0.1


@pytest.fixture(scope="module")
def fe(oracle_mod):
    f = _capi.Frontend(0)
    yield f
    f.close()


@functools.lru_cache(maxsize=None)
def sm_count():
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


# ---- graphs -------------------------------------------------------------------------------------------------------
def _graph(nv, extra=(), fixed=(0,), seed=0, chain=True, isolated=(), loops=0, outliers=(), duplicates=0, weights=(20.0, 300.0),
           trans_noise=0.01, rot_noise_deg=0.5, init_trans=0.03, init_rot_deg=1.5):
    """nv poses along a looping trajectory, the odometry chain (i, i + 1) without the `isolated` vertices, `loops` local loop
    closures 2..8 apart, the `extra` edges, `duplicates` copies of random edges; measurements are the ground-truth relative poses
    with noise, `outliers` (edge indices) carry 0.5 m more (Huber-active); information isotropic, weight U[weights]; the
    initial poses are the ground truth perturbed (fixed vertices too: they must not move)."""
    rng = np.random.default_rng(seed)
    s = np.linspace(0, 5 * np.pi, max(nv, 2))[:nv]
    pos = np.stack([3 * np.cos(s), 2 * np.sin(s), 0.3 * np.sin(3 * s)], 1)
    yaw = s + np.pi / 2
    gt = np.concatenate([pos, np.stack([np.zeros(nv), np.zeros(nv), np.sin(yaw / 2), np.cos(yaw / 2)], 1)], 1)
    iso = set(isolated)
    ij = [(i, i + 1) for i in range(nv - 1) if chain and i not in iso and i + 1 not in iso]
    ij += [(i - 1, i + 1) for i in sorted(iso) if 0 < i < nv - 1 and i - 1 not in iso and i + 1 not in iso]
    cand = [v for v in range(nv) if v not in iso]
    for _ in range(loops):
        a = int(rng.choice(cand))
        b = a + int(rng.integers(2, 9))
        if b < nv and b not in iso:
            ij.append((a, b) if rng.random() < 0.5 else (b, a))
    ij += [tuple(map(int, e)) for e in extra]
    if duplicates:
        ij += [ij[k] for k in rng.integers(0, len(ij), duplicates)]
    ij = np.array(ij, np.int32).reshape(-1, 2)
    ne = len(ij)
    rel = synth.pose_compose(synth.pose_inverse(gt[ij[:, 0]]), gt[ij[:, 1]]) if ne else np.zeros((0, 7))
    meas = synth.pose_compose(rel, _noise(rng, ne, trans_noise, rot_noise_deg)) if ne else rel
    if len(outliers):
        meas[list(outliers), :3] += rng.normal(0, 0.5, (len(outliers), 3))
    info = np.zeros((ne, 36))
    info[:, ::7] = rng.uniform(*weights, ne)[:, None]
    init = synth.pose_compose(gt, _noise(rng, nv, init_trans, init_rot_deg))
    fx = np.zeros(nv, np.uint8)
    fx[list(fixed)] = 1
    return dict(init=init, fixed=fx, ij=ij, meas=meas, info=info)


def _noise(rng, n, trans, rot_deg):
    ax = rng.normal(size=(n, 3))
    ax /= np.linalg.norm(ax, axis=1, keepdims=True)
    ang = np.deg2rad(rot_deg) * rng.normal(size=n)
    return np.concatenate([rng.normal(size=(n, 3)) * trans, ax * np.sin(ang / 2)[:, None], np.cos(ang / 2)[:, None]], 1)


def _spread(rng, v, n, nv, avoid):
    """n edges between v and vertices drawn from all others but `avoid`, v in both roles"""
    others = np.array([u for u in range(nv) if u not in avoid and u != v])
    us = rng.choice(others, n, replace=n > len(others))
    return [(v, int(u)) if k % 2 == 0 else (int(u), v) for k, u in enumerate(us)]


def _cta_incidences(nv, ij, vpc, cta):
    deg = np.bincount(ij.reshape(-1), minlength=nv)
    return int(deg[cta * vpc:min(nv, (cta + 1) * vpc)].sum())


def _cap_case(G, total):
    """vpc = 4: CTA 1 (vertices 4..7) holds exactly `total` incidences; vertex 7 (the CTA's last) owns most of the extra edges,
    so the capacity of 568 falls inside its incidence range"""
    nv, vpc = 4 * G, 4
    rng = np.random.default_rng(total)
    base = _graph(nv, loops=nv, seed=total)
    have = _cta_incidences(nv, base["ij"], vpc, 1)
    n_extra = total - have
    extra = _spread(rng, 5, n_extra // 4, nv, range(4, 8)) + _spread(rng, 7, n_extra - n_extra // 4, nv, range(4, 8))
    g = _graph(nv, loops=nv, seed=total, extra=extra, fixed=(0, 4))
    assert _cta_incidences(nv, g["ij"], vpc, 1) == total
    deg = np.bincount(g["ij"].reshape(-1), minlength=nv)
    assert deg[4:7].sum() < CAP_MAX - 1 and deg[7] > 2  # vertex 7's incidences run across positions 566 .. 568
    return g


def _hub_alone_case(G):
    """vpc = 5 and nv = 5 (G - 1) + 1: the last CTA holds the hub alone, degree > 568, its tail read from global memory"""
    nv = 5 * (G - 1) + 1
    rng = np.random.default_rng(3)
    hub = nv - 1
    extra = _spread(rng, hub, CAP_MAX + 140, nv, ())  # more edges than other vertices: duplicate hub edges
    return _graph(nv, loops=nv, extra=extra, seed=3)


def _two_hubs_case(G):
    """two hubs of degree > 568 in CTA 2 (vpc = 5), one free and one fixed, both roles, duplicate edges"""
    nv = 5 * G
    rng = np.random.default_rng(4)
    extra = _spread(rng, 10, CAP_MAX + 60, nv, ()) + _spread(rng, 12, CAP_MAX + 9, nv, ())
    return _graph(nv, loops=nv, extra=extra, seed=4, fixed=(0, 12), outliers=range(nv - 1, nv + 40))


def _fixed_case(G):
    """vpc = 8: fixed first and last vertex of CTA 3, the whole CTA 5, a fixed hub (vertex 100); Huber-active and duplicate
    edges"""
    nv = 8 * G
    rng = np.random.default_rng(6)
    extra = _spread(rng, 100, 300, nv, ())
    fixed = (0, 24, 31) + tuple(range(40, 48)) + (100,)
    return _graph(nv, loops=2 * nv, extra=extra, fixed=fixed, seed=6, outliers=range(nv, nv + nv // 10, 3), duplicates=nv // 8)


def _ill_chain():
    """a 20-vertex chain with information weights 1e-6 .. 1e6 and initial rotations of the order of 100 degrees: in the first
    iteration PCG runs into its cap (6 nv iterations), LM rejects two trials and the carried _residual sets the next trials'
    tolerances above 1e-6"""
    g = _graph(20, seed=1, weights=(1e-2, 1e6), init_trans=0.5, init_rot_deg=100.0, rot_noise_deg=5.0)
    g["info"][::2, ::7] *= 1e-4
    return g


CASES = {
    "nv1_ne0": lambda G: _graph(1, fixed=()),
    "nv2": lambda G: _graph(2),
    "below_grid_isolated_vertex": lambda G: _graph(G // 2 + 3, loops=G, isolated=(7,), seed=1),
    "grid": lambda G: _graph(G, loops=2 * G, seed=2),
    "grid_plus_1": lambda G: _graph(G + 1, loops=2 * G, seed=3, fixed=(0, G)),
    "vpc16": lambda G: _graph(16 * G, loops=2 * 16 * G, seed=16),
    "vpc17": lambda G: _graph(16 * G + 1, loops=2 * 16 * G, seed=17, fixed=(0, 17, 33)),
    "vpc79": lambda G: _graph(79 * G, loops=2 * 79 * G, seed=79),
    "vpc80": lambda G: _graph(RES_VPC * G, loops=2 * RES_VPC * G, seed=80, fixed=(0, 79, 80)),
    "general_only": lambda G: _graph(RES_VPC * G + 1, loops=2 * RES_VPC * G, seed=81),
    "cta_567": lambda G: _cap_case(G, CAP_MAX - 1),
    "cta_568": lambda G: _cap_case(G, CAP_MAX),
    "cta_569": lambda G: _cap_case(G, CAP_MAX + 1),
    "hub_alone": _hub_alone_case,
    "two_hubs": _two_hubs_case,
    "fixed_patterns": _fixed_case,
    "all_but_one_fixed": lambda G: _graph(40, loops=40, fixed=[v for v in range(40) if v != 17], seed=12, duplicates=5),
    "ill_conditioned_chain": lambda G: _ill_chain(),
}
ITERATIONS = 3
ITERATIONS_SMALL = 5  # graphs below 1000 vertices


@functools.lru_cache(maxsize=None)
def case_graph(name, G):
    return CASES[name](G)


# ---- the oracle side ----------------------------------------------------------------------------------------------
def stop_certified(t):
    """the trial's PCG stop index is certain (module docstring)"""
    dn, tol = t["dn"], t["tol"]
    if not t["ok"]:
        return False
    before, last = dn[:-1], dn[-1]
    if np.any(before <= tol * (1 + CERT_BAND)):
        return False
    nv6 = len(t["dx"]) * 6
    return t["iterations"] == nv6 or last < tol * (1 - CERT_BAND)


def decision_certified(t, chi2):
    """the accept / reject decision is certain, or the step is zero (PCG started below its tolerance): then either decision
    leaves the poses where they were up to the quaternions' renormalisation, and every further trial is again zero"""
    return (abs(t["rho"]) > RHO_BAND and abs(chi2 - t["chi2"]) > CHI2_BAND * abs(chi2)) or not t["ok"] or not t["dx"].any()


def step_bound(g, poses, t):
    """bound on |dx_gpu - dx_oracle| (max norm) of the trial t taken at `poses` (module docstring)"""
    S = co.posegraph_damped_system(poses, g["fixed"], g["ij"], g["meas"], g["info"], t["lam"])
    f = S["free"]
    dx = t["dx"][f].reshape(-1)
    if len(f) == 0:
        return 0.0
    direct = spla.spsolve(S["A"].tocsc(), S["b"][f].reshape(-1)) if dx.size else dx
    deg = np.bincount(g["ij"].reshape(-1), minlength=len(poses)) if len(g["ij"]) else np.zeros(len(poses), int)
    nterms = np.repeat(deg[f], 6) + 1
    absA = abs(S["A"])
    delta = (nterms + 8) * EPS * (S["babs"][f].reshape(-1) + absA @ np.abs(dx))
    floor = float(np.linalg.norm(delta)) / t["lam"] if t["lam"] > 0 else 0.0
    return 8 * float(np.abs(dx - direct).max()) + 1e-12 * float(np.abs(dx).max()) + floor


def chi2_floor(x, g, per_edge):
    """near zero a term e'We is the square of a difference of poses: e carries an absolute rounding of a few ulps of the poses
    (delta = 16 eps max(1, |x|)), which moves the term by up to 2 w |e|_1 delta <= 2 sqrt(6 w e'We) delta (W = w I)"""
    if not len(per_edge):
        return 0.0
    delta = 16 * EPS * max(1.0, float(np.abs(x).max()))
    return 2 * delta * float(np.sqrt(6 * g["info"][:, 0] * per_edge).sum())


def pose_bound(bc, poses):
    return 2 * bc + 8 * EPS * max(1.0, float(np.abs(poses).max()))


def pose_diff(a, b, free):
    if len(free) == 0:
        return 0.0
    dt = np.abs(a[free, :3] - b[free, :3]).max()
    sgn = np.where((a[free, 3:] * b[free, 3:]).sum(1) < 0, -1.0, 1.0)[:, None]
    return float(max(dt, np.abs(a[free, 3:] - sgn * b[free, 3:]).max()))


@functools.lru_cache(maxsize=None)
def oracle_steps(name, G):
    """the oracle's iterations: per iteration (start poses, trace, bound of the accepted step or 0, certified)"""
    g = case_graph(name, G)
    n_it = ITERATIONS_SMALL if len(g["init"]) < 1000 else ITERATIONS
    x = g["init"]
    out = []
    for _ in range(n_it):
        r = co.posegraph_lm_trace(x, g["fixed"], g["ij"], g["meas"], g["info"])
        chi2 = co.posegraph_chi2(x, g["ij"], g["meas"], g["info"])[1]
        cert_stop = all(stop_certified(t) for t in r["trials"])
        cert_dec = all(decision_certified(t, chi2) for t in r["trials"])
        acc = [t for t in r["trials"] if t["accepted"]]
        bc = step_bound(g, x, acc[0]) if acc else 0.0
        out.append(dict(start=x, trace=r, bound=pose_bound(bc, r["poses"]), cert_stop=cert_stop, cert_dec=cert_dec))
        x = r["poses"]
    return out


# ---- tests --------------------------------------------------------------------------------------------------------
def _run(fe, monkeypatch, g, x, resident):
    monkeypatch.setenv("RB200_PG_RESIDENT", "1" if resident else "0")
    return fe.optimize_graph(x, g["fixed"], g["ij"], g["meas"], g["info"], stop=1)


@pytest.mark.parametrize("name", list(CASES))
def test_one_lm_iteration_against_the_oracle_trace(fe, monkeypatch, name):
    G = sm_count()
    g = case_graph(name, G)
    free = np.nonzero(g["fixed"] == 0)[0]
    fixed = np.nonzero(g["fixed"])[0]
    steps = oracle_steps(name, G)
    worst = dict(step=0.0, kernels=0.0, chi2=0.0)
    uncertified = 0
    for k, st in enumerate(steps):
        r = st["trace"]
        cert = st["cert_stop"] and st["cert_dec"]
        uncertified += not cert
        out = {res: _run(fe, monkeypatch, g, st["start"], res) for res in (False, True)}
        for res, (x, chi2, it, cg) in out.items():
            what = (name, k, "resident" if res else "general")
            assert it == 1, what
            assert np.array_equal(x[fixed], st["start"][fixed]), what
            if name == "ill_conditioned_chain":
                pass  # see EXACT_PCG
            elif cert and r["cg_iterations"] <= EXACT_PCG:
                assert cg == r["cg_iterations"], (what, cg, r["cg_iterations"], [t["iterations"] for t in r["trials"]])
            elif cert:
                assert abs(cg - r["cg_iterations"]) <= len(r["trials"]) + LONG_PCG_REL * r["cg_iterations"], (what, cg, r["cg_iterations"])
            if st["cert_dec"]:
                d = pose_diff(x, r["poses"], free)
                assert d <= st["bound"], (what, d, st["bound"])
                worst["step"] = max(worst["step"], d / st["bound"] if st["bound"] else 0.0)
            want = co.posegraph_chi2(x, g["ij"], g["meas"], g["info"])[0]
            got, per_edge = fe.graph_chi2(x, g["ij"], g["meas"], g["info"], per_edge=True)
            assert abs(got - want) <= 1e-12 * want + chi2_floor(x, g, per_edge), (what, got, want)
            rel = abs(got - want) / want if want else abs(got)
            assert chi2 == got, what  # the returned chi2 is the chi2 of the returned poses
            worst["chi2"] = max(worst["chi2"], rel)
        if st["cert_dec"]:
            d = pose_diff(out[True][0], out[False][0], free)
            assert d <= st["bound"], (name, k, "kernels", d, st["bound"])
            worst["kernels"] = max(worst["kernels"], d / st["bound"] if st["bound"] else 0.0)
    print(f"{name}: nv {len(g['init'])} ne {len(g['ij'])} worst step/bound {worst['step']:.3g} kernels/bound {worst['kernels']:.3g} "
          f"chi2 rel {worst['chi2']:.3g} uncertified iterations {uncertified}/{len(steps)} "
          f"pcg {[st['trace']['cg_iterations'] for st in steps]}")
    assert uncertified <= len(steps) // 3, (name, uncertified)
    if name == "ill_conditioned_chain":
        first = steps[0]["trace"]["trials"]
        assert [t["accepted"] for t in first][:2] == [0, 0] and first[0]["iterations"] == 6 * len(g["init"])
        assert first[1]["tol"] > 1e-6


def test_general_kernel_above_the_resident_capacity(fe, monkeypatch):
    """80 x SM count + 1 vertices: the host must take the general kernel whatever RB200_PG_RESIDENT says"""
    G = sm_count()
    g = case_graph("general_only", G)
    x = g["init"]
    a = _run(fe, monkeypatch, g, x, True)
    b = _run(fe, monkeypatch, g, x, False)
    assert np.array_equal(a[0], b[0]) and a[1:] == b[1:]


def test_cases_reach_the_edges_they_name():
    """the fixtures' shapes, checked on the SM count of an H100 SXM (132) and of a B200 (148)"""
    for G in (132, 148):
        for total, name in ((CAP_MAX - 1, "cta_567"), (CAP_MAX, "cta_568"), (CAP_MAX + 1, "cta_569")):
            g = case_graph(name, G)
            assert _cta_incidences(len(g["init"]), g["ij"], 4, 1) == total
            assert max(_cta_incidences(len(g["init"]), g["ij"], 4, c) for c in range(G)) == total
        g = case_graph("hub_alone", G)
        nv = len(g["init"])
        assert -(-nv // G) == 5 and (nv - 1) % 5 == 0 and np.bincount(g["ij"].reshape(-1))[nv - 1] > CAP_MAX
        g = case_graph("two_hubs", G)
        deg = np.bincount(g["ij"].reshape(-1))
        assert deg[10] > CAP_MAX and deg[12] > CAP_MAX and g["fixed"][12]
        assert -(-len(case_graph("vpc80", G)["init"]) // G) == RES_VPC
        assert -(-len(case_graph("general_only", G)["init"]) // G) == RES_VPC + 1
        assert -(-len(case_graph("vpc17", G)["init"]) // G) == 17
