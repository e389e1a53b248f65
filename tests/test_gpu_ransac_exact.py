"""Exact gates on the RANSAC stage (run with -m gpu on an H100).

- Scoring invariant: the returned inlier list of every pair that reports inliers is exactly the float64 errorFunction2
  decision (tests/ransac_exact.scores_f64) under the returned transform, n_inliers is its size, info_scale follows from
  (n_inliers, rmse) bit for bit and rmse is the float64 value to the float32 screen's envelope.
- Near-threshold batches: the same invariant where hundreds of correspondences sit inside the screen's fall-back band, across
  the depth-covariance regimes the product reaches.
- Bookkeeping: planned paths through the reference loop (breaks, +10 jumps across the phase and CTA edges, the identity
  fallback, the 0.75 M clamp, mask-word edges, both kernel instantiations, several ransac_iterations) equal the oracle.
- Stale records: a slot whose hypothesis workspace holds another batch's records gives the same bytes as an unused slot.
"""
import ctypes as C

import numpy as np
import pytest

import ransac_exact as rx

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def fe(built):
    from rgbdslam_v2_b200 import Frontend
    from rgbdslam_v2_b200._capi import default_params
    p = default_params()
    p.depth_cov_z0 = 2.0
    f = Frontend(0, p)
    yield f
    _reinit(f)
    f.close()


def _reinit(fe, **kw):
    from rgbdslam_v2_b200._capi import default_params
    p = default_params()
    p.depth_cov_z0 = 2.0
    for k, v in kw.items():
        setattr(p, k, v)
    fe.params = p
    fe._check(fe.lib.rgbdslam_b200_init(0, C.byref(p)))
    return p


def _run(fe, b, seed):
    return fe.match_pairs_host(b["desc_newer"], b["xyz_newer"], b["n_newer"], b["desc_older"], b["xyz_older"], b["n_older"],
                               b["id_newer"], b["id_older"], seed=seed)


def _czc(fe):
    return None if fe.params.depth_cov_z0 < 0 else rx.cov_const(fe.params.sigma_depth, fe.depth_cov_z0)


def _rows(b, allm, i, n):
    on = int(np.sum(b["n_newer"][:i]))
    oo = int(np.sum(b["n_older"][:i]))
    m = allm[i, :n]
    return b["xyz_newer"][on + m["queryIdx"]], b["xyz_older"][oo + m["trainIdx"]]


def _min_thr(mn, M):  # node.cpp:1094-1099
    return mn if mn <= 0.75 * M else int(0.75 * M)


def _check_invariant(fe, b, res, allm, inl, tie=1e-10):
    """The scoring invariant on every pair that reports inliers; returns the margins of all scored correspondences.  Rows
    within `tie` (relative) of a cut are left out of the mask comparison: there two float64 evaluations in different
    operation orders (this restatement, the kernel's fma chains) may round to different sides.  A pair without inliers must
    have a reason: too few matches for RANSAC, or no hypothesis above the threshold and an identity fallback that float64
    rejects too."""
    czc = _czc(fe)
    prm = fe.params
    md = prm.max_dist_for_inliers
    mm, sm, inside_m, inside_s, checked = [], [], [], [], 0
    for i in range(len(res)):
        r = res[i]
        n, ni = int(r["n_all_matches"]), int(r["n_inliers"])
        frm, to = _rows(b, allm, i, n)
        T = r["ransac_trafo"].reshape(4, 4).T
        s = rx.scores_f64(T, frm, to, max_dist=md, sigma_depth=prm.sigma_depth, czc=czc)
        if ni == 0:
            assert r["id1"] < 0 and r["used_identity"] == 0, i
            if n > prm.min_matches:
                assert np.array_equal(T, np.eye(4, dtype=np.float32)), i
                if r["valid_iterations"] == 0:  # the identity fallback ran and must have been rejected
                    assert not (s["cnt"] > _min_thr(prm.min_matches, n) and s["rmse"] < np.float32(md)), (i, s["cnt"])
            continue
        firm = (s["m_margin"] > tie) & (s["s_margin"] > tie)
        assert (~firm).sum() <= 2, i
        assert abs(ni - s["cnt"]) <= (~firm).sum(), (i, ni, s["cnt"])
        got = np.zeros(n, bool)
        pos = {(int(q), int(t)): k for k, (q, t) in enumerate(zip(allm[i, :n]["queryIdx"], allm[i, :n]["trainIdx"]))}
        if (~firm).sum() == 0:
            assert ni == s["cnt"], (i, ni, s["cnt"])
            assert np.array_equal(inl[i, :ni], allm[i, :n][s["inl"]]), i
        else:
            got[[pos[(int(q), int(t))] for q, t in zip(inl[i, :ni]["queryIdx"], inl[i, :ni]["trainIdx"])]] = True
            assert np.array_equal(got[firm], s["inl"][firm]), i
        assert abs(float(r["rmse"]) / s["rmse"] - 1) < 5e-5, (i, float(r["rmse"]), s["rmse"])
        if r["id1"] >= 0:
            assert r["info_scale"] == np.float64(np.float32(ni) / (np.float32(r["rmse"]) * np.float32(r["rmse"]))), i
        mm.append(s["m_margin"]); sm.append(s["s_margin"])
        inside_m.append(s["inl"]); inside_s.append(s["dsq"] <= s["lim"])
        checked += 1
    assert checked > 0
    return np.concatenate(mm), np.concatenate(sm), np.concatenate(inside_m), np.concatenate(inside_s), checked


# ---- C1: the invariant on the synthetic batches of the older parity tests ------------------------------------------------

SYNTH = [
    ("c2-size", dict(), dict(npairs=256, n_kp=1000, seed0=5000)),
    ("nan-zero-depth", dict(), dict(npairs=3, n_kp=600, seed0=500, overlap=0.7, holes=True)),
    ("max-matches-512", dict(max_matches=512, ransac_iterations=100, max_dist_for_inliers=2.0), dict(npairs=8, n_kp=900, seed0=900)),
    ("z0-2", dict(), dict(npairs=24, n_kp=1000, seed0=0)),
    ("z0-latched", dict(depth_cov_z0=0.0), dict(npairs=6, n_kp=800, seed0=1200)),
    ("per-point", dict(depth_cov_z0=-1.0), dict(npairs=8, n_kp=900, seed0=900)),
]


@pytest.mark.parametrize("name,params,gen", SYNTH, ids=[s[0] for s in SYNTH])
def test_scoring_invariant_on_synthetic_batches(fe, name, params, gen):
    from rgbdslam_v2_b200 import synth
    _reinit(fe, **params)
    gen = dict(gen)
    holes = gen.pop("holes", False)
    b = synth.make_batch(gen.pop("npairs"), gen.pop("n_kp"), **gen)
    if holes:
        x = b["xyz_newer"].copy()
        x[5::17, 2] = np.nan
        x[3::29, :3] = 0.0
        b["xyz_newer"] = x
    res, allm, inl = _run(fe, b, 99)
    _, _, _, _, checked = _check_invariant(fe, b, res, allm, inl)
    assert checked >= 0.8 * len(res)
    _reinit(fe)


# ---- C2: near-threshold batches -------------------------------------------------------------------------------------------

# (name, depth_cov_z0 parameter, point depths, max_dist_for_inliers, far z of match 0 of pair 0 for the latch)
PLANTED = [
    ("z0=2, z 0.3-0.8", 2.0, (0.3, 0.8), 3.0, None),
    ("z0=2, z 0.3-0.8, 1.5 m", 2.0, (0.3, 0.8), 1.5, None),
    ("latched z0=5, z 1-2", 0.0, (1.0, 2.0), 3.0, 5.0),
    ("per-point, z 4-10", -1.0, (4.0, 10.0), 3.0, None),
    ("per-point, z 10-30", -1.0, (10.0, 30.0), 3.0, None),
    ("per-point, z 4-10, 1.5 m", -1.0, (4.0, 10.0), 1.5, None),
]
PLANTED_H = 16  # every one of the first 16 hypotheses draws a gross outlier


def planted_batch(oracle_mod, regime, npairs=8, seed=3):
    """Pairs that end in the identity fallback, with rows planted near both cuts under T = I (the transform the kernel then
    returns exactly, so the planted margins survive)."""
    name, z0p, zr, md, zfar = regime
    rng = np.random.default_rng(sum(map(ord, name)))
    z0 = 2.0 if z0p > 0 else (float(np.float32(zfar)) if zfar else None)
    czc = None if z0 is None else rx.cov_const(0.01, z0)
    pairs = [rx.identity_planted_pair(oracle_mod, rng, zr, czc, seed, i, PLANTED_H, max_dist=md, zfar=zfar if i == 0 else None)
             for i in range(npairs)]
    return rx.concat_batch(pairs), z0


def margin_counts(mm, sm, im, is_):
    near_m, near_s = mm < 3e-2, sm < 3e-2
    return dict(band=int((mm < 1e-3).sum()), near=int(((mm >= 1e-3) & near_m).sum()), s_band=int((sm < 1e-3).sum()),
                m_in=int((near_m & im).sum()), m_out=int((near_m & ~im).sum()), s_in=int((near_s & is_).sum()),
                s_out=int((near_s & ~is_).sum()), tiny=int((mm < 1e-6).sum() + (sm < 1e-6).sum()))


def identity_margins(b, res, allm, md, czc):
    """margin counts over the pairs that ended in the accepted identity fallback (at least 6 of 8: with a large latched
    covariance an occasional fit from a sample with one outlier still converges)"""
    idp = np.nonzero(res["used_identity"] == 1)[0]
    assert len(idp) >= 6 and (res["valid_iterations"][idp] == 1).all(), res["used_identity"]
    parts = [[], [], [], []]
    for i in idp:
        frm, to = _rows(b, allm, i, int(res[i]["n_all_matches"]))
        s = rx.scores_f64(np.eye(4), frm, to, max_dist=md, czc=czc)
        for lst, v in zip(parts, (s["m_margin"], s["s_margin"], s["inl"], s["dsq"] <= s["lim"])):
            lst.append(v)
    return margin_counts(*(np.concatenate(x) for x in parts))


def assert_not_vacuous(c):
    """>= 200 rows inside the screen's 1e-3 fall-back band, >= 200 in [1e-3, 3e-2], >= 50 within 1e-3 of the shortcut limit,
    both sides of both cuts, and >= 100 rows closer to a cut than the screen's own error (~1e-6..1e-5)."""
    assert c["band"] >= 200 and c["near"] >= 200 and c["s_band"] >= 50, c
    assert min(c["m_in"], c["m_out"], c["s_in"], c["s_out"]) >= 20 and c["tiny"] >= 100, c


@pytest.mark.parametrize("regime", PLANTED, ids=[r[0] for r in PLANTED])
def test_scoring_invariant_near_threshold(fe, oracle_mod, regime):
    """Hundreds of rows inside the fall-back band of the float32 screen, scored under a transform the kernel returns
    exactly: the returned inlier list is the float64 decision, so neither the screen nor its float64 fall-back may err."""
    name, z0p, zr, md, zfar = regime
    _reinit(fe, depth_cov_z0=z0p, max_dist_for_inliers=md, ransac_iterations=PLANTED_H)
    b, z0 = planted_batch(oracle_mod, regime)
    res, allm, inl = _run(fe, b, 3)
    if zfar:
        assert fe.depth_cov_z0 == z0
    _, _, _, _, checked = _check_invariant(fe, b, res, allm, inl)
    assert checked == len(res)
    assert_not_vacuous(identity_margins(b, res, allm, md, rx.cov_const(0.01, z0) if z0 else None))
    _reinit(fe)


# ---- C3: exact bookkeeping ------------------------------------------------------------------------------------------------

def _oracle(oracle_mod, b, cfg, seed):
    mn, mm, H = cfg
    prm = oracle_mod.make_params(min_matches=mn, max_matches=mm, ransac_iterations=H, depth_cov_z0=2.0)
    return oracle_mod.match_pairs(prm, b["desc_newer"], b["xyz_newer"], b["n_newer"], b["desc_older"], b["xyz_older"],
                                  b["n_older"], b["id_newer"], b["id_older"], seed=seed)


CERT_MARGIN = 0.05


def _assert_bookkeeping(b, allm, res, inl, ores, oinl, meta, cfg):
    """GPU == oracle on planned paths.  Every correspondence of these scenarios is at least CERT_MARGIN (relative) from both
    cuts under either side's transform (asserted below): far above what the float32 fits' difference (< 2e-5) or the screen's
    error (< 1e-4) can move, so no inlier decision of the returned model can differ between the two.  The only error
    comparisons with equal counts are the refinement loop's converged step (node.cpp:1160), where both branches end with the
    same inlier set; each plan visits a single valid hypothesis, so node.cpp:1177 never compares two equal counts."""
    mn, _, H = cfg
    for i, (name, M, valid, n_in) in enumerate(meta):
        g, o = res[i], ores[i]
        frm, to = _rows(b, allm, i, M)
        for T in (g["ransac_trafo"], o["ransac_trafo"]):
            s = rx.scores_f64(T.reshape(4, 4).T, frm, to, czc=rx.cov_const(0.01, 2.0))
            assert min(s["m_margin"].min(), s["s_margin"].min()) > CERT_MARGIN, name
        real, nvalid, _ = rx.expected_path(set(valid), H, M, n_in, mn)
        assert o["real_iterations"] == real, name  # the oracle took the planned path
        for f in ("n_all_matches", "valid_iterations", "n_inliers", "used_identity", "id1", "id2"):
            assert g[f] == o[f], (name, f, g[f], o[f])
        ni = int(g["n_inliers"])
        assert np.array_equal(inl[i, :ni], oinl[i, :ni]), name
        assert np.abs(g["ransac_trafo"] - o["ransac_trafo"]).max() < 2e-5, name
        if ni:
            assert abs(float(g["rmse"]) / float(o["rmse"]) - 1) < 5e-5, (name, g["rmse"], o["rmse"])


def test_bookkeeping_scenarios_equal_oracle(fe, oracle_mod):
    for cfg, (b, meta, seed) in rx.scenario_batches(oracle_mod).items():
        mn, mm, H = cfg
        _reinit(fe, min_matches=mn, max_matches=mm, ransac_iterations=H)
        res, allm, inl = _run(fe, b, seed)
        ores, oall, oinl = _oracle(oracle_mod, b, cfg, seed)
        for i in range(len(res)):
            n = int(res[i]["n_all_matches"])
            assert np.array_equal(allm[i, :n], oall[i, :n])
        _assert_bookkeeping(b, allm, res, inl, ores, oinl, meta, cfg)
        _check_invariant(fe, b, res, allm, inl)
    _reinit(fe)


# ---- C4: stale hypothesis records -----------------------------------------------------------------------------------------

VICTIMS = ["break@0", "break@3", "jump1@0", "jump1@1", "jump1@2", "jump1@3", "jump2@0", "jump2@3"]


def _poison_batch(oracle_mod, npairs):
    """Every pair: 512 matches, 254 noise-free inliers on the first ranks (49.6 %: no jump, every hypothesis is computed; a
    third of them valid with a large count and a tiny error)."""
    pairs = []
    for i in range(npairs):
        rng = np.random.default_rng(4242 + i)
        qd, xn, td, xo, _ = rx.scenario_pair(oracle_mod, rng, 512, 200, (), 258, 5, i, max_matches=512, noise=0.0,
                                             outliers_last=True)
        pairs.append((qd, xn, td, xo))
    return rx.concat_batch(pairs)


def _submit(fe, slot, b, seed):
    import torch
    from rgbdslam_v2_b200._capi import PAIR_RESULT_DTYPE, DMATCH_DTYPE
    n, mm = len(b["n_newer"]), fe.params.max_matches
    bufs = [torch.zeros(n * PAIR_RESULT_DTYPE.itemsize, dtype=torch.uint8).pin_memory(),
            torch.zeros(n * mm * 16, dtype=torch.uint8).pin_memory(), torch.zeros(n * mm * 16, dtype=torch.uint8).pin_memory()]
    out = (bufs[0].numpy().view(PAIR_RESULT_DTYPE), bufs[1].numpy().view(DMATCH_DTYPE).reshape(n, mm),
           bufs[2].numpy().view(DMATCH_DTYPE).reshape(n, mm))
    pins = {k: torch.from_numpy(b[k]).pin_memory() for k in ("desc_newer", "xyz_newer", "desc_older", "xyz_older")}
    fe.submit_pairs_host(slot, pins["desc_newer"], pins["xyz_newer"], b["n_newer"], pins["desc_older"], pins["xyz_older"],
                         b["n_older"], b["id_newer"], b["id_older"], out, seed=seed)
    fe.wait_slot(slot)
    return tuple(a.copy() for a in out)


def _same(a, b):
    (r, m, i), (rr, rm, ri) = a, b
    assert r.tobytes() == rr.tobytes() and m.tobytes() == rm.tobytes()
    for k in range(len(r)):
        assert np.array_equal(i[k, :r[k]["n_inliers"]], ri[k, :rr[k]["n_inliers"]])


def test_stale_hypothesis_records(fe, oracle_mod):
    """Victim pairs whose phase 1 breaks or jumps leave records unwritten that the sequential loop never reads.  Run on a slot
    that holds another batch's records (same layout, and after an init with a smaller ransac_iterations that changes the
    p * H + n layout), and on unused slots: the same bytes every time, equal to the oracle."""
    ((cfg, (vb, meta, seed)),) = rx.scenario_batches(oracle_mod, names=VICTIMS).items()
    mn, mm, H = cfg
    assert len(meta) == len(VICTIMS) and H == 40
    pb = _poison_batch(oracle_mod, len(VICTIMS))
    # the poison really fills the workspace with valid, high-count records
    _reinit(fe, max_matches=512, ransac_iterations=H)
    pr = _run(fe, pb, 5)[0]
    assert (pr["valid_iterations"] >= 8).all() and (pr["n_inliers"] == 254).all()
    _reinit(fe, min_matches=mn, max_matches=mm, ransac_iterations=H)
    runs = [_run(fe, vb, seed)]                              # slot 0: poisoned, same layout
    _reinit(fe, max_matches=512, ransac_iterations=H)
    _submit(fe, 3, pb, 5)                                     # slot 3: poisoned through the pipelined path
    _reinit(fe, min_matches=mn, max_matches=mm, ransac_iterations=H)
    runs.append(_submit(fe, 3, vb, seed))
    runs.append(_submit(fe, 6, vb, seed))                     # slot 6: unused
    _reinit(fe, max_matches=512, ransac_iterations=200)
    _run(fe, pb, 5)                                           # slot 0: poisoned with 200 records per pair
    _reinit(fe, min_matches=mn, max_matches=mm, ransac_iterations=H)
    runs.append(_run(fe, vb, seed))
    for r in runs[1:]:
        _same(runs[0], r)
    res, allm, inl = runs[0]
    ores, oall, oinl = _oracle(oracle_mod, vb, cfg, seed)
    _assert_bookkeeping(vb, allm, res, inl, ores, oinl, meta, cfg)
    _reinit(fe)


# ---- C5: degenerate samples -----------------------------------------------------------------------------------------------

def degenerate_batch(oracle_mod, seed=11):
    pairs, meta = [], []
    for i, kind in enumerate(["many-to-one", "collinear"] * 3):
        rng = np.random.default_rng(900 + i)
        qd, xn, td, xo, k, n_in, s0 = rx.degenerate_pair(oracle_mod, rng, kind, seed, i)
        pairs.append((qd, xn, td, xo))
        meta.append((kind, k, n_in, s0))
    return rx.concat_batch(pairs), meta


def test_degenerate_samples_reach_the_oracles_outcome(fe, oracle_mod):
    """Hypothesis 0 draws a rank-deficient sample (rank 0: four queries matched to one train row; rank 1: collinear
    from-points).  The kernel's fit reports failure (rank < 2); the oracle fits and scores a rank-deficient R, which explains
    fewer than min_matches correspondences.  Both end with hypothesis 0 invalid and break at the first clean sample."""
    b, meta = degenerate_batch(oracle_mod)
    cfg = (20, 300, 8)
    _reinit(fe, min_matches=20, max_matches=300, ransac_iterations=8)
    res, allm, inl = _run(fe, b, 11)
    ores, oall, oinl = _oracle(oracle_mod, b, cfg, 11)
    for i, (kind, k, n_in, s0) in enumerate(meta):
        frm, to = _rows(b, allm, i, int(res[i]["n_all_matches"]))
        d1 = frm[s0, :3].astype(np.float64) - frm[s0, :3].mean(0)
        d2 = to[s0, :3].astype(np.float64) - to[s0, :3].mean(0)
        assert np.linalg.matrix_rank(d2.T @ d1, tol=1e-6) == (0 if kind == "many-to-one" else 1), kind
        assert ores[i]["real_iterations"] == k + 1 and ores[i]["valid_iterations"] == 1, (kind, ores[i]["real_iterations"], k)
        assert ores[i]["n_inliers"] == n_in, kind
    _assert_bookkeeping(b, allm, res, inl, ores, oinl, [(kind, 300, (k,), n_in) for kind, k, n_in, _ in meta], cfg)
    _reinit(fe)
