"""The shapes of the RANSAC hypothesis kernel's blocking (run with -m gpu on an H100).

ransac_hyp_kernel runs hypotheses [0, 4) in one CTA per pair, then [4, H) in CTAs of 32 consecutive hypotheses whose refit
loops advance in lockstep rounds.  These tests put the block edges where they can break: ransac_iterations on both sides of
a block, the > 80 % break in the first, a middle and the last block of the second phase, both mask-word instantiations,
the fewest matches RANSAC runs on, blocks whose hypotheses all end after their first fit, and batches in flight on several
slots.
"""
import numpy as np
import pytest

import ransac_exact as rx
import test_gpu_frontend as gf
import test_gpu_ransac_exact as gx

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def fe(built):
    from rgbdslam_v2_b200 import Frontend
    from rgbdslam_v2_b200._capi import default_params
    p = default_params()
    p.depth_cov_z0 = 2.0
    f = Frontend(0, p)
    yield f
    gx._reinit(f)
    f.close()


def _synth_vs_oracle(fe, oracle_mod, kw, npairs=8, n_kp=900, seed0=900, seed=21, strict_frac=0.75):
    """The oracle's match lists and edge decisions; the model within test_gpu_frontend's tolerances from 200 hypotheses on,
    below that the exact float64 scoring invariant of the returned model (test_gpu_ransac_exact)."""
    from rgbdslam_v2_b200 import synth
    p = gx._reinit(fe, **kw)
    b = synth.make_batch(npairs, n_kp, seed0=seed0)
    res, allm, inl = gx._run(fe, b, seed)
    ores, oall, oinl = oracle_mod.match_pairs(
        oracle_mod.make_params(min_matches=p.min_matches, max_matches=p.max_matches, ransac_iterations=p.ransac_iterations,
                               depth_cov_z0=p.depth_cov_z0),
        b["desc_newer"], b["xyz_newer"], b["n_newer"], b["desc_older"], b["xyz_older"], b["n_older"], b["id_newer"],
        b["id_older"], seed=seed, threads=8)
    if p.ransac_iterations >= 200:
        gf._compare(res, allm, inl, ores, oall, oinl, strict_frac=strict_frac)
    else:  # short runs may settle on a different one of two near-equal models than the oracle: decisions exact, model exact
        for i in range(len(res)):
            n = int(res[i]["n_all_matches"])
            assert n == ores[i]["n_all_matches"] and np.array_equal(allm[i, :n], oall[i, :n]), i
            for f in ("id1", "id2", "used_identity"):
                assert res[i][f] == ores[i][f], (i, f)
        gx._check_invariant(fe, b, res, allm, inl)
    gx._reinit(fe)
    return res


@pytest.mark.parametrize("H", [1, 4, 5, 31, 32, 33, 36, 37, 200, 1000])
def test_ransac_iterations_across_block_edges(fe, oracle_mod, H):
    """Phase 2 absent (1, 4), one hypothesis (5), one partial / full block (31-36) and a second block (37), the default and
    31 full blocks plus a partial one (1000)."""
    res = _synth_vs_oracle(fe, oracle_mod, dict(ransac_iterations=H))
    assert (res["id1"] >= 0).any()


@pytest.mark.parametrize("mm", [319, 320, 321])
def test_max_matches_around_the_instantiation_edge(fe, oracle_mod, mm):
    _synth_vs_oracle(fe, oracle_mod, dict(max_matches=mm))


# (name, (min_matches, max_matches, H), M, hypotheses that draw all-inlier samples, outliers)
BLOCK_SCENARIOS = [
    *[(f"H200-break@{k}", (20, 300, 200), 300, (k,), 40) for k in (4, 35, 36)],       # first block; first of the second
    *[(f"H40-break@{k}", (20, 300, 40), 300, (k,), 40) for k in (35, 36, 39)],       # last block [36, 40)
    ("H37-break@36", (20, 300, 37), 300, (36,), 40),                                  # last block of one hypothesis
    ("H200-jump1@25", (20, 300, 200), 300, (25, 29, 35), 100),                        # +10 from the first block to 36
    ("H40-maxm512", (20, 512, 40), 512, (37,), 60),                                   # 16 mask words
]


def test_break_and_jump_positions_equal_oracle(fe, oracle_mod):
    groups = {}
    for name, cfg, M, valid, n_out in BLOCK_SCENARIOS:
        groups.setdefault(cfg, []).append((name, M, valid, n_out))
    for cfg, items in groups.items():
        mn, mm, H = cfg
        pairs, meta = [], []
        for i, (name, M, valid, n_out) in enumerate(items):
            rng = np.random.default_rng(sum(map(ord, name)) * 7919 + M)
            qd, xn, td, xo, _ = rx.scenario_pair(oracle_mod, rng, M, H, valid, n_out, 7, i, max_matches=mm)
            pairs.append((qd, xn, td, xo))
            meta.append((name, M, valid, M - n_out))
        b = rx.concat_batch(pairs)
        gx._reinit(fe, min_matches=mn, max_matches=mm, ransac_iterations=H)
        res, allm, inl = gx._run(fe, b, 7)
        ores, oall, oinl = gx._oracle(oracle_mod, b, cfg, 7)
        for i in range(len(res)):
            n = int(res[i]["n_all_matches"])
            assert np.array_equal(allm[i, :n], oall[i, :n])
        gx._assert_bookkeeping(b, allm, res, inl, ores, oinl, meta, cfg)
    gx._reinit(fe)


@pytest.mark.parametrize("H", [1, 5, 200])
def test_blocks_where_every_fit_fails(fe, oracle_mod, H):
    """The degenerate pairs of tests/ransac_exact.degenerate_pair: hypothesis 0 draws a rank-deficient sample and the
    hypotheses up to the first clean sample draw an outlier, so each ends after its first fit.  H = 1: the only hypothesis
    fails and the identity fallback decides; H = 5: the second phase is one block of one hypothesis; H = 200: the break."""
    pairs = []
    for i, kind in enumerate(["many-to-one", "collinear"] * 3):
        rng = np.random.default_rng(900 + i)
        qd, xn, td, xo, _, _, _ = rx.degenerate_pair(oracle_mod, rng, kind, 11, i)
        pairs.append((qd, xn, td, xo))
    b = rx.concat_batch(pairs)
    gx._reinit(fe, min_matches=20, max_matches=300, ransac_iterations=H)
    res, allm, inl = gx._run(fe, b, 11)
    ores, oall, oinl = gx._oracle(oracle_mod, b, (20, 300, H), 11)
    gx._reinit(fe)
    for i in range(len(res)):
        g, o = res[i], ores[i]
        for f in ("n_all_matches", "valid_iterations", "n_inliers", "used_identity", "id1", "id2"):
            assert g[f] == o[f], (i, f, g[f], o[f])
        ni = int(g["n_inliers"])
        assert np.array_equal(inl[i, :ni], oinl[i, :ni]), i
    if H == 1:
        assert (res["used_identity"] == 1).sum() + (res["valid_iterations"] == 0).sum() == len(res)


@pytest.mark.parametrize("M", [21, 22, 33])
def test_fewest_matches_equal_oracle(fe, oracle_mod, M):
    """M just above min_matches = 20: one mask word, every block's hypotheses share a handful of samples."""
    pairs = []
    for i in range(4):
        rng = np.random.default_rng(1300 + 10 * M + i)
        qd, xn, td, xo, _ = rx.scenario_pair(oracle_mod, rng, M, 200, (), 3, 7, i, outliers_last=True)
        pairs.append((qd, xn, td, xo))
    b = rx.concat_batch(pairs)
    gx._reinit(fe, min_matches=20, max_matches=300, ransac_iterations=200)
    res, allm, inl = gx._run(fe, b, 7)
    ores, oall, oinl = gx._oracle(oracle_mod, b, (20, 300, 200), 7)
    gx._reinit(fe)
    assert (res["n_all_matches"] == M).all()
    gf._compare(res, allm, inl, ores, oall, oinl, strict_frac=0.75)
    assert (res["id1"] >= 0).all()


def test_slots_in_flight_equal_synchronous(fe, oracle_mod):
    """Three batches with several blocks per pair in flight on three slots at once give the bytes of the synchronous call."""
    import torch
    from rgbdslam_v2_b200 import synth
    from rgbdslam_v2_b200._capi import PAIR_RESULT_DTYPE, DMATCH_DTYPE
    gx._reinit(fe, ransac_iterations=1000)
    mm = fe.params.max_matches
    batches = [synth.make_batch(16, 1000, seed0=7000 + 100 * j) for j in range(3)]
    sync = [tuple(a.copy() for a in gx._run(fe, b, 13 + j)) for j, b in enumerate(batches)]
    keep, outs = [], []
    for j, b in enumerate(batches):
        n = len(b["n_newer"])
        bufs = [torch.zeros(n * PAIR_RESULT_DTYPE.itemsize, dtype=torch.uint8).pin_memory(),
                torch.zeros(n * mm * DMATCH_DTYPE.itemsize, dtype=torch.uint8).pin_memory(),
                torch.zeros(n * mm * DMATCH_DTYPE.itemsize, dtype=torch.uint8).pin_memory()]
        out = (bufs[0].numpy().view(PAIR_RESULT_DTYPE), bufs[1].numpy().view(DMATCH_DTYPE).reshape(n, mm),
               bufs[2].numpy().view(DMATCH_DTYPE).reshape(n, mm))
        pins = {k: torch.from_numpy(b[k]).pin_memory() for k in ("desc_newer", "xyz_newer", "desc_older", "xyz_older")}
        fe.submit_pairs_host(1 + j, pins["desc_newer"], pins["xyz_newer"], b["n_newer"], pins["desc_older"], pins["xyz_older"],
                             b["n_older"], b["id_newer"], b["id_older"], out, seed=13 + j)
        keep.append((bufs, pins))
        outs.append(out)
    for j in range(3):
        fe.wait_slot(1 + j)
    gx._reinit(fe)
    for j in range(3):
        gx._same(sync[j], outs[j])
        assert (sync[j][0]["id1"] >= 0).sum() >= 12
