"""GPU parity tests (run with -m gpu on an H100): the CUDA path through the C ABI vs the CPU oracle."""
import ctypes as C
from pathlib import Path

import numpy as np
import pytest

pytestmark = pytest.mark.gpu
GOLD = Path(__file__).parent / "golden"


@pytest.fixture(scope="module")
def fe(built):
    from rgbdslam_v2_b200 import Frontend
    from rgbdslam_v2_b200._capi import default_params
    p = default_params()
    p.depth_cov_z0 = 2.0
    f = Frontend(0, p)
    yield f
    f.close()


def _reinit(fe, **kw):
    from rgbdslam_v2_b200._capi import default_params
    import ctypes as C
    p = default_params()
    p.depth_cov_z0 = 2.0
    for k, v in kw.items():
        setattr(p, k, v)
    fe.params = p
    fe._check(fe.lib.rgbdslam_b200_init(0, C.byref(p)))
    return p


def test_native_library_is_loaded(fe):
    maps = open("/proc/self/maps").read()
    assert "librgbdslam_b200.so" in maps


def test_brute_force_golden_vectors(fe):
    """Bit-exact against vectors produced by the reference's own bruteForceSearchORB."""
    g = np.load(GOLD / "brute_force_orb.npz")
    for name in ("a", "b", "c", "d", "ties"):
        hd, idx = fe.brute_force_search_orb(g[f"{name}_q"], g[f"{name}_t"])
        assert np.array_equal(hd, g[f"{name}_hd"]), name
        assert np.array_equal(idx, g[f"{name}_idx"]), name


@pytest.mark.parametrize("nq,nt", [(1, 2), (1, 1), (5, 0), (127, 128), (128, 129), (129, 257), (1000, 1000),
                                   (2000, 1999), (4096, 4096), (333, 3)])
def test_brute_force_vs_oracle_bit_exact(fe, oracle_mod, nq, nt):
    rng = np.random.default_rng(nq * 7919 + nt)
    q = rng.integers(0, 256, (nq, 32), dtype=np.uint8)
    t = rng.integers(0, 256, (nt, 32), dtype=np.uint8)
    if nt > 4 and nq > 4:  # plant exact + near duplicates, incl. the never-examined last row
        q[0] = t[-1]
        q[1] = t[0]
        q[2] = t[nt // 2]
        t[nt // 3] = t[1]  # tie: lowest index wins
        q[3] = t[1]
    hd, idx = fe.brute_force_search_orb(q, t)
    ohd, oidx = oracle_mod.brute_force_orb(q, t)
    assert np.array_equal(hd, ohd)
    assert np.array_equal(idx, oidx)


@pytest.mark.parametrize("nq,nt", [(1, 2), (5, 1), (128, 257), (129, 256), (1000, 1000), (1000, 1001), (1500, 700),
                                   (4096, 4096), (300, 4000)])
def test_hamming_tensor_core_path_equals_simt_path(fe, oracle_mod, nq, nt):
    """wgmma int8 GEMM formulation (hd = (256 - a.b)/2) is exact: identical to the popcount kernel."""
    rng = np.random.default_rng(nq * 31 + nt)
    q = rng.integers(0, 256, (nq, 32), dtype=np.uint8)
    t = rng.integers(0, 256, (nt, 32), dtype=np.uint8)
    if nt > 8 and nq > 8:
        q[0] = t[-1]; q[1] = t[0]; q[2] = ~t[3]; t[nt // 3] = t[1]; q[3] = t[1]
        q[4] = 0; q[5] = 255; t[2] = 0; t[5] = 255
    try:
        fe.set_hamming_path(1)  # default: descriptors expanded to int8 operands inside the kernel, column index in the accumulator
        hd1, idx1 = fe.brute_force_search_orb(q, t)
        fe.set_hamming_path(0)
        hd0, idx0 = fe.brute_force_search_orb(q, t)
    finally:
        fe.set_hamming_path(1)
    ohd, oidx = oracle_mod.brute_force_orb(q, t)
    assert np.array_equal(hd0, ohd) and np.array_equal(idx0, oidx)
    assert np.array_equal(hd1, ohd) and np.array_equal(idx1, oidx)


def test_hamming_expand_kernel_many_items_and_ragged_pairs(fe, oracle_mod):
    """The in-kernel-expansion match kernel over a batch whose work items outnumber the SMs (several items per persistent CTA:
    ring-slot reuse, the producer's look-ahead schedule) with ragged feature counts incl. single-tile and empty train sets."""
    from rgbdslam_v2_b200 import synth
    rng = np.random.default_rng(77)
    sizes = [(1000, 1000), (257, 129), (5, 1), (130, 2), (3, 600), (1000, 128), (999, 1025), (1, 1), (64, 4096), (4096, 64)] * 17
    newer, older, exp = [], [], []
    for i, (nq, nt) in enumerate(sizes):
        q = rng.integers(0, 256, (nq, 32), dtype=np.uint8)
        t = rng.integers(0, 256, (nt, 32), dtype=np.uint8)
        k = min(nq, nt) // 2
        if k:
            q[:k] = t[rng.permutation(nt)[:k]] ^ (1 << rng.integers(0, 8, (k, 32))).astype(np.uint8) * (rng.random((k, 32)) < 0.1)
        xq = np.concatenate([rng.uniform(0.5, 3, (nq, 3)), np.ones((nq, 1))], 1).astype(np.float32)
        xt = np.concatenate([rng.uniform(0.5, 3, (nt, 3)), np.ones((nt, 1))], 1).astype(np.float32)
        newer.append(fe.node_from_features(2 * i + 1, q, xq)); older.append(fe.node_from_features(2 * i, t, xt))
        exp.append((q, t))
    out = {}
    try:
        for path in (1, 0):
            fe.set_hamming_path(path)
            res, allm, _ = fe.match_node_pairs(newer, older, seed=4)
            out[path] = (res["n_all_matches"].copy(), allm.copy())
    finally:
        fe.set_hamming_path(1)
    assert np.array_equal(out[1][0], out[0][0])
    for i in range(len(sizes)):
        n = int(out[1][0][i])
        for f in ("queryIdx", "trainIdx", "distance"):
            assert np.array_equal(out[1][1][i, :n][f], out[0][1][i, :n][f]), (i, sizes[i], f)
    for h in newer + older:
        fe.node_destroy(h)


def _oracle_run(oracle_mod, b, seed, first=0, **kw):
    prm = oracle_mod.make_params(depth_cov_z0=kw.pop("depth_cov_z0", 2.0), **kw)
    return oracle_mod.match_pairs(prm, b["desc_newer"], b["xyz_newer"], b["n_newer"], b["desc_older"], b["xyz_older"],
                                  b["n_older"], b["id_newer"], b["id_older"], seed=seed, first_pair_index=first, threads=8)


def _compare(res, allm, inl, ores, oall, oinl, T_true=None, strict_frac=0.9):
    npairs = len(res)
    same = 0
    for i in range(npairs):
        n = int(res[i]["n_all_matches"])
        assert n == ores[i]["n_all_matches"]
        # integer / byte work is bit exact: match lists incl. the jitter distances
        assert np.array_equal(allm[i, :n], oall[i, :n])
        assert res[i]["id1"] == ores[i]["id1"] and res[i]["id2"] == ores[i]["id2"], i
        assert res[i]["used_identity"] == ores[i]["used_identity"]
        if res[i]["id1"] < 0:
            assert res[i]["n_inliers"] == ores[i]["n_inliers"]
            continue
        ni, no = int(res[i]["n_inliers"]), int(ores[i]["n_inliers"])
        # float tolerance: translation 2 mm, rotation entries 1e-3, rmse 2 % when the two RANSACs settle on different
        # (equally supported) inlier sets; 2e-5 when the inlier sets are identical (checked below)
        Tg = res[i]["ransac_trafo"].reshape(4, 4).T
        To = ores[i]["ransac_trafo"].reshape(4, 4).T
        assert np.abs(Tg[:3, 3] - To[:3, 3]).max() < 2e-3, i
        assert np.abs(Tg[:3, :3] - To[:3, :3]).max() < 1e-3, i
        assert abs(ni - no) <= max(2, 0.02 * no), i
        assert abs(res[i]["rmse"] - ores[i]["rmse"]) <= 0.02 * ores[i]["rmse"] + 1e-4
        assert abs(np.linalg.det(Tg[:3, :3].astype(np.float64)) - 1) < 1e-4
        if ni == no and np.array_equal(inl[i, :ni], oinl[i, :no]) and res[i]["valid_iterations"] == ores[i]["valid_iterations"]:
            same += 1
            assert np.abs(Tg - To).max() < 2e-5
            assert res[i]["info_scale"] == pytest.approx(ores[i]["info_scale"], rel=1e-3)
    valid = int((res["id1"] >= 0).sum())
    if valid:
        assert same >= strict_frac * valid, (same, valid)
    return same, valid


def test_match_pairs_host_vs_oracle(fe, oracle_mod):
    from rgbdslam_v2_b200 import synth
    _reinit(fe)
    b = synth.make_batch(24, 1000, seed0=0)
    res, allm, inl = fe.match_pairs_host(b["desc_newer"], b["xyz_newer"], b["n_newer"], b["desc_older"], b["xyz_older"],
                                         b["n_older"], b["id_newer"], b["id_older"], seed=11)
    ores, oall, oinl = _oracle_run(oracle_mod, b, 11)
    same, valid = _compare(res, allm, inl, ores, oall, oinl)
    assert valid >= 20
    # and both agree with the generator's ground truth
    for i in range(24):
        if res[i]["id1"] >= 0:
            T = res[i]["ransac_trafo"].reshape(4, 4).T
            assert np.abs(T[:3, 3] - b["T_true"][i][:3, 3]).max() < 6e-3


def test_node_handles_equal_host_path_and_sharding(fe, oracle_mod):
    """match_pairs on device-resident nodes == match_pairs_host; splitting the batch with
    first_pair_index reproduces the single-call results (what the multi-GPU sharding relies on)."""
    from rgbdslam_v2_b200 import synth
    _reinit(fe)
    b = synth.make_batch(10, 700, seed0=300)
    res, allm, inl = fe.match_pairs_host(b["desc_newer"], b["xyz_newer"], b["n_newer"], b["desc_older"], b["xyz_older"],
                                         b["n_older"], b["id_newer"], b["id_older"], seed=5)
    newer = [fe.node_from_features(int(b["id_newer"][i]), p["desc_newer"], p["xyz_newer"]) for i, p in enumerate(b["pairs"])]
    older = [fe.node_from_features(int(b["id_older"][i]), p["desc_older"], p["xyz_older"]) for i, p in enumerate(b["pairs"])]
    d, x = fe.node_download(newer[3])
    assert np.array_equal(d, b["pairs"][3]["desc_newer"]) and np.array_equal(x, b["pairs"][3]["xyz_newer"])
    r2, a2, i2 = fe.match_node_pairs(newer, older, seed=5)
    assert r2.tobytes() == res.tobytes() and a2.tobytes() == allm.tobytes()
    for i in range(10):
        assert np.array_equal(i2[i, :r2[i]["n_inliers"]], inl[i, :res[i]["n_inliers"]])
    ra, aa, ia = fe.match_node_pairs(newer[:4], older[:4], seed=5, first_pair_index=0)
    rb, ab, ib = fe.match_node_pairs(newer[4:], older[4:], seed=5, first_pair_index=4)
    assert np.concatenate([ra, rb]).tobytes() == res.tobytes()
    for h in newer + older:
        fe.node_destroy(h)


def test_edge_cases(fe, oracle_mod):
    """Empty / tiny / ragged nodes, hd>=128 everywhere, too few matches (node.cpp:1319,1087,1420)."""
    from rgbdslam_v2_b200 import synth
    _reinit(fe)
    rng = np.random.default_rng(9)
    good = synth.make_pair(77, 400)
    sizes = [(0, 0), (0, 50), (50, 0), (1, 1), (30, 2), (400, 400), (25, 400), (400, 19)]
    dn, xn, do, xo, nn, no = [], [], [], [], [], []
    for a, c in sizes:
        if (a, c) == (400, 400):
            dn.append(good["desc_newer"]); xn.append(good["xyz_newer"]); do.append(good["desc_older"]); xo.append(good["xyz_older"])
        else:
            dn.append(rng.integers(0, 256, (a, 32), dtype=np.uint8)); xn.append(np.concatenate([synth._random_points(rng, a), np.ones((a, 1))], 1).astype(np.float32))
            do.append(rng.integers(0, 256, (c, 32), dtype=np.uint8)); xo.append(np.concatenate([synth._random_points(rng, c), np.ones((c, 1))], 1).astype(np.float32))
        nn.append(a); no.append(c)
    b = dict(desc_newer=np.concatenate(dn), xyz_newer=np.concatenate(xn), desc_older=np.concatenate(do),
             xyz_older=np.concatenate(xo), n_newer=np.array(nn, np.int32), n_older=np.array(no, np.int32),
             id_newer=np.arange(len(sizes), dtype=np.int32) + 10, id_older=np.arange(len(sizes), dtype=np.int32))
    res, allm, inl = fe.match_pairs_host(b["desc_newer"], b["xyz_newer"], b["n_newer"], b["desc_older"], b["xyz_older"],
                                         b["n_older"], b["id_newer"], b["id_older"], seed=2)
    ores, oall, oinl = _oracle_run(oracle_mod, b, 2)
    _compare(res, allm, inl, ores, oall, oinl, strict_frac=0.0)
    assert res[5]["id1"] == 5 and res[5]["id2"] == 15
    assert (res["id1"][[0, 1, 2, 3, 4]] == -1).all()
    assert res[0]["rmse"] == 0 and res[0]["n_all_matches"] == 0


def test_nan_and_zero_depth_points(fe, oracle_mod):
    """NaN z is skipped by the fit (transformation_estimation_euclidean.cpp:22) and rejected by the score
    (misc.cpp:711); z == 0 is skipped by computeInliersAndError (node.cpp:994)."""
    from rgbdslam_v2_b200 import synth
    _reinit(fe)
    b = synth.make_batch(3, 600, seed0=500, overlap=0.7)
    x = b["xyz_newer"].copy()
    x[5::17, 2] = np.nan
    x[3::29, :3] = 0.0
    b["xyz_newer"] = x
    res, allm, inl = fe.match_pairs_host(b["desc_newer"], b["xyz_newer"], b["n_newer"], b["desc_older"], b["xyz_older"],
                                         b["n_older"], b["id_newer"], b["id_older"], seed=4)
    ores, oall, oinl = _oracle_run(oracle_mod, b, 4)
    _compare(res, allm, inl, ores, oall, oinl, strict_frac=0.6)
    assert (res["id1"] >= 0).all()


@pytest.mark.parametrize("kw", [dict(max_matches=128, ransac_iterations=64, min_matches=10),
                                dict(max_matches=512, ransac_iterations=100, max_dist_for_inliers=2.0),
                                dict(depth_cov_z0=-1.0)])
def test_parameter_variants(fe, oracle_mod, kw):
    from rgbdslam_v2_b200 import synth
    p = _reinit(fe, **kw)
    b = synth.make_batch(8, 900, seed0=900)
    res, allm, inl = fe.match_pairs_host(b["desc_newer"], b["xyz_newer"], b["n_newer"], b["desc_older"], b["xyz_older"],
                                         b["n_older"], b["id_newer"], b["id_older"], seed=21)
    okw = dict(kw)
    ores, oall, oinl = oracle_mod.match_pairs(
        oracle_mod.make_params(min_matches=p.min_matches, max_matches=p.max_matches, ransac_iterations=p.ransac_iterations,
                               max_dist_for_inliers=p.max_dist_for_inliers, depth_cov_z0=p.depth_cov_z0),
        b["desc_newer"], b["xyz_newer"], b["n_newer"], b["desc_older"], b["xyz_older"], b["n_older"], b["id_newer"],
        b["id_older"], seed=21, threads=8)
    _compare(res, allm, inl, ores, oall, oinl, strict_frac=0.75)
    _reinit(fe)


def test_depth_cov_static_latch(fe, oracle_mod):
    """depth_cov_z0 = 0: the library latches z0 like the function-static in misc2.h:30-35."""
    from rgbdslam_v2_b200 import synth
    _reinit(fe, depth_cov_z0=0.0)
    assert fe.depth_cov_z0 == 0.0
    b = synth.make_batch(6, 800, seed0=1200)
    res, allm, inl = fe.match_pairs_host(b["desc_newer"], b["xyz_newer"], b["n_newer"], b["desc_older"], b["xyz_older"],
                                         b["n_older"], b["id_newer"], b["id_older"], seed=8)
    # oracle emulation: z of the first scored correspondence of the first pair that reaches RANSAC
    prm0 = oracle_mod.make_params(depth_cov_z0=1.0)
    z0 = 0.0
    for i, p in enumerate(b["pairs"]):
        m = oracle_mod.feature_matching_orb(p["desc_newer"], p["desc_older"], 300, 8, i)
        z0 = oracle_mod.first_depth_z0(prm0, m, len(m), p["xyz_newer"], p["xyz_older"])
        if z0:
            break
    assert fe.depth_cov_z0 == pytest.approx(z0) and z0 > 0
    ores, oall, oinl = _oracle_run(oracle_mod, b, 8, depth_cov_z0=z0)
    _compare(res, allm, inl, ores, oall, oinl, strict_frac=0.75)
    _reinit(fe)


def test_full_size_batch_properties(fe, oracle_mod):
    """BASELINE config C2 size (256 pairs x 1000 kp): size-independent properties + oracle spot check."""
    from rgbdslam_v2_b200 import synth
    _reinit(fe)
    b = synth.make_batch(256, 1000, seed0=5000)
    res, allm, inl = fe.match_pairs_host(b["desc_newer"], b["xyz_newer"], b["n_newer"], b["desc_older"], b["xyz_older"],
                                         b["n_older"], b["id_newer"], b["id_older"], seed=99)
    valid = res["id1"] >= 0
    assert valid.sum() >= 230
    # idempotence / determinism
    res2, allm2, inl2 = fe.match_pairs_host(b["desc_newer"], b["xyz_newer"], b["n_newer"], b["desc_older"], b["xyz_older"],
                                            b["n_older"], b["id_newer"], b["id_older"], seed=99)
    assert res.tobytes() == res2.tobytes() and allm.tobytes() == allm2.tobytes()
    gt_err = []
    for i in np.nonzero(valid)[0]:
        n, ni = res[i]["n_all_matches"], res[i]["n_inliers"]
        assert 20 < n <= 300 and ni <= n
        assert (np.diff(allm[i, :n]["distance"]) >= 0).all()            # sortedness
        assert (np.diff(inl[i, :ni]["distance"]) >= 0).all()
        assert np.isin(inl[i, :ni]["queryIdx"], allm[i, :n]["queryIdx"]).all()
        T = res[i]["ransac_trafo"].reshape(4, 4).T
        assert abs(np.linalg.det(T[:3, :3].astype(np.float64)) - 1) < 1e-4
        gt_err.append(np.abs(T[:3, 3] - b["T_true"][i][:3, 3]).max())
        assert res[i]["info_scale"] == pytest.approx(ni / float(res[i]["rmse"]) ** 2, rel=1e-4)
    # ground truth of the generator: statistical (the early-exit RANSAC of node.cpp:1186-1188 accepts the first
    # model with > 80 % inliers; the CPU oracle shows the same cm-level outliers on this batch)
    assert np.median(gt_err) < 2e-3 and np.max(gt_err) < 3e-2
    sub = slice(100, 132)
    bs = {k: (v[sub] if k in ("n_newer", "n_older", "id_newer", "id_older") else v) for k, v in b.items()}
    bs["desc_newer"] = b["desc_newer"][100 * 1000:132 * 1000]; bs["xyz_newer"] = b["xyz_newer"][100 * 1000:132 * 1000]
    bs["desc_older"] = b["desc_older"][100 * 1000:132 * 1000]; bs["xyz_older"] = b["xyz_older"][100 * 1000:132 * 1000]
    ores, oall, oinl = _oracle_run(oracle_mod, bs, 99, first=100)
    _compare(res[sub], allm[sub], inl[sub], ores, oall, oinl, strict_frac=0.85)


def test_pipelined_submit_wait_equals_synchronous(fe, oracle_mod):
    """rgbdslam_b200_match_pairs_submit / _host_submit / _wait: batches in flight on different slots give exactly the
    results of the synchronous calls."""
    import torch
    from rgbdslam_v2_b200 import synth
    from rgbdslam_v2_b200._capi import PAIR_RESULT_DTYPE, DMATCH_DTYPE
    _reinit(fe)
    batches = [synth.make_batch(12, 800, seed0=7000 + 100 * j) for j in range(3)]
    ref = []
    for j, b in enumerate(batches):
        ref.append(fe.match_pairs_host(b["desc_newer"], b["xyz_newer"], b["n_newer"], b["desc_older"], b["xyz_older"], b["n_older"],
                                       b["id_newer"], b["id_older"], seed=31, first_pair_index=100 * j))
    outs, keep = [], []
    for j, b in enumerate(batches):
        bufs = [torch.zeros(12 * PAIR_RESULT_DTYPE.itemsize, dtype=torch.uint8).pin_memory(),
                torch.zeros(12 * 300 * 16, dtype=torch.uint8).pin_memory(), torch.zeros(12 * 300 * 16, dtype=torch.uint8).pin_memory()]
        keep.append(bufs)
        out = (bufs[0].numpy().view(PAIR_RESULT_DTYPE), bufs[1].numpy().view(DMATCH_DTYPE).reshape(12, 300),
               bufs[2].numpy().view(DMATCH_DTYPE).reshape(12, 300))
        outs.append(out)
        pins = {k: torch.from_numpy(b[k]).pin_memory() for k in ("desc_newer", "xyz_newer", "desc_older", "xyz_older")}
        keep.append(pins)
        fe.submit_pairs_host(1 + j, pins["desc_newer"], pins["xyz_newer"], b["n_newer"], pins["desc_older"], pins["xyz_older"],
                             b["n_older"], b["id_newer"], b["id_older"], out, seed=31, first_pair_index=100 * j)
    for j in range(3):
        fe.wait_slot(1 + j)
    for (r, a, i), (rr, ra, ri) in zip(outs, ref):
        assert r.tobytes() == rr.tobytes() and a.tobytes() == ra.tobytes()
        for k in range(12):
            assert np.array_equal(i[k, :r[k]["n_inliers"]], ri[k, :rr[k]["n_inliers"]])
    # device-resident variant, two slots reused several times
    b = batches[0]
    newer = np.array([fe.node_from_features(int(b["id_newer"][k]), p["desc_newer"], p["xyz_newer"]) for k, p in enumerate(b["pairs"])], np.uint64)
    older = np.array([fe.node_from_features(int(b["id_older"][k]), p["desc_older"], p["xyz_older"]) for k, p in enumerate(b["pairs"])], np.uint64)
    for it in range(5):
        fe.submit_node_pairs(1 + it % 2, newer, older, (outs[it % 2][0], None, None), seed=31, first_pair_index=0)
    fe.wait_slot(1); fe.wait_slot(2)
    assert outs[0][0].tobytes() == ref[0][0].tobytes() and outs[1][0].tobytes() == ref[0][0].tobytes()
    for h in list(newer) + list(older):
        fe.node_destroy(int(h))


def _node_batch(fe, seed0):
    from rgbdslam_v2_b200 import synth
    b = synth.make_batch(4, 600, seed0=seed0)
    newer = np.array([fe.node_from_features(int(b["id_newer"][i]), p["desc_newer"], p["xyz_newer"]) for i, p in enumerate(b["pairs"])],
                     np.uint64)
    older = np.array([fe.node_from_features(int(b["id_older"][i]), p["desc_older"], p["xyz_older"]) for i, p in enumerate(b["pairs"])],
                     np.uint64)
    return newer, older


def _assert_same_results(a, b):
    (r, m, i), (rr, rm, ri) = a, b
    assert r.tobytes() == rr.tobytes() and m.tobytes() == rm.tobytes()
    for k in range(len(r)):  # inlier rows past n_inliers are not written
        assert np.array_equal(i[k, :r[k]["n_inliers"]], ri[k, :rr[k]["n_inliers"]])


def test_argument_and_state_errors_leave_the_library_usable(fe):
    """Bad slots, handles and states are rejected with their codes; a valid call afterwards gives the same bytes as before."""
    from rgbdslam_v2_b200._capi import KEYPOINT_DTYPE, PAIR_RESULT_DTYPE, _ptr
    _reinit(fe)
    lib = fe.lib
    newer, older = _node_batch(fe, 4100)
    ref = fe.match_node_pairs(list(newer), list(older), seed=9)
    res = np.zeros(len(newer), PAIR_RESULT_DTYPE)
    assert lib.rgbdslam_b200_match_pairs_submit(8, _ptr(newer), _ptr(older), len(newer), 9, 0, _ptr(res), None, None) == 1
    assert lib.rgbdslam_b200_match_pairs_wait(-1) == 1
    t = np.zeros(7, np.float32)
    assert lib.rgbdslam_b200_slot_stage_times(7, _ptr(t)) == 3  # slot 7 has never been submitted to
    assert lib.rgbdslam_b200_last_timing_slot(7, None, None) == 3
    bad = newer.copy()
    bad[1] = 0
    assert lib.rgbdslam_b200_match_pairs(_ptr(bad), _ptr(older), len(newer), 9, 0, _ptr(res), None, None) == 1
    comm = fe.comm_init(0, 1, fe.comm_unique_id())
    fe.wait_slot(5)
    assert lib.rgbdslam_b200_allgather_slot_edges(C.c_uint64(comm), 5, 1, _ptr(res)) == 3
    fe.comm_destroy(comm)
    kp = np.zeros(fe.node_num_features(int(newer[0])), KEYPOINT_DTYPE)
    assert lib.rgbdslam_b200_node_download_keypoints(int(newer[0]), _ptr(kp)) == 3
    again = fe.match_node_pairs(list(newer), list(older), seed=9)
    _assert_same_results(ref, again)
    for h in list(newer) + list(older):
        fe.node_destroy(int(h))


def test_rejected_match_calls_launch_nothing(fe):
    """Preconditions that the pair table decides (keypoints for the refinement, clouds for the measurement model, the z0 latch
    of a synchronous first batch) are checked before anything is queued: a rejected call launches no kernel, and the next
    submit on the same slot gives the synchronous results."""
    from rgbdslam_v2_b200._capi import _ptr
    lib = fe.lib
    _reinit(fe)
    newer, older = _node_batch(fe, 4200)
    ref = fe.match_node_pairs(list(newer), list(older), seed=13, first_pair_index=4)
    rejected = [(dict(g2o_transformation_refinement=3), 2, 4), (dict(observability_threshold=0.5), 3, 4),
                (dict(depth_cov_z0=0.0), 0, 4)]
    for kw, slot, first in rejected:
        _reinit(fe, **kw)
        out = fe._alloc_out(len(newer), True)
        launches = fe.launch_count
        rc = lib.rgbdslam_b200_match_pairs_submit(slot, _ptr(newer), _ptr(older), len(newer), 13, first, *(_ptr(a) for a in out))
        assert rc == 3, kw
        if slot == 0:
            assert lib.rgbdslam_b200_match_pairs(_ptr(newer), _ptr(older), len(newer), 13, first, *(_ptr(a) for a in out)) == 3
        assert fe.launch_count == launches, kw
        _reinit(fe)
        fe.submit_node_pairs(slot, newer, older, out, seed=13, first_pair_index=first)
        fe.wait_slot(slot)
        _assert_same_results(ref, out)
    for h in list(newer) + list(older):
        fe.node_destroy(int(h))
