"""The ORB match kernel as a binary GEMM: hd = pa + pb - 2 popcount(a & b), arg-max of the key 4096 (2c - pb) + (4095 - col).
These cases target what only that formulation can get wrong -- equal distances reached through different train popcounts
(the per-column key term), the popcount extremes 0 and 256, the extreme keys 2c - pb = +-256, the masked columns of the last
train tile and the ring of train stages -- against the oracle's bruteForceSearchORB and the SIMT kernel."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu

POPC = np.unpackbits(np.arange(256, dtype=np.uint8)[:, None], axis=1).sum(1)


def _hd(q, t):
    return POPC[q[:, None, :] ^ t[None, :, :]].sum(-1)


def _flip(row, bits):
    r = np.unpackbits(row).copy()
    r[bits] ^= 1
    return np.packbits(r)


def _equal_distance_pair(rng, q, k):
    """Two train rows at Hamming distance k from q: one clears k set bits of q (c = pa - k, pb = pa - k), the other sets k
    clear bits (c = pa, pb = pa + k) -- the same distance with popcounts 2k apart."""
    bits = np.unpackbits(q)
    ones, zeros = np.flatnonzero(bits), np.flatnonzero(bits == 0)
    lo = _flip(q, rng.choice(ones, k, replace=False))
    hi = _flip(q, rng.choice(zeros, k, replace=False))
    return lo, hi


def _crafted(nq, nt, seed):
    """Random rows (distances near 128) with planted pairs of equal distance and different train popcounts, in both orders,
    around every tile boundary, in the last (partly masked) tile and on the never-searched last row; plus rows of popcount
    0 and 256 on both sides."""
    rng = np.random.default_rng(seed)
    q = rng.integers(0, 256, (nq, 32), dtype=np.uint8)
    t = rng.integers(0, 256, (nt, 32), dtype=np.uint8)
    nsearch = nt - 1
    # disjoint column pairs, each planted for one query row, the lower-popcount row first (order 0) or second (order 1)
    pairs = [(0, 1, 0), (nsearch - 2, nsearch - 1, 1), (nsearch - 4, nsearch - 3, 0)]
    for b in range(128, nsearch, 128):
        pairs += [(b - 1, b, 0), (b - 2, b + 1, 1)]  # across the tile boundary
    used, r = set(), 0
    for c0, c1, order in pairs:
        if r >= nq - 4 or min(c0, c1) < 0 or max(c0, c1) >= nsearch or {c0, c1} & used:
            continue
        used |= {c0, c1}
        pa = int(rng.integers(64, 192))  # popcount away from the extremes
        row = np.packbits(rng.permutation(np.r_[np.ones(pa, np.uint8), np.zeros(256 - pa, np.uint8)]))
        lo, hi = _equal_distance_pair(rng, row, 3)
        q[r] = row
        t[c0], t[c1] = (lo, hi) if order == 0 else (hi, lo)
        r += 1
    free = [c for c in range(nsearch) if c not in used]
    if nq > r + 4 and len(free) >= 2:
        q[r], q[r + 1] = 0, 255  # pa = 0 and 256
        q[r + 2], q[r + 3] = 0, 255
        t[free[len(free) // 2]] = 0    # pb = 0: hd 0 for q = 0, hd 256 for q = 255
        t[free[len(free) // 3]] = 255  # pb = 256: hd 256 for q = 0, hd 0 for q = 255
    if nt >= 1:
        t[nt - 1] = q[0]         # the last train row is never examined (features.cpp:174)
    return q, t


def _both_paths(fe, q, t):
    try:
        fe.set_hamming_path(1)
        hd1, idx1 = fe.brute_force_search_orb(q, t)
        fe.set_hamming_path(0)
        hd0, idx0 = fe.brute_force_search_orb(q, t)
    finally:
        fe.set_hamming_path(1)
    return (hd1, idx1), (hd0, idx0)


@pytest.fixture(scope="module")
def fe(built):
    from rgbdslam_v2_b200 import Frontend
    from rgbdslam_v2_b200._capi import default_params
    p = default_params()
    p.depth_cov_z0 = 2.0
    f = Frontend(0, p)
    yield f
    f.close()


@pytest.mark.parametrize("nt", [1, 2, 129, 257, 1000, 4096])
@pytest.mark.parametrize("nq", [1, 300])
def test_equal_distances_with_different_train_popcounts(fe, oracle_mod, nq, nt):
    q, t = _crafted(nq, nt, seed=nq * 10007 + nt)
    if nt > 4 and nq > 1:  # the planted pairs really are ties of distance 3 reached with popcounts 6 apart
        d = _hd(q[:2], t[: nt - 1])
        assert d[0].min() == 3 and (d[0] == 3).sum() >= 2
        ties = np.flatnonzero(d[0] == 3)
        assert len(set(POPC[t[ties]].sum(1))) > 1
    (hd1, idx1), (hd0, idx0) = _both_paths(fe, q, t)
    ohd, oidx = oracle_mod.brute_force_orb(q, t)
    assert np.array_equal(hd1, ohd) and np.array_equal(idx1, oidx)
    assert np.array_equal(hd0, ohd) and np.array_equal(idx0, oidx)


@pytest.mark.parametrize("nt", [2, 129, 257, 4096])
def test_extreme_keys(fe, oracle_mod, nt):
    """2c - pb = +256 (all-ones rows on both sides: hd 0) and -256 (a zero query against all-ones train rows: hd 256, every
    column tied, index 0); all-zero train rows (2c - pb = 0 everywhere: hd = pa, index 0)."""
    q = np.zeros((6, 32), np.uint8)
    q[1] = 255
    q[2:] = np.random.default_rng(nt).integers(0, 256, (4, 32), dtype=np.uint8)
    for fill in (255, 0):
        t = np.full((nt, 32), fill, np.uint8)
        (hd1, idx1), (hd0, idx0) = _both_paths(fe, q, t)
        ohd, oidx = oracle_mod.brute_force_orb(q, t)
        assert np.array_equal(hd1, ohd) and np.array_equal(idx1, oidx), fill
        assert np.array_equal(hd0, ohd) and np.array_equal(idx0, oidx), fill
        assert (idx1 == 0).all()
        if fill == 255:
            assert hd1[0] == 256 and hd1[1] == 0
        else:
            assert np.array_equal(hd1, POPC[q].sum(1))


def test_many_items_per_cta(fe, oracle_mod):
    """A batch with several work items per persistent CTA (the train-stage ring and the A slices wrap across items) of
    crafted pairs: the kernel against the SIMT path, and each pair's query rows against the oracle."""
    sizes = [(300, 4096), (256, 257), (257, 129), (600, 2), (40, 1), (512, 1000)] * 40
    newer, older, crafted = [], [], []
    for i, (nq, nt) in enumerate(sizes):
        q, t = _crafted(nq, nt, seed=9000 + i)
        rng = np.random.default_rng(i)
        xq = np.concatenate([rng.uniform(0.5, 3, (nq, 3)), np.ones((nq, 1))], 1).astype(np.float32)
        xt = np.concatenate([rng.uniform(0.5, 3, (nt, 3)), np.ones((nt, 1))], 1).astype(np.float32)
        newer.append(fe.node_from_features(2 * i + 1, q, xq))
        older.append(fe.node_from_features(2 * i, t, xt))
        crafted.append((q, t))
    out = {}
    try:
        for path in (1, 0):
            fe.set_hamming_path(path)
            res, allm, _ = fe.match_node_pairs(newer, older, seed=5)
            out[path] = (res["n_all_matches"].copy(), allm.copy())
    finally:
        fe.set_hamming_path(1)
    assert np.array_equal(out[1][0], out[0][0])
    for i, (q, t) in enumerate(crafted):
        n = int(out[1][0][i])
        for f in ("queryIdx", "trainIdx", "distance"):
            assert np.array_equal(out[1][1][i, :n][f], out[0][1][i, :n][f]), (i, sizes[i], f)
        if n:  # every listed match is the oracle's best train row of its query row
            ohd, oidx = oracle_mod.brute_force_orb(q, t)
            qi = out[1][1][i, :n]["queryIdx"]
            assert np.array_equal(out[1][1][i, :n]["trainIdx"], oidx[qi]), (i, sizes[i])
    for h in newer + older:
        fe.node_destroy(h)
