"""The SIFT-128 ratio matcher (k_sift_prepare, tc_match256_kernel<1>, k_l2_refine, k_select_sift) against the bit-exact
restatement in sift_exact.py: tile and item edges, ties, persistent CTAs that run many work items, and the ratio
threshold compared in double."""
import ctypes as C
import itertools

import numpy as np
import pytest

import sift_exact as sx

pytestmark = pytest.mark.gpu

SHAPES = [(255, 1), (256, 2), (257, 3), (1, 4), (5, 5), (300, 127), (300, 128), (300, 129), (4095, 257), (4096, 4096),
          (513, 0)]
NODE_SIZES = [0, 1, 3, 255, 256, 257, 1000, 4096, 4096, 3000]


@pytest.fixture(scope="module")
def fe(built):
    from rgbdslam_v2_b200 import Frontend
    from rgbdslam_v2_b200._capi import default_params
    p = default_params()
    p.depth_cov_z0 = 2.0
    f = Frontend(0, p)
    yield f
    f.set_sift_matcher(0)
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


def _bits(x):
    return np.asarray(x, np.float32).view(np.uint32)


def _sift_like(rng, n):
    return np.minimum(rng.gamma(0.6, 30.0, size=(n, 128)), 255.0).astype(np.float32)


def _int_like(rng, n):
    return np.rint(_sift_like(rng, n)).astype(np.float32)


def _rows(rng, nq, nt, integer):
    """Query / train rows with true matches, duplicated train rows (one pair across the 128-column tile edge) and, for
    integer rows, queries whose five nearest train rows are exactly tied."""
    gen = _int_like if integer else _sift_like
    q, t = gen(rng, nq), gen(rng, nt)
    x = gen(rng, 1)[0]
    if nt >= 2:
        t[nt - 1] = t[0]
    if nt > 256:
        t[256] = t[255]
    ties = integer and nt >= 5
    if ties:  # five identical train rows, two of them on either side of the first tile edge when nt > 128
        cols = []
        for c in (2, 127, 128, nt // 3, nt - 3, 0, 1, 3, 4):
            if c < nt and c not in cols and len(cols) < 5:
                cols.append(c)
        t[cols] = x
    elif nt > 128:
        t[128] = t[127]
    k = min(nq, nt) // 2
    if k:
        noise = rng.normal(0, 5.0, (k, 128))
        q[:k] = np.clip(t[rng.permutation(nt)[:k]] + (np.rint(noise) if integer else noise), 0, 255)
    if nq > 0 and nt >= 1:
        q[0] = t[0]
    if nq > 2 and nt > 128:
        q[1], q[2] = t[127], np.clip(t[128] + 1, 0, 255)
    if ties:
        for i in range(3, nq, 97):
            q[i] = x if i % 2 else np.clip(x + rng.integers(-2, 3, 128), 0, 255)  # 5-way exact ties in score and distance
    return q.astype(np.float32), t.astype(np.float32)


@pytest.mark.parametrize("nq,nt", SHAPES)
def test_knn2_integer_rows_bit_exact(fe, nq, nt):
    """use_root_sift = 0 with integer rows <= 255: every bf16 operand, product and partial sum is an integer below 2^24,
    so the tensor-core scores are exact and knn2_l2 is predicted bit for bit, ties and empty slots included."""
    _reinit(fe, use_root_sift=0)
    try:
        q, t = _rows(np.random.default_rng(nq * 31 + nt), nq, nt, integer=True)
        idx, d = fe.knn2_l2(q, t)
        cand, _ = sx.candidates_bf16(q, t)
        eidx, ed = sx.knn2_from_candidates(q, t, cand)
        assert np.array_equal(idx, eidx), np.nonzero((idx != eidx).any(1))[0][:10]
        assert np.array_equal(_bits(d), _bits(ed))
        if nt < 2:
            assert (idx[:, 1] == -1).all() and (_bits(d[:, 1]) == _bits(sx.SENTINEL)).all()
    finally:
        _reinit(fe)


@pytest.mark.parametrize("nq,nt", SHAPES)
def test_knn2_root_sift_bit_exact_on_safe_rows(fe, nq, nt):
    """Default RootSIFT path: where fp32 accumulation on the tensor cores cannot change the 4-candidate set, the result
    (second neighbour included) is bit-identical to the restatement; elsewhere it is the exact fp32 2-NN of one of the
    4-subsets of the restated top 5."""
    q, t = _rows(np.random.default_rng(nq * 37 + nt), nq, nt, integer=False)
    idx, d = fe.knn2_l2(q, t)
    qr, tr = sx.root_sift_f32(q), sx.root_sift_f32(t)
    cand, safe = sx.candidates_bf16(qr, tr)
    eidx, ed = sx.knn2_from_candidates(qr, tr, cand)
    assert np.array_equal(idx[safe], eidx[safe])
    assert np.array_equal(_bits(d[safe]), _bits(ed[safe]))
    uns = np.nonzero(~safe)[0]
    print(f"nq={nq} nt={nt}: {len(uns)} unsafe rows")
    if len(uns):
        top5, _ = sx.candidates_bf16(qr[uns], tr, depth=5)
        for r, i in enumerate(uns):
            options = [sx.knn2_from_candidates(qr[i:i + 1], tr, np.array([s], np.int32))
                       for s in itertools.combinations(top5[r], 4)]
            assert any(np.array_equal(idx[i], oi[0]) and np.array_equal(_bits(d[i]), _bits(od[0])) for oi, od in options), i
    # The flag is a property of the input, computed on the CPU: 103 of the 10,378 query rows of these shapes are unsafe
    # (1.0 %, at most 2.3 % in one shape, 2 of 5 rows at 5 x 5), mostly duplicated train rows tied at ranks 4 and 5.
    # On every one of them ranks 1-3 and ranks 6+ are certain, so the 4-subsets of the top 5 cover the GPU's choice.
    assert len(uns) <= max(2, 0.025 * nq)


def _batch_rows(rng, sizes, integer):
    """Nodes drawn from one pool of scene descriptors plus noise, so every pair of nodes shares true matches."""
    pool = _sift_like(rng, 6000)
    out = []
    for n in sizes:
        noise = rng.normal(0, 4.0, (n, 128))
        d = np.clip(pool[rng.choice(len(pool), n, replace=False)] + noise, 0, 255)
        out.append((np.rint(d) if integer else d).astype(np.float32))
    return out


def _xyz(rng, n):
    return np.concatenate([rng.uniform(0.5, 3, (n, 3)), np.ones((n, 1))], 1).astype(np.float32)


def _sm_count():
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


@pytest.mark.parametrize("integer", [True, False], ids=["int", "root"])
def test_batched_ratio_matcher_equals_single_pair_restatement(fe, integer):
    """One match_node_pairs call of 90 pairs over ragged nodes (486 work items of 256 queries, more than 3 per CTA of the
    persistent grid): every pair's match list equals select_ratio(knn2_l2(q, t)) exactly, at max_matches 512 and 300."""
    rng = np.random.default_rng(11 if integer else 12)
    _reinit(fe, use_root_sift=0 if integer else 1, max_matches=512)
    handles = []
    try:
        desc = _batch_rows(rng, NODE_SIZES, integer)
        handles = [fe.node_from_sift(i, d, _xyz(rng, len(d))) for i, d in enumerate(desc)]
        pairs = [(i, j) for i in range(len(desc)) for j in range(len(desc)) if i != j]
        items = sum((len(desc[i]) + 255) // 256 for i, _ in pairs)
        sm = _sm_count()
        print(f"{len(pairs)} pairs, {items} work items, {min(items, sm)} CTAs")
        assert items > 3 * sm
        knn = [fe.knn2_l2(desc[i], desc[j]) for i, j in pairs]
        assert max(len(sx.select_ratio(k, 0.95, 4096)) for k in knn) > 512  # the cap binds at both settings
        for max_matches in (512, 300):
            _reinit(fe, use_root_sift=0 if integer else 1, max_matches=max_matches)
            res, allm, _ = fe.match_node_pairs([handles[i] for i, _ in pairs], [handles[j] for _, j in pairs], seed=5)
            for p, (i, j) in enumerate(pairs):
                exp = sx.select_ratio(knn[p], 0.95, max_matches)
                n = int(res[p]["n_all_matches"])
                assert n == len(exp), (i, j, max_matches)
                got = allm[p, :n]
                assert np.array_equal(got["queryIdx"], exp["queryIdx"]), (i, j, max_matches)
                assert np.array_equal(got["trainIdx"], exp["trainIdx"]), (i, j, max_matches)
                assert np.array_equal(_bits(got["distance"]), _bits(exp["distance"])), (i, j, max_matches)
    finally:
        for h in handles:
            fe.node_destroy(h)
        _reinit(fe)


def _unit_pool(rng, n):
    d = rng.gamma(0.6, 1.0, size=(n, 128))
    d /= np.linalg.norm(d, axis=1, keepdims=True)
    d = np.minimum(d, 0.2)
    return d / np.linalg.norm(d, axis=1, keepdims=True)


def test_batched_siftgpu_matcher_is_bit_exact(fe):
    """set_sift_matcher(1) on the same ragged batch, 45 pairs: both GetSiftMatch passes give 486 work items, more than
    3 per CTA, and every match list equals the restated SiftMatchGPU + SiftGPUWrapper::match."""
    from oracle import sift_oracle
    rng = np.random.default_rng(13)
    pool = _unit_pool(rng, 6000)
    desc = []
    for n in NODE_SIZES:
        d = np.abs(pool[rng.choice(len(pool), n, replace=False)] + rng.normal(0, 0.01, (n, 128)))
        desc.append(d.astype(np.float32))
    fe.set_sift_matcher(1)
    handles = []
    try:
        handles = [fe.node_from_sift(i, d, _xyz(rng, len(d))) for i, d in enumerate(desc)]
        pairs = list(itertools.combinations(range(len(desc)), 2))
        items = sum((len(desc[i]) + 255) // 256 + (len(desc[j]) + 255) // 256 for i, j in pairs)
        sm = _sm_count()
        print(f"{len(pairs)} pairs, {items} work items, {min(items, sm)} CTAs")
        assert items > 3 * sm
        res, allm, _ = fe.match_node_pairs([handles[i] for i, _ in pairs], [handles[j] for _, j in pairs], seed=3)
        total = 0
        for p, (i, j) in enumerate(pairs):
            exp = sift_oracle.siftgpu_feature_matching(desc[i], desc[j], max_matches=300)
            n = int(res[p]["n_all_matches"])
            assert n == len(exp), (i, j)
            got = allm[p, :n]
            assert np.array_equal(got["queryIdx"], exp["queryIdx"]) and np.array_equal(got["trainIdx"], exp["trainIdx"])
            assert np.array_equal(_bits(got["distance"]), _bits(exp["distance"])), (i, j)
            total += n
        assert total > 3000
    finally:
        fe.set_sift_matcher(0)
        for h in handles:
            fe.node_destroy(h)


def test_ratio_threshold_compared_in_double(fe):
    """Squared distances (19, 20), (20, 21), (18, 19): the ratio fl32(19/20) = fl32(0.95) = 0.949999988 is below the
    double threshold 0.95, so the reference's `double > float` comparison accepts the first query."""
    _reinit(fe, use_root_sift=0)
    handles = []
    try:
        q, t = sx.threshold_rows()
        idx, d = fe.knn2_l2(q, t)
        assert idx.tolist() == [[0, 1], [2, 3], [4, 5]] and d.tolist() == [[19, 20], [20, 21], [18, 19]]
        rng = np.random.default_rng(0)
        handles = [fe.node_from_sift(1, q, _xyz(rng, 3)), fe.node_from_sift(0, t, _xyz(rng, 6))]
        res, allm, _ = fe.match_node_pairs([handles[0]], [handles[1]], seed=1)
        n = int(res[0]["n_all_matches"])
        got = allm[0, :n]
        assert got["queryIdx"].tolist() == [2, 0] and got["trainIdx"].tolist() == [4, 0]
        assert _bits(got["distance"][1]) == _bits(np.float32(0.95))
    finally:
        for h in handles:
            fe.node_destroy(h)
        _reinit(fe)
