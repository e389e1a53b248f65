"""CPU self-tests of tests/sift_exact.py, the bit-exact restatement of the SIFT-128 ratio matcher's GPU stages."""
from fractions import Fraction

import numpy as np
import pytest

import sift_exact as sx


def _bits(x):
    return np.asarray(x, np.float32).view(np.uint32)


def _f32(bits):
    return np.asarray(bits, np.uint32).view(np.float32)


def test_bf16_rne_matches_torch():
    torch = pytest.importorskip("torch")
    rng = np.random.default_rng(0)
    special = _f32([
        0x00000000, 0x80000000,              # +-0
        0x3F808000, 0xBF808000,              # exact tie, even below: rounds down
        0x3F818000, 0xBF818000,              # exact tie, odd below: rounds up
        0x3F808001, 0x3F807FFF,              # just above / below a tie
        0x00008000, 0x00018000, 0x00007FFF,  # subnormal ties and a subnormal that rounds to 0
        0x0000C000, 0x807FFFFF,              # subnormal that rounds up; -largest subnormal (rounds to -smallest normal)
        0x7F7FFFFF, 0xFF7FFFFF,              # largest float: rounds to +-inf
        0x7F800000, 0xFF800000,              # +-inf
    ])
    rand = np.concatenate([
        rng.standard_normal(4000).astype(np.float32) * np.float32(2.0) ** rng.integers(-140, 120, 4000).astype(np.float32),
        _f32(rng.integers(0, 2 ** 32, 4000, dtype=np.uint64).astype(np.uint32)),
    ])
    x = np.concatenate([special, rand])
    x = x[~np.isnan(x)]
    want = torch.from_numpy(x.copy()).to(torch.bfloat16).to(torch.float32).numpy()
    got = sx.bf16_rne(x)
    assert np.array_equal(_bits(got), _bits(want))
    assert _bits(sx.bf16_rne(_f32([0x3F808000])))[0] == 0x3F800000
    assert _bits(sx.bf16_rne(_f32([0x3F818000])))[0] == 0x3F820000
    assert np.isnan(sx.bf16_rne(np.float32(np.nan)))


def _round_exact(x: Fraction) -> np.float32:
    """Independent reference: the float32 nearest to x, ties to even mantissa."""
    f = np.float32(float(x))
    best = None
    for c in (np.nextafter(f, np.float32(-np.inf)), f, np.nextafter(f, np.float32(np.inf))):
        key = (abs(Fraction(float(c)) - x), int(_bits(c)) & 1)
        if best is None or key < best[0]:
            best = (key, c)
    return best[1]


def _check_fma(a, b, c):
    got = sx.fma32(a, b, c)
    for i in range(len(a)):
        want = _round_exact(Fraction(float(a[i])) * Fraction(float(b[i])) + Fraction(float(c[i])))
        assert _bits(got[i]) == _bits(want), (a[i], b[i], c[i], got[i], want)


def test_fma32_random_inputs():
    rng = np.random.default_rng(1)
    n = 3000
    a = (rng.standard_normal(n) * 2.0 ** rng.integers(-30, 30, n)).astype(np.float32)
    b = (rng.standard_normal(n) * 2.0 ** rng.integers(-30, 30, n)).astype(np.float32)
    c = (rng.standard_normal(n) * 2.0 ** rng.integers(-60, 60, n)).astype(np.float32)
    c[::3] = -(a[::3] * b[::3])  # heavy cancellation
    _check_fma(a, b, c)


def test_fma32_double_rounding_midpoints():
    """a * b lands exactly on a float32 midpoint, c nudges it by far less than a float64 ulp: the float64 sum rounds
    back onto the midpoint, and a plain float64 -> float32 conversion would round the wrong way."""
    a, b, c = [], [], []
    for i in (1, 3, 5, 7, 9, 101):
        for j in (1, 3, 5, 11):
            for e in (-20, 0, 17):
                for nudge in (0.0, 2.0 ** -80, -(2.0 ** -80), 2.0 ** -100):
                    s = 2.0 ** e
                    a.append((1 + i * 2.0 ** -12) * s)
                    b.append(1 + j * 2.0 ** -12)
                    c.append(nudge * s)
    a, b, c = (np.array(v, np.float32) for v in (a, b, c))
    p = a.astype(np.float64) * b.astype(np.float64)
    assert (p != p.astype(np.float32).astype(np.float64)).all()  # every product is a float32 midpoint
    plain = (p + c.astype(np.float64)).astype(np.float32)
    got = sx.fma32(a, b, c)
    assert (_bits(got) != _bits(plain)).sum() > 0  # the constructed cases do hit the double-rounding trap
    _check_fma(a, b, c)


def test_root_sift_f32_vs_oracle():
    from oracle import sift_oracle
    rng = np.random.default_rng(2)
    d = np.minimum(rng.gamma(0.6, 30.0, size=(3000, 128)), 255.0).astype(np.float32)
    d[:500] = np.rint(d[:500])
    d[7] = 0.0                                     # zero rows are left alone
    d[8] = -d[9]                                   # abs() first
    got, want = sx.root_sift_f32(d), sift_oracle.root_sift(d)
    a = np.abs(d)
    s_gpu = sx._butterfly((a[:, 0::4] + a[:, 1::4]) + (a[:, 2::4] + a[:, 3::4]))
    s_np = a.sum(1, dtype=np.float32)  # NumPy's pairwise order
    same = s_gpu == s_np
    assert same.sum() > 1000 and (~same).sum() > 100  # both kinds of rows occur
    assert np.array_equal(_bits(got[same]), _bits(want[same]))
    # elsewhere the two sums are a few ulps apart; sqrt(v / s) moves by half of that plus the two roundings
    ulps = np.abs(_bits(got).astype(np.int64) - _bits(want).astype(np.int64)).max(1)
    sum_ulps = np.abs(_bits(s_gpu).astype(np.int64) - _bits(s_np).astype(np.int64))
    assert (ulps <= sum_ulps + 1).all() and sum_ulps.max() <= 2
    assert np.array_equal(got[7], d[7]) and np.array_equal(got[8], got[9])


def test_l2_f32_is_exact_on_integer_rows_and_close_on_root_rows():
    rng = np.random.default_rng(3)
    a = rng.integers(0, 256, (200, 128)).astype(np.float32)
    b = rng.integers(0, 256, (200, 128)).astype(np.float32)
    exact = ((a.astype(np.int64) - b.astype(np.int64)) ** 2).sum(1)
    assert np.array_equal(sx.l2_f32(a, b), exact.astype(np.float32))
    ra, rb = sx.root_sift_f32(a), sx.root_sift_f32(b)
    ex = ((ra.astype(np.float64) - rb.astype(np.float64)) ** 2).sum(1)
    assert np.abs(sx.l2_f32(ra, rb) - ex).max() < 1e-5


def test_candidates_and_refine_ties_on_integer_rows():
    """Equal scores keep the lower column, nt < 4 leaves -1 slots, equal distances keep the lower index."""
    rng = np.random.default_rng(4)
    t = rng.integers(0, 40, (300, 128)).astype(np.float32)
    x = rng.integers(0, 40, 128).astype(np.float32)
    t[[3, 127, 128, 200, 299]] = x                 # five identical rows, two of them across the 128-column tile edge
    q = np.stack([x, x + 1, rng.integers(0, 40, 128).astype(np.float32)])
    cand, _ = sx.candidates_bf16(q, t)
    assert cand[0].tolist() == [3, 127, 128, 200] and cand[1].tolist() == [3, 127, 128, 200]
    idx, d = sx.knn2_from_candidates(q, t, cand)
    assert idx[0].tolist() == [3, 127] and d[0].tolist() == [0.0, 0.0]
    assert idx[1].tolist() == [3, 127] and d[1].tolist() == [128.0, 128.0]
    cand, safe = sx.candidates_bf16(q, t[:2])
    assert (cand[:, 2:] == -1).all() and safe.all()
    idx, d = sx.knn2_from_candidates(q, t[:1], sx.candidates_bf16(q, t[:1])[0])
    assert (idx[:, 0] == 0).all() and (idx[:, 1] == -1).all() and (d[:, 1] == np.float32(3.0e38)).all()
    idx, d = sx.knn2_from_candidates(q, t[:0], sx.candidates_bf16(q, t[:0])[0])
    assert (idx == -1).all() and (d == np.float32(3.0e38)).all()


def _knn(rows):
    idx = np.array([r[0] for r in rows], np.int32)
    d = np.array([r[1] for r in rows], np.float32)
    return idx, d


def test_select_ratio_threshold_in_double():
    m = sx.select_ratio(_knn([([0, 1], [19, 20]), ([2, 3], [20, 21]), ([4, 5], [18, 19]), ([6, 7], [7, 7]),
                              ([8, 9], [0, 0]), ([10, -1], [1, 3e38])]), 0.95, 300)
    # 19/20 rounds to fl32(0.95) = 0.949999988...: below the double 0.95, so the reference accepts it
    assert m["queryIdx"].tolist() == [2, 0]
    assert _bits(m["distance"][1]) == _bits(np.float32(0.95))
    assert m["trainIdx"].tolist() == [4, 0]


def test_select_ratio_first_passing_query_owns_the_train_row():
    m = sx.select_ratio(_knn([([5, 1], [9, 10]), ([3, 1], [1, 10]), ([5, 2], [1, 100]), ([4, 1], [1, 2])]), 0.95, 300)
    # query 2 has the best ratio for train row 5 but query 0 passed first ("FIXME: Keep better", node.cpp:655-656)
    assert m["queryIdx"].tolist() == [1, 3, 0] and m["trainIdx"].tolist() == [3, 4, 5]


def test_select_ratio_cap_orders_equal_ratios_by_query():
    rows = [([100 + i, 0], [3, 4]) for i in range(8)] + [([50, 0], [1, 4]), ([51, 0], [1, 2])]
    m = sx.select_ratio(_knn(rows[::-1]), 0.95, 5)  # queries 0, 1 carry the better ratios, 2..9 tie at 0.75
    assert m["queryIdx"].tolist() == [1, 0, 2, 3, 4]
    assert len(sx.select_ratio(_knn(rows), 0.95, 512)) == 10


def test_select_ratio_and_oracle_accept_the_fl32_threshold_ratio():
    from oracle import sift_oracle
    q, t = sx.threshold_rows()
    idx, d = sx.knn2_from_candidates(q, t, sx.candidates_bf16(q, t)[0])
    assert d.tolist() == [[19, 20], [20, 21], [18, 19]]
    m = sx.select_ratio((idx, d), 0.95, 300)
    o = sift_oracle.feature_matching(q, t, 0.95, 300)
    assert m["queryIdx"].tolist() == [2, 0] and m["trainIdx"].tolist() == [4, 0]
    assert np.array_equal(o["queryIdx"], m["queryIdx"]) and np.array_equal(o["trainIdx"], m["trainIdx"])
    assert np.array_equal(_bits(o["distance"]), _bits(m["distance"]))
