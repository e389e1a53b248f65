"""The planted OctoMap and occupancy-filter cases (tests/octomap_planted.py) reach the edges they are named for, on the C
oracles: a case that misses its edge would let the GPU comparison (tests/test_gpu_octomap_edges.py) pass without testing
anything."""
import numpy as np
import pytest

import octomap_exact as ox
import octomap_planted as op
from test_octomap_oracle_cpu import leaves

F32 = np.float32
CASES = op.CASES


def lo(p):
    return F32(np.log(p / (1 - p)))


def of(name):
    return [c for n, c in CASES.items() if n.startswith(name + "-")]


def write(case, scans=None):
    return op.oracle(case, scans).write()


def morton(k):
    return sum(((k[a] >> b) & 1) << (3 * b + a) for b in range(16) for a in range(3))


def test_every_case_is_checked_here():
    names = {"ray-walk", "long-rays", "corners", "reduction", "clamping", "clamping-exact", "colour-order", "colour-range",
             "max-range", "short-range", "merge", "empty", "empty-after"}
    assert {n.rsplit("-", 1)[0] for n in CASES} == names
    for c in CASES.values():
        assert all(len(s.local) <= op.SLOTS for s in c.scans) and len(c.scans) >= 1
        cl = op.clouds(c.scans[:2])
        assert cl.shape == (min(2, len(c.scans)), op.H, op.W, 8)


@pytest.mark.parametrize("res", op.EXACT + op.INEXACT)
def test_ray_walk_ties_borders_zero_components_and_key_32768(res):
    c = CASES[f"ray-walk-{res:g}"]
    ties, corner, axis, cross, diag, diag_back, tiny = c.scans
    if res in op.EXACT:
        # centre to centre along the tie directions: every tMax ties, and the tie goes to the last tied axis (y before x,
        # z before x or y) on the first step
        for p, d in zip(ties.pts, op.TIE_DIRS):
            r = ox.ray_keys(ties.origin, p, res)
            step = np.flatnonzero(r[1].astype(int) - r[0].astype(int))
            assert len(step) == 1 and step[0] == max(i for i in range(3) if d[i]), d
        # the corner origin sits on a border on every axis
        assert all(float(v) / res == np.floor(float(v) / res) for v in corner.origin)
    for p in corner.pts:
        assert len(ox.ray_keys(corner.origin, p, res)) > 1
    # one and two zero direction components, and an end in the origin's voxel
    same = [int((p == axis.origin).sum()) for p in axis.pts]
    assert 1 in same and 2 in same
    assert op.keys3(res, axis.pts[-1]) == op.keys3(res, axis.origin) and len(ox.ray_keys(axis.origin, axis.pts[-1], res)) == 0
    assert op.keys3(res, axis.pts[-1]) in leaves(write(c, [axis]))
    # rays across coordinate 0: keys 32767 and 32768 on one ray
    for s in (cross, diag, diag_back):
        for p in s.pts:
            r = ox.ray_keys(s.origin, p, res)
            assert any({32767, 32768} <= set(r[:, a].tolist()) for a in range(3))
    # a component that rounds to 0 in the float division, and one that stays subnormal
    d = (tiny.pts - tiny.origin).astype(F32)
    n = np.sqrt((d.astype(F32) ** 2).sum(1, dtype=F32).astype(np.float64)).astype(F32)
    q = (d / n[:, None]).astype(F32)
    assert q[0, 1] == 0 and d[0, 1] != 0 and q[1, 1] == 0 and d[1, 1] != 0
    assert q[2, 1] != 0 and abs(q[2, 1]) < np.finfo(F32).tiny


def test_long_rays():
    c = CASES["long-rays-0.001"]
    s = c.scans[0]
    n = [len(ox.ray_keys(s.origin, p, 0.001)) for p in s.pts]
    assert min(n) >= 10_000 and max(n) >= 50_000 and max(n) <= 60_000


@pytest.mark.parametrize("res", op.EXACT + op.INEXACT)
def test_corners_reach_keys_0_and_65535(res):
    c = CASES[f"corners-{res:g}"]
    lo_, hi = op.key_edges(res)
    if res in op.EXACT:
        assert lo_ == F32(-32768 * res)
    assert op.key(res, lo_) == 0 and op.key(res, hi) == 65535
    assert op.key(res, op.outside(lo_)) is None and op.key(res, op.outside(hi)) is None
    lv = leaves(write(c))
    for k in range(8):
        corner = tuple(65535 if (k >> a) & 1 else 0 for a in range(3))
        assert corner in lv
        pts = c.scans[k].pts
        assert op.keys3(res, pts[0]) == corner  # the corner itself
        assert sum(op.keys3(res, p) is None for p in pts) == 4  # just outside on each axis, and on all three
    # the origin on the low corner
    assert op.keys3(res, c.scans[8].origin) == (0, 0, 0)
    # an origin outside the tree: no ray, the occupied cells stay (log-odds of one hit)
    out = c.scans[9]
    assert op.keys3(res, out.origin) is None
    one = leaves(write(c, [out]))
    assert sorted(one) == sorted(op.keys3(res, p) for p in out.pts)
    assert all(v[0] == lo(0.9) for v in one.values())
    # +-inf and NaN coordinates contribute nothing: the scan leaves the one finite point's ray
    bad = c.scans[10]
    assert (~np.isfinite(bad.pts).all(1)).sum() == 5
    assert leaves(write(c, [bad])) == leaves(write(c, [op.scan(bad.origin, bad.pts[-1:], bad.rgb[-1:])]))


@pytest.mark.parametrize("res", [1.0, 0.05])
def test_per_scan_reduction(res):
    c = CASES[f"reduction-{res:g}"]
    s1, s2, _ = c.scans
    X = op.keys3(res, s1.pts[3])
    through = [p for p in s1.pts if any(tuple(k) == X for k in ox.ray_keys(s1.origin, p, res))]
    assert len(through) >= 3  # freed by several rays and hit by one point in one scan: one hit
    assert leaves(write(c, [s1]))[X][0] == lo(0.9)
    Y = op.keys3(res, s1.pts[6])
    assert sum(op.keys3(res, p) == Y for p in s1.pts) == 3
    # freed in scan 1, hit in scan 2
    K = op.keys3(res, s2.pts[0])
    assert leaves(write(c, [s1]))[K][0] == lo(0.4)
    assert leaves(write(c, [s1, s2]))[K][0] == F32(lo(0.4) + lo(0.9))


def _sum(updates):
    t = F32(0)
    for u in updates:
        t = F32(t + u)
    return t


@pytest.mark.parametrize("name", [n for n in CASES if n.startswith("clamping")])
def test_clamping_depends_on_the_scan_order(name):
    c = CASES[name]
    assert 20 <= len(c.scans) <= 40
    assert write(c) != write(c, c.scans[::-1])
    kw = dict(prob_hit=0.9, prob_miss=0.4, clamping_min=0.001, clamping_max=0.999) | c.kw
    hit, miss, cmin, cmax = lo(kw["prob_hit"]), lo(kw["prob_miss"]), lo(kw["clamping_min"]), lo(kw["clamping_max"])
    lv = leaves(write(c))
    A = op.keys3(c.res, c.scans[0].origin)
    top = op.keys3(c.res, c.scans[0].pts[-1])
    n = len(c.scans)
    assert lv[top][0] == cmax and _sum([hit] * n) != cmax
    assert lv[A][0] == cmin and _sum([miss] * n) != cmin
    if c.kw:  # one update from 0 lands exactly on each clamp value
        assert F32(0 + hit) == cmax and F32(0 + miss) == cmin
    else:  # the cells of the alternation end between the clamps
        H = op.keys3(c.res, c.scans[0].pts[0])
        assert cmin < lv[H][0] < cmax


@pytest.mark.parametrize("res", [1.0, 0.05])
def test_colour_order(res):
    c = CASES[f"colour-order-{res:g}"]
    s = c.scans[0]
    ks = {op.keys3(res, p) for p in s.pts}
    assert len(s.pts) > 4096 and len(ks) == 1 and len(np.unique(s.rgb & 0xFFFFFF)) > 4000
    assert (s.rgb == op.WHITE).any() and (s.rgb == 0x80FFFFFF).any() and ((s.rgb >> 24) == 0xFF).any()
    assert op.slots(len(s.pts))[-1] >= 4 * 1024
    rev = op.scan(s.origin, s.pts[::-1], s.rgb[::-1])
    assert write(c) != write(c, [rev] + c.scans[1:])


@pytest.mark.parametrize("res", [1.0, 0.05])
def test_colour_and_max_range(res):
    c = CASES[f"colour-range-{res:g}"]
    s1, s2, s3 = c.scans
    o = s1.origin
    p1, p2, p3 = s1.pts
    # p1 beyond max_range, its cell on p2's free ray: its colour lands in that scan
    assert op._norm(o, p1) > c.max_range >= op._norm(o, p2)
    k1 = op.keys3(res, p1)
    assert any(tuple(k) == k1 for k in ox.ray_keys(o, p2, res))
    lv = leaves(write(c, [s1]))
    assert lv[k1][1] == tuple(int(v) for v in ((s1.rgb[0] >> 16) & 255, (s1.rgb[0] >> 8) & 255, s1.rgb[0] & 255))
    # p3's cell has no leaf in its scan; scan 2 makes it, and the same cell's colour of scan 3 lands
    k3 = op.keys3(res, p3)
    assert op._norm(o, p3) > c.max_range and k3 not in lv
    assert op.keys3(res, s2.pts[0]) == k3 == op.keys3(res, s3.pts[0])
    a, b = leaves(write(c, [s1, s2]))[k3][1], leaves(write(c))[k3][1]
    assert a != b and b != (255, 255, 255)


@pytest.mark.parametrize("res", [1.0, 0.05])
def test_max_range_edges(res):
    c = CASES[f"max-range-{res:g}"]
    eq, above, far = c.scans
    assert op._norm(eq.origin, eq.pts[0]) == c.max_range
    assert op.keys3(res, eq.pts[0]) in leaves(write(c, [eq]))
    assert op._norm(above.origin, above.pts[0]) > c.max_range  # shortened: the point's own cell is not hit
    got = leaves(write(c, [above]))
    assert op.keys3(res, above.pts[0]) not in got and len(got) >= 2
    assert op.keys3(res, far.pts[0]) is None and len(leaves(write(c, [far]))) >= 3
    sr = CASES[f"short-range-{res:g}"]
    s = sr.scans[0]
    assert sorted(leaves(write(sr))) == [op.keys3(res, s.origin)]  # every shortened ray ends in the origin's voxel
    assert sum(op._norm(s.origin, p) > sr.max_range for p in s.pts) == 3


@pytest.mark.parametrize("res", [1.0, 0.0625, 0.05])
def test_merge_order_and_full_parents(res):
    c = CASES[f"merge-{res:g}"]
    seen = []
    for i, s in enumerate(c.scans[:10]):
        k = morton(op.keys3(res, s.pts[0]))
        assert len(ox.ray_keys(s.origin, s.pts[0], res)) == 0
        if i == 2:
            assert k < min(seen)
        elif i == 3:
            assert k > max(seen)
        elif i >= 4:
            assert min(seen) < k < max(seen)
        seen.append(k)
    assert len(set(seen)) == 10
    _, _, rec = ox.parse(write(c))
    kids = np.unpackbits(rec["children"][:, None], axis=1).sum(1)
    assert (kids == 8).sum() >= 8
    # each block's parent: the int mean of its 1..8 coloured children
    lv = leaves(write(c))
    for j, s in enumerate(c.scans[10:]):
        cols = [lv[op.keys3(res, p)][1] for p in s.pts]
        set_ = [x for x in cols if x != (255, 255, 255)]
        assert len(set_) == j + 1
        if j:
            mean = tuple(sum(x[i] for x in set_) // len(set_) for i in range(3))
            assert mean != set_[0]


@pytest.mark.parametrize("res", [1.0, 0.0625, 0.05])
def test_empty_scans_insert_nothing(res):
    c = CASES[f"empty-{res:g}"]
    m = op.oracle(c)
    assert m.stats() == (0, 0) and m.write() == ox.Oracle(res).write()
    # the last scan has points with keys: entries on the device, no leaf
    assert all(op.keys3(res, p) is not None for p in c.scans[-1].pts)
    a = CASES[f"empty-after-{res:g}"]
    assert op.oracle(a).write() == write(a, a.scans[:1]) and op.oracle(a, a.scans[:1]).stats()[1] == 1


# ---- the occupancy filter --------------------------------------------------------------------------------------------------

@pytest.fixture(scope="module", params=[1.0, 0.05])
def fmap(request):
    res = request.param
    m = op.filter_oracle(res)
    lv = leaves(m.write())
    return res, m, lv, op.filter_cases(res, lv)


def test_filter_map_is_the_insert_map(fmap):
    res, m, lv, _ = fmap
    assert m.write() == op.oracle(op.filter_map(res)).write()


def test_filter_wraps_reach_the_far_side(fmap):
    res, m, lv, fc = fmap
    f = fc[f"wrap-{res:g}"]
    far = zwrap = 0
    for p in f.pts:
        own = [op.key(res, v) for v in p]
        for c in op.visited(res, f.sensor7, p):
            if c in lv and any(abs(a - b) > 32768 for a, b in zip(c, own)):
                far += 1
        kz = own[2]
        zwrap += kz == 65535 and (kz - 1 + 2) & 0xFFFF == 0 and (op.visited(res, f.sensor7, p)[2] in lv)
    assert far >= 8 and zwrap >= 1
    keep = m.occupancy_filter(f.pts, f.sensor7[:4], f.sensor7[4:], f.thresholds[2])
    assert 0 < keep.sum() < len(keep)


def test_filter_int_range_nan_and_no_leaf(fmap):
    res, m, lv, fc = fmap
    f = fc[f"int-range-{res:g}"]
    v = np.floor((1.0 / res) * f.pts.astype(np.float64))
    assert ((np.abs(v) >= 2.0 ** 31) & np.isfinite(v)).any() and np.isinf(f.pts).any()
    assert ((v >= -(2.0 ** 31)) & (v < 2.0 ** 31) & (np.abs(v) > 2.0 ** 31 - 2 ** 9)).sum() >= 2  # the ends inside int range
    keep = m.occupancy_filter(f.pts, f.sensor7[:4], f.sensor7[4:], np.inf)
    assert keep[:3].any()  # a key from INT_MIN finds a leaf
    nan_x = np.flatnonzero(np.isnan(f.pts[:, 0]))[0]
    assert np.isfinite(f.pts[nan_x, 2]) and op.visited(res, f.sensor7, f.pts[nan_x]) is None and not keep[nan_x]
    lonely = f.pts[-1]
    assert not any(c in lv for c in op.visited(res, f.sensor7, lonely)) and not keep[-1]
    t = fc[f"int-range-turned-{res:g}"]
    assert not np.array_equal(t.sensor7, op.IDENTITY7)


def test_filter_near_points_decide_both_ways(fmap):
    res, m, lv, fc = fmap
    for name in (f"near-{res:g}", f"near-turned-{res:g}"):
        f = fc[name]
        n = [int(m.occupancy_filter(f.pts, f.sensor7[:4], f.sensor7[4:], t).sum()) for t in f.thresholds]
        assert any(0 < k < len(f.pts) for k in n) and len(set(n)) >= 3, (name, n)


def test_filter_tie_is_exact(fmap):
    res, m, lv, fc = fmap
    f = fc[f"tie-{res:g}"]
    so, sw = op.filter_sums(res, lv, f.sensor7, f.pts[0])
    thr, above = f.thresholds
    assert so == thr * sw and above == np.nextafter(thr, np.inf)
    assert not m.occupancy_filter(f.pts, f.sensor7[:4], f.sensor7[4:], thr)[0]
    assert m.occupancy_filter(f.pts, f.sensor7[:4], f.sensor7[4:], above)[0]
