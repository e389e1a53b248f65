"""Planted scans for the colour OctoMap and its occupancy filter (DESIGN.md 4.14, 4.15): named cases of a few points each,
placed where the rules turn -- exact tMax ties, voxel borders, zero and vanishing direction components, the key range's
ends, the per-scan reduction, clamping, colour order, max_range, the merge and the writer, scans that insert nothing --
and the builders that turn a case into Node-constructor input.

A scan is a ray origin and its points, planted in map coordinates.  Its node is an organised PointXYZRGB cloud of W x H
slots, NaN but for the planted points (spread over the slots in order, so that they fall in several 1024-point blocks),
which hold p - o in float32 under the float 3 x 4 [I | o]; the map points are map_point's ((1 x + 0 y) + 0 z) + o of
those, which is p itself wherever the cases need it (the edge tests in test_octomap_planted_cpu.py check that).
W x H is the smallest frame the Node constructor takes with the ungridded detector: level 7 of its one ORB cell keeps
40 px."""
from dataclasses import dataclass, field

import numpy as np

import octomap_exact as ox
import octomap_filter_exact as fx

F32 = np.float32
W = H = 144
SLOTS = W * H
WHITE = 0xFFFFFF
EXACT = (1.0, 0.0625)  # resolutions whose cell borders and centres are float32 values
INEXACT = (0.05, 0.08, 0.001)


@dataclass
class Scan:
    origin: np.ndarray  # (3,) float32, the transform's translation
    local: np.ndarray  # (n, 3) float32 points as the node stores them
    rgb: np.ndarray  # (n,) uint32 colour words

    @property
    def pts(self):
        """the map points the device and the oracle read (ox.transform of the stored points)"""
        return ox.transform(stored(self), transform(self))


@dataclass
class Case:
    name: str
    res: float
    scans: list
    kw: dict = field(default_factory=dict)  # octomap parameters besides the resolution
    max_range: float | None = None  # None: no limit
    calls: list | None = None  # the case's own split of its scans into octomap_insert calls (counts)

    @property
    def params(self):
        return dict(resolution=self.res, **self.kw)


def scan(origin, pts, rgb=None):
    pts = np.asarray(pts, F32).reshape(-1, 3)
    o = np.asarray(origin, F32).reshape(3)
    if rgb is None:
        rgb = (np.arange(len(pts), dtype=np.uint32) * np.uint32(0x9E3779B1) >> np.uint32(8)) % np.uint32(WHITE)
    with np.errstate(invalid="ignore"):
        local = (pts - o).astype(F32)
    return Scan(o, local, np.asarray(rgb, np.uint32).reshape(-1))


# ---- keys and the tree's borders -------------------------------------------------------------------------------------------

def key(res, c):
    """coordToKeyChecked of one float32 coordinate: the key, or None outside [0, 65536)"""
    with np.errstate(invalid="ignore"):
        v = np.floor((1.0 / res) * np.float64(F32(c)))
    return int(v) + 32768 if -32768.0 <= v < 32768.0 else None


def keys3(res, p):
    k = [key(res, c) for c in p]
    return None if None in k else tuple(k)


def key_edges(res):
    """(lo, hi): the smallest and the largest float32 coordinate with a key"""
    up, down = F32(np.inf), F32(-np.inf)
    lo = F32(-32768 * res)
    while key(res, lo) is None:
        lo = np.nextafter(lo, up)
    while key(res, np.nextafter(lo, down)) is not None:
        lo = np.nextafter(lo, down)
    hi = F32(32768 * res)
    while key(res, hi) is None:
        hi = np.nextafter(hi, down)
    while key(res, np.nextafter(hi, up)) is not None:
        hi = np.nextafter(hi, up)
    return lo, hi


def outside(c):
    """the next float32 away from 0"""
    return np.nextafter(F32(c), F32(np.copysign(np.inf, c)))


# ---- the builders ----------------------------------------------------------------------------------------------------------

def slots(n):
    """the slots of a scan's n points, in order and spread over the frame"""
    assert n <= SLOTS
    return np.arange(n) * (SLOTS // max(n, 1))


def transform(s):
    T = np.zeros((3, 4), F32)
    T[:, :3] = np.eye(3, dtype=F32)
    T[:, 3] = s.origin
    return T


def stored(s):
    """the cloud dict (x, y, z, rgb) of the planted points as the node stores them"""
    xyz = s.local
    return dict(x=xyz[:, 0].copy(), y=xyz[:, 1].copy(), z=xyz[:, 2].copy(), rgb=s.rgb.copy())


def clouds(scans):
    """(n, H, W, 8) float32 PointXYZRGB clouds: NaN but for the planted points"""
    out = np.full((len(scans), H * W, 8), np.nan, F32)
    out[..., 3] = 1.0
    out[..., 4] = 0.0
    for k, s in enumerate(scans):
        pc, at = stored(s), slots(len(s.pts))
        out[k, at, 0], out[k, at, 1], out[k, at, 2] = pc["x"], pc["y"], pc["z"]
        out[k, at, 4] = pc["rgb"].view(F32)
    return out.reshape(len(scans), H, W, 8)


def transforms(scans):
    return np.stack([transform(s) for s in scans])


def oracle(case, scans=None, cls=ox.Oracle):
    """the oracle's map after the case's scans, in order"""
    m = cls(**case.params)
    mr = -1.0 if case.max_range is None else case.max_range
    for s in case.scans if scans is None else scans:
        m.insert(s.pts, s.rgb, s.origin, mr)
    return m


def device_max_range(case):
    return float("inf") if case.max_range is None else case.max_range


# ---- the cases -------------------------------------------------------------------------------------------------------------

def _c(res, *cells):
    """map points at cell coordinates (cells of the resolution), as float32"""
    return (np.asarray(cells, np.float64).reshape(-1, 3) * res).astype(F32)


TIE_DIRS = [(1, 1, 0), (1, 0, 1), (0, 1, 1), (1, 1, 1), (-1, 1, 0), (1, -1, 0), (-1, 0, -1), (0, -1, 1), (-1, -1, -1), (1, -1, 1)]


def ray_walk(res):
    A = (0.5, 0.5, 0.5)
    ties = [np.add(A, np.multiply(d, 3)) for d in TIE_DIRS]
    corner_ends = [np.multiply(d, 3) for d in TIE_DIRS] + [(2, 3, 0), (3, 0, 2)]
    axis = [np.add(A, d) for d in [(4, 0, 0), (0, -4, 0), (0, 0, 5), (3, 2, 0), (0, 3, -2), (-2, 0, 3)]]
    scans = [
        scan(_c(res, A)[0], _c(res, *ties)),  # centre to centre: every tMax ties
        scan(_c(res, (0, 0, 0))[0], _c(res, *corner_ends)),  # corner to corners: the origin on a border on every axis
        scan(_c(res, A)[0], _c(res, *axis, (0.8, 0.1, 0.9))),  # zero direction components; an end in the origin's voxel
        scan(_c(res, (-2.5, -1.5, 0.5))[0], _c(res, (2.5, 1.5, 0.5), (2.5, -1.5, -3.5), (-2.5, 2.5, 0.5))),  # across key 32768
        scan(_c(res, (-2.5, -2.5, -2.5))[0], _c(res, (2.5, 2.5, 2.5), (2.5, -2.5, 2.5))),  # a tie across 0 on all axes
        scan(_c(res, (2.5, 2.5, 2.5))[0], _c(res, (-2.5, -2.5, -2.5), (-2.5, 2.5, -1.5))),
    ]
    # a direction component that vanishes in the float division (1e-45 / ~3.5) and one that stays subnormal
    o = np.array([0.5 * res, 0.0, 0.5 * res], F32)
    tiny = np.array([[3.5, 1e-45, 0.5 * res], [3.5, -1e-45, 2.5 * res], [3.5, 1e-39, 0.5 * res], [0.5 * res, 1e-45, 3.5]], F32)
    scans.append(scan(o, tiny))
    return Case(f"ray-walk-{res:g}", res, scans)


def long_rays():
    res = 0.001
    pts = np.array([[10.5, 0.0004, 0.0007], [-20.0, 20.0, 20.0], [25.0, -15.0, 5.0], [0.0003, -32.5, 0.0002]], F32)
    return Case("long-rays-0.001", res, [scan(np.zeros(3, F32), pts)])


def corners(res):
    """a scan near each of the tree's 8 corners: ends at the first and last keyed float of each axis and just outside; an
    origin on the low corner; an origin just outside with points inside; ±inf and NaN coordinates"""
    lo, hi = key_edges(res)
    scans = []
    for c in range(8):
        e = np.array([hi if (c >> a) & 1 else lo for a in range(3)], F32)
        inward = np.where(e > 0, -1.0, 1.0)
        o = (e + F32(1.5 * res) * inward).astype(F32)
        pts = [e.copy()]
        for a in range(3):
            p = e.copy()
            p[a] = outside(e[a])
            pts.append(p)
            p = e.copy()
            p[a] = F32(e[a] + F32(res) * F32(inward[a]))
            pts.append(p)
        pts.append(np.array([outside(v) for v in e], F32))
        scans.append(scan(o, pts))
    # an origin exactly on the low corner
    L = np.array([lo, lo, lo], F32)
    scans.append(scan(L, [L + F32(2 * res) * np.array([1, 0.5, 1.5], F32), L + F32(res) * np.array([0, 0, 3], F32)]))
    # an origin just outside the tree: no rays, the occupied cells and colours stay
    Hh = np.array([hi, hi, hi], F32)
    o = np.array([outside(hi), hi - F32(2 * res), hi - F32(2 * res)], F32)
    scans.append(scan(o, [Hh - F32(res) * np.array([1, 2, 3], F32), Hh - F32(res) * np.array([0.5, 0.25, 4], F32)]))
    # +-inf and NaN in one coordinate
    o = _c(res, (0.5, 0.5, 0.5))[0]
    bad = np.array([[np.inf, 0, 0], [0, -np.inf, 0], [0, 0, np.nan], [np.nan, 0, 0], [-np.inf, 0, 3 * res]], F32) + o
    scans.append(scan(o, np.concatenate([bad, _c(res, (2.5, 0.5, 0.5))])))
    return Case(f"corners-{res:g}", res, scans)


def reduction(res):
    A = (0.5, 0.5, 0.5)
    s1 = [(6.5, 0.5, 0.5), (7.2, 0.3, 0.7), (7.9, 0.6, 0.4), (3.5, 0.5, 0.5), (4.4, 0.5, 0.5), (6.1, 0.45, 0.55),  # (3, 0, 0)
          (2.1, 2.2, 0.3), (2.5, 2.5, 0.5), (4.5, 4.5, 0.5), (2.9, 2.8, 0.9)]  # (2, 2, 0): hit three times, and on a ray
    s2 = [(5.5, 0.5, 0.5), (8.5, 0.5, 0.5), (2.4, 2.6, 0.1)]  # (5, 0, 0) freed in scan 1, hit here
    s3 = [(6.5, 0.5, 0.5), (3.5, 0.5, 0.5)]
    return Case(f"reduction-{res:g}", res, [scan(_c(res, A)[0], _c(res, *s)) for s in (s1, s2, s3)])


CLAMP_SEQ = "HHHHHH" + "M" * 20 + "HM" * 4 + "HHMM"


def clamping(res, kw=None, seq=CLAMP_SEQ, tag=""):
    """scans that alternate hits and misses on the same cells: H hits (2, 0, 0) and (4, 0, 0), M frees them; every scan
    hits (0, 0, 3) and frees the origin's cell"""
    A = _c(res, (0.5, 0.5, 0.5))[0]
    scans = []
    for i, c in enumerate(seq):
        pts = [(2.5, 0.5, 0.5), (4.5, 0.5, 0.5)] if c == "H" else [(6.5, 0.5, 0.5)]
        pts.append((0.5, 0.5, 3.5))
        scans.append(scan(A, _c(res, *pts), np.arange(len(pts), dtype=np.uint32) + np.uint32(0x10203 * (i + 1))))
    return Case(f"clamping{tag}-{res:g}", res, scans, kw=kw or {})


# clamping thresholds equal to the hit and miss probabilities: one update from 0 lands exactly on a clamp value
EXACT_CLAMP = dict(prob_hit=0.7, prob_miss=0.4, clamping_min=0.4, clamping_max=0.7)
EXACT_SEQ = "HHMHMMMHHMHMHHHMMHMHMMHH"


def colour_order(res):
    A = _c(res, (0.5, 0.5, 0.5))[0]
    n = 5000
    rng = np.random.default_rng(7)
    u = rng.uniform(0.1, 0.9, (n, 3))
    pts = ((np.array([2.0, 0.0, 0.0]) + u) * res).astype(F32)  # one leaf, (2, 0, 0)
    rgb = (rng.permutation(WHITE)[:n]).astype(np.uint32)
    rgb[::97] = WHITE  # white is unset
    rgb[5::89] |= np.uint32(0xFF000000)  # alpha is not colour
    rgb[11::101] = 0x80FFFFFF  # white with alpha
    s2 = ((np.array([2.0, 0.0, 0.0]) + rng.uniform(0.1, 0.9, (5, 3))) * res).astype(F32)
    return Case(f"colour-order-{res:g}", res, [scan(A, pts, rgb), scan(A, s2, np.arange(5, dtype=np.uint32) * 0x30507 + 3)])


def colour_range(res):
    """max_range 3.45 cells from (0.5, 0.5, 0.5): a point beyond it whose cell is on another point's free ray; a colour whose
    leaf comes only in a later scan"""
    A = _c(res, (0.5, 0.5, 0.5))[0]
    s1 = _c(res, (3.99, 0.5, 0.5), (3.9, 1.05, 0.5), (0.5, 3.99, 0.5))
    s2 = _c(res, (0.5, 3.2, 0.5))
    s3 = _c(res, (0.5, 3.99, 0.45), (3.98, 0.55, 0.5))
    rgb = [np.array([0x112233, 0x445566, 0x778899], np.uint32), np.array([0xA0B0C0], np.uint32), np.array([0x0D0E0F, 0x102030], np.uint32)]
    return Case(f"colour-range-{res:g}", res, [scan(A, s, c) for s, c in zip((s1, s2, s3), rgb)], max_range=3.45 * res)


def _norm(o, p):
    d = (np.asarray(p, F32) - np.asarray(o, F32)).astype(F32)
    return float(np.sqrt(np.float64(F32(F32(F32(d[0] * d[0]) + F32(d[1] * d[1])) + F32(d[2] * d[2])))))


def max_range(res):
    """max_range equal to one point's |p - o|; the next float above it; a shortened ray of a point without a key"""
    lo, hi = key_edges(res)
    A = _c(res, (0.5, 0.5, 0.5))[0]
    p = _c(res, (3.5, 0.5, 0.5))[0]
    mr = _norm(A, p)
    B = _c(res, (0.5, 10.5, 0.5))[0]
    q = B + (p - A)
    q[0] = np.nextafter(q[0], F32(np.inf))
    O = np.array([hi - F32(5 * res), F32(0.5 * res), F32(0.5 * res)], F32)
    far = np.array([outside(hi), F32(0.5 * res), F32(0.5 * res)], F32)
    return Case(f"max-range-{res:g}", res, [scan(A, [p]), scan(B, [q]), scan(O, [far])], max_range=mr)


def short_range(res):
    """max_range 0.3 cells: shortened rays that end in the origin's voxel; a point inside it"""
    A = _c(res, (0.5, 0.5, 0.5))[0]
    pts = _c(res, (5.5, 0.5, 0.5), (0.5, -4.5, 2.5), (0.6, 0.4, 0.55), (0.5, 0.5, 9.5))
    return Case(f"short-range-{res:g}", res, [scan(A, pts)], max_range=0.3 * res)


def merge(res):
    """one leaf per scan (each point in its origin's voxel, so no ray): later scans land before the smallest Morton key,
    after the largest and between every pair; 2x2x2 blocks whose parent has all eight children, with 1..8 coloured"""
    cells = [(0, 0, 0), (8, 8, 8), (-8, -8, -8), (20, 20, 20), (4, 4, 4), (-4, -4, -4), (14, 14, 14), (-6, -6, -6),
             (2, 2, 2), (-2, 6, -2)]
    scans = [scan(_c(res, np.add(c, 0.5))[0], _c(res, np.add(c, 0.3)), [0x101010 * (i + 1)]) for i, c in enumerate(cells)]
    for j in range(8):
        base = np.array([4 * j - 16, 12, -12])
        cs = [base + [a & 1, (a >> 1) & 1, a >> 2] for a in range(8)]
        rgb = [(((10 + 7 * j + 13 * a) & 255) << 16) | (((200 - 9 * a) & 255) << 8) | ((31 * a + j) & 255) for a in range(8)]
        rgb = [c if a <= j else WHITE for a, c in enumerate(rgb)]
        scans.append(scan(_c(res, base + 0.5)[0], _c(res, *[c + 0.5 for c in cs]), rgb))
    return Case(f"merge-{res:g}", res, scans, calls=[2, 3, 1, len(scans) - 6])


def empty(res, after=False):
    """scans that insert nothing: NaN, ±inf and keyless points, an origin outside the tree, and (max_range 0.3 cells)
    shortened rays inside the origin's voxel, one of them with a keyed end: a colour entry and no leaf.  after: first a
    scan that makes one leaf"""
    lo, hi = key_edges(res)
    A = _c(res, (0.5, 0.5, 0.5))[0]
    scans = [
        scan(A, np.zeros((0, 3), F32)),
        scan(A, np.array([[np.inf, 0, 0], [0, -np.inf, 0], [0, 0, np.nan], [np.nan, np.nan, np.nan]], F32) + A),
        scan(A, np.array([[outside(hi), A[1], A[2]], [A[0], outside(lo), A[2]], [A[0], A[1], F32(40000 * res)]], F32)),
        scan(np.array([outside(lo), A[1], A[2]], F32), np.array([[outside(lo), A[1], A[2]], [outside(outside(lo)), 0, 0]], F32)),
        scan(A, _c(res, (6.5, 0.5, 0.5), (0.5, 0.5, -7.5))),
    ]
    if after:
        scans.insert(0, scan(A, _c(res, (0.7, 0.6, 0.4))))
    return Case(f"empty{'-after' if after else ''}-{res:g}", res, scans, max_range=0.3 * res,
                calls=[1, len(scans) - 1] if after else None)


def cases():
    out = []
    for r in EXACT + INEXACT:
        out += [ray_walk(r), corners(r)]
    out.append(long_rays())
    for r in (1.0, 0.05):
        out += [reduction(r), colour_order(r), colour_range(r), max_range(r), short_range(r)]
    for r in (1.0, 0.0625):
        out += [clamping(r), clamping(r, EXACT_CLAMP, EXACT_SEQ, "-exact")]
    out.append(clamping(0.05))
    for r in (1.0, 0.0625, 0.05):
        out += [merge(r), empty(r), empty(r, True)]
    return {c.name: c for c in out}


CASES = cases()


# ---- the occupancy filter --------------------------------------------------------------------------------------------------

IDENTITY7 = np.array([0, 0, 0, 1, 0, 0, 0], F32)


def turned7(res):
    """cloud_sensor_pose of a quarter turn about z and a shift of a few cells"""
    from rgbdslam_v2_b200._capi import cloud_sensor_pose
    T = np.eye(4)
    T[:3, :3] = [[0.0, -1.0, 0.0], [1.0, 0.0, 0.0], [0.0, 0.0, 1.0]]
    T[:3, 3] = np.array([0.5, -0.25, 0.75]) * res
    q, t = cloud_sensor_pose(T)
    return np.concatenate([q, t]).astype(F32)


def filter_map(res):
    """the map the filter cases read: the corner, ray-walk and reduction scans"""
    scans = corners(res).scans + ray_walk(res).scans + reduction(res).scans
    return Case(f"filter-map-{res:g}", res, scans)


def filter_oracle(res):
    c = filter_map(res)
    return oracle(c, cls=fx.FilterOracle)


@dataclass
class FilterCase:
    name: str
    res: float
    pts: np.ndarray  # (n, 3) float32 points as stored
    sensor7: np.ndarray  # (7,) float32
    thresholds: list


def visited(res, sensor7, p):
    """the three cells occupancyFilter looks at for stored point p (uint16 keys), or None when in.z is NaN"""
    inn = fx.sensor_transform(sensor7[:4], sensor7[4:], p)
    if np.isnan(inn[2]):
        return None

    def k(c):
        with np.errstate(invalid="ignore"):
            v = np.floor((1.0 / res) * np.float64(c))
        i = int(v) if -2.0 ** 31 <= v < 2.0 ** 31 else -2 ** 31
        return (i + 32768) & 0xFFFF

    kx, ky, kz = ((k(c) - 1) & 0xFFFF for c in inn)
    return [(kx, ky, (kz + d) & 0xFFFF) for d in range(3)]


def libm_occupancy(lo):
    import ctypes as C
    libm = C.CDLL("libm.so.6")
    libm.exp.restype = C.c_double
    libm.exp.argtypes = [C.c_double]
    return 1.0 - 1.0 / (1.0 + libm.exp(float(lo)))


def filter_sums(res, leaves, sensor7, p):
    """(sum_occ, sum_w) of occupancyFilter for stored point p against the map's {key: (lo, colour)}"""
    inn = fx.sensor_transform(sensor7[:4], sensor7[4:], p).astype(np.float64)
    so = sw = 0.0
    for c in visited(res, sensor7, p) or []:
        if c in leaves:
            d = [((k - 32768) + 0.5) * res - v for k, v in zip(c, inn)]
            w = (d[0] * d[0] + d[1] * d[1]) + d[2] * d[2]
            so += libm_occupancy(leaves[c][0]) / w
            sw += w
    return so, sw


def tie_point(res, leaves, sensor7):
    """a stored point whose sums tie exactly at threshold so / sw (searched on a fixed grid near the map's origin)"""
    for a in np.linspace(0.05, 0.95, 19):
        for b in np.linspace(0.05, 0.95, 19):
            p = (np.array([1.0 + a, 1.0 + b, 1.0 + (a + b) / 2]) * res).astype(F32)
            so, sw = filter_sums(res, leaves, sensor7, p)
            if sw > 0 and so > 0 and (so / sw) * sw == so:
                return p, so / sw
    raise AssertionError("no tie")


def filter_cases(res, leaves):
    lo, hi = key_edges(res)
    r = F32(res)
    ext = [lo, F32(lo + r), F32(hi - r), hi]
    wrap = np.array([[x, y, z] for x in ext for y in ext for z in ext], F32)  # keys 0, 1, 65534, 65535 on every axis
    big = 2.0 ** 31 * res
    wide = np.array([[1e12, 0.5 * res, 0.5 * res], [0.5 * res, -1e12, 0.5 * res], [0.5 * res, 0.5 * res, 3e38],
                     [F32(big), 0.5 * res, 0.5 * res], [np.nextafter(F32(big), F32(0)), 0.5 * res, 0.5 * res],
                     [-F32(big), 0.5 * res, 0.5 * res], [np.nextafter(-F32(big), F32(0)), 0.5 * res, 0.5 * res],
                     [np.inf, 0.5 * res, 0.5 * res], [0.5 * res, -np.inf, 0.5 * res], [0.5 * res, 0.5 * res, np.inf],
                     [np.nan, 0.5 * res, 0.5 * res], [0.5 * res, 0.5 * res, np.nan], [100.5 * res, 100.5 * res, 100.5 * res]], F32)
    rng = np.random.default_rng(11)
    near = (rng.uniform(-3, 5, (300, 3)) * res).astype(F32)  # around the ray-walk and reduction leaves
    thr = [0.0, 0.05, 0.3, np.inf] if res == 1.0 else [3e3, 3e4, 3e5, np.inf]
    T7 = turned7(res)
    out = [FilterCase(f"wrap-{res:g}", res, wrap, IDENTITY7, thr),
           FilterCase(f"int-range-{res:g}", res, wide, IDENTITY7, thr),
           FilterCase(f"int-range-turned-{res:g}", res, wide, T7, thr),
           FilterCase(f"near-{res:g}", res, near, IDENTITY7, thr),
           FilterCase(f"near-turned-{res:g}", res, near, T7, thr)]
    p, t = tie_point(res, leaves, IDENTITY7)
    out.append(FilterCase(f"tie-{res:g}", res, p[None], IDENTITY7, [t, float(np.nextafter(t, np.inf))]))
    return {c.name: c for c in out}
