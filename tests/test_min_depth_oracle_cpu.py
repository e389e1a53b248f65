"""use_feature_min_depth without a GPU: the restated getMinDepthInNeighborhood (misc.cpp:774-791) pinned against cv2.minMaxLoc
on windows of rendered depth, the engineered corners of the rule, and the parameter that switches it on."""
import ctypes as C

import cv2
import numpy as np
import pytest

import min_depth_oracle as md
from oracle import orb_oracle

ORB_SIZES = [np.float32(31) * orb_oracle.layer_scale(l) for l in range(8)]
SIZES = ORB_SIZES + [np.float32(7)]  # FAST keypoints have size 7


@pytest.fixture(scope="module")
def depths():
    """(NaN-free depth, the same frame with the renderer's NaN holes) for three rendered frames"""
    from rgbdslam_v2_b200 import synth
    poses = synth.trajectory(40)
    return [(synth.render_frame(poses[k], seed=k, nan_frac=0.0)[1], synth.render_frame(poses[k], seed=k)[1]) for k in (0, 5, 9)]


def _cv2_min(win: np.ndarray) -> np.float32:
    """getMinDepthInNeighborhood with cv2's minMaxLoc, as the reference calls it"""
    m = np.float32(cv2.minMaxLoc(win)[0])
    return md.NAN if m == 0 else m


def _centres(rng, W, H, n):
    """sub-pixel centres like those of ORB keypoints on higher octaves, plus centres on and next to every image border"""
    xs = list(rng.uniform(0, W - 1, n).astype(np.float32))
    ys = list(rng.uniform(0, H - 1, n).astype(np.float32))
    for e in (0.0, 0.5, 2.7, 14.3, 30.999, 54.6):
        for x, y in ((e, H / 2), (W - 1 - e, H / 2), (W / 2, e), (W / 2, H - 1 - e), (e, e), (W - 1 - e, H - 1 - e)):
            xs.append(np.float32(x)); ys.append(np.float32(y))
    return list(zip(xs, ys))


def test_radii():
    assert [md.radius(s) for s in ORB_SIZES] == [15, 18, 21, 26, 31, 38, 45, 55]
    assert md.radius(np.float32(7)) == 3


def test_rule_equals_cv2_on_nan_free_windows(depths):
    """At every ORB radius and the FAST radius, including windows clipped at each border: the rule == cv2.minMaxLoc."""
    rng = np.random.default_rng(3)
    clipped = 0
    for full, _ in depths:
        assert not np.isnan(full).any()
        H, W = full.shape
        for size in SIZES:
            for x, y in _centres(rng, W, H, 40):
                win = md.window(full, x, y, size)
                assert win.base is full or np.shares_memory(win, full)  # a view into the frame, as cv::Mat(depth, Range, Range)
                r = md.radius(size)
                clipped += win.shape != (2 * r, 2 * r)
                got, want = md.min_depth(full, x, y, size), _cv2_min(win)
                assert got.tobytes() == want.tobytes()
    assert clipped > 100


def test_zero_in_the_window_gives_nan(depths):
    full = depths[0][0].copy()
    x, y, size = np.float32(200.4), np.float32(150.6), ORB_SIZES[2]
    assert not np.isnan(md.min_depth(full, x, y, size))
    for z in (0.0, -0.0):
        d = full.copy()
        d[150, 205] = z
        assert np.isnan(md.min_depth(d, x, y, size)) and np.isnan(_cv2_min(md.window(d, x, y, size)))
    d = full.copy()
    d[150, 205] = 0.0
    d[151, 206] = -1.0  # a negative depth is an ordinary value: it is the minimum, not 0
    assert md.min_depth(d, x, y, size) == np.float32(-1.0)


def test_all_nan_window_gives_nan(depths):
    d = depths[0][0].copy()
    x, y = np.float32(300.0), np.float32(200.0)
    top, left = 200 - 3, 300 - 3
    d[top:top + 6, left:left + 6] = np.nan
    assert np.isnan(md.min_depth(d, x, y, 7))
    d[top + 6, left + 6] = 0.5  # row / column +3: outside the window
    assert np.isnan(md.min_depth(d, x, y, 7))
    d[top, left] = 0.5  # row / column -3: inside
    assert md.min_depth(d, x, y, 7) == np.float32(0.5)


def test_fast_window_is_6x6_and_not_centred(depths):
    d = depths[0][0]
    x, y = np.float32(100.0), np.float32(80.0)
    win = md.window(d, x, y, 7)
    assert win.shape == (6, 6)
    assert np.array_equal(win, d[77:83, 97:103])
    e = d.copy()
    e[83, 100] = 0.01  # y + 3
    e[80, 103] = 0.01  # x + 3
    assert md.min_depth(e, x, y, 7) == d[77:83, 97:103].min()
    e[77, 97] = 0.02  # y - 3, x - 3
    assert md.min_depth(e, x, y, 7) == np.float32(0.02)


def test_sub_pixel_truncation(depths):
    """int() truncates toward zero: a centre in (r - 1, r) gives top 0 (floor would give -1 and the clamp 0 as well); a
    centre whose y - r and y + r have fractions gives [int(y - r), int(y + r)), which is 2r rows, not centred on round(y)."""
    d = depths[1][0]
    for size in SIZES:
        r = md.radius(size)
        for frac in (0.01, 0.5, 0.99):
            y = np.float32(r - 1 + frac)
            x = np.float32(3 * r + 10 + frac)
            win = md.window(d, x, y, size)
            assert int(np.float32(y) - np.float32(r)) == 0 and np.floor(np.float32(y) - np.float32(r)) == -1
            assert win.shape[0] == int(y + np.float32(r))
            assert np.array_equal(win, d[0:int(y + np.float32(r)), int(x - np.float32(r)):int(x + np.float32(r))])
            assert win.shape[1] == 2 * r
            assert md.min_depth(d, x, y, size).tobytes() == _cv2_min(win).tobytes()
        y = np.float32(3 * r + 20.7)
        win = md.window(d, np.float32(200.3), y, size)
        assert win.shape == (2 * r, 2 * r) and np.array_equal(win, d[3 * r + 20 - r:3 * r + 20 + r, 200 - r:200 + r])


def test_nan_windows_never_above_cv2(depths):
    """With NaN in the window cv2 4.13's vectorised minMaxLoc is not defined by the pixel values alone (it returns NaN or a
    value above the finite minimum, depending on the lane layout); the rule takes the finite minimum, so it is never above
    any non-NaN cv2 answer.  cv2's values are not asserted."""
    rng = np.random.default_rng(5)
    n = 0
    for _, holed in depths:
        H, W = holed.shape
        for size in SIZES:
            for x, y in _centres(rng, W, H, 60):
                win = md.window(holed, x, y, size)
                if not np.isnan(win).any() or np.isnan(win).all():
                    continue
                got = md.min_depth(holed, x, y, size)
                assert got == np.nanmin(win)
                c = np.float32(cv2.minMaxLoc(win)[0])
                if not np.isnan(c):
                    assert got <= c
                n += 1
    assert n > 500


def test_min_depth_parameter(built):
    """use_feature_min_depth keeps its offset; init accepts 0 and 1 (here it only fails for want of a device) and rejects
    other values and allow_features_without_depth before it looks for a device."""
    from rgbdslam_v2_b200 import _capi
    P = _capi.Params
    assert C.sizeof(P) == 128
    assert P.use_feature_min_depth.offset == 124 and P.allow_features_without_depth_.offset == 125
    assert P.feature_detector_type.offset == 126
    p = _capi.default_params()
    assert p.use_feature_min_depth == 0
    lib = _capi.load_library()
    for bad in (2, 255):
        p.use_feature_min_depth = bad
        assert lib.rgbdslam_b200_init(0, C.byref(p)) == 1
        assert b"use_feature_min_depth" in lib.rgbdslam_b200_last_error()
    p.use_feature_min_depth = 1
    p.allow_features_without_depth_ = 1
    assert lib.rgbdslam_b200_init(0, C.byref(p)) == 1
    assert b"allow_features_without_depth" in lib.rgbdslam_b200_last_error()
    p.allow_features_without_depth_ = 0
    rc = lib.rgbdslam_b200_init(0, C.byref(p))
    assert rc in (0, 2)  # 2 = ERR_CUDA: no device on this host
    if rc == 0:  # a host with a GPU: leave the library with the default parameters again
        q = _capi.default_params()
        assert lib.rgbdslam_b200_get_params(C.byref(q)) == 0 and q.use_feature_min_depth == 1
        assert lib.rgbdslam_b200_init(0, C.byref(_capi.default_params())) == 0
