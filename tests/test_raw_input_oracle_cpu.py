"""The restatements of the listener's raw-image conversions (tests/raw_input_oracle.py) against cv2 4.13 itself, without a
GPU: 16-bit depth -> metres and -> detection mask on all 65536 values, Bayer GRBG -> RGB -> grey on every pixel."""
import cv2
import numpy as np
import pytest

import raw_input_oracle as ro

ALL = np.arange(65536, dtype=np.uint16).reshape(256, 256)


def _convert_to(src, scale, shift, dtype):
    """Mat::convertTo(dtype, scale, shift), reached through normalize(NORM_MINMAX) on a source whose range is [0, 65535]"""
    assert src.min() == 0 and src.max() == 65535
    return cv2.normalize(src, None, shift, shift + scale * 65535.0, cv2.NORM_MINMAX, dtype=dtype)


def test_depth_plane_equals_convert_to_on_all_values():
    want = _convert_to(ALL, 0.001, 0.0, cv2.CV_32F)
    got = ro.depth_u16_to_m(ALL)
    assert got.dtype == np.float32 and np.array_equal(got.view(np.uint32), want.view(np.uint32))
    assert got[0, 0] == 0.0  # a hole is 0 m, not NaN


def test_mask_equals_convert_to_on_all_values():
    want = _convert_to(ALL, 0.05, -25.0, cv2.CV_8U)
    got = ro.depth_u16_mask(ALL)
    assert np.array_equal(got, want)
    assert np.array_equal(got.ravel() != 0, np.arange(65536) >= 510)


def test_unfused_mask_differs_only_where_expected():
    fused, unfused = ro.depth_u16_mask(ALL).ravel(), ro.depth_u16_mask_unfused(ALL).ravel()
    assert np.nonzero(fused != unfused)[0].tolist() == list(range(510, 791, 40))
    assert np.nonzero((fused != 0) != (unfused != 0))[0].tolist() == [510]


SIZES = [(4, 4), (5, 7), (12, 16), (13, 16), (12, 17), (13, 17), (31, 30), (96, 97), (481, 641), (480, 640)]


@pytest.mark.parametrize("shape", SIZES, ids=[f"{h}x{w}" for h, w in SIZES])
def test_bayer_equals_cvtcolor_on_every_pixel(shape):
    rng = np.random.default_rng(shape[0] * 1000 + shape[1])
    for _ in range(3):
        raw = rng.integers(0, 256, shape, dtype=np.uint8)
        rgb = cv2.cvtColor(raw, cv2.COLOR_BayerGR2RGB)
        assert np.array_equal(ro.bayer_gr_to_rgb(raw), rgb)
        assert np.array_equal(ro.bayer_gr_to_gray(raw), cv2.cvtColor(rgb, cv2.COLOR_RGB2GRAY))


def test_bayer_layout_and_fused_gray_differs():
    """the mosaic of a colour image holds G B on even rows and R G on odd rows as cv2 reads BayerGR; cv2's fused
    BayerGR2GRAY rounds differently from the two calls the listener and the Node make"""
    rng = np.random.default_rng(5)
    rgb = rng.integers(0, 256, (12, 16, 3), dtype=np.uint8)
    raw = ro.mosaic_gr(rgb)
    back = cv2.cvtColor(raw, cv2.COLOR_BayerGR2RGB)
    for y, x in ((4, 4), (4, 5), (5, 4), (5, 5)):
        own = {(0, 0): 1, (0, 1): 2, (1, 0): 0, (1, 1): 1}[(y % 2, x % 2)]
        assert back[y, x, own] == rgb[y, x, own]
    raw = rng.integers(0, 256, (12, 16), dtype=np.uint8)
    fused = cv2.cvtColor(raw, cv2.COLOR_BayerGR2GRAY)
    assert (fused != ro.bayer_gr_to_gray(raw)).sum() > 0


def test_to_millimetres():
    d = np.array([np.nan, -1.0, 0.0, 0.0004, 0.0006, 0.51, 65.535, 65.536, np.inf], np.float32)
    assert ro.to_millimetres(d).tolist() == [0, 0, 0, 0, 1, 510, 65535, 0, 0]
