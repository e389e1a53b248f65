"""Numpy restatements of the listener's conversions of raw sensor images (openni_listener.cpp:633-659) -- TEST
INFRASTRUCTURE, not product code.  test_raw_input_oracle_cpu.py pins them to cv2 4.13; the GPU tests feed them to the float /
grey / caller-mask path as the reference for RGBDSLAM_B200_DEPTH_U16 and RGBDSLAM_B200_VISUAL_BAYER_GR.
  depth_u16_to_m    depth.convertTo(CV_32FC1, 0.001): (float)d * 0.001f
  depth_u16_mask    depthToCV8UC1 (misc.cpp:414-425): convertTo(CV_8UC1, 0.05, -25) = saturate_cast<uchar>(fmaf(d, 0.05f, -25))
  bayer_gr_to_rgb   cvtColor(COLOR_BayerGR2RGB): G B on even rows, R G on odd rows, bilinear, borders repeated
  bayer_gr_to_gray  the RGB above rounded to u8, then CV_RGB2GRAY (node.cpp:139-144)
"""
import numpy as np

F32 = np.float32


def depth_u16_to_m(d):
    return np.asarray(d, np.uint16).astype(F32) * F32(0.001)


def _saturate_u8(v):
    return np.clip(np.rint(v), 0, 255).astype(np.uint8)  # cvRound (half to even), then saturate


def depth_u16_mask(d):
    """fmaf(d, 0.05f, -25.f) rounded once: the float64 product of a 16-bit integer and a float is exact, and so is the sum"""
    v = np.asarray(d, np.uint16).astype(np.float64) * np.float64(F32(0.05)) - 25.0
    return _saturate_u8(v.astype(F32))


def depth_u16_mask_unfused(d):
    """d * 0.05f - 25.f rounded twice: what a non-fused build would compute"""
    return _saturate_u8(np.asarray(d, np.uint16).astype(F32) * F32(0.05) - F32(25.0))


def bayer_gr_to_rgb(raw):
    """An interior pixel keeps its own channel; the other two are the mean of a pair, (a + b + 1) >> 1, or of a quad (the
    cross or the diagonals), (a + b + c + d + 2) >> 2.  Rows 0 / H-1 repeat rows 1 / H-2, then columns 0 / W-1 repeat
    columns 1 / W-2."""
    H, W = raw.shape
    p = np.asarray(raw, np.int32)
    c = p[1:-1, 1:-1]
    up, dn, lf, rt = p[:-2, 1:-1], p[2:, 1:-1], p[1:-1, :-2], p[1:-1, 2:]
    pair_v, pair_h = (up + dn + 1) >> 1, (lf + rt + 1) >> 1
    cross = (up + dn + lf + rt + 2) >> 2
    diag = (p[:-2, :-2] + p[:-2, 2:] + p[2:, :-2] + p[2:, 2:] + 2) >> 2
    yy, xx = np.mgrid[1:H - 1, 1:W - 1]
    ey, ex = yy % 2 == 0, xx % 2 == 0
    where = [ey & ex, ey & ~ex, ~ey & ex, ~ey & ~ex]  # G (B to the sides), B, R, G (R to the sides)
    r = np.select(where, [pair_v, diag, c, pair_h])
    g = np.select(where, [c, cross, cross, c])
    b = np.select(where, [pair_h, c, diag, pair_v])
    out = np.zeros((H, W, 3), np.uint8)
    out[1:-1, 1:-1] = np.stack([r, g, b], -1)
    out[0], out[-1] = out[1], out[-2]
    out[:, 0], out[:, -1] = out[:, 1], out[:, -2]
    return out


def rgb_to_gray(rgb):
    """cv::cvtColor(CV_RGB2GRAY) of cv2 4.13: (R * 9798 + G * 19235 + B * 3735 + 2^14) >> 15, channel 0 = R."""
    r, g, b = (rgb[..., i].astype(np.uint32) for i in range(3))
    return ((r * 9798 + g * 19235 + b * 3735 + (1 << 14)) >> 15).astype(np.uint8)


def bayer_gr_to_gray(raw):
    return rgb_to_gray(bayer_gr_to_rgb(raw))


def mosaic_gr(rgb):
    """the bayer_grbg8 image a sensor would send for a colour image (channel 0 = R): G B on even rows, R G on odd rows"""
    H, W = rgb.shape[:2]
    yy, xx = np.mgrid[0:H, 0:W]
    ch = np.where(yy % 2 == 0, np.where(xx % 2 == 0, 1, 2), np.where(xx % 2 == 0, 0, 1))
    return np.ascontiguousarray(np.take_along_axis(rgb, ch[..., None], -1)[..., 0])


def to_millimetres(depth_m):
    """a float depth image quantised as a 16UC1 sensor image: millimetres, holes (NaN, <= 0, too far) -> 0"""
    d = np.asarray(depth_m, np.float64) * 1000.0
    ok = np.isfinite(d) & (d > 0) & (d < 65535.5)
    return np.where(ok, np.rint(np.where(ok, d, 0)), 0).astype(np.uint16)
