"""The ORB pyramids as cv2 4.13 builds them, and numpy restatements of the device's arithmetic on them -- TEST
INFRASTRUCTURE, shared by tests/test_orb_pyramid_oracle_cpu.py and tests/test_gpu_orb_textures.py.

  extractor pyramid   cv::ORB's image pyramid (orb.cpp): level l = resize(level l-1, INTER_LINEAR_EXACT) to the sides
                      orb_oracle.level_side gives; the descriptor reads each level blurred by GaussianBlur(7x7, sigma 2,
                      BORDER_REFLECT_101), the float separable filter = cv2.sepFilter2D with getGaussianKernel(7, 2, CV_32F)
  cell pyramids       the same chain per grid cell of the detector; the mask pyramid is the binarised cell mask (255 where
                      non-zero) at level 0, resize then THRESH_TOZERO(254) above
  blur(fused)         the separable filter with every multiply-add fused (cv2's SIMD path on x86-64 with FMA) or with each
                      product and sum rounded to float (an unfused evaluation)
  resize_table        INTER_LINEAR_EXACT's first tap and 8-bit weight of the second per destination index, with cv2's scale
                      1 / (dst / src) or with src / dst
  orb_candidates      what the ORB detector's candidate buffer holds for one cell: every strict 3x3 maximum of the
                      threshold-free FAST score with score >= 2, at least 15 px inside its level, under the mask
"""
import cv2
import numpy as np

import fast_oracle
import node_helpers as nh
from oracle import orb_oracle as oo

LEVELS = 8
GAUSS = cv2.getGaussianKernel(7, 2, ktype=cv2.CV_32F).ravel().astype(np.float32)
ORB_EDGE = 15  # ORB's edgeThreshold as the detector passes it (feature_adjuster.cpp:94): FAST corners 15 px inside a level


def resize_exact(img, w, h):
    return cv2.resize(img, (w, h), interpolation=cv2.INTER_LINEAR_EXACT)


def pyramid(img):
    """cv::ORB's chained pyramid of img: LEVELS levels"""
    h, w = img.shape
    out = [np.ascontiguousarray(img)]
    for l in range(1, LEVELS):
        out.append(resize_exact(out[-1], oo.level_side(w, l), oo.level_side(h, l)))
    return out


def blurred(levels):
    return [cv2.sepFilter2D(p, -1, GAUSS, GAUSS, borderType=cv2.BORDER_REFLECT_101) for p in levels]


def mask_pyramid(mask):
    """the cell mask pyramid: (mask != 0) * 255, then resize and THRESH_TOZERO(254) per level"""
    h, w = mask.shape
    out = [np.where(mask != 0, 255, 0).astype(np.uint8)]
    for l in range(1, LEVELS):
        m = resize_exact(out[-1], oo.level_side(w, l), oo.level_side(h, l))
        out.append(cv2.threshold(m, 254, 0, cv2.THRESH_TOZERO)[1])
    return out


def cell_pyramids(gray, mask, grid=3):
    """[(image pyramid, mask pyramid)] of the detector's grid cells (orb_oracle._cells)"""
    H, W = gray.shape
    out = []
    for y0, y1, x0, x1 in oo._cells(W, H, grid):
        out.append((pyramid(gray[y0:y1, x0:x1]), mask_pyramid(mask[y0:y1, x0:x1])))
    return out


def blur(img, fused, row_tail=None):
    """The 7-tap separable Gaussian in float: the row pass accumulated left to right, the column pass symmetric (the centre
    row times its weight, then each pair of rows summed and multiplied in), rounded half to even to uint8.  fused: each
    multiply-add rounded once, except (row_tail = n) in the row pass of the columns past the last whole n-column block, where
    each product and sum is rounded.  cv2 4.13 on x86-64 with FMA is fused=True, row_tail=32: its SIMD row filter takes
    32 columns at a time and leaves the rest to a scalar loop.  The operands are floats, so each product is exact in the
    64-bit significand of long double, and so is each sum for this filter's ranges (every non-zero addend within 2^17 of
    the other): one rounding to float32, as a fused multiply-add."""
    assert np.finfo(np.longdouble).nmant >= 63
    ld, f32 = np.longdouble, np.float32
    k = GAUSS
    h, w = img.shape
    p = np.pad(img.astype(f32), 3, mode="reflect")  # reflect = BORDER_REFLECT_101
    unfused_cols = np.full(w, not fused)
    if fused and row_tail:
        unfused_cols[w // row_tail * row_tail:] = True

    def mad(c, a, b, unfused):  # c + a * b
        return np.where(unfused, f32(c + f32(a * b)), f32(ld(a) * ld(b) + ld(c)))

    acc = np.zeros((h + 6, w), f32)
    for j in range(7):
        acc = mad(acc, k[j], p[:, j:j + w], unfused_cols)
    c = f32(k[3] * acc[3:3 + h])
    for j in range(1, 4):
        c = mad(c, k[3 + j], f32(acc[3 + j:3 + j + h] + acc[3 - j:3 - j + h]), not fused)
    return np.clip(np.rint(c), 0, 255).astype(np.uint8)


def resize_table(src, dst, reciprocal=True):
    """(first tap, weight of the second tap x 256) per destination index; reciprocal: scale = 1 / (dst / src) as
    cv::resize computes it, else src / dst"""
    scale = 1.0 / (dst / src) if reciprocal else src / dst
    f = (np.arange(dst, dtype=np.float64) + 0.5) * scale - 0.5
    i = np.floor(f).astype(np.int64)
    fr = f - i
    lo, hi = i < 0, i >= src - 1
    i[lo], fr[lo] = 0, 0.0
    i[hi], fr[hi] = src - 1, 0.0
    return i, np.rint(fr * 256).astype(np.int64)


def resize_rows(img, dst, reciprocal=True):
    """img resized along its rows only with resize_table's taps (8.8 fixed point, rounded to nearest)"""
    src = img.shape[1]
    i, w1 = resize_table(src, dst, reciprocal)
    a = img[:, i].astype(np.int64)
    b = img[:, np.minimum(i + 1, src - 1)].astype(np.int64)
    return ((a * (256 - w1) + b * w1 + 128) >> 8).astype(np.uint8)


def orb_candidates(img_levels, mask_levels):
    """per level, {(x, y): score} of the ORB detector's candidates in one cell"""
    out = []
    for img, m in zip(img_levels, mask_levels):
        h, w = img.shape
        inner = np.zeros(img.shape, np.uint8)
        inner[ORB_EDGE:h - ORB_EDGE, ORB_EDGE:w - ORB_EDGE] = 255
        out.append(fast_oracle.fast_nms(img, inner & m, 2))
    return out


# -- the texture corpus: frames where the pyramids, the blur and the quotas are exercised at every pixel -----------------
def checkerboard(h, w, s=3):
    y, x = np.indices((h, w))
    return (((y // s + x // s) % 2) * 255).astype(np.uint8)


def steps_and_lines(h, w):
    """0/255 steps every 37 columns and 29 rows, with one-pixel lines of the opposite value every 11 columns and 13 rows"""
    y, x = np.indices((h, w))
    img = (((x // 37 + y // 29) % 2) * 255).astype(np.uint8)
    line = (x % 11 == 5) | (y % 13 == 6)
    img[line] = 255 - img[line]
    return img


def tiled(h, w, seed=3):
    """a 24 x 24 patch of band-limited noise tiled over the frame: corners repeat with bit-identical scores and responses"""
    patch = nh.textured(24, 24, 1, seed, 0.8)[0]
    return np.ascontiguousarray(np.tile(patch, (h // 24 + 1, w // 24 + 1))[:h, :w])


def corpus(h, w, seed=0):
    """{name: frame} of the texture corpus at h x w"""
    rng = np.random.default_rng(seed + 1)
    return {
        "noise1": nh.textured(h, w, 1, seed, 1.0)[0],
        "noise2": nh.textured(h, w, 1, seed, 2.0)[0],
        "iid": rng.integers(0, 256, (h, w), dtype=np.uint8),
        "checker": checkerboard(h, w),
        "steps": steps_and_lines(h, w),
        "constant": np.full((h, w), 128, np.uint8),
        "tiled": tiled(h, w),
    }


# the frame sizes orb_prepare accepts that the tests cover: both sides of the 1023 / 1024 boundary, grid columns whose
# level-1 side cvRound(n * (1.f / 1.2f)) differs from cvRound(n / 1.2f) (633), 3993 (the one side where resize's two scale
# rules differ) and the widest frame
SIZES = [(333, 333), (480, 633), (480, 640), (481, 641), (1023, 1023), (768, 1024), (360, 3993), (360, 4095)]
