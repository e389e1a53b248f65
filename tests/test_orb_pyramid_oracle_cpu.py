"""The ORB pyramid oracle pinned to cv2 4.13 on the texture corpus: the blur is cv2's float separable filter with every
multiply-add fused, and INTER_LINEAR_EXACT takes its scale as 1 / (dst / src).  These are the two rules k_blur and
build_table (api_orb.cu) follow; tests/test_gpu_orb_textures.py compares the device's planes with cv2 itself."""
import numpy as np
import pytest

cv2 = pytest.importorskip("cv2")

import orb_pyramid_oracle as po  # noqa: E402
from oracle import orb_oracle as oo  # noqa: E402

NO_FMA = ("cv2.sepFilter2D differs from the fused multiply-add emulation: this host's cv2 is not dispatching fused "
          "multiply-adds (an x86-64 CPU or build without FMA), so cv2 here is not the arithmetic the device restates and "
          "the GPU tests' blurred planes and descriptors cannot be compared with it")


_ALL_FUSED = {}  # size -> pixels where fusing the row pass's last partial 32-column block too differs from cv2


@pytest.mark.parametrize("hw", po.SIZES, ids=[f"{w}x{h}" for h, w in po.SIZES])
def test_cv2_blur_is_the_fused_separable_filter(hw):
    """every pixel of every level of every corpus frame equals the fused rule with cv2's unfused row remainder; at 640x480
    the unfused rule differs from cv2 somewhere"""
    h, w = hw
    unfused_diff = all_fused = 0
    for name, img in po.corpus(h, w).items():
        levels = po.pyramid(img)
        for l, (lev, ref) in enumerate(zip(levels, po.blurred(levels))):
            bad = np.argwhere(po.blur(lev, True, row_tail=32) != ref)
            assert len(bad) == 0, f"{NO_FMA}: {name} level {l}, {len(bad)} pixels, first (y, x) {tuple(bad[0])}"
            all_fused += int((po.blur(lev, True) != ref).sum())
            if hw == (480, 640):
                unfused_diff += int((po.blur(lev, False) != ref).sum())
    _ALL_FUSED[hw] = all_fused
    if hw == (480, 640):
        assert unfused_diff > 0


def test_the_row_remainder_is_unfused():
    """the corpus has pixels where only the unfused row remainder gives cv2's value: 633x480 (tiled, level 5, 254 px wide,
    column 227) and 1023x1023 (level 1, 852 px wide, columns 837 and 838)"""
    for hw in ((480, 633), (1023, 1023)):
        if hw not in _ALL_FUSED:
            test_cv2_blur_is_the_fused_separable_filter(hw)
        assert _ALL_FUSED[hw] > 0, hw


def test_the_extractor_pyramid_is_chained_at_the_orb_level_sides():
    h, w = 480, 633
    levels = po.pyramid(po.corpus(h, w)["noise1"])
    assert [p.shape for p in levels] == [(oo.level_side(h, l), oo.level_side(w, l)) for l in range(8)]
    assert oo.level_side(489, 1) == 408  # cvRound(489 * (1.f / 1.2f)); cvRound(489 / 1.2f) = 407


def test_resize_scale_is_the_reciprocal_of_the_inverse_scale():
    """every side 41..4095 and every chained level: the taps with scale 1 / (dst / src) equal cv2.resize; src / dst differs
    only at 3993 -> 3328 (level 1).  The rows vary, the row count stays (a vertical scale of 1 takes row y from row y)."""
    rng = np.random.default_rng(1)
    wrong = set()
    for n in range(41, 4096):
        prev = n
        for l in range(1, 8):
            m = oo.level_side(n, l)
            img = rng.integers(0, 256, (8, prev), dtype=np.uint8)
            ref = po.resize_exact(img, m, 8)
            assert np.array_equal(po.resize_rows(img, m, True), ref), (n, l, prev, m)
            if not np.array_equal(po.resize_rows(img, m, False), ref):
                wrong.add((n, l))
            prev = m
    assert wrong == {(3993, 1)}
    assert oo.level_side(3993, 1) == 3328
    i_new, w_new = po.resize_table(3993, 3328, True)
    i_old, w_old = po.resize_table(3993, 3328, False)
    assert np.array_equal(i_new, i_old) and (w_new != w_old).sum() >= 1


def test_cell_and_mask_pyramids():
    """the mask pyramid keeps 255 only where every tap of the resize is 255 (TOZERO 254), and level 0 is the binarised
    mask; the cell pyramids are the pyramids of the cells' sub-images"""
    h, w = 480, 640
    img = po.corpus(h, w)["noise1"]
    mask = np.full((h, w), 7, np.uint8)
    mask[100:140, 200:330] = 0
    cells = po.cell_pyramids(img, mask)
    y0, y1, x0, x1 = oo._cells(w, h, 3)[4]
    lev, mlev = cells[4]
    assert np.array_equal(lev[0], img[y0:y1, x0:x1]) and set(np.unique(mlev[0])) == {0, 255}
    for l in range(1, 8):
        assert lev[l].shape == mlev[l].shape == (oo.level_side(y1 - y0, l), oo.level_side(x1 - x0, l))
        assert set(np.unique(mlev[l])) <= {0, 255}
        assert (mlev[l] == 0).sum() > (mlev[0] == 0).sum() / po.oo.layer_scale(l) ** 2  # the hole grows by the taps around it
