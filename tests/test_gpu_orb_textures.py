"""The ORB extractor and detector on dense textures against cv2 4.13, byte for byte (tests/orb_pyramid_oracle.py): the
extractor pyramid raw and blurred, the cell and mask pyramids, descriptors on the pixels where the blur's rounding
matters, and nodes where cv::ORB's per-level quotas decide what the frame keeps.  The rendered frames of the other tests
are smooth; these textures reach the rounding and the quotas at every frame size the tests cover."""
import numpy as np
import pytest

import node_helpers as nh
import orb_pyramid_oracle as po

pytestmark = pytest.mark.gpu

CAND_CAP = 12288  # candidates per (frame, cell) up to 1023 px per side (kOrbCandCap)
NAMES = list(po.corpus(96, 96))


@pytest.fixture(scope="module")
def fe(built):
    from rgbdslam_v2_b200 import Frontend
    f = Frontend(0, nh.params())
    yield f
    f.close()


def _holes(h, w):
    """a detection mask with holes: 48 px blocks, one in four kept"""
    y, x = np.indices((h, w))
    return np.where((y // 48 + x // 48) % 4 == 0, 255, 0).astype(np.uint8)


def _narrow(h, w):
    return max(h, w) <= 1023


@pytest.mark.parametrize("name", NAMES)
@pytest.mark.parametrize("hw", po.SIZES, ids=[f"{w}x{h}" for h, w in po.SIZES])
def test_extractor_planes(fe, hw, name):
    """planes 3 and 4 after orb_compute: the 8-level extractor pyramid and its blurred levels equal cv2's"""
    from oracle import orb_oracle
    h, w = hw
    img = po.corpus(h, w)[name]
    nh.reinit(fe, 0)
    kp = orb_oracle.records_to_array([dict(x=np.float32(w // 2), y=np.float32(h // 2), size=np.float32(31), angle=np.float32(0),
                                           response=np.float32(0), octave=7)])
    fe.orb_compute(img, kp)
    levels = po.pyramid(img)
    for l, (raw, blr) in enumerate(zip(levels, po.blurred(levels))):
        assert np.array_equal(fe.orb_debug_plane(3, 0, l), raw), (name, l)
        got = fe.orb_debug_plane(4, 0, l)
        assert got.shape == blr.shape and np.array_equal(got, blr), (name, l, np.argwhere(got != blr)[:4].tolist())


@pytest.mark.parametrize("name", NAMES)
@pytest.mark.parametrize("hw", po.SIZES, ids=[f"{w}x{h}" for h, w in po.SIZES])
def test_cell_planes(fe, hw, name):
    """planes 0 and 1 after orb_detect with a mask that has holes: every cell's pyramid and mask pyramid at every level"""
    h, w = hw
    img, mask = po.corpus(h, w)[name], _holes(h, w)
    det = nh.make_detector(fe, 0)
    fe.orb_detect(det, img, mask)
    if _narrow(h, w):
        assert all(len(fe.orb_debug_candidates(c)[0]) < CAND_CAP for c in range(9))
    for c, (levels, masks) in enumerate(po.cell_pyramids(img, mask)):
        for l in range(8):
            assert np.array_equal(fe.orb_debug_plane(0, c, l), levels[l]), (name, c, l)
            assert np.array_equal(fe.orb_debug_plane(1, c, l), masks[l]), (name, c, l)
    fe.detector_destroy(det)


ANGLES = [0.0, 17.5, 45.0, 90.0, 133.25, 180.0, 222.0, 270.0, 359.0]


def _kps(points):
    """keypoints at (level x, level y, octave), the angles cycling through ANGLES"""
    from oracle import orb_oracle
    rec = []
    for i, (lx, ly, o) in enumerate(points):
        s = orb_oracle.layer_scale(o)
        rec.append(dict(x=np.float32(lx) * s, y=np.float32(ly) * s, size=np.float32(31) * s, angle=np.float32(ANGLES[i % len(ANGLES)]),
                        response=np.float32(1), octave=o))
    return orb_oracle.records_to_array(rec)


def _probe_points(img):
    """level positions around every pixel where the unfused or the all-fused blur differs from cv2, plus a grid at every
    octave"""
    pts = []
    levels = po.pyramid(img)
    for l, (lev, ref) in enumerate(zip(levels, po.blurred(levels))):
        lh, lw = lev.shape
        bad = np.argwhere((po.blur(lev, False) != ref) | (po.blur(lev, True) != ref))
        for y, x in bad[:40]:
            pts += [(x + dx, y + dy, l) for dy in range(-12, 13, 6) for dx in range(-12, 13, 6)]
        pts += [(x, y, l) for y in range(20, lh - 20, max(8, lh // 6)) for x in range(20, lw - 20, max(8, lw // 6))]
    return pts


@pytest.mark.parametrize("hw", po.SIZES, ids=[f"{w}x{h}" for h, w in po.SIZES])
def test_descriptors(fe, hw):
    """orb_compute equals cv2's compute (border filter, octave order, descriptors) on every corpus frame, with keypoints
    whose patches read the pixels where the blur's rounding rules part, at all 8 octaves and a sweep of angles; at
    3993 px, keypoints along the level-1 column whose resize weight depends on the scale rule"""
    from oracle import orb_oracle
    h, w = hw
    nh.reinit(fe, 0)
    for name, img in po.corpus(h, w).items():
        pts = _probe_points(img)
        if w == 3993:
            i_new, w_new = po.resize_table(3993, 3328, True)
            d = int(np.argmax(w_new != po.resize_table(3993, 3328, False)[1]))
            pts += [(d + dx, y, 1) for dx in range(-14, 15, 2) for y in range(20, 280, 16)]
        kp = _kps(pts)
        gk, gd = fe.orb_compute(img, kp)
        ok, od = orb_oracle.orb_compute(img, kp)
        assert len(gk) == len(ok) > 0
        assert gk.tobytes() == ok.tobytes(), name
        bad = np.nonzero((gd != od).any(1))[0]
        assert len(bad) == 0, (name, len(bad), [tuple(ok[i][["x", "y", "angle", "octave"]]) for i in bad[:4]])


_SEQ = {}


def _sequence(h, w):
    """3 frames of band-limited noise (sigma 1.0) with the rendered scene's depth and its mask; at 1023x1023 the mask keeps
    one 48 px block in three, so that no cell stores more than CAND_CAP candidates"""
    from oracle import orb_oracle
    from rgbdslam_v2_b200 import synth
    if (h, w) not in _SEQ:
        poses = synth.trajectory(240)
        depth = np.stack([synth.render_frame(poses[k], seed=k, shape=(h, w))[1] for k in range(3)])
        mask = np.stack([orb_oracle.depth_to_mask(d) for d in depth])
        if h > 480:
            y, x = np.indices((h, w))
            mask = np.where((y // 48 + x // 48) % 3 == 0, mask, 0).astype(np.uint8)
        _SEQ[(h, w)] = nh.textured(h, w, 3, 0, 1.0), depth, mask, synth.intrinsics(w, h)
    return _SEQ[(h, w)]


NODE_SIZES = [(480, 640), (1023, 1023)]


@pytest.mark.parametrize("iters", [1, 5])
@pytest.mark.parametrize("K", [600, 2000])
@pytest.mark.parametrize("detector", [0, 1], ids=["ORB", "FAST"])
@pytest.mark.parametrize("hw", NODE_SIZES, ids=[f"{w}x{h}" for h, w in NODE_SIZES])
def test_nodes_on_dense_texture(fe, hw, detector, K, iters):
    """Node::Node over a 3-frame sequence, thresholds carried: keypoints, descriptors, points and thresholds equal the
    oracle, no cell overflowing the candidate buffer.  ORB: cv::ORB's per-level quotas bind in every cell of the first
    frame.  The FAST detector has no quotas."""
    import fast_oracle
    from oracle import orb_oracle
    h, w = hw
    gray, depth, mask, K4 = _sequence(h, w)
    construct = orb_oracle.node_construct if detector == 0 else fast_oracle.node_construct
    det = nh.make_detector(fe, detector, max_keypoints=K, adjuster_max_iterations=iters)
    st = orb_oracle.DetectorState()
    got = []
    for k in range(3):
        hs, _ = fe.nodes_create(det, gray[k:k + 1], depth[k:k + 1], mask[k:k + 1], K4)
        assert all(len(fe.orb_debug_candidates(c)[0]) < CAND_CAP for c in range(9)), k
        okp, odesc, oxyz = construct(gray[k], depth[k], mask[k], K4, st, max_keypoints=K, max_iters=iters)
        gkp = fe.node_keypoints(hs[0])
        gdesc, gxyz = fe.node_download(hs[0])
        assert len(gkp) == len(okp) > 0, k
        assert gkp.tobytes() == okp.tobytes(), k
        assert np.array_equal(gdesc, odesc), k
        assert np.array_equal(gxyz.view(np.uint32), oxyz.view(np.uint32)), k
        assert np.array_equal(fe.detector_thresholds(det)[:9], np.array(st.thresh[:9])), k
        got.append(gkp.tobytes())
        nh.destroy(fe, hs)
    fe.detector_destroy(det)
    if detector == 0:  # frame 0 (threshold 20 everywhere): cv::ORB's quotas cull keypoints in every cell
        import orb_quota_oracle as qo
        for c, (y0, y1, x0, x1) in enumerate(orb_oracle._cells(w, h, 3)):
            sub, smask = np.ascontiguousarray(gray[0, y0:y1, x0:x1]), np.ascontiguousarray(mask[0, y0:y1, x0:x1])
            assert len(qo.detect(sub, smask, 20, 10000)) < len(qo.detect(sub, smask, 20, qo.UNBOUND)), c
    nh.reinit(fe, 0)
