"""GPU tests of the listener's raw inputs to the Node constructor: RGBDSLAM_B200_DEPTH_U16 (16UC1 millimetres, converted and
optionally masked on the device) and RGBDSLAM_B200_VISUAL_BAYER_GR (debayered on the device).  Each is pinned bit for bit to
the existing float-depth / grey / colour path fed the restatements of tests/raw_input_oracle.py, with the detector thresholds
compared after the call."""
import cv2
import numpy as np
import pytest

import node_helpers as nh
import raw_input_oracle as ro

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def fe(built):
    from rgbdslam_v2_b200 import Frontend
    f = Frontend(0, nh.params(0))
    yield f
    f.close()


def _colour(gray):
    """a colour image whose channels differ (channel 0 = R)"""
    return np.ascontiguousarray(np.stack([gray, np.roll(gray, 3, axis=-1), np.roll(gray, 5, axis=-2)], -1))


def _plant(u16, k):
    """patches below 0.51 m, values at and around 510, and (frame 1) every one of the 65536 values"""
    d = u16.copy()
    rng = np.random.default_rng(k)
    d[40:130, 60:220] = rng.integers(1, 510, (90, 160))
    d[200:280, 300:440] = rng.integers(505, 516, (80, 140))
    d[300:380, 40:200] = 510
    if k == 1:
        d[100:356, 200:456] = rng.permutation(65536).reshape(256, 256)
    return d


def _millimetres(depth):
    return np.stack([_plant(ro.to_millimetres(d), k) for k, d in enumerate(depth)])


@pytest.fixture(scope="module")
def planted():
    gray, depth = nh.stack(nh.render(range(4)))
    return gray, _millimetres(depth)


def _run(fe, detector, fn, **kw):
    """nodes of fn(det) with a fresh detector: (node dumps, thresholds, launches)"""
    det = nh.make_detector(fe, detector, **kw)
    l0 = fe.lib.rgbdslam_b200_launch_count()
    hs = fn(det)
    launches = fe.lib.rgbdslam_b200_launch_count() - l0
    out = (nh.node_dump(fe, hs), fe.detector_thresholds(det).copy(), launches)
    fe.detector_destroy(det)
    nh.destroy(fe, hs)
    return out


def _same(a, b, min_features=100):
    assert nh.same_nodes(a[0], b[0]) and min(len(k) for k, _, _ in a[0]) > min_features
    assert np.array_equal(a[1], b[1])


@pytest.mark.parametrize("min_depth", [0, 1])
@pytest.mark.parametrize("mask_mode", ["from_depth", "caller", "none"])
@pytest.mark.parametrize("detector", [0, 1], ids=["ORB", "FAST"])
def test_u16_nodes_equal_float_path(fe, planted, detector, mask_mode, min_depth):
    """DEPTH_U16 == nodes_create_ex fed (float)d * 0.001f and, with MASK_FROM_DEPTH, the restated 16-bit mask as a caller
    mask; grey and colour visuals; one launch more (k_depth_u16)."""
    from oracle import orb_oracle as oo
    gray, u16 = planted
    zf = ro.depth_u16_to_m(u16)
    caller = np.stack([oo.depth_to_mask(d) for d in zf])
    K4 = nh.K4()
    zeros = 0
    for vis in (gray, np.stack([_colour(g) for g in gray])):
        if mask_mode == "from_depth":
            a = _run(fe, detector, lambda det: fe.nodes_create(det, vis, u16, None, K4, mask_from_depth=True)[0],
                     use_feature_min_depth=min_depth)
            b = _run(fe, detector, lambda det: fe.nodes_create(det, vis, zf, ro.depth_u16_mask(u16), K4)[0],
                     use_feature_min_depth=min_depth)
        else:
            m = caller if mask_mode == "caller" else None
            a = _run(fe, detector, lambda det: fe.nodes_create(det, vis, u16, m, K4)[0], use_feature_min_depth=min_depth)
            b = _run(fe, detector, lambda det: fe.nodes_create(det, vis, zf, m, K4)[0], use_feature_min_depth=min_depth)
        _same(a, b, 20 if min_depth else 100)  # with the minimum rule the planted frames lose most keypoints to holes
        assert a[2] == b[2] + 1
        zeros += sum(int((x[:, 2] == 0).sum()) for _, _, x in a[0])
    if min_depth:  # a neighbourhood that touches a hole has minimum 0 -> NaN -> dropped
        assert zeros == 0
    print(f"points with z = 0: {zeros}")


def test_u16_mask_rejects_the_near_range(fe, planted):
    """with MASK_FROM_DEPTH no keypoint sits in the patches below 0.51 m, which the float rule accepts; the patch at exactly
    510 mm is accepted (the fused rule; an unfused one would reject it)"""
    gray, u16 = planted
    K4 = nh.K4()
    det = nh.make_detector(fe, 1)  # FAST: every keypoint is on level 0, at its pixel
    hs = fe.nodes_create(det, gray, u16, None, K4, mask_from_depth=True)[0]
    at_510 = 0
    for k, h in enumerate(hs):
        kp = fe.node_keypoints(h)
        x, y = np.rint(kp["x"]).astype(int), np.rint(kp["y"]).astype(int)
        assert len(kp) > 100 and (u16[k][y, x] >= 510).all()
        at_510 += int((u16[k][y, x] == 510).sum())
    assert at_510 > 0
    fe.detector_destroy(det)
    nh.destroy(fe, hs)


@pytest.mark.parametrize("detector", [0, 1], ids=["ORB", "FAST"])
def test_bayer_equals_rgb_path_fed_cvtcolor(fe, planted, detector):
    """VISUAL_BAYER_GR, with float or 16-bit depth, == VISUAL_RGB fed cv2.cvtColor(COLOR_BayerGR2RGB); the Bayer kernel
    takes the place of k_rgb_to_gray"""
    gray, u16 = planted
    raw = np.stack([ro.mosaic_gr(_colour(g)) for g in gray])
    rgb = np.stack([cv2.cvtColor(r, cv2.COLOR_BayerGR2RGB) for r in raw])
    K4 = nh.K4()
    for dep in (u16, ro.depth_u16_to_m(u16)):
        a = _run(fe, detector, lambda det: fe.nodes_create(det, raw, dep, None, K4, mask_from_depth=True, bayer=True)[0])
        b = _run(fe, detector, lambda det: fe.nodes_create(det, rgb, dep, None, K4, mask_from_depth=True)[0])
        _same(a, b)
        assert a[2] == b[2]


def _pad(a, W, H):
    pad = ((0, 0), (0, H - a.shape[1]), (0, W - a.shape[2])) + ((0, 0),) * (a.ndim - 3)
    return np.ascontiguousarray(np.pad(a, pad, mode="edge"))


@pytest.fixture(scope="module")
def seq70():
    """70 frames (more than one 64-frame chunk): 24 rendered frames, repeated"""
    gray, depth = nh.stack(nh.render(range(24)))
    idx = np.arange(70) % 24
    return gray[idx], _millimetres(depth)[idx]


CONFIGS = {"gray_u16_maskdepth_ORB": ("gray", True, "depth", 0), "bayer_u16_caller_FAST": ("bayer", True, "caller", 1),
           "bayer_float_maskdepth_ORB": ("bayer", False, "depth", 0)}


@pytest.mark.parametrize("size", [(640, 480), (641, 481)], ids=["640x480", "641x481"])
@pytest.mark.parametrize("config", list(CONFIGS))
def test_pipeline_variants_identical(fe, seq70, config, size):
    """70 frames in one call (two chunks) == one chunk per frame == from pinned memory == 1-rank sharded; at 641 px the 16-bit
    and Bayer rows are not 4-byte aligned"""
    import torch

    from oracle import orb_oracle as oo
    vis_kind, u16_depth, mask_kind, detector = CONFIGS[config]
    W, H = size
    gray, u16 = _pad(seq70[0], W, H), _pad(seq70[1], W, H)
    n = len(gray)
    vis = np.stack([ro.mosaic_gr(_colour(g)) for g in gray]) if vis_kind == "bayer" else gray
    dep = u16 if u16_depth else ro.depth_u16_to_m(u16)
    mask = np.stack([oo.depth_to_mask(d) for d in ro.depth_u16_to_m(u16)]) if mask_kind == "caller" else None
    kw = dict(mask_from_depth=mask_kind == "depth", bayer=vis_kind == "bayer")
    K4 = nh.K4()
    ref = _run(fe, detector, lambda det: fe.nodes_create(det, vis, dep, mask, K4, **kw)[0])
    assert len(ref[0]) == n

    def one_by_one(det):
        hs = []
        for k in range(n):
            hs += fe.nodes_create(det, vis[k:k + 1], dep[k:k + 1], None if mask is None else mask[k:k + 1], K4, ids=[k], **kw)[0]
        return hs
    _same(ref, _run(fe, detector, one_by_one))
    pv, pd = torch.from_numpy(vis).pin_memory(), torch.from_numpy(dep).pin_memory()
    pm = None if mask is None else torch.from_numpy(mask).pin_memory()
    _same(ref, _run(fe, detector, lambda det: fe.nodes_create(det, pv, pd, pm, K4, **kw)[0]))
    comm = fe.comm_init(0, 1, fe.comm_unique_id())
    _same(ref, _run(fe, detector, lambda det: fe.nodes_create_sharded(det, comm, n, vis, dep, mask, K4, **kw)[0]))
    fe.comm_destroy(comm)


def test_measurement_model_counts_equal_float_nodes(fe, planted):
    """pairs of 16-bit nodes: the measurement model runs on the converted plane, so its counts (and the gate) equal those of
    the float-path nodes"""
    gray, u16 = planted
    K4 = nh.K4()
    zf = ro.depth_u16_to_m(u16)
    out = []
    for dep, m, kw in ((u16, None, {"mask_from_depth": True}), (zf, ro.depth_u16_mask(u16), {})):
        det = nh.make_detector(fe, 0, observability_threshold=0.75)
        hs = fe.nodes_create(det, gray, dep, m, K4, **kw)[0]
        res, _, _ = fe.match_node_pairs(hs[1:] + hs[2:], hs[:-1] + hs[:-2], seed=3)
        out.append(res.copy())
        fe.detector_destroy(det)
        nh.destroy(fe, hs)
    nh.reinit(fe, 0)
    a, b = out
    for f in ("id1", "id2", "n_all_matches", "n_inliers", "inlier_points", "outlier_points", "occluded_points", "all_points"):
        assert np.array_equal(a[f], b[f]), f
    assert np.array_equal(a["ransac_trafo"], b["ransac_trafo"])
    assert (a["all_points"] > 0).any()


def test_matcher_on_points_with_zero_depth(fe, oracle_mod):
    """points with z = 0 (a 16-bit hole under a kept keypoint): RANSAC's scoring skips them and a sample holding one fits a
    non-finite transformation, on the device as in the oracle -- matches equal, validity equal, no such point among the
    inliers, inlier counts within the float tolerance of the smoke test.  The transformations are refitted on inlier sets
    that may differ by those rows: on these batches their translations differ by up to 2.4e-3 m (one pair of six), hence
    5e-3 here against the smoke test's 2e-3."""
    from rgbdslam_v2_b200 import synth
    b = synth.make_batch(6, 500, seed0=300)
    for key, step in (("xyz_newer", 7), ("xyz_older", 11)):
        b[key][::step, 2] = 0.0
    res, allm, inl = fe.match_pairs_host(b["desc_newer"], b["xyz_newer"], b["n_newer"], b["desc_older"], b["xyz_older"],
                                         b["n_older"], b["id_newer"], b["id_older"], seed=7)
    op = oracle_mod.make_params(depth_cov_z0=2.0)
    ores, oall, oinl = oracle_mod.match_pairs(op, b["desc_newer"], b["xyz_newer"], b["n_newer"], b["desc_older"], b["xyz_older"],
                                              b["n_older"], b["id_newer"], b["id_older"], seed=7)
    assert (res["id1"] >= 0).any()
    for i in range(len(res)):
        n = int(res[i]["n_all_matches"])
        assert n == ores[i]["n_all_matches"] and np.array_equal(allm[i, :n], oall[i, :n])
        assert res[i]["id1"] == ores[i]["id1"] and res[i]["id2"] == ores[i]["id2"]
        if res[i]["id1"] < 0:
            continue
        for r, lst in ((res[i], inl[i]), (ores[i], oinl[i])):
            m = lst[:int(r["n_inliers"])]
            zq = b["xyz_newer"][500 * i + m["queryIdx"], 2]
            zt = b["xyz_older"][500 * i + m["trainIdx"], 2]
            assert (zq != 0).all() and (zt != 0).all()
        assert abs(int(res[i]["n_inliers"]) - int(ores[i]["n_inliers"])) <= 2
        assert np.abs(res[i]["ransac_trafo"] - ores[i]["ransac_trafo"]).max() < 5e-3


def test_rejected_combinations_launch_nothing(fe, planted):
    from rgbdslam_v2_b200._capi import (CLOUD_XYZ, CLOUD_XYZRGB, DEPTH_U16, MASK_FROM_DEPTH, VISUAL_BAYER_GR, VISUAL_RGB,
                                        _ptr)
    gray, u16 = planted
    det = nh.make_detector(fe, 0)
    K4 = np.array(nh.K4(), np.float32)
    H, W = gray.shape[1:]
    buf = np.zeros((1, H, W, 8), np.float32)  # large enough for every reading of the flags
    vis = np.zeros((1, H, W, 3), np.uint8)
    handles = np.zeros(1, np.uint64)
    nf = np.zeros(1, np.int32)
    comm = fe.comm_init(0, 1, fe.comm_unique_id())
    cases = ((DEPTH_U16 | CLOUD_XYZRGB, b"DEPTH_U16"), (DEPTH_U16 | CLOUD_XYZ | MASK_FROM_DEPTH, b"MASK_FROM_DEPTH"),
             (VISUAL_BAYER_GR | VISUAL_RGB, b"exclusive"), (VISUAL_BAYER_GR | CLOUD_XYZ, b"VISUAL_BAYER_GR"),
             (VISUAL_BAYER_GR | DEPTH_U16 | CLOUD_XYZRGB, b"DEPTH_U16"), (1024, b"unknown"), (DEPTH_U16 | 2048, b"unknown"))
    for flags, word in cases:
        for sharded in (False, True):
            l0 = fe.lib.rgbdslam_b200_launch_count()
            if sharded:
                rc = fe.lib.rgbdslam_b200_nodes_create_sharded(det, comm, 1, _ptr(vis), _ptr(buf), None, W, H, _ptr(K4), None, flags,
                                                               _ptr(handles), _ptr(nf))
            else:
                rc = fe.lib.rgbdslam_b200_nodes_create_ex(det, 1, _ptr(vis), _ptr(buf), None, W, H, _ptr(K4), None, flags,
                                                          _ptr(handles), _ptr(nf))
            assert fe.lib.rgbdslam_b200_launch_count() == l0
            assert rc == 1 and word in fe.lib.rgbdslam_b200_last_error(), (flags, sharded)
    fe.comm_destroy(comm)
    fe.detector_destroy(det)
