"""GPU tests of the Node constructor for depth images of another size than the visual (include/rgbdslam_b200/depth_resize.h):
nodes_create_resized must be bit-identical to nodes_create_ex on the same visuals and cv2.resize(depth, (w, h), INTER_NEAREST)
-- the listener's resize (openni_listener.cpp:651-656), the oracle -- in features, 3-D points, detector thresholds, stored
clouds and measurement-model counts, for smaller, larger, non-integer-ratio and tiny depth images."""
import cv2
import numpy as np
import pytest

import node_helpers as nh
import raw_input_oracle as ro

pytestmark = pytest.mark.gpu

# (w, h, dw, dh): visual and depth sizes -- depth smaller, larger, at non-integer ratios and tiny; sensor pairs
PAIRS = [(640, 480, 320, 240), (640, 480, 1280, 960), (640, 480, 512, 424), (640, 480, 97, 61), (1280, 1024, 640, 480),
         (1920, 1080, 512, 424), (1280, 720, 640, 480)]


def _pid(p):
    return "{}x{}-{}x{}".format(*p)


@pytest.fixture(scope="module")
def fe(built):
    from rgbdslam_v2_b200 import Frontend
    f = Frontend(0, nh.params(0))
    yield f
    f.close()


_RENDERED = {}


def _render(h, w, k):
    """frame k of the 240-pose trajectory rendered at h x w (the 640x480 camera's field of view)"""
    from rgbdslam_v2_b200 import synth
    if (h, w, k) not in _RENDERED:
        _RENDERED[h, w, k] = synth.render_frame(synth.trajectory(240)[k], seed=k, shape=(h, w))
    return _RENDERED[h, w, k]


def frames(w, h, dw, dh, n=3, u16=False):
    """n frames: the visual rendered at w x h, the depth rendered at dw x dh (float metres or 16-bit millimetres), the depth
    cv2 resizes to w x h, and the visual camera"""
    from rgbdslam_v2_b200 import synth
    gray = np.stack([_render(h, w, k)[0] for k in range(n)])
    depth = np.stack([_render(dh, dw, k)[1] for k in range(n)])
    if u16:
        depth = np.stack([ro.to_millimetres(d) for d in depth])
    big = np.stack([cv2.resize(d, (w, h), interpolation=cv2.INTER_NEAREST) for d in depth])
    return gray, depth, big, synth.intrinsics(w, h)


def _run(fe, fn, clouds=False, **kw):
    """nodes of fn(det) with a fresh detector of the parameters kw: (node dumps, thresholds, launches, stored clouds)"""
    det = nh.make_detector(fe, 0, **kw)
    l0 = fe.lib.rgbdslam_b200_launch_count()
    hs = fn(det)
    launches = fe.lib.rgbdslam_b200_launch_count() - l0
    cl = [(fe.node_cloud(h, 16), fe.node_cloud(h, 32)) for h in hs] if clouds else None
    out = (nh.node_dump(fe, hs), fe.detector_thresholds(det).copy(), launches, cl)
    fe.detector_destroy(det)
    nh.destroy(fe, hs)
    return out


def _same(a, b, min_features=50):
    assert nh.same_nodes(a[0], b[0]) and min(len(k) for k, _, _ in a[0]) > min_features
    assert np.array_equal(a[1], b[1])
    if a[3] is not None or b[3] is not None:
        for (a16, a32), (b16, b32) in zip(a[3], b[3]):
            assert a16.tobytes() == b16.tobytes() and a32.tobytes() == b32.tobytes()


def _caller_mask(big, u16):
    from oracle import orb_oracle as oo
    z = ro.depth_u16_to_m(big) if u16 else big
    return np.stack([oo.depth_to_mask(d) for d in z])


@pytest.mark.parametrize("mask_mode", ["none", "caller", "from_depth"])
@pytest.mark.parametrize("u16", [False, True], ids=["float", "u16"])
@pytest.mark.parametrize("pair", PAIRS, ids=_pid)
def test_resized_equals_host_resize(fe, pair, u16, mask_mode):
    """nodes_create_resized == nodes_create_ex on cv2.resize(INTER_NEAREST)'d depth; the resize costs one launch per chunk
    for float depth and none for 16-bit depth, whose conversion kernel does it"""
    gray, depth, big, K4 = frames(*pair, u16=u16)
    mask = _caller_mask(big, u16) if mask_mode == "caller" else None
    kw = dict(mask_from_depth=mask_mode == "from_depth")
    ref = _run(fe, lambda det: fe.nodes_create(det, gray, big, mask, K4, **kw)[0])
    got = _run(fe, lambda det: fe.nodes_create_resized(det, gray, depth, mask, K4, **kw)[0])
    _same(got, ref)
    assert got[2] == ref[2] + (0 if u16 else 1)


@pytest.mark.parametrize("visual", ["rgb", "bayer"])
def test_colour_and_bayer_visuals(fe, visual):
    pair = (1280, 1024, 640, 480) if visual == "rgb" else (640, 480, 512, 424)
    gray, depth, big, K4 = frames(*pair, u16=True)
    col = np.stack([np.stack([g, np.roll(g, 3, axis=-1), np.roll(g, 5, axis=-2)], -1) for g in gray])
    vis = np.ascontiguousarray(col) if visual == "rgb" else np.stack([ro.mosaic_gr(c) for c in col])
    kw = dict(mask_from_depth=True, bayer=visual == "bayer")
    ref = _run(fe, lambda det: fe.nodes_create(det, vis, big, None, K4, **kw)[0])
    _same(_run(fe, lambda det: fe.nodes_create_resized(det, vis, depth, None, K4, **kw)[0]), ref)


@pytest.mark.parametrize("encoding_rgb", [False, True], ids=["bgr", "rgb"])
@pytest.mark.parametrize("pair,u16", [((640, 480, 320, 240), False), ((1280, 720, 640, 480), True)], ids=["float", "u16"])
def test_store_cloud(fe, pair, u16, encoding_rgb):
    """STORE_CLOUD: the stored colour clouds, downloaded at 16 and 32 bytes per point, equal the host-resized nodes'"""
    gray, depth, big, K4 = frames(*pair, u16=u16)
    col = np.ascontiguousarray(np.stack([np.stack([g, 255 - g, g // 2], -1) for g in gray]))
    kw = dict(mask_from_depth=True, store_cloud=True, encoding_rgb=encoding_rgb)
    ref = _run(fe, lambda det: fe.nodes_create(det, col, big, None, K4, **kw)[0], clouds=True)
    _same(_run(fe, lambda det: fe.nodes_create_resized(det, col, depth, None, K4, **kw)[0], clouds=True), ref)
    assert any(np.isfinite(c32["z"]).any() for _, c32 in ref[3])


@pytest.mark.parametrize("setting", ["use_feature_min_depth", "depth_scaling_factor"])
def test_min_depth_and_depth_scaling(fe, setting):
    """float depth with use_feature_min_depth (a 16-bit hole reads as 0 m, which empties a neighbourhood's minimum), 16-bit
    depth with depth_scaling_factor != 1"""
    pair, u16, prm = (((640, 480, 512, 424), False, {"use_feature_min_depth": 1}) if setting == "use_feature_min_depth" else
                      ((1280, 1024, 640, 480), True, {"depth_scaling_factor": 1.07}))
    gray, depth, big, K4 = frames(*pair, u16=u16)
    ref = _run(fe, lambda det: fe.nodes_create(det, gray, big, None, K4, mask_from_depth=True)[0], **prm)
    _same(_run(fe, lambda det: fe.nodes_create_resized(det, gray, depth, None, K4, mask_from_depth=True)[0], **prm), ref,
          min_features=10)
    nh.reinit(fe, 0)


@pytest.mark.parametrize("config", ["u16_maskdepth", "float_caller"])
def test_chunks_pinned_and_sharded(fe, config):
    """70 frames in one call (two chunks of 64) == the host-resized call == one call per frame == from pinned memory == a 1-rank
    _sharded_resized call"""
    import torch
    u16 = config.startswith("u16")
    gray, depth, big, K4 = frames(640, 480, 320, 240, n=70, u16=u16)
    mask = _caller_mask(big, u16) if config.endswith("caller") else None
    kw = dict(mask_from_depth=mask is None)
    n = len(gray)
    ref = _run(fe, lambda det: fe.nodes_create(det, gray, big, mask, K4, **kw)[0])
    assert len(ref[0]) == n
    got = _run(fe, lambda det: fe.nodes_create_resized(det, gray, depth, mask, K4, **kw)[0])
    _same(got, ref)
    assert got[2] == ref[2] + (0 if u16 else 2)  # one gather launch per chunk

    def one_by_one(det):
        hs = []
        for k in range(n):
            hs += fe.nodes_create_resized(det, gray[k:k + 1], depth[k:k + 1], None if mask is None else mask[k:k + 1], K4, ids=[k],
                                          **kw)[0]
        return hs
    _same(_run(fe, one_by_one), ref)
    pg, pd = torch.from_numpy(gray).pin_memory(), torch.from_numpy(depth).pin_memory()
    pm = None if mask is None else torch.from_numpy(mask).pin_memory()
    _same(_run(fe, lambda det: fe.nodes_create_resized(det, pg, pd, pm, K4, **kw)[0]), ref)
    comm = fe.comm_init(0, 1, fe.comm_unique_id())
    _same(_run(fe, lambda det: fe.nodes_create_sharded_resized(det, comm, n, gray, depth, mask, K4, **kw)[0]), ref)
    fe.comm_destroy(comm)


def test_measurement_model_counts(fe):
    """observability_threshold > 0: the model reads the resized plane, so match_node_pairs on resized nodes returns the
    host-resized nodes' results and counts"""
    gray, depth, big, K4 = frames(640, 480, 320, 240, n=4, u16=True)
    out = []
    for dep, fn in ((big, fe.nodes_create), (depth, fe.nodes_create_resized)):
        det = nh.make_detector(fe, 0, observability_threshold=0.75)
        hs = fn(det, gray, dep, None, K4, mask_from_depth=True)[0]
        res, _, _ = fe.match_node_pairs(hs[1:] + hs[2:], hs[:-1] + hs[:-2], seed=3)
        out.append(res.copy())
        fe.detector_destroy(det)
        nh.destroy(fe, hs)
    nh.reinit(fe, 0)
    a, b = out
    for f in ("id1", "id2", "n_all_matches", "n_inliers", "inlier_points", "outlier_points", "occluded_points", "all_points"):
        assert np.array_equal(a[f], b[f]), f
    assert np.array_equal(a["ransac_trafo"].view(np.uint32), b["ransac_trafo"].view(np.uint32))
    assert (a["all_points"] > 0).any() and (a["id1"] >= 0).any()


@pytest.mark.parametrize("u16", [False, True], ids=["float", "u16"])
def test_equal_sizes_are_nodes_create_ex(fe, u16):
    """depth_w == w and depth_h == h: the call is nodes_create_ex, launches included"""
    gray, depth, big, K4 = frames(640, 480, 640, 480, u16=u16)
    assert np.array_equal(depth.view(np.uint8), big.view(np.uint8))
    ref = _run(fe, lambda det: fe.nodes_create(det, gray, depth, None, K4, mask_from_depth=True)[0])
    got = _run(fe, lambda det: fe.nodes_create_resized(det, gray, depth, None, K4, mask_from_depth=True)[0])
    _same(got, ref)
    assert got[2] == ref[2]


def test_rejections_launch_nothing(fe):
    from rgbdslam_v2_b200._capi import (CLOUD_XYZ, CLOUD_XYZRGB, DEPTH_U16, ENCODING_RGB, KEEP_CLOUD, MASK_FROM_CLOUD,
                                        STORE_CLOUD, VISUAL_BAYER_GR, VISUAL_RGB, _ptr)
    det = nh.make_detector(fe, 0)
    W, H = 640, 480
    K4 = np.array(nh.K4(), np.float32)
    vis = np.zeros((1, H, W, 3), np.uint8)
    buf = np.zeros((1, 4095, 4095), np.float32)  # large enough for every depth size below
    handles = np.zeros(1, np.uint64)
    nf = np.zeros(1, np.int32)
    comm = fe.comm_init(0, 1, fe.comm_unique_id())
    # (flags, depth_w, depth_h, w, h, error word, sharded only)
    cases = [(0, 0, 240, W, H, b"depth_w", False), (0, 320, 0, W, H, b"depth_w", False), (0, -1, 240, W, H, b"depth_w", False),
             (0, 4096, 240, W, H, b"depth_w", False), (0, 320, 4096, W, H, b"depth_w", False),
             (CLOUD_XYZRGB, 320, 240, W, H, b"depth images only", False), (CLOUD_XYZ, 320, 240, W, H, b"depth images only", False),
             (MASK_FROM_CLOUD, 320, 240, W, H, b"depth images only", False), (KEEP_CLOUD, 320, 240, W, H, b"depth images only", False),
             (DEPTH_U16 | CLOUD_XYZ, 320, 240, W, H, b"depth images only", False),
             (VISUAL_BAYER_GR | VISUAL_RGB, 320, 240, W, H, b"exclusive", False), (1024, 320, 240, W, H, b"unknown", False),
             (ENCODING_RGB, 320, 240, W, H, b"ENCODING_RGB", False), (0, 320, 240, 95, H, b"image size", False),
             (0, 320, 240, W, 4096, b"image size", False), (STORE_CLOUD, 320, 240, W, H, b"STORE_CLOUD", True)]
    nh.reinit(fe, 0, cloud_creation_skip_step=2)
    cases.append((STORE_CLOUD, 320, 240, 641, H, b"skip_step", False))
    for flags, dw, dh, w, h, word, sharded_only in cases:
        for sharded in (False, True) if not sharded_only else (True,):
            if flags == STORE_CLOUD and w == 641 and sharded:
                continue
            l0 = fe.lib.rgbdslam_b200_launch_count()
            if sharded:
                rc = fe.lib.rgbdslam_b200_nodes_create_sharded_resized(det, comm, 1, _ptr(vis), _ptr(buf), dw, dh, None, w, h, _ptr(K4),
                                                                       None, flags, _ptr(handles), _ptr(nf))
            else:
                rc = fe.lib.rgbdslam_b200_nodes_create_resized(det, 1, _ptr(vis), _ptr(buf), dw, dh, None, w, h, _ptr(K4), None, flags,
                                                               _ptr(handles), _ptr(nf))
            assert fe.lib.rgbdslam_b200_launch_count() == l0
            assert rc == 1 and word in fe.lib.rgbdslam_b200_last_error(), (flags, dw, dh, w, h, sharded,
                                                                          fe.lib.rgbdslam_b200_last_error())
    nh.reinit(fe, 0)
    fe.comm_destroy(comm)
    fe.detector_destroy(det)
