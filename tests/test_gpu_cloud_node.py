"""GPU parity tests of the point-cloud Node constructor (node.cpp:252-369) and of colour input to both constructors, checked
bit for bit against tests/cloud_oracle.py (on top of the cv2-based ORB and FAST detection oracles), with the detector
thresholds compared after every frame."""
import copy

import cv2
import numpy as np
import pytest

import node_helpers as nh
from node_helpers import MAXK

pytestmark = pytest.mark.gpu

SCENARIOS = ["mask", "no_mask", "mask_from_cloud", "planted", "trunc"]


@pytest.fixture(scope="module")
def fe(built):
    from rgbdslam_v2_b200 import Frontend
    f = Frontend(0, nh.params(0))
    yield f
    f.close()


def _colour(gray):
    """a colour image whose channels differ (channel 0 = R)"""
    return np.ascontiguousarray(np.stack([gray, np.roll(gray, 3, axis=-1), np.roll(gray, 5, axis=-2)], -1))


def _render(n):
    return nh.stack(nh.render(range(n)))


@pytest.fixture(scope="module")
def frames():
    return _render(4)


@pytest.fixture(scope="module")
def seq24():
    """24 frames: several chunks of the constructor's pipeline with cloud input"""
    return _render(24)


def _plant_values(cloud, seed):
    """blobs where only x is NaN, where z is NaN, where z is +inf"""
    c = cloud.copy()
    H, W = c.shape[:2]
    rng = np.random.default_rng(seed)
    for k in range(90):
        y, x = int(rng.integers(0, H - 8)), int(rng.integers(0, W - 8))
        s = int(rng.integers(2, 8))
        if k % 3 == 0:
            c[y:y + s, x:x + s, 0] = np.nan
        elif k % 3 == 1:
            c[y:y + s, x:x + s, 2] = np.nan
        else:
            c[y:y + s, x:x + s, 2] = np.inf
    return c


def _plant_trunc(cloud, rec):
    """for keypoints whose truncated and rounded pixels differ: NaN at the truncated pixel of every other one, NaN at the
    rounded pixel of the rest; for the others NaN under every fourth keypoint"""
    c = cloud.copy()
    at_round = []
    for i, r in enumerate(rec):
        x, y = np.float32(r["x"]), np.float32(r["y"])
        tx, ty = int(x), int(y)
        rx, ry = int(np.floor(x + np.float32(0.5))), int(np.floor(y + np.float32(0.5)))
        if (tx, ty) != (rx, ry):
            if i % 2:
                c[ty, tx, 1] = np.nan
            else:
                c[ry, rx, 2] = np.nan
                at_round.append((rx, ry))
        elif i % 4 == 0:
            c[ty, tx, 2] = np.nan
    return c, at_round


@pytest.mark.parametrize("scenario", SCENARIOS)
@pytest.mark.parametrize("detector", [0, 1], ids=["ORB", "FAST"])
def test_cloud_nodes_vs_oracle(fe, frames, scenario, detector):
    """Node(visual, detector, extractor, point_cloud, detection_mask), frame by frame: keypoints, descriptors and points
    bit-identical to the oracle, thresholds equal after every frame; consecutive nodes give edges of > 50 inliers."""
    import cloud_oracle as co
    from oracle import orb_oracle as oo
    gray, depth = frames
    det = nh.make_detector(fe, detector)
    st = oo.DetectorState()
    ptype = "XYZ" if scenario in ("no_mask", "planted") else "XYZRGB"
    handles, kept_inf, kept_nan_round = [], 0, 0
    for k in range(len(gray)):
        d = depth[k].copy()
        if scenario == "mask_from_cloud":  # depths below 0.02 m and in the 5.12 m band read as "no mask"
            d[40:200, 60:300] = np.float32(0.015)
            d[250:420, 340:600] = np.float32(5.125)
        cloud = co.cloud_from_depth(d, nh.K4(), ptype, _colour(gray[k]))
        mask = None
        if scenario in ("mask", "trunc"):
            mask = oo.depth_to_mask(depth[k])  # kinectCallback's depthToCV8UC1
        elif scenario == "mask_from_cloud":
            mask = co.cloud_mask(cloud[..., 2])  # calculateDepthMask
            assert not mask[40:200, 60:300].any() and not mask[250:420, 340:600].any()
        at_round = []
        if scenario == "planted":
            cloud = _plant_values(cloud, k)
        elif scenario == "trunc":
            rec = co.detect(gray[k], mask, copy.deepcopy(st), MAXK, detector=nh.name(detector))
            cloud, at_round = _plant_trunc(cloud, rec)
        hs, nf = fe.nodes_create(det, gray[k:k + 1], cloud[None], None if scenario == "mask_from_cloud" else (None if mask is None else mask[None]),
                                 None, ids=[k], mask_from_cloud=scenario == "mask_from_cloud")
        handles += hs
        okp, odesc, oxyz = co.node_construct(gray[k], cloud, mask, st, MAXK, detector=nh.name(detector))
        gkp = fe.node_keypoints(hs[0])
        gdesc, gxyz = fe.node_download(hs[0])
        assert nf[0] == len(okp) and 300 < len(okp) <= MAXK
        assert gkp.tobytes() == okp.tobytes()
        assert np.array_equal(gdesc, odesc)
        assert np.array_equal(gxyz.view(np.uint32), oxyz.view(np.uint32))
        assert np.array_equal(fe.detector_thresholds(det)[:9], np.array(st.thresh[:9]))
        assert not np.isnan(gxyz).any() and (gxyz[:, 3] == 1).all()
        kept_inf += int(np.isinf(gxyz[:, 2]).sum())
        pos = {(int(np.floor(x + np.float32(0.5))), int(np.floor(y + np.float32(0.5)))) for x, y in zip(gkp["x"], gkp["y"])}
        kept_nan_round += len(pos & set(at_round))
    if scenario == "planted":
        assert kept_inf > 0  # maximum_depth is +inf: a +inf z is kept
    if scenario == "trunc" and detector == 0:
        assert kept_nan_round > 0  # the rounded pixel is not read
    if scenario != "planted":  # (planted nodes hold +inf points)
        res, _, _ = fe.match_node_pairs(handles[1:], handles[:-1], seed=3)
        assert (res["id1"] == np.arange(len(handles) - 1)).all() and (res["id2"] == np.arange(1, len(handles))).all()
        assert (res["n_inliers"] > 50).all()
    fe.detector_destroy(det)
    nh.destroy(fe, handles)


@pytest.mark.parametrize("detector", [0, 1], ids=["ORB", "FAST"])
def test_colour_input_equals_cvtcolor(fe, frames, detector):
    """Colour input on both constructors gives the nodes of the grey path fed with cv2.cvtColor(RGB2GRAY), with one more
    launch per chunk."""
    import cloud_oracle as co
    from oracle import orb_oracle as oo
    gray, depth = frames
    rgb = np.stack([_colour(g) for g in gray])
    conv = np.stack([cv2.cvtColor(c, cv2.COLOR_RGB2GRAY) for c in rgb])
    mask = np.stack([oo.depth_to_mask(d) for d in depth])
    clouds = np.stack([co.cloud_from_depth(d, nh.K4(), "XYZRGB", c) for d, c in zip(depth, rgb)])
    for dep, m, kw in ((depth, mask, {}), (depth, None, {"mask_from_depth": True}), (clouds, mask, {}),
                       (clouds, None, {"mask_from_cloud": True})):
        out = {}
        for name, vis in (("rgb", rgb), ("gray", conv)):
            det = nh.make_detector(fe, detector)
            l0 = fe.lib.rgbdslam_b200_launch_count()
            hs = fe.nodes_create(det, vis, dep, m, nh.K4(), **kw)[0]
            out[name] = (nh.node_dump(fe, hs), fe.detector_thresholds(det).copy(), fe.lib.rgbdslam_b200_launch_count() - l0)
            fe.detector_destroy(det)
            nh.destroy(fe, hs)
        assert nh.same_nodes(out["rgb"][0], out["gray"][0]) and min(len(x[0]) for x in out["rgb"][0]) > 300
        assert np.array_equal(out["rgb"][1], out["gray"][1])
        assert out["rgb"][2] == out["gray"][2] + 1  # k_rgb_to_gray, one chunk


CONFIGS = {"rgb_xyzrgb_maskcloud": ("rgb", "XYZRGB", "cloud"), "gray_xyz_mask": ("gray", "XYZ", "caller")}


@pytest.mark.parametrize("config", list(CONFIGS))
@pytest.mark.parametrize("detector", [0, 1], ids=["ORB", "FAST"])
def test_cloud_pipeline_variants_identical(fe, seq24, config, detector):
    """24 frames in one call (several chunks) == frame by frame == from pinned memory == 1-rank sharded."""
    import torch

    import cloud_oracle as co
    from oracle import orb_oracle as oo
    vis_kind, ptype, mask_kind = CONFIGS[config]
    gray, depth = seq24
    n = len(gray)
    vis = np.stack([_colour(g) for g in gray]) if vis_kind == "rgb" else gray
    clouds = np.stack([co.cloud_from_depth(d, nh.K4(), ptype) for d in depth])
    mask = np.stack([oo.depth_to_mask(d) for d in depth]) if mask_kind == "caller" else None
    mfc = mask_kind == "cloud"

    def run(fn):
        det = nh.make_detector(fe, detector)
        out = fn(det)
        thr = fe.detector_thresholds(det).copy()
        fe.detector_destroy(det)
        dump = nh.node_dump(fe, out)
        nh.destroy(fe, out)
        return dump, thr

    ref, thr_ref = run(lambda det: fe.nodes_create(det, vis, clouds, mask, None, mask_from_cloud=mfc)[0])
    assert len(ref) == n and min(len(k) for k, _, _ in ref) > 300

    def one_by_one(det):
        hs = []
        for k in range(n):
            hs += fe.nodes_create(det, vis[k:k + 1], clouds[k:k + 1], None if mask is None else mask[k:k + 1], None, ids=[k],
                                  mask_from_cloud=mfc)[0]
        return hs
    a, thr_a = run(one_by_one)
    assert nh.same_nodes(ref, a) and np.array_equal(thr_ref, thr_a)
    pv, pc = torch.from_numpy(vis).pin_memory(), torch.from_numpy(clouds).pin_memory()
    pm = None if mask is None else torch.from_numpy(mask).pin_memory()
    b, thr_b = run(lambda det: fe.nodes_create(det, pv, pc, pm, None, mask_from_cloud=mfc)[0])
    assert nh.same_nodes(ref, b) and np.array_equal(thr_ref, thr_b)
    comm = fe.comm_init(0, 1, fe.comm_unique_id())
    c, thr_c = run(lambda det: fe.nodes_create_sharded(det, comm, n, vis, clouds, mask, None, mask_from_cloud=mfc)[0])
    fe.comm_destroy(comm)
    assert nh.same_nodes(ref, c) and np.array_equal(thr_ref, thr_c)


@pytest.mark.parametrize("detector", [0, 1], ids=["ORB", "FAST"])
def test_cloud_and_depth_calls_interleaved(fe, seq24, detector):
    """One detector serves both constructors: alternating cloud and depth-image calls gives each oracle's nodes, with one
    threshold state."""
    import cloud_oracle as co
    import fast_oracle
    from oracle import orb_oracle as oo
    gray, depth = seq24
    K4 = nh.K4()
    det = nh.make_detector(fe, detector)
    st = oo.DetectorState()
    depth_node = fast_oracle.node_construct if detector == 1 else oo.node_construct
    for i, a in enumerate(range(0, 8, 2)):
        b = a + 2
        mask = np.stack([oo.depth_to_mask(d) for d in depth[a:b]])
        if i % 2 == 0:
            clouds = np.stack([co.cloud_from_depth(d, K4, "XYZRGB") for d in depth[a:b]])
            hs = fe.nodes_create(det, gray[a:b], clouds, mask, None)[0]
            want = [co.node_construct(gray[k], clouds[k - a], mask[k - a], st, MAXK, detector=nh.name(detector)) for k in range(a, b)]
        else:
            hs = fe.nodes_create(det, gray[a:b], depth[a:b], mask, K4)[0]
            want = [depth_node(gray[k], depth[k], mask[k - a], K4, st, max_keypoints=MAXK) for k in range(a, b)]
        got = nh.node_dump(fe, hs)
        for (gk, gd, gx), (ok, od, ox) in zip(got, want):
            assert gk.tobytes() == ok.tobytes() and np.array_equal(gd, od) and np.array_equal(gx.view(np.uint32), ox.view(np.uint32))
        assert np.array_equal(fe.detector_thresholds(det)[:9], np.array(st.thresh[:9]))
        nh.destroy(fe, hs)
    fe.detector_destroy(det)


@pytest.mark.parametrize("detector", [0, 1], ids=["ORB", "FAST"])
def test_depth_parameters_do_not_touch_cloud_nodes(fe, frames, detector):
    """use_feature_min_depth and depth_scaling_factor are not read by the point-cloud constructor."""
    import cloud_oracle as co
    gray, depth = frames
    clouds = np.stack([co.cloud_from_depth(d, nh.K4(), "XYZRGB") for d in depth])
    out = []
    for kw in ({}, {"use_feature_min_depth": 1}, {"depth_scaling_factor": 1.25}):
        det = nh.make_detector(fe, detector, **kw)
        hs = fe.nodes_create(det, gray, clouds, None, None, mask_from_cloud=True)[0]
        out.append((nh.node_dump(fe, hs), fe.detector_thresholds(det).copy()))
        fe.detector_destroy(det)
        nh.destroy(fe, hs)
    for dump, thr in out[1:]:
        assert nh.same_nodes(out[0][0], dump) and np.array_equal(out[0][1], thr)


def test_rejected_combinations_launch_nothing(fe, frames):
    from rgbdslam_v2_b200._capi import CLOUD_XYZ, CLOUD_XYZRGB, MASK_FROM_CLOUD, MASK_FROM_DEPTH, VISUAL_RGB, _ptr
    import cloud_oracle as co
    gray, depth = frames
    det = nh.make_detector(fe, 0)
    cloud = np.ascontiguousarray(co.cloud_from_depth(depth[0], nh.K4(), "XYZRGB")[None])
    rgb = np.ascontiguousarray(_colour(gray[0])[None])
    K4 = np.array(nh.K4(), np.float32)
    handles = np.zeros(1, np.uint64)
    nf = np.zeros(1, np.int32)
    H, W = gray.shape[1:]

    def call(vis, dep, flags, k4=K4):
        l0 = fe.lib.rgbdslam_b200_launch_count()
        rc = fe.lib.rgbdslam_b200_nodes_create_ex(det, 1, _ptr(vis), _ptr(dep), None, W, H, _ptr(k4), None, flags, _ptr(handles), _ptr(nf))
        assert fe.lib.rgbdslam_b200_launch_count() == l0
        return rc, fe.lib.rgbdslam_b200_last_error()

    for flags, word in ((CLOUD_XYZRGB | CLOUD_XYZ, b"exclusive"), (MASK_FROM_CLOUD, b"MASK_FROM_CLOUD"),
                        (MASK_FROM_CLOUD | VISUAL_RGB, b"MASK_FROM_CLOUD"), (MASK_FROM_DEPTH | CLOUD_XYZRGB, b"MASK_FROM_DEPTH"),
                        (32, b"unknown"), (VISUAL_RGB | 64, b"unknown")):
        rc, msg = call(rgb if flags & VISUAL_RGB else gray[:1], cloud, flags)
        assert rc == 1 and word in msg, (flags, msg)
    # the environment measurement model is not built for cloud nodes
    nh.reinit(fe, 0, observability_threshold=0.5)
    rc, msg = call(gray[:1], cloud, CLOUD_XYZRGB, None)
    assert rc == 3 and b"measurement model" in msg
    nh.reinit(fe, 0)
    # K4 may be NULL for cloud input, but not for a depth image
    rc, _ = call(gray[:1], np.ascontiguousarray(depth[:1]), 0, None)
    assert rc == 1
    l0 = fe.lib.rgbdslam_b200_launch_count()
    assert fe.lib.rgbdslam_b200_nodes_create_ex(det, 1, _ptr(gray[:1]), _ptr(cloud), None, W, H, None, None, CLOUD_XYZRGB,
                                                _ptr(handles), _ptr(nf)) == 0
    assert fe.lib.rgbdslam_b200_launch_count() > l0 and nf[0] > 300
    fe.node_destroy(int(handles[0]))
    fe.detector_destroy(det)


def _pad(a, W, H):
    """frames [n, 480, 640] padded to [n, H, W] by repeating the last row / column"""
    return np.ascontiguousarray(np.pad(a, ((0, 0), (0, H - a.shape[1]), (0, W - a.shape[2])), mode="edge"))


@pytest.fixture(scope="module")
def seq20():
    return _render(20)


@pytest.mark.parametrize("size", [(641, 481), (642, 481)], ids=["641x481", "642x481"])
def test_colour_input_at_sizes_not_a_multiple_of_4(fe, seq20, size):
    """W * H % 4 != 0: the conversion's last pixels of a call (_ex), and buffers that are not 4-byte aligned (every chunk after
    the first of _sharded: 9 XYZRGB frames per chunk) give the nodes of the grey path fed with cv2.cvtColor."""
    import cloud_oracle as co
    W, H = size
    gray, depth = _pad(seq20[0], W, H), _pad(seq20[1], W, H)
    assert (W * H) % 4 != 0
    rgb = np.stack([_colour(g) for g in gray])
    conv = np.stack([cv2.cvtColor(c, cv2.COLOR_RGB2GRAY) for c in rgb])
    clouds = np.stack([co.cloud_from_depth(d, nh.K4(), "XYZRGB") for d in depth])
    n = len(gray)

    def run(fn):
        det = nh.make_detector(fe, 0)
        hs = fn(det)
        out = (nh.node_dump(fe, hs), fe.detector_thresholds(det).copy())
        fe.detector_destroy(det)
        nh.destroy(fe, hs)
        return out

    # _ex, depth image: 3 frames in one chunk, the last (W * H * 3) % 4 pixels take the tail path
    a = run(lambda det: fe.nodes_create(det, rgb[:3], depth[:3], None, nh.K4(), mask_from_depth=True)[0])
    b = run(lambda det: fe.nodes_create(det, conv[:3], depth[:3], None, nh.K4(), mask_from_depth=True)[0])
    assert nh.same_nodes(a[0], b[0]) and np.array_equal(a[1], b[1]) and min(len(k) for k, _, _ in a[0]) > 300
    # _sharded (1 rank), XYZRGB clouds: 3 chunks at frames 0, 9, 18 of the rank's device buffers
    comm = fe.comm_init(0, 1, fe.comm_unique_id())
    c = run(lambda det: fe.nodes_create_sharded(det, comm, n, rgb, clouds, None, None, mask_from_cloud=True)[0])
    d = run(lambda det: fe.nodes_create_sharded(det, comm, n, conv, clouds, None, None, mask_from_cloud=True)[0])
    fe.comm_destroy(comm)
    e = run(lambda det: fe.nodes_create(det, rgb, clouds, None, None, mask_from_cloud=True)[0])
    assert nh.same_nodes(c[0], d[0]) and np.array_equal(c[1], d[1]) and min(len(k) for k, _, _ in c[0]) > 300
    assert nh.same_nodes(c[0], e[0]) and np.array_equal(c[1], e[1])
