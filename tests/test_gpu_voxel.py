"""GPU tests of the voxel filter of the stored clouds (rgbdslam_b200_reduce_clouds, Node::reducePointCloud), byte for byte
against the restatement of tests/voxel_exact.py."""
import ctypes as C

import numpy as np
import pytest

import map_cloud_exact as mx
import node_helpers as nh
import raw_input_oracle as ro
import voxel_exact as vx

pytestmark = pytest.mark.gpu
ERR_ARG, ERR_STATE = 1, 3


@pytest.fixture(scope="module")
def fe(built):
    from rgbdslam_v2_b200 import Frontend
    f = Frontend(0, nh.params(0))
    yield f
    f.close()


@pytest.fixture(scope="module")
def frames():
    return nh.stack(nh.render(range(5)))


def _colour(gray):
    return np.ascontiguousarray(np.stack([gray, np.roll(gray, 3, axis=-1), np.roll(gray, 5, axis=-2)], -1))


def _cloud(depth, vis, stride):
    """the organised cloud (H, W, stride) a registered sensor would give: back-projected depth, NaN holes, colour bits"""
    fx, fy, cx, cy = nh.K4()
    h, w = depth.shape
    u, v = np.meshgrid(np.arange(w, dtype=np.float32), np.arange(h, dtype=np.float32))
    c = np.zeros((h, w, stride), np.float32)
    c[..., 0], c[..., 1], c[..., 2] = (u - cx) * depth / fx, (v - cy) * depth / fy, depth
    c[..., 4 if stride == 8 else 3] = mx.colour_words(vis).astype(np.uint32).view(np.float32)
    return c


def _same(a, b):
    return a.shape == b.shape and np.array_equal(a.view(np.uint8), b.view(np.uint8))


def _expect(pc, vfs):
    """the restated cloud after reduce_clouds: the reduced one, or the cloud itself when the leaf size is too small"""
    out = vx.reduce_cloud(pc, vfs)
    return pc if out is None else out


def _check_nodes(fe, hs, pcs, tag=""):
    for pb in (32, 16):
        for k, (h, pc) in enumerate(zip(hs, pcs)):
            assert _same(fe.node_cloud(h, pb), mx.organised(pc, pb)), (tag, pb, k)


@pytest.mark.parametrize("visual,step", [("grey", 2), ("colour-bgr", 2), ("colour-rgb", 2), ("bayer-u16", 2), ("grey", 1), ("colour-bgr", 4)])
def test_depth_image_nodes_equal_the_restatement(fe, frames, visual, step):
    """every visual and depth encoding, skip steps 1 / 2 / 4, 32- and 16-byte records; the rest of the node stays"""
    gray, depth = (a[:3] for a in frames)
    nh.reinit(fe, 0, cloud_creation_skip_step=step)
    det = fe.detector_create()
    K4 = nh.K4()
    bgr = visual != "colour-rgb"
    if visual == "bayer-u16":
        u16 = np.stack([ro.to_millimetres(d) for d in depth])
        raw = np.stack([ro.mosaic_gr(c) for c in _colour(gray)])
        hs, _ = fe.nodes_create(det, raw, u16, None, K4, bayer=True, store_cloud=True)
        vis, dref = [ro.bayer_gr_to_rgb(r) for r in raw], ro.depth_u16_to_m(u16)
    else:
        vis = gray if visual == "grey" else np.stack([_colour(g) for g in gray])
        hs, _ = fe.nodes_create(det, vis, depth, None, K4, store_cloud=True, encoding_rgb=not bgr)
        dref = depth
    before = nh.node_dump(fe, hs), fe.detector_thresholds(det).copy()
    vfs = 0.05 if step > 1 else 0.03
    pcs = [mx.create_cloud(dref[k], vis[k], K4, step, 1.0, fe.params.minimum_depth, bgr) for k in range(len(hs))]
    exp = [vx.reduce_cloud(pc, vfs) for pc in pcs]
    counts = fe.reduce_clouds(hs, vfs)
    assert list(counts) == [e["w"] for e in exp] and all(0 < e["w"] < len(pc["x"]) // 3 for e, pc in zip(exp, pcs))
    _check_nodes(fe, hs, exp, visual)
    assert fe.node_cloud(hs[0]).shape == (1, exp[0]["w"])
    assert nh.same_nodes(nh.node_dump(fe, hs), before[0]) and np.array_equal(fe.detector_thresholds(det), before[1])
    nh.destroy(fe, hs)
    fe.detector_destroy(det)
    nh.reinit(fe, 0)


@pytest.mark.parametrize("stride", [8, 4])
def test_cloud_nodes_equal_the_restatement(fe, frames, stride):
    gray, depth = frames
    nh.reinit(fe, 0)
    det = fe.detector_create()
    clouds = np.stack([_cloud(d, _colour(g), stride) for g, d in zip(gray[:3], depth[:3])])
    clouds[1, 100:110, 200:210, 0] = np.inf  # not NaN: such points reach the map, but take no part in the grid
    clouds[1, 120:130, 200:210, 2] = -np.inf
    hs, _ = fe.nodes_create(det, gray[:3], clouds, None, None, store_cloud=True)
    fe.detector_destroy(det)
    exp = [vx.reduce_cloud(mx.cloud_points(c), 0.04) for c in clouds]
    assert list(fe.reduce_clouds(hs, 0.04)) == [e["w"] for e in exp]
    _check_nodes(fe, hs, exp)
    nh.destroy(fe, hs)


def _stored(fe, gray, depth):
    det = fe.detector_create()
    hs, _ = fe.nodes_create(det, gray, depth, None, nh.K4(), store_cloud=True)
    fe.detector_destroy(det)
    return hs


def test_one_call_equals_one_call_per_node_and_a_chunked_call(fe, frames, monkeypatch):
    """5 nodes (384000 points): in one call; one call each; chunks of 2 + 2 + 1 nodes; chunks of one node (a limit below one
    cloud's size)"""
    gray, depth = frames
    nh.reinit(fe, 0)
    outs = []
    for mode in ("one", "each", "200000", "1"):
        hs = _stored(fe, gray, depth)
        if mode == "each":
            counts = np.concatenate([fe.reduce_clouds([h], 0.02) for h in hs])
        else:
            if mode.isdigit():
                monkeypatch.setenv("RB200_VOX_CHUNK_POINTS", mode)
            n0 = fe.launch_count
            counts = fe.reduce_clouds(hs, 0.02)
            launches = fe.launch_count - n0
            monkeypatch.delenv("RB200_VOX_CHUNK_POINTS", raising=False)
            outs.append(launches)
        outs.append((counts, [fe.node_cloud(h) for h in hs]))
        nh.destroy(fe, hs)
    l_one, one, each, l_three, three, l_five, five = outs
    assert l_one < l_three < l_five  # the chunk limit was read
    for other in (each, three, five):
        assert np.array_equal(one[0], other[0]) and all(_same(a, b) for a, b in zip(one[1], other[1]))
    exp = vx.reduce_cloud(mx.create_cloud(depth[4], gray[4], nh.K4(), 2, 1.0, fe.params.minimum_depth), 0.02)
    assert _same(one[1][4], mx.organised(exp))


def test_a_reduced_node_is_reduced_again(fe, frames):
    gray, depth = frames
    nh.reinit(fe, 0)
    hs = _stored(fe, gray[:2], depth[:2])
    pcs = [mx.create_cloud(depth[k], gray[k], nh.K4(), 2, 1.0, fe.params.minimum_depth) for k in range(2)]
    fe.reduce_clouds(hs, 0.02)
    fe.reduce_clouds(hs[1:], 0.1)
    exp = [vx.reduce_cloud(pcs[0], 0.02), vx.reduce_cloud(vx.reduce_cloud(pcs[1], 0.02), 0.1)]
    assert exp[1]["w"] < vx.reduce_cloud(pcs[1], 0.02)["w"]
    _check_nodes(fe, hs, exp)
    nh.destroy(fe, hs)


def _special_clouds(frames):
    """cloud 0 ordinary; cloud 1 with a far point that makes a 0.01 leaf too small; cloud 2 without a finite point"""
    gray, depth = frames
    clouds = np.stack([_cloud(d, _colour(g), 8) for g, d in zip(gray[:3], depth[:3])])
    clouds[1, 17, 33, :3] = (3000.0, 2500.0, 900.0)
    clouds[2, ..., 2] = np.nan
    return clouds


def test_too_small_a_leaf_leaves_that_node_and_an_empty_cloud_is_empty(fe, frames):
    gray, depth = frames
    clouds = _special_clouds(frames)
    nh.reinit(fe, 0)
    det = fe.detector_create()
    hs, _ = fe.nodes_create(det, gray[:3], clouds, None, None, store_cloud=True)
    fe.detector_destroy(det)
    pcs = [mx.cloud_points(c) for c in clouds]
    assert vx.reduce_cloud(pcs[1], 0.01) is None
    counts = fe.reduce_clouds(hs, 0.01)
    exp = [_expect(pc, 0.01) for pc in pcs]
    assert list(counts) == [exp[0]["w"], -1, 0] and exp[0]["w"] > 1000
    _check_nodes(fe, hs, exp)
    assert fe.node_cloud(hs[1]).shape == (480, 640) and fe.node_cloud(hs[2]).shape == (1, 0)
    # the untouched node still reduces at a leaf that fits it, and the map takes all three
    T = np.stack([np.eye(4)[:3]] * 3)
    got, _ = fe.render_cloud(hs, T)
    assert _same(got, mx.render(exp, T))
    assert list(fe.reduce_clouds(hs[1:2], 2.0)) == [vx.reduce_cloud(pcs[1], 2.0)["w"]]
    nh.destroy(fe, hs)


def _transforms(n):
    from rgbdslam_v2_b200 import synth
    return np.array([mx.world2cam(p) for p in synth.trajectory(40)[::7][:n]])


@pytest.mark.parametrize("maximum_depth,preserve,point_bytes", [(np.inf, False, 32), (3.0, False, 16), (3.0, True, 32)])
def test_render_of_reduced_and_unreduced_nodes(fe, frames, maximum_depth, preserve, point_bytes):
    """reduced depth-image node, unreduced depth-image node, reduced cloud node, unreduced cloud node, in one map"""
    gray, depth = frames
    nh.reinit(fe, 0)
    det = fe.detector_create()
    vis = np.stack([_colour(g) for g in gray])
    hd, _ = fe.nodes_create(det, vis[:2], depth[:2], None, nh.K4(), store_cloud=True)
    clouds = np.stack([_cloud(d, v, 8) for v, d in zip(vis[2:4], depth[2:4])])
    hc, _ = fe.nodes_create(det, gray[2:4], clouds, None, None, store_cloud=True)
    fe.detector_destroy(det)
    pcs = [mx.create_cloud(depth[k], vis[k], nh.K4(), 2, 1.0, fe.params.minimum_depth) for k in range(2)]
    pcs += [mx.cloud_points(c) for c in clouds]
    fe.reduce_clouds([hd[0], hc[0]], 0.05)
    pcs[0], pcs[2] = vx.reduce_cloud(pcs[0], 0.05), vx.reduce_cloud(pcs[2], 0.05)
    T = _transforms(4)
    got, _ = fe.render_cloud(hd + hc, T, maximum_depth, preserve, point_bytes)
    assert _same(got, mx.render(pcs, T, maximum_depth, preserve, point_bytes))
    nh.destroy(fe, hd + hc)


def test_reduced_map_stays_within_half_a_voxel_diagonal_of_the_raw_map(fe):
    """ground-truth poses: every point of the reduced map has a point of the raw map within half the voxel's diagonal (the
    centroid of points in a cube is no farther than that from the nearest of them)"""
    from scipy.spatial import cKDTree

    from rgbdslam_v2_b200 import synth
    poses = synth.trajectory(240)
    ks = [0, 4, 8]
    fr = [synth.render_frame(poses[k], seed=k) for k in ks]
    gray, depth = np.stack([f[0] for f in fr]), np.stack([f[1] for f in fr])
    nh.reinit(fe, 0)
    hs = _stored(fe, gray, depth)
    T = np.stack([poses[k][:3] for k in ks])
    raw, _ = fe.render_cloud(hs, T)
    vfs = 0.05
    fe.reduce_clouds(hs, vfs)
    red, _ = fe.render_cloud(hs, T)
    assert 0 < len(red) < len(raw) // 4
    xyz = lambda r: np.stack([r["x"], r["y"], r["z"]], 1).astype(np.float64)
    dist, _ = cKDTree(xyz(raw)).query(xyz(red))
    assert dist.max() <= 0.5 * np.sqrt(3.0) * vfs + 1e-5, dist.max()
    nh.destroy(fe, hs)


def test_rejected_calls_launch_nothing_and_change_nothing(fe, frames):
    gray, depth = frames
    nh.reinit(fe, 0)
    hs = _stored(fe, gray[:2], depth[:2])
    det = fe.detector_create()
    plain, _ = fe.nodes_create(det, gray[:1], depth[:1], None, nh.K4())
    kept, _ = fe.nodes_create(det, gray[:1], _cloud(depth[0], gray[0], 8)[None], None, None, keep_cloud=True)
    fe.detector_destroy(det)
    before = [fe.node_cloud(h) for h in hs]
    lib = fe.lib
    harr = np.array(hs, np.uint64)
    counts = np.full(2, 77, np.int32)
    n0 = fe.launch_count

    def call(handles, vfs, n=None):
        a = np.ascontiguousarray(handles, np.uint64)
        return lib.rgbdslam_b200_reduce_clouds(len(a) if n is None else n, a.ctypes.data, vfs, counts.ctypes.data)

    for vfs in (0.0, -1.0, np.nan, np.inf, -np.inf, 1e-60, 1e60):  # 1e-60 is 0 and 1e60 is inf as a float
        assert call(harr, vfs) == ERR_ARG, vfs
    assert b"voxelfilter_size" in lib.rgbdslam_b200_last_error()
    assert call(harr, 0.05, -1) == ERR_ARG
    assert lib.rgbdslam_b200_reduce_clouds(2, None, 0.05, None) == ERR_ARG
    assert call([hs[0], hs[1], hs[0]], 0.05) == ERR_ARG and b"twice" in lib.rgbdslam_b200_last_error()
    assert call([hs[0], 0], 0.05) == ERR_ARG  # not a handle
    for other in (plain[0], kept[0]):  # no colour plane
        assert call([hs[0], other], 0.05) == ERR_STATE and b"STORE_CLOUD" in lib.rgbdslam_b200_last_error()
    assert fe.launch_count == n0 and (counts == 77).all()
    assert all(_same(fe.node_cloud(h), b) for h, b in zip(hs, before))
    n0 = fe.launch_count
    assert call(harr, 0.05, 0) == 0 and fe.launch_count == n0  # no node: nothing to do
    assert lib.rgbdslam_b200_reduce_clouds(2, harr.ctypes.data, 0.05, None) == 0  # n_points may be NULL
    assert fe.node_cloud(hs[0]).shape[0] == 1
    nh.destroy(fe, hs + plain + kept)


def test_a_reduced_cloud_does_not_feed_the_measurement_model(fe, frames):
    gray, depth = frames
    nh.reinit(fe, 0)
    hs = _stored(fe, gray[:3], depth[:3])
    fe.reduce_clouds(hs[:1], 0.05)
    nh.reinit(fe, 0, observability_threshold=0.5)
    lib = fe.lib
    T = np.eye(4, dtype=np.float32)
    cnt = np.zeros(4, np.uint32)
    fe.match_node_pairs(hs[2:], hs[1:2], seed=3)  # unreduced nodes feed it
    n0 = fe.launch_count
    for a, b in ((hs[0], hs[1]), (hs[1], hs[0])):
        assert lib.rgbdslam_b200_observation_likelihood(C.c_uint64(a), C.c_uint64(b), T.ctypes.data, cnt.ctypes.data) == ERR_STATE
        assert b"voxel-filtered" in lib.rgbdslam_b200_last_error()
    from rgbdslam_v2_b200._capi import B200Error
    for newer, older in ((hs[1], hs[0]), (hs[0], hs[1])):
        with pytest.raises(B200Error, match="error 3: .*voxel-filtered"):
            fe.match_node_pairs([newer], [older], seed=3)
    K = np.array(nh.K4(), np.float32)
    d0 = np.ascontiguousarray(depth[0])
    assert lib.rgbdslam_b200_node_set_depth(C.c_uint64(hs[0]), d0.ctypes.data, 640, 480, K.ctypes.data) == ERR_STATE
    assert fe.launch_count == n0
    # with the model off the reduced node matches as before
    nh.reinit(fe, 0)
    r, _, _ = fe.match_node_pairs(hs[1:2], hs[:1], seed=3)
    assert r[0]["n_all_matches"] > 0
    nh.destroy(fe, hs)


def test_destroying_nodes_in_any_order_frees_both_allocations(fe, frames):
    import torch
    gray, depth = frames
    nh.reinit(fe, 0)

    def cycle(order, reduce_which):
        hs = _stored(fe, gray, depth)
        fe.reduce_clouds([hs[k] for k in reduce_which], 0.05)
        for k in order:
            fe.node_destroy(hs[k])
        fe.synchronize()
        return torch.cuda.mem_get_info()[0]

    base = cycle(range(5), range(5))  # warm-up: the grow-only tables exist from here on
    for order, which in (([4, 2, 0, 1, 3], [1, 3]), ([0, 1, 2, 3, 4], [0]), ([3, 4, 0, 2, 1], [0, 1, 2, 3, 4])):
        assert cycle(order, which) >= base - (1 << 20), (order, which)
    # the stored clouds of a call are released when its last node has been reduced
    hs = _stored(fe, np.concatenate([gray] * 8), np.concatenate([depth] * 8))  # 40 nodes, 24.6 MB of clouds
    fe.synchronize()
    full = torch.cuda.mem_get_info()[0]
    fe.reduce_clouds(hs[:39], 0.05)
    fe.synchronize()
    part = torch.cuda.mem_get_info()[0]
    fe.reduce_clouds(hs[39:], 0.05)
    fe.synchronize()
    done = torch.cuda.mem_get_info()[0]
    assert part < full and done - full > 15 << 20, (full, part, done)
    nh.destroy(fe, hs)
