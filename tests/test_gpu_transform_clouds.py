"""GPU tests of the in-place transform of the stored clouds (rgbdslam_b200_transform_clouds, transform_individual_clouds,
DESIGN.md 4.16): every node's 32- and 16-byte records after the call equal the restatement of tests/cloud_export_exact.py
applied to its records before, for depth-image nodes of every visual kind, XYZRGB / XYZ cloud nodes with NaN and +inf points,
voxel-reduced and occupancy-filtered nodes; a second call transforms again; how many nodes one call takes does not matter; the
map reads transformed clouds as any other; refused calls change nothing, and the measurement model and ICP refuse transformed
nodes."""
import ctypes as C

import numpy as np
import pytest

import cloud_export_exact as ex
import map_cloud_exact as mx
import node_helpers as nh
import raw_input_oracle as ro
from rgbdslam_v2_b200._capi import B200Error, cloud_sensor_pose, octomap_pose

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
    return nh.stack(nh.render(range(6)))


def _colour(gray):
    return np.ascontiguousarray(np.stack([gray, np.roll(gray, 3, axis=-1), np.roll(gray, 5, axis=-2)], -1))


def _cloud(depth, vis, stride, rng):
    """an organised cloud (H, W, stride) with NaN holes (from the depth) and +inf / -inf coordinates sprinkled in"""
    fx, fy, cx, cy = nh.K4()
    h, w = depth.shape
    u, v = np.meshgrid(np.arange(w, dtype=np.float32), np.arange(h, dtype=np.float32))
    c = np.zeros((h, w, stride), np.float32)
    c[..., 0], c[..., 1], c[..., 2] = (u - cx) * depth / fx, (v - cy) * depth / fy, depth
    flat = c.reshape(-1, stride)
    for axis, val in ((0, np.inf), (1, -np.inf), (2, np.inf)):
        flat[rng.choice(len(flat), 500, replace=False), axis] = val
    c[..., 4 if stride == 8 else 3] = mx.colour_words(vis).astype(np.uint32).view(np.float32)
    return c


def _records(fe, h):
    return fe.node_cloud(h, 32), fe.node_cloud(h, 16)


def _restated(records, T):
    """the records after transformPointCloud by T, from the records before"""
    out = []
    for r in records:
        pc = ex.transform_cloud(dict(x=r["x"].reshape(-1), y=r["y"].reshape(-1), z=r["z"].reshape(-1)), T)
        e = r.copy()
        for k in "xyz":
            e[k] = pc[k].reshape(r.shape)
        out.append(e)
    return out


def _same(a, b):
    return a.shape == b.shape and a.tobytes() == b.tobytes()


def _transforms(n, seed=0):
    from rgbdslam_v2_b200 import synth
    rng = np.random.default_rng(seed)
    poses = synth.trajectory(60)[::9][:n]
    T = np.array([P[:3, :] for P in poses])
    T[:, :, 3] += rng.normal(0, 0.5, (len(T), 3))
    return T


def _check(fe, hs, T, calls=1):
    """transform the nodes `calls` times; each time every node's records equal the restatement of its records before"""
    for _ in range(calls):
        before = [_records(fe, h) for h in hs]
        fe.transform_clouds(hs, T)
        for h, b, t in zip(hs, before, T):
            got, exp = _records(fe, h), _restated(b, t)
            assert _same(got[0], exp[0]) and _same(got[1], exp[1])
            assert not _same(got[0], b[0])


@pytest.mark.parametrize("visual", ["grey", "colour-bgr", "colour-rgb", "bayer-u16"])
def test_depth_image_nodes_equal_the_restatement(fe, frames, visual):
    gray, depth = frames
    nh.reinit(fe, 0)
    det = fe.detector_create()
    K4 = nh.K4()
    if visual == "bayer-u16":
        u16 = np.stack([ro.to_millimetres(d) for d in depth])
        raw = np.stack([ro.mosaic_gr(c) for c in _colour(gray)])
        hs, _ = fe.nodes_create(det, raw, u16, None, K4, bayer=True, store_cloud=True)
    else:
        vis = gray if visual == "grey" else np.stack([_colour(g) for g in gray])
        hs, _ = fe.nodes_create(det, vis, depth, None, K4, store_cloud=True, encoding_rgb=visual == "colour-rgb")
    fe.detector_destroy(det)
    hs = list(hs)
    assert all(np.isnan(fe.node_cloud(h)["z"]).any() for h in hs)  # holes
    before = [fe.node_cloud(h) for h in hs]
    _check(fe, hs, _transforms(len(hs)))
    # the holes keep the 1 m ray of createXYZRGBPointCloud, the raster stays
    for h, b in zip(hs, before):
        a = fe.node_cloud(h)
        hole = np.isnan(b["z"])
        assert a.shape == b.shape and a[hole].tobytes() == b[hole].tobytes()
    nh.destroy(fe, hs)


@pytest.mark.parametrize("stride", [8, 4], ids=["xyzrgb", "xyz"])
def test_cloud_nodes_with_nan_and_inf_points_equal_the_restatement(fe, frames, stride):
    gray, depth = frames
    nh.reinit(fe, 0)
    rng = np.random.default_rng(stride)
    clouds = np.stack([_cloud(d, _colour(g), stride, rng) for g, d in zip(gray[:3], depth[:3])])
    det = fe.detector_create()
    hs, _ = fe.nodes_create(det, gray[:3], clouds, None, None, store_cloud=True)
    fe.detector_destroy(det)
    hs = list(hs)
    inf_before = [np.isinf(fe.node_cloud(h)["x"]) for h in hs]
    assert all(m.sum() == 500 for m in inf_before)
    _check(fe, hs, _transforms(3, 1), calls=2)  # a second call transforms the transformed cloud again
    for h, m in zip(hs, inf_before):
        assert (fe.node_cloud(h)["x"][m] == np.inf).all()
    nh.destroy(fe, hs)


def test_voxel_reduced_and_occupancy_filtered_nodes_equal_the_restatement(fe):
    from rgbdslam_v2_b200 import synth
    gray, depth = nh.stack(nh.render(range(0, 24, 4)))
    nh.reinit(fe, 0)
    det = fe.detector_create()
    hs, _ = fe.nodes_create(det, np.stack([_colour(g) for g in gray]), depth, None, nh.K4(), store_cloud=True)
    fe.detector_destroy(det)
    hs = list(hs)
    fe.reduce_clouds(hs[:2], 0.05)
    poses = synth.trajectory(240)[0:24:4]
    om = fe.octomap_create()
    fe.octomap_insert(om, hs[2:], [octomap_pose(P) for P in poses[2:]])
    S = np.stack([np.concatenate(cloud_sensor_pose(P)) for P in poses[2:]]).astype(np.float32)
    counts = fe.octomap_filter_clouds(om, hs[2:], S, 3e5)
    fe.octomap_destroy(om)
    assert any(0 < c < 320 * 240 for c in counts)
    assert all(fe.node_cloud(h).shape[0] == 1 for h in hs[:2])
    _check(fe, hs, _transforms(len(hs), 2))
    nh.destroy(fe, hs)


def test_render_reduce_and_octomap_read_the_transformed_cloud(fe, frames):
    gray, depth = frames
    nh.reinit(fe, 0)
    det = fe.detector_create()
    hs, _ = fe.nodes_create(det, np.stack([_colour(g) for g in gray[:3]]), depth[:3], None, nh.K4(), store_cloud=True)
    fe.detector_destroy(det)
    hs = list(hs)
    T = _transforms(3, 3)
    fe.transform_clouds(hs, T)
    r32 = [fe.node_cloud(h, 32).reshape(-1) for h in hs]
    r16 = [fe.node_cloud(h, 16).reshape(-1) for h in hs]
    pcs = [dict(x=a["x"], y=a["y"], z=a["z"], rgb=a["rgb"], w16=b["w"]) for a, b in zip(r32, r16)]
    M = _transforms(3, 4)
    for preserve in (False, True):
        for pb in (32, 16):
            got, _ = fe.render_cloud(hs, M, 4.0, preserve, pb)
            assert _same(got, mx.render(pcs, M, 4.0, preserve, pb))
    # the OctoMap and the voxel filter take it as any stored cloud: the same as a cloud node holding these points
    import octomap_filter_exact as fx
    om = fe.octomap_create()
    Tf = [octomap_pose(np.eye(4))] * 3
    fe.octomap_insert(om, hs, Tf)
    m = fx.FilterOracle()
    for pc, t in zip(pcs, Tf):
        m.insert_cloud(pc, t)
    assert fe.octomap_write(om) == m.write()
    fe.octomap_destroy(om)
    n = fe.reduce_clouds(hs, 0.1)
    assert (n > 0).all()
    nh.destroy(fe, hs)


def test_one_call_of_300_nodes_equals_300_one_node_calls(fe, frames):
    """300 depth-image nodes, 23 M points: two slabs"""
    gray, depth = frames
    nh.reinit(fe, 0)
    idx = np.arange(300) % len(gray)
    rng = np.random.default_rng(7)
    T = np.concatenate([np.eye(3)[None].repeat(300, 0) + rng.normal(0, 0.01, (300, 3, 3)), rng.normal(0, 1, (300, 3, 1))], 2)
    out = []
    for batched in (True, False):
        det = fe.detector_create()
        hs, _ = fe.nodes_create(det, gray[idx], depth[idx], None, nh.K4(), store_cloud=True)
        fe.detector_destroy(det)
        hs = list(hs)
        if batched:
            fe.transform_clouds(hs, T)
        else:
            for k, h in enumerate(hs):
                fe.transform_clouds([h], T[k:k + 1])
        out.append([fe.node_cloud(h, 16).tobytes() for h in hs])
        nh.destroy(fe, hs)
    assert out[0] == out[1]
    exp = mx.organised(ex.transform_cloud(mx.create_cloud(depth[idx[299]], gray[idx[299]], nh.K4(), 2, 1.0, fe.params.minimum_depth),
                                          T[299]), 16)
    assert out[0][299] == exp.tobytes()


def test_refused_calls_change_nothing_and_transformed_nodes_leave_the_model_and_icp(fe, frames):
    gray, depth = frames
    nh.reinit(fe, 0)
    det = fe.detector_create()
    hs, _ = fe.nodes_create(det, gray[:3], depth[:3], None, nh.K4(), store_cloud=True)
    plain, _ = fe.nodes_create(det, gray[:1], depth[:1], None, nh.K4())
    fe.detector_destroy(det)
    hs, plain = list(hs), list(plain)
    lib = fe.lib
    before = [_records(fe, h) for h in hs]
    T = np.ascontiguousarray(_transforms(3, 5).reshape(3, 12))

    def call(handles, t=T, n=None):
        h = np.ascontiguousarray(np.asarray(handles, np.uint64))
        return lib.rgbdslam_b200_transform_clouds(len(h) if n is None else n, h.ctypes.data, np.ascontiguousarray(t).ctypes.data)

    n0 = fe.launch_count
    assert call(hs, n=-1) == ERR_ARG
    assert lib.rgbdslam_b200_transform_clouds(2, None, T.ctypes.data) == ERR_ARG
    assert call([hs[0], hs[1], hs[0]]) == ERR_ARG and b"twice" in lib.rgbdslam_b200_last_error()
    assert call([hs[0], 0]) == ERR_ARG  # not a handle
    for bad in (np.nan, np.inf, -np.inf):
        Tb = T.copy()
        Tb[2, 7] = bad
        assert call(hs, Tb) == ERR_ARG and b"non-finite" in lib.rgbdslam_b200_last_error()
    assert call([hs[0], plain[0]]) == ERR_STATE and b"STORE_CLOUD" in lib.rgbdslam_b200_last_error()
    assert fe.launch_count == n0
    assert all(_same(a[0], b[0]) and _same(a[1], b[1]) for a, b in zip((_records(fe, h) for h in hs), before))
    n0 = fe.launch_count  # the downloads above launch
    assert call([], n=0) == 0 and fe.launch_count == n0
    # the measurement model and ICP refuse a pair with a transformed node, before any device work
    fe.transform_clouds(hs[:1], T[:1])
    nh.reinit(fe, 0, observability_threshold=0.5)
    fe.match_node_pairs(hs[2:], hs[1:2], seed=3)  # untransformed nodes feed it
    n0 = fe.launch_count
    cnt = np.zeros(4, np.uint32)
    I = np.eye(4, dtype=np.float32)
    for a, b in ((hs[0], hs[1]), (hs[1], hs[0])):
        assert lib.rgbdslam_b200_observation_likelihood(C.c_uint64(a), C.c_uint64(b), I.ctypes.data, cnt.ctypes.data) == ERR_STATE
        assert b"transform_clouds" in lib.rgbdslam_b200_last_error()
        with pytest.raises(B200Error, match="error 3: .*transform_clouds"):
            fe.match_node_pairs([a], [b], seed=3)
        with pytest.raises(B200Error, match="error 3: .*transform_clouds"):
            fe.icp_align([a], [b])
    assert fe.launch_count == n0
    nh.reinit(fe, 0)
    r = fe.icp_align([hs[2]], [hs[1]])  # untransformed nodes still align
    assert len(r) == 1
    nh.destroy(fe, hs + plain)
