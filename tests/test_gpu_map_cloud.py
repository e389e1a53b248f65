"""GPU tests of the stored colour clouds (RGBDSLAM_B200_STORE_CLOUD, node_download_cloud) and the registered map
(render_cloud), byte for byte against the restatement of tests/map_cloud_exact.py."""
import ctypes as C

import numpy as np
import pytest

import map_cloud_exact as mx
import node_helpers as nh
import raw_input_oracle as ro

pytestmark = pytest.mark.gpu


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


def _clouds(fe, hs, pb=32):
    return [fe.node_cloud(h, pb) for h in hs]


@pytest.mark.parametrize("visual", ["grey", "colour-bgr", "colour-rgb", "bayer-u16", "grey-scaled"])
def test_depth_image_clouds_equal_the_restatement(fe, frames, visual):
    gray, depth = frames
    scaling = 1.03 if visual == "grey-scaled" else 1.0
    nh.reinit(fe, 0, depth_scaling_factor=scaling)
    det = fe.detector_create()
    K4 = nh.K4()
    bgr = visual != "colour-rgb"
    if visual == "bayer-u16":
        u16 = np.stack([ro.to_millimetres(d) for d in depth])
        raw = np.stack([ro.mosaic_gr(c) for c in _colour(gray)])
        hs, _ = fe.nodes_create(det, raw, u16, None, K4, bayer=True, store_cloud=True)
        vis, dref = [ro.bayer_gr_to_rgb(r) for r in raw], ro.depth_u16_to_m(u16)
    else:
        vis = gray if visual.startswith("grey") else np.stack([_colour(g) for g in gray])
        hs, _ = fe.nodes_create(det, vis, depth, None, K4, store_cloud=True, encoding_rgb=not bgr)
        dref = depth
    for pb in (32, 16):
        for k, h in enumerate(hs):
            exp = mx.organised(mx.create_cloud(dref[k], vis[k], K4, 2, scaling, fe.params.minimum_depth, bgr), pb)
            assert _same(fe.node_cloud(h, pb), exp), (visual, pb, k)
            assert np.isnan(exp["z"]).any() and (exp["rgb" if pb == 32 else "w"] != (0 if pb == 32 else 0x3F800000)).any()
    nh.destroy(fe, hs)
    fe.detector_destroy(det)


@pytest.mark.parametrize("stride", [8, 4])
def test_cloud_input_keeps_its_points_and_colour(fe, frames, stride):
    gray, depth = frames
    nh.reinit(fe, 0)
    det = fe.detector_create()
    clouds = np.stack([_cloud(d, _colour(g), stride) for g, d in zip(gray, depth)])
    hs, _ = fe.nodes_create(det, gray, clouds, None, None, store_cloud=True)
    for h, c in zip(hs, clouds):
        exp = mx.organised(mx.cloud_points(c))
        assert _same(fe.node_cloud(h), exp)
    nh.destroy(fe, hs)
    fe.detector_destroy(det)


def test_pinned_input_and_chunking_do_not_change_the_clouds(fe, built):
    """70 colour frames (two chunks) from pinned memory == one call per frame from pageable memory"""
    import torch
    gray, depth = nh.stack(nh.render(range(70)))
    vis = np.stack([_colour(g) for g in gray])
    nh.reinit(fe, 0)
    det = fe.detector_create()
    hs, _ = fe.nodes_create(det, torch.from_numpy(vis).pin_memory(), torch.from_numpy(depth).pin_memory(), None, nh.K4(),
                            store_cloud=True)
    a = _clouds(fe, hs)
    nh.destroy(fe, hs)
    fe.detector_destroy(det)
    det = fe.detector_create()
    b = []
    for k in range(len(vis)):
        h1, _ = fe.nodes_create(det, vis[k:k + 1], depth[k:k + 1], None, nh.K4(), store_cloud=True)
        b += _clouds(fe, h1)
        nh.destroy(fe, h1)
    fe.detector_destroy(det)
    assert all(_same(x, y) for x, y in zip(a, b)) and len(a) == len(b) == 70


@pytest.mark.parametrize("cloud_input", [False, True])
def test_features_thresholds_and_model_counts_do_not_change(fe, frames, cloud_input):
    gray, depth = frames
    kw = dict(observability_threshold=0.5)
    out = []
    for flags in ({}, dict(store_cloud=True)):
        nh.reinit(fe, 0, **kw)
        det = fe.detector_create()
        if cloud_input:
            clouds = np.stack([_cloud(d, g, 8) for g, d in zip(gray, depth)])
            hs, nf = fe.nodes_create(det, gray, clouds, None, nh.K4(), keep_cloud=True, **flags)
        else:
            hs, nf = fe.nodes_create(det, gray, depth, None, nh.K4(), **flags)
        res, _, _ = fe.match_node_pairs(hs[1:], hs[:-1], seed=3)
        out.append((nh.node_dump(fe, hs), fe.detector_thresholds(det).copy(), res.copy()))
        nh.destroy(fe, hs)
        fe.detector_destroy(det)
    assert nh.same_nodes(out[0][0], out[1][0]) and np.array_equal(out[0][1], out[1][1])
    assert out[0][2].tobytes() == out[1][2].tobytes() and out[0][2]["all_points"].sum() > 0


def _mixed_nodes(fe, frames):
    """three depth-image nodes (colour) and two point-cloud nodes, with their restated pc_col"""
    gray, depth = frames
    nh.reinit(fe, 0)
    det = fe.detector_create()
    vis = np.stack([_colour(g) for g in gray])
    hd, _ = fe.nodes_create(det, vis[:3], depth[:3], None, nh.K4(), store_cloud=True)
    clouds = np.stack([_cloud(d, v, 8) for v, d in zip(vis[3:], depth[3:])])
    hc, _ = fe.nodes_create(det, gray[3:], clouds, None, None, store_cloud=True)
    fe.detector_destroy(det)
    pcs = [mx.create_cloud(depth[k], vis[k], nh.K4(), 2, 1.0, fe.params.minimum_depth) for k in range(3)]
    pcs += [mx.cloud_points(c) for c in clouds]
    return hd + hc, pcs


def _transforms(n, seed=0):
    from rgbdslam_v2_b200 import synth
    poses = synth.trajectory(40)[::7][:n]
    return np.array([mx.world2cam(p) for p in poses])


@pytest.mark.parametrize("preserve", [False, True])
@pytest.mark.parametrize("maximum_depth", [np.inf, 3.0, -1.0])
@pytest.mark.parametrize("point_bytes", [32, 16])
def test_render_equals_the_restatement(fe, frames, preserve, maximum_depth, point_bytes):
    hs, pcs = _mixed_nodes(fe, frames)
    T = _transforms(len(hs))
    got, used = fe.render_cloud(hs, T, maximum_depth, preserve, point_bytes)
    exp = mx.render(pcs, T, maximum_depth, preserve, point_bytes)
    assert _same(got, exp), (len(got), len(exp))
    for k in range(len(hs)):
        assert np.array_equal(used[k][:3].view(np.uint32), mx.transform_as_matrix(T[k]).view(np.uint32))
        assert np.array_equal(used[k][3], [0, 0, 0, 1])
    nh.destroy(fe, hs)


def test_render_across_staging_pieces_equals_one_node_calls(fe, frames):
    """300 depth-image nodes (23 M points, 11 staging pieces) in one call == the concatenation of 300 one-node calls"""
    import torch
    gray, depth = frames
    nh.reinit(fe, 0)
    det = fe.detector_create()
    idx = np.arange(300) % len(gray)
    hs, _ = fe.nodes_create(det, gray[idx], depth[idx], None, nh.K4(), store_cloud=True)
    fe.detector_destroy(det)
    rng = np.random.default_rng(5)
    T = np.concatenate([np.eye(3)[None].repeat(300, 0) + rng.normal(0, 0.01, (300, 3, 3)), rng.normal(0, 1, (300, 3, 1))], 2)
    n = fe.render_cloud(hs, T, 6.0, count_only=True)
    assert n > 2 * (1 << 21) * 5
    pinned = torch.empty(n * 32, dtype=torch.uint8).pin_memory()
    got, _ = fe.render_cloud(hs, T, 6.0, out=pinned)
    got = got.numpy()
    parts = [fe.render_cloud([h], T[k:k + 1], 6.0)[0] for k, h in enumerate(hs)]
    assert np.array_equal(got, np.concatenate(parts).view(np.uint8))
    exp = mx.render([mx.create_cloud(depth[idx[k]], gray[idx[k]], nh.K4(), 2, 1.0, fe.params.minimum_depth) for k in (0, 299)],
                    T[[0, 299]], 6.0)
    assert _same(np.concatenate([parts[0], parts[299]]), exp)
    nh.destroy(fe, hs)


def test_count_capacity_and_state_errors(fe, frames):
    from rgbdslam_v2_b200._capi import ENCODING_RGB, STORE_CLOUD
    gray, depth = frames
    hs, pcs = _mixed_nodes(fe, frames)
    T = np.ascontiguousarray(_transforms(len(hs)).reshape(len(hs), 12))
    harr = np.array(hs, np.uint64)
    lib = fe.lib
    n = C.c_int64(-1)
    assert lib.rgbdslam_b200_render_cloud(len(hs), harr.ctypes.data, T.ctypes.data, 4.0, 0, 32, None, 0, C.byref(n), None) == 0
    need = n.value
    assert need == len(mx.render(pcs, T.reshape(-1, 3, 4), 4.0))
    buf = np.full((need - 1) * 32 + 64, 0xA5, np.uint8)
    n2 = C.c_int64(-1)
    rc = lib.rgbdslam_b200_render_cloud(len(hs), harr.ctypes.data, T.ctypes.data, 4.0, 0, 32, buf.ctypes.data, need - 1, C.byref(n2), None)
    assert rc == 1 and n2.value == need and (buf == 0xA5).all()
    assert lib.rgbdslam_b200_render_cloud(len(hs), harr.ctypes.data, T.ctypes.data, 4.0, 0, 24, buf.ctypes.data, need, C.byref(n2), None) == 1
    Tbad = T.copy()
    Tbad[2, 5] = np.nan
    assert lib.rgbdslam_b200_render_cloud(len(hs), harr.ctypes.data, Tbad.ctypes.data, 4.0, 0, 32, buf.ctypes.data, need, C.byref(n2), None) == 1
    assert (buf == 0xA5).all()
    # a node without a stored cloud
    nh.reinit(fe, 0)
    det = fe.detector_create()
    plain, _ = fe.nodes_create(det, gray[:1], depth[:1], None, nh.K4())
    both = np.array([hs[0], plain[0]], np.uint64)
    assert lib.rgbdslam_b200_render_cloud(2, both.ctypes.data, T.ctypes.data, 4.0, 0, 32, buf.ctypes.data, need, C.byref(n2), None) == 3
    w, h = C.c_int(), C.c_int()
    assert lib.rgbdslam_b200_node_download_cloud(C.c_uint64(plain[0]), 32, None, C.byref(w), C.byref(h)) == 3
    # rejected before any device work
    hh = np.zeros(1, np.uint64)
    nf = np.zeros(1, np.int32)
    K = np.array(nh.K4(), np.float32)
    g0, d0 = np.ascontiguousarray(gray[:1]), np.ascontiguousarray(depth[:1])
    assert lib.rgbdslam_b200_nodes_create_ex(det, 1, g0.ctypes.data, d0.ctypes.data, None, 640, 480, K.ctypes.data, None,
                                             ENCODING_RGB, hh.ctypes.data, nf.ctypes.data) == 1  # without STORE_CLOUD
    nh.reinit(fe, 0, cloud_creation_skip_step=7)
    assert lib.rgbdslam_b200_nodes_create_ex(det, 1, g0.ctypes.data, d0.ctypes.data, None, 640, 480, K.ctypes.data, None,
                                             STORE_CLOUD, hh.ctypes.data, nf.ctypes.data) == 1  # 7 divides neither 640 nor 480
    assert b"skip_step" in lib.rgbdslam_b200_last_error()
    fe.detector_destroy(det)
    nh.destroy(fe, hs + plain)
    nh.reinit(fe, 0)


def test_map_points_land_on_the_other_frames_depth(fe):
    """ground-truth poses, noise-free depth: points of frame i, put into the map with pose i, project into frame j onto its
    depth (1 / z interpolated between four pixels that agree) within 1 mm"""
    from rgbdslam_v2_b200 import synth
    poses = synth.trajectory(240)
    ks = [0, 4, 8]
    frames = [synth.render_frame(poses[k], seed=k, nan_frac=0.0) for k in ks]
    gray, depth = np.stack([f[0] for f in frames]), np.stack([f[1] for f in frames])
    nh.reinit(fe, 0)
    det = fe.detector_create()
    hs, _ = fe.nodes_create(det, gray, depth, None, nh.K4(), store_cloud=True)
    fe.detector_destroy(det)
    fx, fy, cx, cy = nh.K4()
    checked = 0
    for a in range(len(ks)):
        pts, _ = fe.render_cloud([hs[a]], poses[ks[a]][None, :3, :])
        P = np.stack([pts["x"], pts["y"], pts["z"]], 1).astype(np.float64)
        for b in range(len(ks)):
            if a == b:
                continue
            R, t = poses[ks[b]][:3, :3], poses[ks[b]][:3, 3]
            q = (P - t) @ R
            u, v = fx * q[:, 0] / q[:, 2] + cx, fy * q[:, 1] / q[:, 2] + cy
            ok = (q[:, 2] > 0.3) & (u >= 0) & (v >= 0) & (u < 639) & (v < 479)
            u0, v0 = np.floor(u[ok]).astype(int), np.floor(v[ok]).astype(int)
            fu, fv = u[ok] - u0, v[ok] - v0
            D = depth[b].astype(np.float64)
            z4 = np.stack([D[v0, u0], D[v0, u0 + 1], D[v0 + 1, u0], D[v0 + 1, u0 + 1]], 1)
            same = np.isfinite(z4).all(1) & (z4.max(1) - z4.min(1) < 0.01 * z4.min(1))
            inv = 1 / z4
            zi = 1 / ((inv[:, 0] * (1 - fu) + inv[:, 1] * fu) * (1 - fv) + (inv[:, 2] * (1 - fu) + inv[:, 3] * fu) * fv)
            err = np.abs(zi - q[ok, 2])[same]
            checked += len(err)
            assert len(err) > 10000 and np.quantile(err, 0.995) < 1e-3 and np.median(err) < 1e-4, (a, b, np.quantile(err, 0.995))
    assert checked > 50000
    nh.destroy(fe, hs)
