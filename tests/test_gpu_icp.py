"""GPU tests of the ICP fallback of matchNodePair (rgbdslam_b200_icp_align_ex), byte for byte in every field against the
restatements of tests/icp_exact.py (icp_method "icp") and tests/icp_nl_exact.py ("icp_nl")."""
import numpy as np
import pytest

import icp_exact as ix
import icp_nl_exact as nx
import map_cloud_exact as mx
import node_helpers as nh
import raw_input_oracle as ro
import voxel_exact as vx

pytestmark = pytest.mark.gpu
ERR_ARG, ERR_STATE = 1, 3
F32 = np.float32
METHODS = {"icp": ix, "icp_nl": nx}


@pytest.fixture(scope="module")
def fe(built):
    from rgbdslam_v2_b200 import Frontend
    f = Frontend(0, nh.params(0))
    yield f
    f.close()


@pytest.fixture(scope="module")
def frames():
    return nh.stack(nh.render(range(4)))


def _colour(gray):
    return np.ascontiguousarray(np.stack([gray, np.roll(gray, 3, axis=-1), np.roll(gray, 5, axis=-2)], -1))


def _record(r):
    """a restatement result as an ICP_RESULT_DTYPE record"""
    from rgbdslam_v2_b200._capi import ICP_RESULT_DTYPE
    out = np.zeros(1, ICP_RESULT_DTYPE)
    out["T"][0] = np.asarray(r["T"], F32).T.ravel()  # column-major
    for k in ("converged", "iterations", "criterion", "n_source", "n_target", "n_correspondences", "mse"):
        out[k][0] = r[k]
    return out[0]


def _check(got, pcs_src, pcs_tgt, mcs=10000, tag="", method="icp"):
    """the device's records against the method's restatement; returns the restatement's results"""
    assert len(got) == len(pcs_src)
    exps = []
    for k, (s, t) in enumerate(zip(pcs_src, pcs_tgt)):
        r = METHODS[method].align(s, t, mcs)
        exp = _record(r)
        assert got[k].tobytes() == exp.tobytes(), (tag, k, got[k], exp)
        exps.append(r)
    return exps


def _stored(fe, gray, depth, **kw):
    det = fe.detector_create()
    hs, _ = fe.nodes_create(det, gray, depth, None, kw.pop("K4", nh.K4()), store_cloud=True, **kw)
    fe.detector_destroy(det)
    return hs


def _planted_nodes(fe, gray, clouds):
    """cloud nodes whose organised 480 x 640 clouds hold the given (3, n) points first, in order, and NaN everywhere else"""
    H, W = gray.shape
    cl = np.full((len(clouds), H, W, 4), np.nan, F32)
    for k, p in enumerate(clouds):
        flat = cl[k].reshape(-1, 4)
        flat[:p.shape[1], :3] = p.T
        flat[:, 3] = 0
    hs = _stored(fe, np.repeat(gray[None], len(clouds), 0), cl, K4=None)
    return hs, [mx.cloud_points(c) for c in cl]


@pytest.mark.parametrize("method", METHODS)
@pytest.mark.parametrize("visual,step", [("grey", 2), ("colour", 2), ("bayer-u16", 2), ("grey", 1), ("grey", 4)])
def test_rendered_adjacent_frames_equal_the_restatement(fe, frames, visual, step, method):
    gray, depth = frames
    nh.reinit(fe, 0, cloud_creation_skip_step=step)
    K4 = nh.K4()
    if visual == "bayer-u16":
        u16 = np.stack([ro.to_millimetres(d) for d in depth])
        raw = np.stack([ro.mosaic_gr(c) for c in _colour(gray)])
        hs = _stored(fe, raw, u16, bayer=True)
        vis, dref = [ro.bayer_gr_to_rgb(r) for r in raw], ro.depth_u16_to_m(u16)
    else:
        vis = gray if visual == "grey" else np.stack([_colour(g) for g in gray])
        hs = _stored(fe, vis, depth)
        dref = depth
    pcs = [mx.create_cloud(dref[k], vis[k], K4, step, 1.0, fe.params.minimum_depth) for k in range(len(hs))]
    got = fe.icp_align(hs[:-1], hs[1:], method=method)  # older -> newer, as matchNodePair
    exps = _check(got, pcs[:-1], pcs[1:], tag=visual, method=method)
    assert all(e["converged"] == 1 and e["n_correspondences"] > 1000 and (method == "icp" or e["lm"]) for e in exps)
    nh.destroy(fe, hs)
    nh.reinit(fe, 0)


def _cloud(depth, vis, stride):
    fx, fy, cx, cy = nh.K4()
    h, w = depth.shape
    u, v = np.meshgrid(np.arange(w, dtype=F32), np.arange(h, dtype=F32))
    c = np.zeros((h, w, stride), F32)
    c[..., 0], c[..., 1], c[..., 2] = (u - cx) * depth / fx, (v - cy) * depth / fy, depth
    c[..., 4 if stride == 8 else 3] = mx.colour_words(vis).astype(np.uint32).view(F32)
    return c


@pytest.mark.parametrize("method", METHODS)
@pytest.mark.parametrize("stride", [8, 4])
def test_cloud_nodes_with_nan_and_inf_points(fe, frames, stride, method):
    gray, depth = frames
    nh.reinit(fe, 0)
    clouds = np.stack([_cloud(d, _colour(g), stride) for g, d in zip(gray[:3], depth[:3])])
    clouds[1, 100:110, 200:210, 0] = np.inf  # kept by filterCloud, no part in the correspondences
    clouds[1, 120:130, 200:210, 2] = -np.inf
    clouds[2, 200:205, 300:340, 1] = np.nan
    hs = _stored(fe, gray[:3], clouds, K4=None)
    pcs = [mx.cloud_points(c) for c in clouds]
    _check(fe.icp_align(hs[:2] + [hs[2]], hs[1:] + [hs[1]], method=method), pcs[:2] + [pcs[2]], pcs[1:] + [pcs[1]], tag=stride,
           method=method)
    nh.destroy(fe, hs)


@pytest.mark.parametrize("method", METHODS)
def test_voxel_reduced_nodes(fe, frames, method):
    gray, depth = frames
    nh.reinit(fe, 0, cloud_creation_skip_step=2)
    hs = _stored(fe, gray[:3], depth[:3])
    pcs = [mx.create_cloud(depth[k], gray[k], nh.K4(), 2, 1.0, fe.params.minimum_depth) for k in range(3)]
    fe.reduce_clouds(hs[:2], 0.02)
    red = [vx.reduce_cloud(pc, 0.02) for pc in pcs[:2]] + [pcs[2]]
    # reduced -> reduced, reduced -> unreduced, unreduced -> reduced
    _check(fe.icp_align([hs[0], hs[1], hs[2]], [hs[1], hs[2], hs[1]], method=method), [red[0], red[1], red[2]],
           [red[1], red[2], red[1]], method=method)
    nh.destroy(fe, hs)
    nh.reinit(fe, 0)


@pytest.mark.parametrize("method", METHODS)
@pytest.mark.parametrize("mcs", [1, 2, 3, 4, 5, 6, 500, 9999, 1000000])
def test_max_cloud_size(fe, frames, mcs, method):
    gray, depth = frames
    nh.reinit(fe, 0, cloud_creation_skip_step=4)
    hs = _stored(fe, gray[:2], depth[:2])
    pcs = [mx.create_cloud(depth[k], gray[k], nh.K4(), 4, 1.0, fe.params.minimum_depth) for k in range(2)]
    got = fe.icp_align([hs[0]], [hs[1]], max_cloud_size=mcs, method=method)
    e = _check(got, [pcs[0]], [pcs[1]], mcs, method=method)[0]
    n_valid = int((~np.isnan(pcs[0]["z"])).sum())
    assert e["n_source"] == (n_valid if mcs >= n_valid else len(ix.filter_indices(pcs[0]["z"], mcs)))
    nh.destroy(fe, hs)
    nh.reinit(fe, 0)


def test_planted_criteria_ties_and_distances(fe, frames):
    import test_icp_exact_cpu as tc
    gray = frames[0][0]
    src, tgt = tc._scene(2)
    far = (tgt + F32(0.5)).astype(F32)
    rng = np.random.default_rng(1)
    p10k = (rng.uniform(-0.3, 0.3, (3, 40)) + 1e4).astype(F32)
    tsrc, ttgt = tc.tie_clouds()
    clouds = [src, tgt, far, p10k, tsrc, ttgt, src[:, :2], np.zeros((3, 0), F32)]
    hs, pcs = _planted_nodes(fe, gray, clouds)
    pairs = [(0, 1, 4), (2, 1, 0), (1, 1, 2), (3, 3, 3), (4, 5, None), (6, 1, 0), (7, 1, 0), (1, 7, 0)]
    got = fe.icp_align([hs[a] for a, _, _ in pairs], [hs[b] for _, b, _ in pairs])
    exps = _check(got, [pcs[a] for a, _, _ in pairs], [pcs[b] for _, b, _ in pairs], tag="planted")
    for e, (_, _, c) in zip(exps, pairs):
        assert c is None or e["criterion"] == c
    assert exps[2]["converged"] == 1 and exps[1]["converged"] == 0 and np.array_equal(got[1]["T"], np.eye(4, dtype=F32).ravel())
    nh.destroy(fe, hs)


@pytest.mark.parametrize("method", METHODS)
def test_one_call_equals_calls_per_pair_and_nodes_may_repeat(fe, frames, method):
    gray, depth = frames
    nh.reinit(fe, 0, cloud_creation_skip_step=4)
    hs = _stored(fe, gray, depth)
    src = [hs[0], hs[1], hs[2], hs[1], hs[2], hs[3], hs[0]]
    tgt = [hs[1], hs[2], hs[3], hs[0], hs[2], hs[0], hs[3]]  # both sides, and a node as its own partner
    before = [fe.node_cloud(h).tobytes() for h in hs]
    one = fe.icp_align(src, tgt, method=method)
    for k in range(len(src)):
        assert fe.icp_align([src[k]], [tgt[k]], method=method)[0].tobytes() == one[k].tobytes(), k
    assert [fe.node_cloud(h).tobytes() for h in hs] == before  # the call changes no node
    pcs = [mx.create_cloud(depth[k], gray[k], nh.K4(), 4, 1.0, fe.params.minimum_depth) for k in range(4)]
    idx = {h: k for k, h in enumerate(hs)}
    _check(one, [pcs[idx[h]] for h in src], [pcs[idx[h]] for h in tgt], method=method)
    nh.destroy(fe, hs)
    nh.reinit(fe, 0)


def test_plain_icp_is_unchanged_after_icp_nl(fe, frames):
    gray, depth = frames
    nh.reinit(fe, 0, cloud_creation_skip_step=4)
    hs = _stored(fe, gray, depth)
    src = [hs[0], hs[1], hs[2], hs[1], hs[2], hs[3], hs[0]]
    tgt = [hs[1], hs[2], hs[3], hs[0], hs[2], hs[0], hs[3]]
    plain_before = fe.icp_align(src, tgt)
    fe.icp_align(src, tgt, method="icp_nl")
    assert fe.icp_align(src, tgt).tobytes() == plain_before.tobytes()  # icp after icp_nl in the same process
    pcs = [mx.create_cloud(depth[k], gray[k], nh.K4(), 4, 1.0, fe.params.minimum_depth) for k in range(4)]
    idx = {h: k for k, h in enumerate(hs)}
    for k in (0, 4):  # and plain ICP still equals its own restatement
        assert plain_before[k].tobytes() == _record(ix.align(pcs[idx[src[k]]], pcs[idx[tgt[k]]])).tobytes()
    nh.destroy(fe, hs)
    nh.reinit(fe, 0)


def test_rejected_calls_launch_nothing(fe, frames):
    import ctypes as C
    from rgbdslam_v2_b200._capi import ICP_RESULT_DTYPE, B200Error
    gray, depth = frames
    nh.reinit(fe, 0, cloud_creation_skip_step=4)
    hs = _stored(fe, gray[:1], depth[:1])
    det = fe.detector_create()
    bare, _ = fe.nodes_create(det, gray[1:2], depth[1:2], None, nh.K4())  # no stored cloud
    fe.detector_destroy(det)
    lib = fe.lib
    out = np.zeros(2, ICP_RESULT_DTYPE)
    h = np.array([hs[0], hs[0]], np.uint64)
    l0 = fe.launch_count
    assert lib.rgbdslam_b200_icp_align(-1, h.ctypes.data, h.ctypes.data, 10000, out.ctypes.data) == ERR_ARG
    assert lib.rgbdslam_b200_icp_align(1, h.ctypes.data, h.ctypes.data, 0, out.ctypes.data) == ERR_ARG
    assert lib.rgbdslam_b200_icp_align(1, None, h.ctypes.data, 10000, out.ctypes.data) == ERR_ARG
    bad = np.array([hs[0], 0], np.uint64)  # not a handle
    assert lib.rgbdslam_b200_icp_align(2, h.ctypes.data, bad.ctypes.data, 10000, out.ctypes.data) == ERR_ARG
    nb = np.array([hs[0], bare[0]], np.uint64)
    assert lib.rgbdslam_b200_icp_align(2, h.ctypes.data, nb.ctypes.data, 10000, out.ctypes.data) == ERR_STATE
    assert lib.rgbdslam_b200_icp_align(0, None, None, 10000, None) == 0
    assert fe.launch_count == l0 and out.tobytes() == bytes(out.nbytes)
    with pytest.raises(B200Error):
        fe.icp_align([bare[0]], [hs[0]])
    assert len(fe.icp_align([], [])) == 0
    nh.destroy(fe, hs + bare)
    nh.reinit(fe, 0)


def _sparse(seed, n, ang=0.01):
    """n points 0.2 m apart or more, and the same points moved by up to 1 cm: every correspondence is known"""
    rng = np.random.default_rng(seed)
    g = np.stack(np.meshgrid(np.arange(6), np.arange(6), np.arange(4)), -1).reshape(-1, 3)[:n] * 0.2
    tgt = (g + rng.uniform(-0.02, 0.02, g.shape)).T
    import test_icp_exact_cpu as tc
    R = tc._rot(rng.normal(size=3), ang)
    src = R @ tgt + rng.uniform(-0.01, 0.01, (3, 1))
    return src.astype(F32), tgt.astype(F32)


def test_planted_sparse_clouds_isolate_the_estimator(fe, frames):
    import test_icp_exact_cpu as tc
    gray = frames[0][0]
    clouds, pairs = [], []
    for k, n in enumerate((3, 4, 5, 6, 7, 40, 144)):
        s, t = _sparse(k, n)
        clouds += [s, t]
        pairs.append((2 * k, 2 * k + 1))
    src, tgt = tc._scene(2)
    tsrc, ttgt = tc.tie_clouds()
    base = len(clouds)
    clouds += [src, tgt, (tgt + F32(0.5)).astype(F32), tsrc, ttgt, np.zeros((3, 0), F32)]
    pairs += [(base, base + 1), (base + 2, base + 1), (base + 1, base + 1), (base + 3, base + 4), (base + 5, base + 1),
              (base + 1, base + 5)]
    hs, pcs = _planted_nodes(fe, gray, clouds)
    got = fe.icp_align([hs[a] for a, _ in pairs], [hs[b] for _, b in pairs], method="icp_nl")
    exps = _check(got, [pcs[a] for a, _ in pairs], [pcs[b] for _, b in pairs], tag="planted", method="icp_nl")
    assert [e["criterion"] for e in exps[:3]] == [0, 2, 2] and exps[0]["n_correspondences"] == 3
    assert exps[1]["lm"] == [(nx.IMPROPER, 0, 0)] and exps[3]["lm"][0][0] != nx.IMPROPER
    assert exps[len(pairs) - 5]["converged"] == 0 and exps[len(pairs) - 4]["converged"] == 1
    nh.destroy(fe, hs)


def test_unknown_method_launches_nothing(fe, frames):
    from rgbdslam_v2_b200._capi import ICP_RESULT_DTYPE
    gray, depth = frames
    nh.reinit(fe, 0, cloud_creation_skip_step=4)
    hs = _stored(fe, gray[:2], depth[:2])
    lib = fe.lib
    out = np.zeros(1, ICP_RESULT_DTYPE)
    s, t = np.array([hs[0]], np.uint64), np.array([hs[1]], np.uint64)
    l0 = fe.launch_count
    for method in (-1, 2, 7):
        assert lib.rgbdslam_b200_icp_align_ex(1, s.ctypes.data, t.ctypes.data, 10000, method, out.ctypes.data) == ERR_ARG
    assert lib.rgbdslam_b200_icp_align_ex(0, None, None, 10000, 5, None) == ERR_ARG
    assert fe.launch_count == l0 and out.tobytes() == bytes(out.nbytes)
    with pytest.raises(ValueError):
        fe.icp_align([hs[0]], [hs[1]], method="gicp")
    assert lib.rgbdslam_b200_icp_align_ex(1, s.ctypes.data, t.ctypes.data, 10000, 1, out.ctypes.data) == 0
    assert fe.launch_count > l0
    nh.destroy(fe, hs)
    nh.reinit(fe, 0)


def test_icp_recovers_a_known_motion(fe, frames):
    """a rendered frame's cloud and the same points moved by a known rigid motion M: T is closer to M than the identity is.
    (Between two rendered frames of the box room, whose walls are planes, two iterations of point-to-point ICP slide along
    the walls and do not beat the identity; DESIGN 4.12 gives the numbers.)"""
    import test_icp_exact_cpu as tc
    gray, depth = frames
    nh.reinit(fe, 0)
    c0 = _cloud(depth[0], gray[0], 4)
    ang, t = 0.003, (0.004, -0.003, 0.002)
    R = tc._rot([0.3, 1.0, 0.2], ang)
    M = np.eye(4)
    M[:3, :3], M[:3, 3] = R, t
    c1 = c0.copy()
    with np.errstate(invalid="ignore"):
        c1[..., :3] = (c0[..., :3].astype(np.float64) @ R.T + np.asarray(t)).astype(F32)
    hs = _stored(fe, gray[:2], np.stack([c0, c1]), K4=None)
    got = fe.icp_align([hs[0]], [hs[1]])
    _check(got, [mx.cloud_points(c0)], [mx.cloud_points(c1)])
    r = got[0]
    T = r["T"].reshape(4, 4).T.astype(np.float64)
    assert r["converged"] == 1 and np.abs(T - M).max() < np.abs(np.eye(4) - M).max(), (T, M)
    nh.destroy(fe, hs)
