"""GPU tests of icp_method "icp_nl" (rgbdslam_b200_icp_align_ex with RGBDSLAM_B200_ICP_METHOD_ICP_NL), byte for byte in every
field against the restatement of tests/icp_nl_exact.py, on the corpus of test_gpu_icp.py."""
import numpy as np
import pytest

import icp_exact as ix
import icp_nl_exact as nx
import map_cloud_exact as mx
import node_helpers as nh
import raw_input_oracle as ro
import voxel_exact as vx
from test_gpu_icp import _cloud, _colour, _planted_nodes, _record, _stored

pytestmark = pytest.mark.gpu
ERR_ARG = 1
F32 = np.float32


@pytest.fixture(scope="module")
def fe(built):
    from rgbdslam_v2_b200 import Frontend
    f = Frontend(0, nh.params(0))
    yield f
    f.close()


@pytest.fixture(scope="module")
def frames():
    return nh.stack(nh.render(range(4)))


def _check(got, pcs_src, pcs_tgt, mcs=10000, tag=""):
    assert len(got) == len(pcs_src)
    exps = []
    for k, (s, t) in enumerate(zip(pcs_src, pcs_tgt)):
        r = nx.align(s, t, mcs)
        exp = _record(r)
        assert got[k].tobytes() == exp.tobytes(), (tag, k, got[k], exp)
        exps.append(r)
    return exps


@pytest.mark.parametrize("visual,step", [("grey", 2), ("colour", 2), ("bayer-u16", 2), ("grey", 1), ("grey", 4)])
def test_rendered_adjacent_frames_equal_the_restatement(fe, frames, visual, step):
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
    got = fe.icp_align(hs[:-1], hs[1:], method="icp_nl")  # older -> newer, as matchNodePair
    exps = _check(got, pcs[:-1], pcs[1:], tag=visual)
    assert all(e["converged"] == 1 and e["n_correspondences"] > 1000 and e["lm"] for e in exps)
    nh.destroy(fe, hs)
    nh.reinit(fe, 0)


@pytest.mark.parametrize("stride", [8, 4])
def test_cloud_nodes_with_nan_and_inf_points(fe, frames, stride):
    gray, depth = frames
    nh.reinit(fe, 0)
    clouds = np.stack([_cloud(d, _colour(g), stride) for g, d in zip(gray[:3], depth[:3])])
    clouds[1, 100:110, 200:210, 0] = np.inf  # kept by filterCloud, no part in the correspondences
    clouds[1, 120:130, 200:210, 2] = -np.inf
    clouds[2, 200:205, 300:340, 1] = np.nan
    hs = _stored(fe, gray[:3], clouds, K4=None)
    pcs = [mx.cloud_points(c) for c in clouds]
    _check(fe.icp_align(hs[:2] + [hs[2]], hs[1:] + [hs[1]], method="icp_nl"), pcs[:2] + [pcs[2]], pcs[1:] + [pcs[1]],
           tag=stride)
    nh.destroy(fe, hs)


def test_voxel_reduced_nodes(fe, frames):
    gray, depth = frames
    nh.reinit(fe, 0, cloud_creation_skip_step=2)
    hs = _stored(fe, gray[:3], depth[:3])
    pcs = [mx.create_cloud(depth[k], gray[k], nh.K4(), 2, 1.0, fe.params.minimum_depth) for k in range(3)]
    fe.reduce_clouds(hs[:2], 0.02)
    red = [vx.reduce_cloud(pc, 0.02) for pc in pcs[:2]] + [pcs[2]]
    _check(fe.icp_align([hs[0], hs[1], hs[2]], [hs[1], hs[2], hs[1]], method="icp_nl"), [red[0], red[1], red[2]],
           [red[1], red[2], red[1]])
    nh.destroy(fe, hs)
    nh.reinit(fe, 0)


@pytest.mark.parametrize("mcs", [1, 2, 3, 4, 5, 6, 500, 9999, 1000000])
def test_max_cloud_size(fe, frames, mcs):
    gray, depth = frames
    nh.reinit(fe, 0, cloud_creation_skip_step=4)
    hs = _stored(fe, gray[:2], depth[:2])
    pcs = [mx.create_cloud(depth[k], gray[k], nh.K4(), 4, 1.0, fe.params.minimum_depth) for k in range(2)]
    got = fe.icp_align([hs[0]], [hs[1]], max_cloud_size=mcs, method="icp_nl")
    _check(got, [pcs[0]], [pcs[1]], mcs)
    nh.destroy(fe, hs)
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
    exps = _check(got, [pcs[a] for a, _ in pairs], [pcs[b] for _, b in pairs], tag="planted")
    assert [e["criterion"] for e in exps[:3]] == [0, 2, 2] and exps[0]["n_correspondences"] == 3
    assert exps[1]["lm"] == [(nx.IMPROPER, 0, 0)] and exps[3]["lm"][0][0] != nx.IMPROPER
    assert exps[len(pairs) - 5]["converged"] == 0 and exps[len(pairs) - 4]["converged"] == 1
    nh.destroy(fe, hs)


def test_one_call_equals_calls_per_pair_and_plain_icp_is_unchanged(fe, frames):
    gray, depth = frames
    nh.reinit(fe, 0, cloud_creation_skip_step=4)
    hs = _stored(fe, gray, depth)
    src = [hs[0], hs[1], hs[2], hs[1], hs[2], hs[3], hs[0]]
    tgt = [hs[1], hs[2], hs[3], hs[0], hs[2], hs[0], hs[3]]  # both sides, and a node as its own partner
    plain_before = fe.icp_align(src, tgt)
    before = [fe.node_cloud(h).tobytes() for h in hs]
    one = fe.icp_align(src, tgt, method="icp_nl")
    for k in range(len(src)):
        assert fe.icp_align([src[k]], [tgt[k]], method="icp_nl")[0].tobytes() == one[k].tobytes(), k
    assert [fe.node_cloud(h).tobytes() for h in hs] == before  # the call changes no node
    assert fe.icp_align(src, tgt).tobytes() == plain_before.tobytes()  # icp after icp_nl in the same process
    pcs = [mx.create_cloud(depth[k], gray[k], nh.K4(), 4, 1.0, fe.params.minimum_depth) for k in range(4)]
    idx = {h: k for k, h in enumerate(hs)}
    _check(one, [pcs[idx[h]] for h in src], [pcs[idx[h]] for h in tgt])
    for k in (0, 4):  # and plain ICP still equals its own restatement
        assert plain_before[k].tobytes() == _record(ix.align(pcs[idx[src[k]]], pcs[idx[tgt[k]]])).tobytes()
    nh.destroy(fe, hs)
    nh.reinit(fe, 0)


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
