"""GPU tests of the occupancy filter (rgbdslam_b200_octomap_filter_clouds, DESIGN.md 4.15): after inserts that equal the C
oracle's map byte for byte, every node's kept 16- and 32-byte records equal those of the oracle's om_occupancy_filter (tests/octomap_filter_oracle.c), for
depth-image, point-cloud and voxel-reduced nodes, several thresholds and sensor poses, an empty map, a second call and any
chunking; a node that keeps every point keeps its raster; the readers of a filtered cloud equal their restatements fed its
records; refused calls change nothing."""
import ctypes as C

import numpy as np
import pytest

import icp_exact as ix
import map_cloud_exact as mx
import node_helpers as nh
import octomap_exact as ox
import octomap_filter_exact as fx
from rgbdslam_v2_b200._capi import B200Error, cloud_sensor_pose, octomap_pose

pytestmark = pytest.mark.gpu

N = 6
IDENTITY7 = np.array([0, 0, 0, 1, 0, 0, 0], np.float32)


@pytest.fixture(scope="module")
def fe(built):
    from rgbdslam_v2_b200 import Frontend
    f = Frontend(0, nh.params(0))
    yield f
    f.close()


@pytest.fixture(scope="module")
def scene():
    from rgbdslam_v2_b200 import synth
    gray, depth = nh.stack(nh.render(range(0, 4 * N, 4)))
    poses = synth.trajectory(240)[0:4 * N:4]
    return gray, depth, poses


def _colour(gray):
    return np.ascontiguousarray(np.stack([gray, np.roll(gray, 3, axis=-1), np.roll(gray, 5, axis=-2)], -1))


def _depth_nodes(fe, scene, k=N):
    det = fe.detector_create()
    hs, _ = fe.nodes_create(det, np.stack([_colour(g) for g in scene[0][:k]]), scene[1][:k], None, nh.K4(), store_cloud=True)
    fe.detector_destroy(det)
    return list(hs)


def _cloud_nodes(fe, scene, k=3):
    gray, depth, _ = scene
    fx, fy, cx, cy = nh.K4()
    h, w = depth.shape[1:]
    u, v = np.meshgrid(np.arange(w, dtype=np.float32), np.arange(h, dtype=np.float32))
    clouds = np.zeros((k, h, w, 8), np.float32)
    for i in range(k):
        d = depth[i]
        clouds[i, ..., 0], clouds[i, ..., 1], clouds[i, ..., 2] = (u - cx) * d / fx, (v - cy) * d / fy, d
        clouds[i, ..., 4] = mx.colour_words(_colour(gray[i])).astype(np.uint32).view(np.float32)
    det = fe.detector_create()
    hs, _ = fe.nodes_create(det, gray[:k], clouds, None, None, store_cloud=True)
    fe.detector_destroy(det)
    return list(hs)


def _records(fe, h):
    """(32-byte, 16-byte) records of the node's cloud, flat"""
    return fe.node_cloud(h, 32).reshape(-1), fe.node_cloud(h, 16).reshape(-1)


def _pc(fe, h):
    r32, r16 = _records(fe, h)
    return dict(x=r32["x"].copy(), y=r32["y"].copy(), z=r32["z"].copy(), rgb=r32["rgb"].copy(), w16=r16["w"].copy())


def _maps(fe, hs, T, kw=None):
    """the device map and the oracle's after inserting the nodes' clouds under T, checked byte for byte"""
    kw = kw or {}
    om = fe.octomap_create(**kw)
    fe.octomap_insert(om, hs, T)
    m = fx.FilterOracle(**kw)
    for h, t in zip(hs, T):
        m.insert_cloud(_pc(fe, h), t)
    assert fe.octomap_write(om) == m.write()
    return om, m


def _sensor(poses, identity):
    return np.stack([IDENTITY7 if identity else np.concatenate(cloud_sensor_pose(P)) for P in poses]).astype(np.float32)


def _expected(fe, m, hs, S, thr):
    """per node the oracle's kept 32- and 16-byte records of its current cloud"""
    out = []
    for h, s in zip(hs, S):
        r32, r16 = _records(fe, h)
        keep = m.occupancy_filter(np.stack([r32["x"], r32["y"], r32["z"]], 1), s[:4], s[4:], thr)
        out.append((r32[keep].tobytes(), r16[keep].tobytes(), len(r32)))
    return out


def _check(fe, hs, exp, counts):
    for h, (e32, e16, P), c in zip(hs, exp, counts):
        r32, r16 = _records(fe, h)
        assert r32.tobytes() == e32 and r16.tobytes() == e16 and c == len(r32)
        shape = fe.node_cloud(h).shape
        if c < P:
            assert shape == (1, c)


THRESHOLDS = [0.9, 0.5, 0.0, np.inf, 3e3, 3e5]


@pytest.mark.parametrize("identity", [True, False], ids=["identity", "sensor-pose"])
@pytest.mark.parametrize("thr", THRESHOLDS)
def test_depth_image_nodes_equal_the_oracle(fe, scene, thr, identity):
    poses = scene[2]
    hs = _depth_nodes(fe, scene)
    T = [octomap_pose(P) for P in poses]
    om, m = _maps(fe, hs, T)
    S = _sensor(poses, identity)
    exp = _expected(fe, m, hs, S, thr)
    counts = fe.octomap_filter_clouds(om, hs, S, thr)
    _check(fe, hs, exp, counts)
    if thr in (3e3, 3e5) and not identity:  # thresholds where the decisions are mixed
        assert any(0 < c < P for c, (_, _, P) in zip(counts, exp))
    fe.octomap_destroy(om)
    nh.destroy(fe, hs)


def test_point_cloud_and_reduced_nodes_equal_the_oracle(fe, scene):
    poses = scene[2]
    hs = _cloud_nodes(fe, scene) + _depth_nodes(fe, scene, 3)
    fe.reduce_clouds(hs[3:5], 0.02)  # two reduced depth-image nodes, one not
    T = [octomap_pose(P) for P in poses]
    om, m = _maps(fe, hs, T)
    for thr in (3e4, 0.9):
        S = _sensor(poses, False)
        exp = _expected(fe, m, hs, S, thr)
        _check(fe, hs, exp, fe.octomap_filter_clouds(om, hs, S, thr))
    fe.octomap_destroy(om)
    nh.destroy(fe, hs)


def test_an_empty_map_empties_every_cloud(fe, scene):
    hs = _depth_nodes(fe, scene, 2) + _cloud_nodes(fe, scene, 1)
    om = fe.octomap_create()
    counts = fe.octomap_filter_clouds(om, hs, _sensor(scene[2][:3], False), np.inf)
    assert counts.tolist() == [0, 0, 0]
    for h in hs:
        assert fe.node_cloud(h).shape == (1, 0) and fe.node_cloud(h, 16).shape == (1, 0)
    fe.octomap_destroy(om)
    nh.destroy(fe, hs)


def test_chunkings_second_calls_and_repeated_runs_are_identical(fe, scene, monkeypatch):
    poses = scene[2]
    T = [octomap_pose(P) for P in poses]
    S = _sensor(poses, False)
    results = []
    for chunk, splits in ((None, [N]), ("1", [N]), ("50000", [N]), (None, [1] * N), (None, [2, 4]), (None, [N])):
        if chunk:
            monkeypatch.setenv("RB200_OCF_CHUNK_POINTS", chunk)
        else:
            monkeypatch.delenv("RB200_OCF_CHUNK_POINTS", raising=False)
        hs = _depth_nodes(fe, scene)
        om, m = _maps(fe, hs, T)
        k = 0
        for s in splits:
            fe.octomap_filter_clouds(om, hs[k:k + s], S[k:k + s], 3e5)
            k += s
        first = [_records(fe, h)[0].tobytes() for h in hs]
        exp = _expected(fe, m, hs, S, 3e4)  # a second call on the filtered clouds
        _check(fe, hs, exp, fe.octomap_filter_clouds(om, hs, S, 3e4))
        results.append((first, [e[0] for e in exp]))
        fe.octomap_destroy(om)
        nh.destroy(fe, hs)
    assert all(r == results[0] for r in results)


def _cover_node(fe, pts, shape, res=0.05):
    """a point-cloud node whose points are the centres of the three cells occupancyFilter visits for each of pts"""
    k = np.floor((1.0 / res) * pts.astype(np.float64)).astype(np.int64) - 1
    cells = np.concatenate([k + np.array([0, 0, d]) for d in range(3)])
    c = ((cells + 0.5) * res).astype(np.float32)
    h, w = 3 * shape[0] * shape[1] // 640, 640  # an image the ORB pyramid accepts
    cloud = np.zeros((1, h, w, 8), np.float32)
    cloud[0, ..., :3] = c.reshape(h, w, 3)
    det = fe.detector_create()
    hs, _ = fe.nodes_create(det, np.zeros((1, h, w), np.uint8), cloud, None, None, store_cloud=True)
    fe.detector_destroy(det)
    return hs[0]


def test_a_node_that_keeps_every_point_keeps_its_raster_and_the_measurement_model(fe, scene):
    gray, depth, poses = scene
    full = np.where(np.isfinite(depth) & (depth >= 0.5), depth, np.float32(2.0)).astype(np.float32)  # a depth at every point
    hs = _depth_nodes(fe, (gray, full, poses), 2)
    r = fe.node_cloud(hs[0])
    shape = r.shape
    assert not np.isnan(r["z"]).any()
    cover = _cover_node(fe, np.stack([r["x"].ravel(), r["y"].ravel(), r["z"].ravel()], 1), shape)
    eye = np.eye(4)
    om, m = _maps(fe, [cover], [octomap_pose(eye)])
    before = [x.tobytes() for x in _records(fe, hs[0])]
    T = np.eye(4)
    like_before = fe.observation_likelihood(hs[0], hs[1], T)
    counts = fe.octomap_filter_clouds(om, hs[:1], IDENTITY7[None], np.inf)
    assert counts[0] == r.size
    assert fe.node_cloud(hs[0]).shape == shape and [x.tobytes() for x in _records(fe, hs[0])] == before
    assert fe.observation_likelihood(hs[0], hs[1], T).tolist() == like_before.tolist()
    # the other node loses points: no raster, the measurement model refuses it
    fe.octomap_filter_clouds(om, hs[1:], IDENTITY7[None], np.inf)
    assert fe.node_cloud(hs[1]).shape[0] == 1 and fe.node_cloud(hs[1]).size < r.size
    with pytest.raises(B200Error):
        fe.observation_likelihood(hs[0], hs[1], T)
    fe.octomap_destroy(om)
    nh.destroy(fe, hs + [cover])


def test_reads_after_filtering_equal_their_restatements(fe, scene):
    poses = scene[2]
    nh.reinit(fe, 0, cloud_creation_skip_step=4)
    hs = _depth_nodes(fe, scene, 4)
    T = [octomap_pose(P) for P in poses[:4]]
    om, m = _maps(fe, hs, T)
    fe.octomap_filter_clouds(om, hs, _sensor(poses[:4], False), 3e5)
    fe.octomap_destroy(om)
    pcs = [_pc(fe, h) for h in hs]
    assert all(0 < len(pc["x"]) for pc in pcs)
    # render_cloud
    T12 = [np.asarray(P, np.float64)[:3].ravel() for P in poses[:4]]
    for pb in (32, 16):
        got, _ = fe.render_cloud(hs, T12, point_bytes=pb)
        assert got.tobytes() == mx.render(pcs, T12, point_bytes=pb).tobytes()
    # octomap_insert
    om = fe.octomap_create()
    fe.octomap_insert(om, hs, T)
    m = ox.Oracle()
    for pc, t in zip(pcs, T):
        m.insert_cloud(pc, t)
    assert fe.octomap_write(om) == m.write()
    fe.octomap_destroy(om)
    # icp_align
    import test_gpu_icp as tg
    res = fe.icp_align(hs[:3], hs[1:4])
    for k in range(3):
        assert res[k].tobytes() == tg._record(ix.align(pcs[k], pcs[k + 1])).tobytes(), k
    nh.destroy(fe, hs)
    nh.reinit(fe, 0)


def test_refused_calls_change_no_node(fe, scene):
    hs = _depth_nodes(fe, scene, 2)
    om = fe.octomap_create()
    before = [_records(fe, h)[0].tobytes() for h in hs]
    S = _sensor(scene[2][:2], False)
    bad = S.copy()
    bad[1, 2] = np.nan
    det = fe.detector_create()
    plain, _ = fe.nodes_create(det, scene[0][:1], scene[1][:1], None, nh.K4())
    fe.detector_destroy(det)
    lib = fe.lib
    for args, rc in (((hs, bad, 0.9), 1), ((hs, S, float("nan")), 1), (([hs[0], hs[0]], S, 0.9), 1),
                     (([hs[0], 0], S, 0.9), 1), (([hs[0], plain[0]], S, 0.9), 3)):
        h = np.ascontiguousarray(np.asarray(args[0], np.uint64))
        s = np.ascontiguousarray(np.asarray(args[1], np.float32))
        assert lib.rgbdslam_b200_octomap_filter_clouds(C.c_uint64(om), len(h), h.ctypes.data, s.ctypes.data, args[2], None) == rc
        assert [_records(fe, x)[0].tobytes() for x in hs] == before
    assert lib.rgbdslam_b200_octomap_filter_clouds(C.c_uint64(0), 1, np.array(hs[:1], np.uint64).ctypes.data, S.ctypes.data, 0.9,
                                                   None) == 1
    assert [_records(fe, x)[0].tobytes() for x in hs] == before
    fe.octomap_destroy(om)
    nh.destroy(fe, hs + list(plain))
