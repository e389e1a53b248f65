"""GPU tests of the colour OctoMap (include/rgbdslam_b200/octomap.h): the device .ot bytes equal the C oracle's
(tests/octomap_oracle.c) for depth-image, point-cloud and voxel-reduced nodes, whatever the batching, across repeated inserts
and clear; stats equal the oracle's; repeated runs are bit-identical; bad arguments are refused before any device work."""
import ctypes as C

import numpy as np
import pytest

import map_cloud_exact as mx
import node_helpers as nh
import octomap_exact as ox
from rgbdslam_v2_b200._capi import B200Error, octomap_pose

pytestmark = pytest.mark.gpu

N = 6


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
    return gray, depth, [octomap_pose(P) for P in poses]


def _colour(gray):
    return np.ascontiguousarray(np.stack([gray, np.roll(gray, 3, axis=-1), np.roll(gray, 5, axis=-2)], -1))


def _pc(fe, h):
    """the node's stored cloud as the oracle reads it"""
    r = fe.node_cloud(h).reshape(-1)
    return dict(x=r["x"].copy(), y=r["y"].copy(), z=r["z"].copy(), rgb=r["rgb"].copy())


def _oracle(fe, hs, T, max_range=-1.0, m=None):
    m = m or ox.Oracle()
    for h, t in zip(hs, T):
        m.insert_cloud(_pc(fe, h), t, max_range)
    return m


def _device(fe, hs, T, max_range=float("inf"), splits=None, **kw):
    om = fe.octomap_create(**kw)
    splits = splits or [len(hs)]
    k = 0
    for s in splits:
        fe.octomap_insert(om, hs[k:k + s], T[k:k + s], max_range)
        k += s
    data, st = fe.octomap_write(om), fe.octomap_stats(om)
    fe.octomap_destroy(om)
    return data, st


@pytest.fixture(scope="module")
def depth_nodes(fe, scene):
    gray, depth, _ = scene
    det = fe.detector_create()
    hs, _ = fe.nodes_create(det, np.stack([_colour(g) for g in gray]), depth, None, nh.K4(), store_cloud=True)
    fe.detector_destroy(det)
    yield hs
    nh.destroy(fe, hs)


def test_depth_image_nodes_equal_the_oracle(fe, scene, depth_nodes):
    T = scene[2]
    data, st = _device(fe, depth_nodes, T)
    m = _oracle(fe, depth_nodes, T)
    ref = m.write()
    size, res, rec = ox.parse(data)
    assert data == ref and st == m.stats() and size > 1000 and res == "0.05"
    assert (rec["r"] != 255).any() and (rec["lo"] > 0).any() and (rec["lo"] < 0).any()


@pytest.mark.parametrize("splits,batch", [([1] * N, None), ([2, 4], None), ([N], "300000"), ([3, 3], "1")],
                         ids=["one-by-one", "2+4", "small-batches", "one-node-batches"])
def test_batching_does_not_change_the_bytes(fe, scene, depth_nodes, monkeypatch, splits, batch):
    T = scene[2]
    ref, _ = _device(fe, depth_nodes, T)
    if batch:
        monkeypatch.setenv("RB200_OCT_BATCH_ENTRIES", batch)
    got, _ = _device(fe, depth_nodes, T, splits=splits)
    assert got == ref


def test_max_range_and_parameters_equal_the_oracle(fe, scene, depth_nodes):
    T = scene[2]
    kw = dict(resolution=0.08, prob_hit=0.7, prob_miss=0.45, clamping_min=0.12, clamping_max=0.97)
    data, st = _device(fe, depth_nodes[:3], T[:3], max_range=1.5, **kw)
    m = _oracle(fe, depth_nodes[:3], T[:3], 1.5, ox.Oracle(**kw))
    assert data == m.write() and st == m.stats()


def test_repeated_inserts_clear_and_repeated_runs(fe, scene, depth_nodes):
    T = scene[2]
    om = fe.octomap_create()
    fe.octomap_insert(om, depth_nodes[:2], T[:2])
    fe.octomap_insert(om, depth_nodes[:2], T[:2])  # the same scans again: sequential updates
    m = _oracle(fe, depth_nodes[:2], T[:2])
    _oracle(fe, depth_nodes[:2], T[:2], m=m)
    assert fe.octomap_write(om) == m.write()
    fe.octomap_clear(om)
    assert fe.octomap_stats(om) == (0, 0) and fe.octomap_write(om) == ox.Oracle().write()
    fe.octomap_insert(om, depth_nodes[2:], T[2:])
    first = fe.octomap_write(om)
    assert first == _oracle(fe, depth_nodes[2:], T[2:]).write()
    fe.octomap_destroy(om)
    again, _ = _device(fe, depth_nodes[2:], T[2:])
    assert again == first


def test_point_cloud_and_reduced_nodes_equal_the_oracle(fe, scene):
    gray, depth, T = scene
    fx, fy, cx, cy = nh.K4()
    h, w = depth.shape[1:]
    u, v = np.meshgrid(np.arange(w, dtype=np.float32), np.arange(h, dtype=np.float32))
    clouds = np.zeros((3, h, w, 8), np.float32)
    for k in range(3):
        d = depth[k]
        clouds[k, ..., 0], clouds[k, ..., 1], clouds[k, ..., 2] = (u - cx) * d / fx, (v - cy) * d / fy, d
        clouds[k, ..., 4] = mx.colour_words(_colour(gray[k])).astype(np.uint32).view(np.float32)
    det = fe.detector_create()
    hs, _ = fe.nodes_create(det, gray[:3], clouds, None, None, store_cloud=True)
    d_hs, _ = fe.nodes_create(det, gray[3:], depth[3:], None, nh.K4(), store_cloud=True)
    fe.detector_destroy(det)
    fe.reduce_clouds(d_hs[:2], 0.02)  # two reduced depth-image nodes, one unreduced
    allh = list(hs) + list(d_hs)
    data, st = _device(fe, allh, T)
    m = _oracle(fe, allh, T)
    assert data == m.write() and st == m.stats()
    nh.destroy(fe, allh)


def test_bad_arguments_are_refused(fe, scene, depth_nodes):
    T = np.array(scene[2][:1])
    lib = fe.lib
    from rgbdslam_v2_b200._capi import OctomapParams
    for bad in (dict(resolution=0.0), dict(prob_hit=1.0), dict(prob_miss=0.0), dict(clamping_min=0.9, clamping_max=0.8),
                dict(resolution=float("nan"))):
        with pytest.raises(B200Error):
            fe.octomap_create(**bad)
    om = fe.octomap_create()
    Tn = T.copy()
    Tn[0, 1, 2] = np.inf
    with pytest.raises(B200Error):
        fe.octomap_insert(om, depth_nodes[:1], Tn)
    with pytest.raises(B200Error):
        fe.octomap_insert(om, depth_nodes[:1], T, max_range=float("nan"))
    det = fe.detector_create()
    plain, _ = fe.nodes_create(det, scene[0][:1], scene[1][:1], None, nh.K4())
    fe.detector_destroy(det)
    rc = lib.rgbdslam_b200_octomap_insert(C.c_uint64(om), 1, np.array(plain, np.uint64).ctypes.data,
                                          np.ascontiguousarray(T, np.float32).ctypes.data, -1.0)
    assert rc == 3  # ERR_STATE: no stored cloud
    assert fe.octomap_stats(om) == (0, 0)
    n = C.c_int64()
    assert lib.rgbdslam_b200_octomap_write(C.c_uint64(om), np.zeros(4, np.uint8).ctypes.data, 4, C.byref(n)) == 1
    assert n.value == len(ox.Oracle().write())
    nh.destroy(fe, plain)
    fe.octomap_destroy(om)
    p = OctomapParams()
    lib.rgbdslam_b200_octomap_default_params(C.byref(p))
    assert (p.resolution, p.prob_hit, p.prob_miss, p.clamping_min, p.clamping_max) == (0.05, 0.9, 0.4, 0.001, 0.999)
