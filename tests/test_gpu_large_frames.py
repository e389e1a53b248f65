"""The Node constructor on frames wider or taller than 1023 px (DESIGN.md 4.5.5): 12-bit positions, a candidate buffer sized
from the largest grid cell, chunks sized by bytes per 640x480 frame and cv::ORB's per-level quotas, against the cv2 oracles
of the 640x480 tests on rendered frames at sensor sizes (the 640x480 camera's field of view, max_keypoints scaled with the
area)."""
import ctypes as C

import numpy as np
import pytest

import node_helpers as nh

pytestmark = pytest.mark.gpu

# (h, w): the 1023 / 1024 boundary, common RGB-D sensor sizes, the widest frame (a 3x3 grid needs cells of >= 143 rows for
# an 8-level pyramid of >= 40 px at level 7, so the shortest 3x3 frame is 333 rows)
SIZES = [(1023, 1023), (1023, 1024), (1024, 1023), (768, 1024), (720, 1280), (1024, 1280), (1080, 1920), (360, 4095)]


def _k(h, w):
    """max_keypoints scaled with the area from 600 at 640x480, within 1.5 K <= 4096"""
    return int(min(2700, round(600 * h * w / (640 * 480))))


@pytest.fixture(scope="module")
def fe(built):
    from rgbdslam_v2_b200 import Frontend
    f = Frontend(0, nh.params())
    yield f
    f.close()


_FRAMES = {}


def frames(h, w, n=3, first=0):
    """n rendered frames (gray, depth, the reference's mask from depth) at h x w and the camera"""
    from oracle import orb_oracle
    from rgbdslam_v2_b200 import synth
    key = (h, w, n, first)
    if key not in _FRAMES:
        poses = synth.trajectory(240)
        fr = [synth.render_frame(poses[k], seed=k, shape=(h, w)) for k in range(first, first + n)]
        gray, depth = np.stack([f[0] for f in fr]), np.stack([f[1] for f in fr])
        _FRAMES[key] = gray, depth, np.stack([orb_oracle.depth_to_mask(d) for d in depth])
    return (*_FRAMES[key], synth.intrinsics(w, h))


def _check_node(fe, h, o, det, st, nmin=1):
    """node h equals the oracle's (keypoints, descriptors, points); the detector's thresholds equal st's unless det is None"""
    okp, odesc, oxyz = o
    gkp = fe.node_keypoints(h)
    gdesc, gxyz = fe.node_download(h)
    assert len(gkp) == len(okp) >= nmin
    assert gkp.tobytes() == okp.tobytes()
    assert np.array_equal(gdesc, odesc)
    assert np.array_equal(gxyz.view(np.uint32), oxyz.view(np.uint32))
    if det is not None:
        assert np.array_equal(fe.detector_thresholds(det)[:9], np.array(st.thresh[:9]))


@pytest.mark.parametrize("detector", [0, 1], ids=["ORB", "FAST"])
@pytest.mark.parametrize("hw", SIZES, ids=[f"{w}x{h}" for h, w in SIZES])
def test_nodes_vs_oracle(fe, hw, detector):
    """Node::Node frame by frame over a sequence (thresholds carried): keypoints, descriptors, points and thresholds
    bit-identical to the cv2 oracle, the mask derived from depth on the device."""
    import fast_oracle
    from oracle import orb_oracle
    h, w = hw
    gray, depth, mask, K4 = frames(h, w)
    K = _k(h, w)
    det = nh.make_detector(fe, detector, max_keypoints=K)
    st = orb_oracle.DetectorState()
    construct = orb_oracle.node_construct if detector == 0 else fast_oracle.node_construct
    for k in range(len(gray)):
        hs, _ = fe.nodes_create(det, gray[k:k + 1], depth[k:k + 1], None, K4, mask_from_depth=True)
        _check_node(fe, hs[0], construct(gray[k], depth[k], mask[k], K4, st, max_keypoints=K), det, st, nmin=K // 2)
        nh.destroy(fe, hs)
    fe.detector_destroy(det)


def test_level_sides_follow_cv_orb_on_a_small_frame(fe):
    """633x480: the middle grid column is 273 px wide, one of the sides whose level 1 cv::ORB sizes as
    cvRound(273 * (1.f / 1.2f)) = 228 where cvRound(273 / 1.2f) = 227; ORB nodes over a sequence equal the oracle"""
    from oracle import orb_oracle
    h, w = 480, 633
    assert [x1 - x0 for _, _, x0, x1 in orb_oracle._cells(w, h, 3)][1] == 273
    gray, depth, mask, K4 = frames(h, w)
    det = nh.make_detector(fe, 0, max_keypoints=600)
    st = orb_oracle.DetectorState()
    for k in range(len(gray)):
        hs, _ = fe.nodes_create(det, gray[k:k + 1], depth[k:k + 1], None, K4, mask_from_depth=True)
        _check_node(fe, hs[0], orb_oracle.node_construct(gray[k], depth[k], mask[k], K4, st, max_keypoints=600), det, st, nmin=300)
        nh.destroy(fe, hs)
    fe.detector_destroy(det)


def test_input_kinds_at_1280x720(fe):
    """colour, Bayer with 16-bit depth, an XYZRGB cloud with its mask, use_feature_min_depth: each equal to its oracle"""
    import cloud_oracle as co
    import min_depth_oracle as md
    import raw_input_oracle as ro
    from oracle import orb_oracle
    h, w = 720, 1280
    gray, depth, mask, K4 = frames(h, w)
    K = _k(h, w)
    colour = np.stack([np.stack([g, np.roll(g, 7, 1), 255 - g], -1) for g in gray])

    def seq(run, construct, **kw):
        det = nh.make_detector(fe, 0, max_keypoints=K, **kw)
        st = orb_oracle.DetectorState()
        for k in range(len(gray)):
            hs, _ = run(det, k)
            _check_node(fe, hs[0], construct(k, st), det, st, nmin=K // 2)
            nh.destroy(fe, hs)
        fe.detector_destroy(det)

    sl = lambda a, k: a[k:k + 1]  # noqa: E731
    seq(lambda det, k: fe.nodes_create(det, sl(colour, k), sl(depth, k), sl(mask, k), K4),
        lambda k, st: orb_oracle.node_construct(co.rgb_to_gray(colour[k]), depth[k], mask[k], K4, st, max_keypoints=K))
    raw = np.stack([ro.mosaic_gr(c) for c in colour])
    u16 = np.stack([ro.to_millimetres(d) for d in depth])
    seq(lambda det, k: fe.nodes_create(det, sl(raw, k), sl(u16, k), None, K4, mask_from_depth=True, bayer=True),
        lambda k, st: orb_oracle.node_construct(ro.bayer_gr_to_gray(raw[k]), ro.depth_u16_to_m(u16[k]), ro.depth_u16_mask(u16[k]),
                                                K4, st, max_keypoints=K))
    fx, fy, cx, cy = K4
    uu, vv = np.meshgrid(np.arange(w, dtype=np.float32), np.arange(h, dtype=np.float32))
    cloud = np.zeros((len(gray), h, w, 8), np.float32)
    cloud[..., 0], cloud[..., 1], cloud[..., 2] = (uu - cx) * depth / fx, (vv - cy) * depth / fy, depth
    seq(lambda det, k: fe.nodes_create(det, sl(gray, k), sl(cloud, k), None, None, mask_from_cloud=True),
        lambda k, st: co.node_construct(gray[k], cloud[k], co.cloud_mask(cloud[k][..., 2]), st, max_keypoints=K))
    seq(lambda det, k: fe.nodes_create(det, sl(gray, k), sl(depth, k), sl(mask, k), K4),
        lambda k, st: md.node_construct(gray[k], depth[k], mask[k], K4, st, max_keypoints=K), use_feature_min_depth=1)


@pytest.mark.parametrize("detector", [0, 1], ids=["ORB", "FAST"])
def test_quotas_decide_the_nodes_when_the_adjuster_ends_on_too_many(fe, detector, monkeypatch):
    """1920x1080 frames of dense texture with adjuster_max_iterations 1: every detection ends on "too many", the nodes equal
    the oracle, which runs cv2's ORB itself.  ORB: the per-level quotas decide what the nodes hold -- in every cell of frame 0
    the keepStrongest survivors with and without the quotas differ, the FAST-score cut of the centre cell falls inside a
    tie, and no node equals the oracle's without the quotas.  The FAST detector has no quotas."""
    import fast_oracle
    import orb_quota_oracle as qo
    from oracle import orb_oracle
    h, w = 1080, 1920
    # at threshold 20 cv::ORB's per-level quotas change which keypoints every cell keeps, and a 702 x 422 cell under the
    # rendered mask has at most about 39 000 FAST / NMS candidates (the buffer holds 59 648)
    gray = nh.textured(h, w, 3)
    _, depth, mask, K4 = frames(h, w)
    K = 2000
    per_cell = int(K * 1.5) // 9
    det = nh.make_detector(fe, detector, max_keypoints=K, adjuster_max_iterations=1)
    st = orb_oracle.DetectorState()
    construct = orb_oracle.node_construct if detector == 0 else fast_oracle.node_construct
    hs, _ = fe.nodes_create(det, gray, depth, mask, K4)
    for k in range(3):
        st_before = list(st.thresh)
        o = construct(gray[k], depth[k], mask[k], K4, st, max_keypoints=K, max_iters=1)
        assert all(b * 1.3 == a or a == 10000.0 for a, b in zip(st.thresh[:9], st_before[:9]))  # "too many" everywhere
        _check_node(fe, hs[k], o, None, st, nmin=K // 2)
    assert np.array_equal(fe.detector_thresholds(det)[:9], np.array(st.thresh[:9]))
    if detector == 0:
        def strongest(kps):  # keepStrongest(per_cell), canonical ties (orb_oracle.grid_detect)
            r = sorted(kps, key=lambda q: (-abs(q.response), q.octave, q.pt[1], q.pt[0]))
            return {qo.key(q) for q in r[:per_cell]}
        for c, (y0, y1, x0, x1) in enumerate(orb_oracle._cells(w, h, 3)):  # frame 0: every threshold is 20
            sub, smask = np.ascontiguousarray(gray[0, y0:y1, x0:x1]), np.ascontiguousarray(mask[0, y0:y1, x0:x1])
            assert strongest(qo.detect(sub, smask, 20, 10000)) != strongest(qo.detect(sub, smask, 20, qo.UNBOUND)), c
            if c == 4:
                _, stats = qo.quota_rule(sub, smask, 20)
                assert any(f > 0 for _, f, _, _ in stats)  # ties at the 2 n_l cut, all kept
        monkeypatch.setattr(orb_oracle, "cv2", nh.UnboundOrb())
        st_free = orb_oracle.DetectorState()
        for k in range(3):
            okp, _, _ = orb_oracle.node_construct(gray[k], depth[k], mask[k], K4, st_free, max_keypoints=K, max_iters=1)
            assert okp.tobytes() != fe.node_keypoints(hs[k]).tobytes()
    nh.destroy(fe, hs)
    fe.detector_destroy(det)


def test_one_call_chunks_pinned_and_sharded_are_identical(fe):
    """12 frames of 1920x1080 (two chunks of 9 and 3) in one call == one call per frame == pinned input == a 1-rank
    _sharded call: nodes and final thresholds"""
    import torch
    gray, depth, mask, K4 = frames(1080, 1920, 12)
    K = _k(1080, 1920)
    nh.reinit(fe, 0, max_keypoints=K)

    def run(fn):
        det = fe.detector_create()
        hs = fn(det)
        thr = fe.detector_thresholds(det).copy()
        fe.detector_destroy(det)
        dump = nh.node_dump(fe, hs)
        nh.destroy(fe, hs)
        return dump, thr

    ref, thr = run(lambda det: fe.nodes_create(det, gray, depth, mask, K4)[0])
    assert min(len(k) for k, _, _ in ref) > K // 2
    one = run(lambda det: sum((fe.nodes_create(det, gray[k:k + 1], depth[k:k + 1], mask[k:k + 1], K4)[0] for k in range(12)), []))
    pg, pd, pm = (torch.from_numpy(x).pin_memory() for x in (gray, depth, mask))
    pinned = run(lambda det: fe.nodes_create(det, pg, pd, pm, K4)[0])
    comm = fe.comm_init(0, 1, fe.comm_unique_id())
    sharded = run(lambda det: fe.nodes_create_sharded(det, comm, 12, gray, depth, mask, K4)[0])
    fe.comm_destroy(comm)
    for dump, t in (one, pinned, sharded):
        assert nh.same_nodes(ref, dump) and np.array_equal(thr, t)


def test_sizes_and_geometries_outside_the_limits_launch_nothing(fe):
    """4096 px in either dimension, an ungridded detector above 1023 px and round(1.5 K / cells) >= 606 above 1023 px
    (grid 2 from K = 1615; grid 3 reaches it only beyond 1.5 K = 4096): ERR_ARG before any device work"""
    from rgbdslam_v2_b200._capi import B200Error
    lib = fe.lib
    nh.reinit(fe, 0, max_keypoints=2000)
    det = fe.detector_create()
    for (h, w), kw in [((720, 4096), {}), ((4096, 720), {}), ((720, 1280), dict(detector_grid_resolution=1)),
                       ((720, 1280), dict(max_keypoints=1615, detector_grid_resolution=2)),
                       ((1024, 768), dict(max_keypoints=2500, detector_grid_resolution=2))]:
        nh.reinit(fe, 0, **{"max_keypoints": 2000, **kw})
        g = np.zeros((1, h, w), np.uint8)
        d = np.ones((1, h, w), np.float32)
        l0 = lib.rgbdslam_b200_launch_count()
        with pytest.raises(B200Error):
            fe.nodes_create(det, g, d, None, (500.0, 500.0, w / 2, h / 2))
        comm = fe.comm_init(0, 1, fe.comm_unique_id())
        with pytest.raises(B200Error):
            fe.nodes_create_sharded(det, comm, 1, g, d, None, (500.0, 500.0, w / 2, h / 2))
        fe.comm_destroy(comm)
        assert lib.rgbdslam_b200_launch_count() == l0, (h, w, kw)
    fe.detector_destroy(det)
    nh.reinit(fe, 0)


def test_store_cloud_render_and_model_counts_at_1280x720(fe):
    """STORE_CLOUD clouds and render_cloud equal the restatement; the measurement model's counts on these nodes equal
    its restatement"""
    import emm_exact as ee
    import map_cloud_exact as mx
    h, w = 720, 1280
    gray, depth, mask, K4 = frames(h, w)
    nh.reinit(fe, 0, max_keypoints=_k(h, w))
    det = fe.detector_create()
    hs, _ = fe.nodes_create(det, gray, depth, mask, K4, store_cloud=True)
    pcs = []
    for k, hd in enumerate(hs):
        pc = mx.create_cloud(depth[k], gray[k], K4, 2, 1.0, fe.params.minimum_depth)
        exp = mx.organised(pc, 32)
        got = fe.node_cloud(hd, 32)
        assert got.shape == exp.shape and np.array_equal(got.view(np.uint8), exp.view(np.uint8))
        pcs.append(pc)
    from rgbdslam_v2_b200 import synth
    T = np.array([mx.world2cam(p) for p in synth.trajectory(40)[::7][:len(hs)]])
    got, _ = fe.render_cloud(hs, T)
    exp = mx.render(pcs, T)
    assert got.shape == exp.shape and np.array_equal(got.view(np.uint8), exp.view(np.uint8))
    nh.destroy(fe, hs)
    fe.detector_destroy(det)
    # the environment measurement model on 1280x720 nodes
    p = nh.params(0, max_keypoints=_k(h, w), observability_threshold=0.5)
    fe.params = p
    fe._check(fe.lib.rgbdslam_b200_init(0, C.byref(p)))
    det = fe.detector_create()
    hs, _ = fe.nodes_create(det, gray, depth, mask, K4)
    step, scale, md = p.cloud_creation_skip_step, p.depth_scaling_factor, p.minimum_depth
    czc = None if p.depth_cov_z0 < 0 else ee.cov_const(p.sigma_depth, fe.depth_cov_z0)
    seen = np.zeros(3, np.int64)
    for a, b in ((1, 0), (2, 1), (2, 0)):
        Ta, Tb = synth.trajectory(240)[a], synth.trajectory(240)[b]
        T = (np.linalg.inv(Tb) @ Ta).astype(np.float32)  # newer camera -> older camera
        got = fe.observation_likelihood(hs[a], hs[b], T)
        exp = ee.pairwise(T, ee.cloud_z(depth[a], step, scale, md), K4, ee.cloud_z(depth[b], step, scale, md), K4,
                          cloud_step=step, skip_step=p.emm_skip_step, sigma_depth=p.sigma_depth, czc=czc)
        n_loose = int(exp["loose"].sum())
        assert np.abs(np.asarray(got, np.int64) - exp["counts"]).max() <= n_loose, (a, b, got, exp["counts"])
        seen += exp["counts"][:3]
    assert seen[0] > 0
    nh.destroy(fe, hs)
    fe.detector_destroy(det)
    nh.reinit(fe, 0)
