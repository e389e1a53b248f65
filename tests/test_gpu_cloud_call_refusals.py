"""GPU tests of how the five calls that read many nodes' stored clouds refuse bad input: render_cloud, reduce_clouds,
transform_clouds, octomap_insert and octomap_filter_clouds.  Every fault alone, and every pair of faults whose order of
checks decides the outcome, gives a fixed return code and message and launches nothing.  The order is: the call's own
arguments, then a non-finite transform or sensor pose entry, then the nodes in order (an unknown handle gives ERR_ARG, a
node without a stored cloud ERR_STATE), then a node listed twice, for the three calls that rebuild clouds."""
import ctypes as C

import numpy as np
import pytest

import node_helpers as nh

pytestmark = pytest.mark.gpu

ERR_ARG, ERR_STATE = 1, 3
UNKNOWN = 0  # not a node handle
NO_CLOUD = "has no stored cloud (nodes_create_ex with RGBDSLAM_B200_STORE_CLOUD)"
IDENTITY12 = np.array([1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1, 0], np.float64)
IDENTITY7 = np.array([0, 0, 0, 1, 0, 0, 0], np.float64)

# call: (noun of its per-node values, one node's valid values, their dtype, whether a node may be listed only once)
CALLS = {
    "render_cloud": ("transform", IDENTITY12, np.float64, False),
    "reduce_clouds": (None, None, None, True),
    "transform_clouds": ("transform", IDENTITY12, np.float64, True),
    "octomap_insert": ("transform", IDENTITY12, np.float32, False),
    "octomap_filter_clouds": ("sensor pose", IDENTITY7, np.float32, True),
}


@pytest.fixture(scope="module")
def fe(built):
    from rgbdslam_v2_b200 import Frontend
    f = Frontend(0, nh.params(0))
    yield f
    f.close()


@pytest.fixture(scope="module")
def scene(fe):
    """two nodes with a stored cloud, one without, and an empty OctoMap"""
    gray, depth = nh.stack(nh.render(range(3)))
    det = fe.detector_create()
    hs, _ = fe.nodes_create(det, gray[:2], depth[:2], None, nh.K4(), store_cloud=True)
    plain, _ = fe.nodes_create(det, gray[2:], depth[2:], None, nh.K4())
    fe.detector_destroy(det)
    om = fe.octomap_create()
    yield [int(h) for h in hs], int(plain[0]), om
    fe.octomap_destroy(om)
    nh.destroy(fe, list(hs) + list(plain))


def _invoke(lib, name, om, n, hp, vp, point_bytes=32, leaf=0.05, max_range=np.inf, threshold=0.9):
    if name == "render_cloud":
        n_out = C.c_int64()
        return lib.rgbdslam_b200_render_cloud(n, hp, vp, np.inf, 0, point_bytes, None, 0, C.byref(n_out), None)
    if name == "reduce_clouds":
        return lib.rgbdslam_b200_reduce_clouds(n, hp, leaf, None)
    if name == "transform_clouds":
        return lib.rgbdslam_b200_transform_clouds(n, hp, vp)
    if name == "octomap_insert":
        return lib.rgbdslam_b200_octomap_insert(C.c_uint64(om), n, hp, vp, max_range)
    return lib.rgbdslam_b200_octomap_filter_clouds(C.c_uint64(om), n, hp, vp, threshold, None)


def _call(fe, name, handles, om, bad=None, n=None, null_handles=False, null_values=False, **kw):
    """the return code and last_error of one call on `handles`; bad = (node, entry, value) plants a value in its values"""
    _, one, dtype, _ = CALLS[name]
    h = np.ascontiguousarray(np.asarray(handles, np.uint64))
    v = None
    if one is not None:
        v = np.ascontiguousarray(np.tile(one, (len(h), 1)).astype(dtype))
        if bad is not None:
            v[bad[0], bad[1]] = bad[2]
    hp = None if null_handles else h.ctypes.data
    vp = None if null_values or v is None else v.ctypes.data
    rc = _invoke(fe.lib, name, om, len(h) if n is None else n, hp, vp, **kw)
    return rc, fe.lib.rgbdslam_b200_last_error().decode()


def _check(fe, scene, name, cases):
    hs, _, om = scene
    before = [fe.node_cloud(h, 16).tobytes() for h in hs]
    for handles, kw, rc, message in cases:
        n0 = fe.launch_count
        got, err = _call(fe, name, handles, **{"om": om, **kw})
        assert got == rc and message in err, (name, handles, kw, got, err)
        assert fe.launch_count == n0, (name, handles, kw)
    assert [fe.node_cloud(h, 16).tobytes() for h in hs] == before


def _arg_message(name):
    """the start of the call's message for a bad n, a null pointer or a bad scalar argument"""
    return "render_cloud: bad arguments" if name == "render_cloud" else f"{name}: n >= 0"


def _own_faults(name, hs):
    """the faults of the call's own arguments besides n and the pointers"""
    if name == "render_cloud":
        return [([hs[0]], dict(point_bytes=pb), ERR_ARG, "render_cloud: point_bytes must be 16") for pb in (0, 24, 64)]
    if name == "reduce_clouds":
        return [([hs[0]], dict(leaf=x), ERR_ARG, _arg_message(name)) for x in (0.0, -0.05, np.nan, np.inf, 1e-50)]
    if name == "octomap_insert":
        return [([hs[0]], dict(max_range=np.nan), ERR_ARG, _arg_message(name)),
                ([hs[0]], dict(om=0), ERR_ARG, "invalid octomap handle")]
    if name == "octomap_filter_clouds":
        return [([hs[0]], dict(threshold=np.nan), ERR_ARG, _arg_message(name)),
                ([hs[0]], dict(om=0), ERR_ARG, "invalid octomap handle")]
    return []


@pytest.mark.parametrize("name", list(CALLS))
def test_each_fault_alone(fe, scene, name):
    hs, plain, _ = scene
    noun, one, _, distinct = CALLS[name]
    cases = [
        ([hs[0]], dict(n=-1), ERR_ARG, _arg_message(name)),
        ([hs[0]], dict(null_handles=True), ERR_ARG, _arg_message(name)),
        ([hs[0], UNKNOWN], {}, ERR_ARG, "invalid node handle"),
        ([hs[0], plain], {}, ERR_STATE, f"{name}: node 1 {NO_CLOUD}"),
    ]
    if distinct:
        cases.append(([hs[0], hs[1], hs[0]], {}, ERR_ARG, f"{name}: a node is listed twice"))
    if noun:
        cases.append(([hs[0]], dict(null_values=True), ERR_ARG, _arg_message(name)))
        for j in (0, len(one) - 1):
            for bad in (np.nan, np.inf, -np.inf):
                cases.append(([hs[0], hs[1]], dict(bad=(1, j, bad)), ERR_ARG, f"{name}: {noun} 1 has a non-finite entry"))
    _check(fe, scene, name, cases + _own_faults(name, hs))


@pytest.mark.parametrize("name", list(CALLS))
def test_the_order_of_checks(fe, scene, name):
    hs, plain, _ = scene
    noun, _, _, _ = CALLS[name]
    cases = [
        # the nodes in order: an unknown handle before a node without a cloud, and the other way round
        ([UNKNOWN, plain], {}, ERR_ARG, "invalid node handle"),
        ([plain, UNKNOWN], {}, ERR_STATE, f"{name}: node 0 {NO_CLOUD}"),
        # a node listed twice is looked for only once every node has passed
        ([plain, hs[0], hs[0]], {}, ERR_STATE, f"{name}: node 0 {NO_CLOUD}"),
        ([hs[0], hs[0], plain], {}, ERR_STATE, f"{name}: node 2 {NO_CLOUD}"),
        ([hs[1], hs[1], UNKNOWN], {}, ERR_ARG, "invalid node handle"),
    ]
    if noun:
        cases += [
            # the values come before the nodes
            ([hs[0], UNKNOWN], dict(bad=(0, 0, np.nan)), ERR_ARG, f"{name}: {noun} 0 has a non-finite entry"),
            ([UNKNOWN, hs[0]], dict(bad=(1, 2, np.inf)), ERR_ARG, f"{name}: {noun} 1 has a non-finite entry"),
            ([hs[0], plain], dict(bad=(1, 0, -np.inf)), ERR_ARG, f"{name}: {noun} 1 has a non-finite entry"),
            ([hs[0], hs[0]], dict(bad=(0, 1, np.nan)), ERR_ARG, f"{name}: {noun} 0 has a non-finite entry"),
        ]
    # the call's own arguments come first
    cases.append(([UNKNOWN, plain], dict(n=-1, bad=(0, 0, np.nan) if noun else None), ERR_ARG, _arg_message(name)))
    _check(fe, scene, name, cases)
