"""The C oracle of the colour OctoMap (tests/octomap_oracle.c) on hand-computed cases, and the pose chain of saveOctomap
(rgbdslam_v2_b200._capi.octomap_pose).  Resolution 1 m unless noted, so that key(c) = floor(c) + 32768."""
import numpy as np
import pytest

import octomap_exact as ox
from rgbdslam_v2_b200._capi import octomap_pose_steps

F32 = np.float32
Z = 32768


def lo(p):
    return F32(np.log(p / (1 - p)))


HIT, MISS, CMIN, CMAX = lo(0.9), lo(0.4), lo(0.001), lo(0.999)


def keys(*cells):
    return np.array([[Z + a, Z + b, Z + c] for a, b, c in cells], np.uint16).reshape(-1, 3)


def leaves(data):
    """{(x, y, z) keys: (log-odds, (r, g, b))} of the leaves of an .ot file"""
    _, _, rec = ox.parse(data)
    out = {}

    def walk(node, depth, k):
        r, kids = node
        if depth == 16:
            out[tuple(k)] = (r["lo"], (int(r["r"]), int(r["g"]), int(r["b"])))
        for c, child in kids:
            bit = 15 - depth
            walk(child, depth + 1, [k[0] | ((c & 1) << bit), k[1] | (((c >> 1) & 1) << bit), k[2] | (((c >> 2) & 1) << bit)])

    root = ox.tree(rec)
    if root is not None:
        walk(root, 0, [0, 0, 0])
    return out


def test_axis_aligned_ray():
    assert np.array_equal(ox.ray_keys([0.5, 0.5, 0.5], [3.5, 0.5, 0.5], 1.0), keys((0, 0, 0), (1, 0, 0), (2, 0, 0)))
    assert np.array_equal(ox.ray_keys([0.5, 0.5, 3.5], [0.5, 0.5, 0.5], 1.0), keys((0, 0, 3), (0, 0, 2), (0, 0, 1)))


def test_exact_tmax_ties_advance_y_then_z():
    # direction (1, 1, 0) / sqrt 2: tMax x == tMax y, and the tie goes to y (tMax[0] < tMax[1] fails, tMax[1] < tMax[2] holds)
    assert np.array_equal(ox.ray_keys([0.5, 0.5, 0.5], [2.5, 2.5, 0.5], 1.0), keys((0, 0, 0), (0, 1, 0), (1, 1, 0), (1, 2, 0)))
    # x == z tie: tMax[0] < tMax[2] fails -> z
    assert np.array_equal(ox.ray_keys([0.5, 0.5, 0.5], [1.5, 0.5, 1.5], 1.0), keys((0, 0, 0), (0, 0, 1)))


def test_negative_coordinates_and_voxel_borders():
    # floor: -1.0 and -0.0001 share key -1, 1.0 starts key 1
    assert len(ox.ray_keys([-1.0, 0.5, 0.5], [-0.0001, 0.5, 0.5], 1.0)) == 0
    assert np.array_equal(ox.ray_keys([-1.0001, 0.5, 0.5], [-0.5, 0.5, 0.5], 1.0), keys((-2, 0, 0)))
    assert np.array_equal(ox.ray_keys([-0.5, -0.5, -0.5], [1.0, -0.5, -0.5], 1.0), keys((-1, -1, -1), (0, -1, -1)))


def test_origin_and_end_in_one_voxel():
    r = ox.ray_keys([0.01, 0.01, 0.01], [0.04, 0.02, 0.049], 0.05)
    assert r is not None and len(r) == 0


@pytest.mark.parametrize("end", [[40000.0, 0.5, 0.5], [-32769.0, 0.5, 0.5], [np.inf, 0.5, 0.5], [0.5, -np.inf, 0.5],
                                 [0.5, 0.5, np.nan]])
def test_out_of_range_ends_have_no_ray(end):
    assert ox.ray_keys([0.5, 0.5, 0.5], end, 1.0) is None


def test_key_both_free_and_occupied_is_occupied():
    m = ox.Oracle(1.0)
    m.insert([[3.5, 0.5, 0.5], [1.5, 0.5, 0.5]], [0, 0], [0.5, 0.5, 0.5])
    lv = leaves(m.write())
    assert {k: v[0] for k, v in lv.items()} == {(Z, Z, Z): MISS, (Z + 1, Z, Z): HIT, (Z + 2, Z, Z): MISS, (Z + 3, Z, Z): HIT}


def test_clamping_from_both_sides():
    m = ox.Oracle(1.0)
    exp_hit, exp_miss = F32(0), F32(0)
    for _ in range(20):
        m.insert([[2.5, 0.5, 0.5]], [0], [0.5, 0.5, 0.5])
        exp_hit = min(max(F32(exp_hit + HIT), CMIN), CMAX)
        exp_miss = min(max(F32(exp_miss + MISS), CMIN), CMAX)
    lv = leaves(m.write())
    assert lv[(Z + 2, Z, Z)][0] == exp_hit == CMAX
    assert lv[(Z + 1, Z, Z)][0] == lv[(Z, Z, Z)][0] == exp_miss == CMIN


def test_cell_freed_then_hit():
    m = ox.Oracle(1.0)
    m.insert([[3.5, 0.5, 0.5]], [0], [0.5, 0.5, 0.5])
    m.insert([[1.5, 0.5, 0.5]], [0], [0.5, 0.5, 0.5])
    lv = leaves(m.write())
    assert lv[(Z + 1, Z, Z)][0] == F32(MISS + HIT)
    assert lv[(Z, Z, Z)][0] == F32(MISS + MISS) and lv[(Z + 3, Z, Z)][0] == HIT


def word(r, g, b):
    return (r << 16) | (g << 8) | b


def test_white_is_unset_and_int_mean_rounds_down():
    m = ox.Oracle(1.0)
    pts = [[2.2, 0.5, 0.5], [2.4, 0.5, 0.5], [2.6, 0.5, 0.5], [2.8, 0.5, 0.5]]
    m.insert(pts, [word(255, 255, 255), word(10, 20, 31), word(11, 21, 32), word(0xff, 0, 0) | 0xff000000], [0.5, 0.5, 0.5])
    lv = leaves(m.write())
    # white leaves the leaf unset, so (10, 20, 31) replaces it; then ((10 + 11) / 2, ...) and ((10 + 255) / 2, ...) in int;
    # the alpha byte is not colour
    assert lv[(Z + 2, Z, Z)][1] == (132, 10, 15)
    assert lv[(Z, Z, Z)][1] == lv[(Z + 1, Z, Z)][1] == (255, 255, 255)
    _, _, rec = ox.parse(m.write())
    # every ancestor of the coloured leaf has it as its only coloured descendant: same colour up to the root
    assert (int(rec[0]["r"]), int(rec[0]["g"]), int(rec[0]["b"])) == (132, 10, 15)


def test_inner_colour_is_the_int_mean_of_the_set_children_and_log_odds_the_max():
    m = ox.Oracle(1.0)
    # leaves (2, 0, 0) and (3, 0, 0) share their parent; (3, 0, 0) ends a ray, (2, 0, 0) too in the second point's scan
    m.insert([[2.5, 0.5, 0.5], [3.5, 0.5, 0.5]], [word(1, 2, 3), word(4, 6, 9)], [0.5, 0.5, 0.5])
    _, _, rec = ox.parse(m.write())
    root = ox.tree(rec)
    node = root
    for _ in range(15):  # down the path of key x = 32770 >> 1
        node = [c for _, c in node[1]][-1]
    r, kids = node
    assert len(kids) == 2 and (int(r["r"]), int(r["g"]), int(r["b"])) == ((1 + 4) // 2, (2 + 6) // 2, (3 + 9) // 2)
    assert r["lo"] == max(k[1][0]["lo"] for k in kids) == HIT


def test_out_of_range_and_infinite_points_contribute_nothing():
    m = ox.Oracle(1.0)
    m.insert([[40000.0, 0.5, 0.5], [np.inf, 0.5, 0.5], [0.5, -np.inf, 0.5], [np.nan, 0.5, 0.5]], [word(9, 9, 9)] * 4, [0.5, 0.5, 0.5])
    assert m.stats() == (0, 0) and ox.parse(m.write())[0] == 0


def test_finite_max_range_frees_the_shortened_ray_only():
    m = ox.Oracle(1.0)
    # |p - o| = 3 > 1.5: the ray ends at o + 1.5 x = 2.0, key 2 -- cells 0 and 1 free, nothing occupied, the colour finds no leaf
    m.insert([[3.5, 0.5, 0.5]], [word(7, 7, 7)], [0.5, 0.5, 0.5], max_range=1.5)
    lv = leaves(m.write())
    assert lv == {(Z, Z, Z): (MISS, (255, 255, 255)), (Z + 1, Z, Z): (MISS, (255, 255, 255))}
    m.clear()
    m.insert([[3.5, 0.5, 0.5]], [word(7, 7, 7)], [0.5, 0.5, 0.5], max_range=3.0)  # |p - o| <= max_range: a normal ray
    assert leaves(m.write())[(Z + 3, Z, Z)] == (HIT, (7, 7, 7))


def test_header_size_and_records_parse_back():
    m = ox.Oracle(0.05)
    empty = m.write()
    assert empty == ox.HEADER + b"size 0\nres 0.05\ndata\n"
    rng = np.random.default_rng(0)
    pts = rng.uniform(-1, 1, (200, 3)).astype(F32)
    m.insert(pts, rng.integers(0, 1 << 24, 200).astype(np.uint32), [0.01, -0.02, 0.03])
    data = m.write()
    size, res, rec = ox.parse(data)
    nodes, nleaves = m.stats()
    assert res == "0.05" and size == nodes == len(rec) and nleaves > 100
    ox.tree(rec)  # the child bits account for every record, in pre-order
    assert sum(1 for _ in leaves(data)) == nleaves
    assert ox.Oracle(0.1).write().endswith(b"size 0\nres 0.1\ndata\n")


# ---- the pose chain --------------------------------------------------------------------------------------------------------

def steps(R, t=(0.25, -1.5, 2.0)):
    T = np.eye(4)
    T[:3, :3] = R
    T[:3, 3] = t
    return octomap_pose_steps(T)


def bits(a):
    return [int(v) for v in np.asarray(a, F32).ravel().view(np.uint32)]


def test_pose_chain_identity_and_half_turns_are_exact():
    st = steps(np.eye(3))
    assert np.array_equal(st["T"][:, :3], np.eye(3, dtype=F32)) and st["eigen_branch"] == st["tf_branch"] == -1
    assert np.array_equal(st["T"][:, 3], np.array([0.25, -1.5, 2.0], F32))
    for i, d in enumerate(([1, -1, -1], [-1, 1, -1], [-1, -1, 1])):  # 180 degrees: the largest-diagonal branch on both sides
        st = steps(np.diag(d).astype(float))
        assert st["eigen_branch"] == st["tf_branch"] == i
        assert np.array_equal(st["T"][:, :3], np.diag(d).astype(F32))


def test_pose_chain_quarter_turn_by_hand():
    """90 degrees about z.  Eigen: trace 0 + (0 + 1) = 1 > 0, t = sqrtf(2), w = 0.5 t and z = (1 - -1) (0.5 / t) are both
    float(1 / sqrt 2) = 0x3f3504f3, which is below 1 / sqrt 2.  tf's double round trip gives that quaternion back, and
    toRotationMatrix forms 2 z z = 2 z w = 1 - 2^-24 in float: the diagonal is 2^-24, not 0, and the off-diagonal
    -(1 - 2^-24), not -1 -- unlike the float cast of the rotation."""
    R = np.array([[0.0, -1.0, 0.0], [1.0, 0.0, 0.0], [0.0, 0.0, 1.0]])
    st = steps(R)
    a = F32(np.sqrt(F32(2))) * F32(0.5)
    assert bits(a) == [0x3F3504F3] and bits(st["q_eigen"]) == bits([0, 0, a, a])
    assert st["eigen_branch"] == st["tf_branch"] == -1
    assert np.array_equal(st["q_tf"].astype(F32), np.array([0, 0, a, a], F32))
    tzz = F32(F32(2) * a) * a
    assert tzz == F32(1) - F32(2.0 ** -24)
    exp = np.array([[F32(1) - tzz, -tzz, 0], [tzz, F32(1) - tzz, 0], [0, 0, 1]], F32)
    assert bits(st["T"][:, :3]) == bits(exp) and not np.array_equal(exp, R.astype(F32))


# Rotations where Eigen's float decision and tf's double decision part ways: the trace is near 0 (a positive float trace
# against a non-positive double one, or the reverse), or two diagonal entries tie in float -- Eigen keeps the first under its
# strict >, tf's rebuilt double matrix orders them.  T: the float32 bits of the rotation the chain gives.
DIVERGING = {
    "float-trace-positive-tf-diagonal-0": (
        [[0.43750407432468497, -0.8858387862309618, 0.15453099934368147], [-0.41680490255005975, -0.04750040961356777, 0.9077540329278513],
         [-0.7967834449582494, -0.4615553660130056, -0.3900035717080865]], -1, 0,
        [0x3EE00088, 0xBF62C655, 0x3E1E3D5A, 0xBED56776, 0xBD429000, 0x3F686291, 0xBF4BFA00, 0xBEEC50FA, 0xBEC7AE90]),
    "float-diagonal-0-tf-trace-positive": (
        [[0.9083653573492179, 0.3176658694197086, -0.2719572999087323], [0.390379043125717, -0.41100898391374785, 0.823817830488293],
         [0.14992191386210726, -0.8544940084915804, -0.4973564206843153]], 0, -1,
        [0x3F688AA2, 0x3EA2A518, 0xBE8B3DFD, 0x3EC7DFC2, 0xBED26FC0, 0x3F52E5BA, 0x3E198521, 0xBF5AC01E, 0xBEFEA57C]),
    "equal-diagonal-0-2": (
        [[-0.0014347147854341627, 0.03815027020477623, 0.9992709835058691], [0.07508027208130147, -0.9964474444884187, 0.03815027020477623],
         [0.9971764609825495, 0.07508027208130147, -0.0014347147854341627]], 0, 2,
        [0xBABC1000, 0x3D1C4374, 0x3F7FD03A, 0x3D99C3B0, 0xBF7F1730, 0x3D1C4376, 0x3F7F46F6, 0x3D99C3B0, 0xBABC0C00]),
    "equal-diagonal-0-1": (
        [[-0.04116788215055062, 0.9555587136083679, 0.29191223051862697], [0.9618644135134504, -0.04116788215055062, 0.2704109012145495],
         [0.2704109012145495, 0.29191223051862697, -0.9174231271218181]], 0, 1,
        [0xBD289FC0, 0x3F749F7F, 0x3E957585, 0x3F763CBF, 0xBD289FA0, 0x3E8A734C, 0x3E8A734B, 0x3E957586, 0xBF6ADC40]),
}


@pytest.mark.parametrize("name", sorted(DIVERGING))
def test_pose_chain_where_eigen_and_tf_branch_differently(name):
    R, eb, tb, exp = DIVERGING[name]
    R = np.array(R)
    Rf = R.astype(F32)
    if name.startswith("equal"):
        i, j = eb, tb
        assert Rf[i, i] == Rf[j, j] and st_diag_order(R, i, j)
    st = steps(R)
    assert (st["eigen_branch"], st["tf_branch"]) == (eb, tb)
    if tb >= 0:  # tf's choice follows from its double matrix
        M = st["M"]
        assert (M[0, 0] + M[1, 1]) + M[2, 2] <= 0.0 and M[tb, tb] == max(M[0, 0], M[1, 1], M[2, 2])
    assert bits(st["T"][:, :3]) == exp
    assert not np.array_equal(st["T"][:, :3], Rf)  # the chain is not the float cast
    assert np.abs(st["T"][:, :3].astype(np.float64) - R).max() < 1e-6


def st_diag_order(R, i, j):
    """Eigen's strict > keeps the lower index on a float tie"""
    st = steps(R)
    return st["eigen_branch"] == min(i, j)


@pytest.mark.parametrize("axis,deg", [([1, 0, 0], 179.99), ([0, 1, 0], -179.9), ([1, 1, 0], 179.999), ([1, 2, 3], 180.0),
                                      ([0, 0, 1], 90.0), ([1, 1, 1], 120.0), ([1, 1, 1], 240.0), ([1, -1, 0], 180.0)])
def test_pose_chain_stays_a_rotation(axis, deg):
    from scipy.spatial.transform import Rotation
    R = Rotation.from_rotvec(np.radians(deg) * np.asarray(axis, float) / np.linalg.norm(axis)).as_matrix()
    M = steps(R)["T"][:, :3].astype(np.float64)
    assert np.abs(M - R).max() < 2e-6 and np.abs(M @ M.T - np.eye(3)).max() < 2e-6
