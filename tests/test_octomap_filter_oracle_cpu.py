"""The C oracle of ColorOctomapServer::occupancyFilter (om_occupancy_filter in tests/octomap_filter_oracle.c, DESIGN.md 4.15) on
hand-built maps, and the sensor pose updateCloudOrigin stores (rgbdslam_v2_b200._capi.cloud_sensor_pose).  Resolution 1 m,
so that key(c) = floor(c) + 32768 and keyToCoord(k) = k - 32768 + 0.5."""
import numpy as np
import pytest

import octomap_filter_exact as fx
from rgbdslam_v2_b200._capi import cloud_sensor_pose, octomap_pose_steps

F32 = np.float32
I = (np.array([0, 0, 0, 1], F32), np.zeros(3, F32))  # PCL's default sensor pose
OCC_HIT = 1.0 - 1.0 / (1.0 + np.exp(np.float64(F32(np.log(0.9 / 0.1)))))


def occupied(*cells):
    """a map with one occupied leaf (log-odds logodds(0.9)) at each cell centre: a scan whose origin is its own point"""
    m = fx.FilterOracle(resolution=1.0)
    for c in cells:
        p = np.asarray(c, F32) + F32(0.5)
        m.insert(p[None], np.zeros(1, np.uint32), p)
    return m


def keep(m, pts, thr=0.9, pose=I):
    return m.occupancy_filter(np.asarray(pts, F32).reshape(-1, 3), pose[0], pose[1], thr)


def test_only_the_three_cells_of_the_loop_quirk_count():
    p = [0.25, 0.5, 0.75]  # cell (0, 0, 0)
    visited = [(-1, -1, -1), (-1, -1, 0), (-1, -1, 1)]
    # the rest of the 27-cell neighbourhood, the point's own cell included, is never looked at
    others = [(a, b, c) for a in (-1, 0, 1) for b in (-1, 0, 1) for c in (-1, 0, 1) if (a, b, c) not in visited]
    for cell in others:
        assert not keep(occupied(cell), p, thr=np.inf)[0], cell
    for cell in visited:
        assert keep(occupied(cell), p, thr=np.inf)[0], cell
    assert not keep(occupied(*others), p, thr=np.inf)[0]


def test_inverse_distance_sums_and_the_strict_comparison():
    p = np.array([0.25, 0.5, 0.75], F32)
    m = occupied((-1, -1, -1), (-1, -1, 1))
    so = sw = 0.0
    for cz in (-1, 1):
        d = np.array([-0.5, -0.5, cz + 0.5]) - p.astype(np.float64)
        w = (d[0] * d[0] + d[1] * d[1]) + d[2] * d[2]
        so += OCC_HIT / w
        sw += w
    tie = so / sw
    assert tie * sw == so  # the threshold below reproduces sum_occ exactly: a tie
    assert not keep(m, p, thr=tie)[0]
    assert keep(m, p, thr=np.nextafter(tie, np.inf))[0]
    for thr in (0.9, 0.5, 0.3, 0.0, np.inf):
        assert keep(m, p, thr)[0] == (so < thr * sw), thr


def test_points_without_a_visited_leaf_and_the_empty_map_are_dropped():
    rng = np.random.default_rng(3)
    pts = rng.uniform(-4, 4, (200, 3)).astype(F32)
    for thr in (0.0, 0.9, 1e30, np.inf, -1.0):
        assert not keep(fx.FilterOracle(resolution=1.0), pts, thr).any()
        assert not keep(occupied((50, 50, 50)), pts, thr).any()


def test_nan_z_is_dropped_and_other_nans_follow_the_rule():
    m = occupied((-1, -1, -1))
    assert keep(m, [0.5, 0.5, 0.5], np.inf)[0]
    assert not keep(m, [0.5, 0.5, np.nan], np.inf)[0]
    # a NaN x spreads into in.z through the rotation; with the identity it does not, and its key is (uint16)(INT_MIN + 32768)
    assert not keep(m, [np.nan, 0.5, 0.5], np.inf)[0]


def test_keys_wrap_at_zero():
    p = [-32767.5, 0.5, 0.5]  # key (0, 32768, 32768): x_a = -1 is key 65535, keyToCoord 32767.5
    assert not keep(occupied((-1, -1, -1)), p, np.inf)[0]
    m = occupied((32767, -1, -1))  # key 65535 on x
    assert keep(m, p, 0.9)[0]  # w = 65535^2 + ...: occ / w < 0.9 w


def _eigen(q, t, p):
    """numpy float32 restatement of q * p + t in Eigen's order"""
    x, y, z, w = (F32(v) for v in q)
    px, py, pz = (F32(v) for v in p)
    u = [y * pz - z * py, z * px - x * pz, x * py - y * px]
    u = [a + a for a in u]
    c = [y * u[2] - z * u[1], z * u[0] - x * u[2], x * u[1] - y * u[0]]
    return np.array([((pp + w * uu) + cc) + tt for pp, uu, cc, tt in zip((px, py, pz), u, c, t)], F32)


def test_sensor_transform_follows_eigens_order():
    from scipy.spatial.transform import Rotation
    rng = np.random.default_rng(5)
    differs = 0
    for R in Rotation.random(400, random_state=9).as_matrix():
        T = np.eye(4)
        T[:3, :3], T[:3, 3] = R, rng.uniform(-3, 3, 3)
        q, t = cloud_sensor_pose(T)
        p = rng.uniform(-4, 4, 3).astype(F32)
        got = fx.sensor_transform(q, t, p)
        assert got.view(np.uint32).tolist() == _eigen(q, t, p).view(np.uint32).tolist()
        # the product with the rotation matrix of q (toRotationMatrix), summed (r0 p0 + r1 p1) + r2 p2, + t
        M = _rotation_matrix(q)
        mat = np.array([((M[r, 0] * p[0] + M[r, 1] * p[1]) + M[r, 2] * p[2]) + t[r] for r in range(3)], F32)
        differs += mat.view(np.uint32).tolist() != got.view(np.uint32).tolist()
    assert differs > 50  # the order is visible in the bits


def _rotation_matrix(q):
    x, y, z, w = (F32(v) for v in q)
    tx, ty, tz = F32(2) * x, F32(2) * y, F32(2) * z
    return np.array([[F32(1) - (ty * y + tz * z), ty * x - tz * w, tz * x + ty * w],
                     [ty * x + tz * w, F32(1) - (tx * x + tz * z), tz * y - tx * w],
                     [tz * x - ty * w, tz * y + tx * w, F32(1) - (tx * x + ty * y)]], F32)


def test_the_sensor_pose_moves_the_decision():
    m = occupied((9, -1, -1))  # the visited cells of a point in cell (10, 0, 0)
    T = np.eye(4)
    T[:3, 3] = [10.0, 0.0, 0.0]
    assert keep(m, [0.5, 0.5, 0.5], np.inf, cloud_sensor_pose(T))[0]
    assert not keep(m, [0.5, 0.5, 0.5], np.inf)[0]


@pytest.mark.parametrize("seed", range(4))
def test_cloud_sensor_pose_is_the_first_step_of_octomap_pose(seed):
    from scipy.spatial.transform import Rotation
    rng = np.random.default_rng(seed)
    for R in list(Rotation.random(200, random_state=seed).as_matrix()) + [np.diag([1.0, -1, -1]), np.diag([-1.0, -1, 1])]:
        T = np.eye(4)
        T[:3, :3], T[:3, 3] = R, rng.uniform(-5, 5, 3)
        q, t = cloud_sensor_pose(T)
        assert q.dtype == np.float32 and t.dtype == np.float32
        assert q.view(np.uint32).tolist() == octomap_pose_steps(T)["q_eigen"].view(np.uint32).tolist()
        assert t.tolist() == T[:3, 3].astype(F32).tolist()
