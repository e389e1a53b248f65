"""ctypes binding of include/rgbdslam_b200.h + a small host-side mirror of the reference interface.

Only plumbing lives here.  Every compute call goes through the C ABI into the CUDA library; if the
library cannot be loaded the import of this module still works (so CPU-only tests can inspect the
header), but any attempt to use it raises :class:`LibraryMissingError` -- there is no CPU fallback.
"""
from __future__ import annotations

import ctypes as C
import re
from pathlib import Path

import numpy as np

from .build import library_path

MAX_MATCHES_CAP = 512


class LibraryMissingError(RuntimeError):
    pass


class B200Error(RuntimeError):
    pass


class KeyPoint(C.Structure):  # == cv::KeyPoint
    _fields_ = [("x", C.c_float), ("y", C.c_float), ("size", C.c_float), ("angle", C.c_float),
                ("response", C.c_float), ("octave", C.c_int32), ("class_id", C.c_int32)]


class DMatch(C.Structure):  # == cv::DMatch
    _fields_ = [("queryIdx", C.c_int32), ("trainIdx", C.c_int32), ("imgIdx", C.c_int32), ("distance", C.c_float)]


class Params(C.Structure):
    _fields_ = [
        ("max_keypoints", C.c_int32), ("min_matches", C.c_int32), ("max_matches", C.c_int32),
        ("ransac_iterations", C.c_int32), ("max_dist_for_inliers", C.c_double), ("sigma_depth", C.c_double),
        ("depth_cov_z0", C.c_double), ("depth_scaling_factor", C.c_double),
        ("detector_grid_resolution", C.c_int32), ("adjuster_max_iterations", C.c_int32),
        ("min_translation_meter", C.c_double), ("min_rotation_degree", C.c_double),
        ("max_translation_meter", C.c_double), ("max_rotation_degree", C.c_double),
        ("nn_distance_ratio", C.c_double), ("use_root_sift", C.c_int32), ("g2o_transformation_refinement", C.c_int32), ("observability_threshold", C.c_double), ("emm_skip_step", C.c_int32),
        ("cloud_creation_skip_step", C.c_int32), ("minimum_depth", C.c_float),
        ("use_feature_min_depth", C.c_uint8), ("allow_features_without_depth_", C.c_uint8),
        ("feature_detector_type", C.c_uint8), ("reserved_", C.c_uint8),
    ]


DETECTOR_ORB, DETECTOR_FAST = 0, 1  # Params.feature_detector_type (RGBDSLAM_B200_DETECTOR_*)
# flags of rgbdslam_b200_nodes_create_ex / _sharded (RGBDSLAM_B200_*)
MASK_FROM_DEPTH, VISUAL_RGB, CLOUD_XYZRGB, CLOUD_XYZ, MASK_FROM_CLOUD, KEEP_CLOUD = 1, 2, 4, 8, 16, 128
DEPTH_U16, VISUAL_BAYER_GR = 256, 512
STORE_CLOUD, ENCODING_RGB = 4096, 8192
# records of rgbdslam_b200_node_download_cloud / render_cloud: pcl::PointXYZRGB (32 bytes) and pcl::PointXYZ (16 bytes, colour
# word in data[3]); the colour word holds b, g, r, a bytes
POINT32_DTYPE = np.dtype([("x", "<f4"), ("y", "<f4"), ("z", "<f4"), ("w", "<u4"), ("rgb", "<u4"), ("pad", "<u4", (3,))])
POINT16_DTYPE = np.dtype([("x", "<f4"), ("y", "<f4"), ("z", "<f4"), ("w", "<u4")])


def _is_u16(a) -> bool:
    """a uint16 numpy array or torch tensor"""
    return str(a.dtype) in ("uint16", "torch.uint16")


def node_input_flags(gray_shape, depth_shape, mask_from_depth=False, mask_from_cloud=False, keep_cloud=False,
                     depth_u16=False, bayer=False, store_cloud=False, encoding_rgb=False) -> int:
    """The nodes_create flags the array shapes select: gray (F,H,W) or (F,H,W,3) colour; depth (F,H,W) depth image, or an
    organised cloud (F,H,W,8) of PointXYZRGB / (F,H,W,4) of PointXYZ as float32.  keep_cloud: the nodes keep their cloud
    for the environment measurement model (cloud input only).  depth_u16: the depth image is uint16 millimetres; bayer: gray
    (F,H,W) holds bayer_grbg8 mosaics.  store_cloud: the nodes keep their colour cloud (pc_col) for the map; encoding_rgb: its
    colour reads channel 0 as red (encoding_bgr = false)."""
    flags = (MASK_FROM_DEPTH if mask_from_depth else 0) | (MASK_FROM_CLOUD if mask_from_cloud else 0)
    flags |= (STORE_CLOUD if store_cloud else 0) | (ENCODING_RGB if encoding_rgb else 0)
    flags |= (KEEP_CLOUD if keep_cloud else 0) | (DEPTH_U16 if depth_u16 else 0) | (VISUAL_BAYER_GR if bayer else 0)
    if len(gray_shape) == 4:
        if gray_shape[3] != 3:
            raise ValueError(f"gray must be (F,H,W) or (F,H,W,3), got {tuple(gray_shape)}")
        flags |= VISUAL_RGB
    if len(depth_shape) == 4:
        if depth_shape[3] not in (4, 8):
            raise ValueError(f"depth must be (F,H,W), (F,H,W,4) or (F,H,W,8), got {tuple(depth_shape)}")
        flags |= CLOUD_XYZRGB if depth_shape[3] == 8 else CLOUD_XYZ
    if tuple(gray_shape[:3]) != tuple(depth_shape[:3]):
        raise ValueError(f"gray {tuple(gray_shape)} and depth {tuple(depth_shape)} differ in frames or image size")
    return flags


def resized_input_flags(gray_shape, depth_shape, **kw) -> int:
    """node_input_flags for nodes_create_resized: gray (F,H,W) or (F,H,W,3), depth (F,dh,dw) a depth image of any size with
    the same frame count (clouds of another size than the visual are not taken)."""
    if len(depth_shape) != 3:
        raise ValueError(f"depth must be a depth image (F,dh,dw) (clouds of another size are not taken), got {tuple(depth_shape)}")
    if depth_shape[0] != gray_shape[0]:
        raise ValueError(f"gray {tuple(gray_shape)} and depth {tuple(depth_shape)} differ in frames")
    return node_input_flags(gray_shape, tuple(gray_shape[:3]), **kw)


class PairResult(C.Structure):
    _fields_ = [
        ("id1", C.c_int32), ("id2", C.c_int32), ("n_all_matches", C.c_int32), ("n_inliers", C.c_int32),
        ("rmse", C.c_float), ("valid_iterations", C.c_int32), ("ransac_trafo", C.c_float * 16),
        ("info_scale", C.c_double), ("used_identity", C.c_int32), ("inlier_points", C.c_uint32), ("outlier_points", C.c_uint32),
        ("occluded_points", C.c_uint32), ("all_points", C.c_uint32), ("reserved_", C.c_int32),
    ]


DMATCH_DTYPE = np.dtype([("queryIdx", "<i4"), ("trainIdx", "<i4"), ("imgIdx", "<i4"), ("distance", "<f4")])
KEYPOINT_DTYPE = np.dtype([("x", "<f4"), ("y", "<f4"), ("size", "<f4"), ("angle", "<f4"), ("response", "<f4"),
                           ("octave", "<i4"), ("class_id", "<i4")])
PAIR_RESULT_DTYPE = np.dtype([
    ("id1", "<i4"), ("id2", "<i4"), ("n_all_matches", "<i4"), ("n_inliers", "<i4"), ("rmse", "<f4"),
    ("valid_iterations", "<i4"), ("ransac_trafo", "<f4", (16,)), ("info_scale", "<f8"), ("used_identity", "<i4"),
    ("inlier_points", "<u4"), ("outlier_points", "<u4"), ("occluded_points", "<u4"), ("all_points", "<u4"), ("reserved_", "<i4"),
])
class IcpResult(C.Structure):  # == rgbdslam_b200_icp_result (include/rgbdslam_b200/icp.h)
    _fields_ = [("T", C.c_float * 16), ("converged", C.c_int32), ("iterations", C.c_int32), ("criterion", C.c_int32),
                ("n_source", C.c_int32), ("n_target", C.c_int32), ("n_correspondences", C.c_int32), ("mse", C.c_double)]


ICP_RESULT_DTYPE = np.dtype([("T", "<f4", (16,)), ("converged", "<i4"), ("iterations", "<i4"), ("criterion", "<i4"),
                             ("n_source", "<i4"), ("n_target", "<i4"), ("n_correspondences", "<i4"), ("mse", "<f8")],
                            align=True)
assert ICP_RESULT_DTYPE.itemsize == C.sizeof(IcpResult) == 96
ICP_METHODS = {"icp": 0, "icp_nl": 1}  # RGBDSLAM_B200_ICP_METHOD_* (include/rgbdslam_b200/icp.h)
assert PAIR_RESULT_DTYPE.itemsize == C.sizeof(PairResult) == 120
assert DMATCH_DTYPE.itemsize == C.sizeof(DMatch) == 16
assert KEYPOINT_DTYPE.itemsize == C.sizeof(KeyPoint) == 28

class OctomapParams(C.Structure):  # == rgbdslam_b200_octomap_params (include/rgbdslam_b200/octomap.h)
    _fields_ = [("resolution", C.c_double), ("prob_hit", C.c_double), ("prob_miss", C.c_double), ("clamping_min", C.c_double),
                ("clamping_max", C.c_double)]


def _eigen_quaternion(T):
    """Eigen's Quaternion(Matrix3f) of T's rotation cast to float: (q (x, y, z, w) float32, branch) -- the trace as its unrolled
    reduction m00 + (m11 + m22), then the positive-trace (branch -1) or the largest-diagonal branch (strict >), in float."""
    f = np.float32
    R = np.asarray(T, np.float64)[:3, :3].astype(f)
    tr = R[0, 0] + (R[1, 1] + R[2, 2])
    q = np.zeros(4, f)  # x, y, z, w
    if tr > f(0):
        eb = -1
        t = np.sqrt(tr + f(1))
        q[3] = f(0.5) * t
        t = f(0.5) / t
        q[0], q[1], q[2] = (R[2, 1] - R[1, 2]) * t, (R[0, 2] - R[2, 0]) * t, (R[1, 0] - R[0, 1]) * t
    else:
        i = 0
        if R[1, 1] > R[0, 0]:
            i = 1
        if R[2, 2] > R[i, i]:
            i = 2
        eb = i
        j, k = (i + 1) % 3, (i + 2) % 3
        t = np.sqrt(((R[i, i] - R[j, j]) - R[k, k]) + f(1))
        q[i] = f(0.5) * t
        t = f(0.5) / t
        q[3] = (R[k, j] - R[j, k]) * t
        q[j] = (R[j, i] + R[i, j]) * t
        q[k] = (R[k, i] + R[i, k]) * t
    return q, eb


def cloud_sensor_pose(T) -> tuple[np.ndarray, np.ndarray]:
    """What GraphManager::updateCloudOrigin stores in a node's cloud for a VertexSE3 estimate T (4 x 4 or 3 x 4, double):
    sensor_orientation_, Eigen's Quaternionf of the rotation cast to float (x, y, z, w), and sensor_origin_, the translation
    as float -- the sensor pose occupancyFilter applies (Frontend.octomap_filter_clouds), and the first step of octomap_pose."""
    return _eigen_quaternion(T)[0], np.asarray(T, np.float64)[:3, 3].astype(np.float32)


def octomap_pose_steps(T) -> dict:
    """The pose chain of saveOctomap step by step (see octomap_pose): q_eigen (x, y, z, w, float32) and eigen_branch of
    Eigen's Quaternion(Matrix3f), M (the tf::Matrix3x3 of setRotation, float64), q_tf and tf_branch of its getRotation,
    and T, the float 3 x 4.  A branch is -1 for the positive-trace formula, else the index of the diagonal entry used."""
    f, d = np.float32, np.float64
    T = np.asarray(T, d)
    q, eb = _eigen_quaternion(T)
    # tf::Matrix3x3::setRotation in double
    x, y, z, w = (d(v) for v in q)
    s = d(2.0) / (((x * x + y * y) + z * z) + w * w)
    xs, ys, zs = x * s, y * s, z * s
    wx, wy, wz = w * xs, w * ys, w * zs
    xx, xy, xz = x * xs, x * ys, x * zs
    yy, yz, zz = y * ys, y * zs, z * zs
    M = np.array([[d(1.0) - (yy + zz), xy - wz, xz + wy], [xy + wz, d(1.0) - (xx + zz), yz - wx],
                  [xz - wy, yz + wx, d(1.0) - (xx + yy)]])
    # tf::Matrix3x3::getRotation (strict <, in double)
    tr = (M[0, 0] + M[1, 1]) + M[2, 2]
    g = np.zeros(4, d)
    if tr > 0.0:
        tb = -1
        sq = np.sqrt(tr + 1.0)
        g[3] = sq * 0.5
        sq = 0.5 / sq
        g[0], g[1], g[2] = (M[2, 1] - M[1, 2]) * sq, (M[0, 2] - M[2, 0]) * sq, (M[1, 0] - M[0, 1]) * sq
    else:
        i = (2 if M[1, 1] < M[2, 2] else 1) if M[0, 0] < M[1, 1] else (2 if M[0, 0] < M[2, 2] else 0)
        tb = i
        j, k = (i + 1) % 3, (i + 2) % 3
        sq = np.sqrt(((M[i, i] - M[j, j]) - M[k, k]) + 1.0)
        g[i] = sq * 0.5
        sq = 0.5 / sq
        g[3] = (M[k, j] - M[j, k]) * sq
        g[j] = (M[j, i] + M[i, j]) * sq
        g[k] = (M[k, i] + M[i, k]) * sq
    # Quaternionf::toRotationMatrix in float
    x, y, z, w = (f(v) for v in g)
    tx, ty, tz = f(2) * x, f(2) * y, f(2) * z
    twx, twy, twz = tx * w, ty * w, tz * w
    txx, txy, txz = tx * x, ty * x, tz * x
    tyy, tyz, tzz = ty * y, tz * y, tz * z
    out = np.zeros((3, 4), f)
    out[:, :3] = [[f(1) - (tyy + tzz), txy - twz, txz + twy], [txy + twz, f(1) - (txx + tzz), tyz - twx],
                  [txz - twy, tyz + twx, f(1) - (txx + tyy)]]
    out[:, 3] = T[:3, 3].astype(f)
    return dict(q_eigen=q, eigen_branch=eb, M=M, q_tf=g, tf_branch=tb, T=out)


def octomap_pose(T) -> np.ndarray:
    """The float 3 x 4 (row-major, node -> map) that the reference's saveOctomap applies to a node whose VertexSE3 estimate is
    T (4 x 4 or 3 x 4, double): updateCloudOrigin stores the rotation cast to float as an Eigen Quaternionf and the translation
    as float; insertCloudCallback widens the quaternion to tf (double), builds a tf::Matrix3x3 from it (setRotation) and
    pcl_ros::transformPointCloud takes it back with getRotation, narrows it to a Quaternionf and uses toRotationMatrix.  The
    ray origin is the translation column.  Every operation is one numpy operation on float32 or float64 scalars; the C++ shim's
    octomapPose (include/rgbdslam_b200/graph_manager.hpp) is the same chain in native arithmetic."""
    return octomap_pose_steps(T)["T"]


_lib = None


def header_path() -> Path:
    return Path(__file__).resolve().parent.parent / "include" / "rgbdslam_b200.h"


def declared_symbols() -> list[str]:
    """All function names declared in include/*.h (used by the CPU-only export test)."""
    names = []
    for h in sorted(header_path().parent.glob("*.h")):
        txt = re.sub(r"/\*.*?\*/", "", h.read_text(), flags=re.S)
        names += re.findall(r"\b(rgbdslam_b200_[a-z0-9_]+)\s*\(", txt)
    return sorted(set(names))


def load_library(path: str | Path | None = None) -> C.CDLL:
    """dlopen the CUDA library and set up prototypes.  Raises LibraryMissingError if it is absent."""
    global _lib
    if _lib is not None and path is None:
        return _lib
    p = Path(path) if path else library_path()
    if not p.exists():
        raise LibraryMissingError(
            f"{p} not found: build it with `python -c 'import __graft_entry__ as g; g.build()'` "
            "(nvcc, sm_90a).  rgbdslam_v2_b200 has no CPU fallback.")
    lib = C.CDLL(str(p))
    u64, i64, i32p = C.c_uint64, C.c_int64, C.POINTER(C.c_int32)
    vp = C.c_void_p
    lib.rgbdslam_b200_default_params.argtypes = [C.POINTER(Params)]
    lib.rgbdslam_b200_default_params.restype = None
    lib.rgbdslam_b200_init.argtypes = [C.c_int, C.POINTER(Params)]
    lib.rgbdslam_b200_shutdown.argtypes = []
    lib.rgbdslam_b200_get_params.argtypes = [C.POINTER(Params)]
    lib.rgbdslam_b200_set_stream.argtypes = [vp]
    lib.rgbdslam_b200_synchronize.argtypes = []
    lib.rgbdslam_b200_last_error.argtypes = []
    lib.rgbdslam_b200_last_error.restype = C.c_char_p
    lib.rgbdslam_b200_launch_count.argtypes = []
    lib.rgbdslam_b200_launch_count.restype = i64
    lib.rgbdslam_b200_depth_cov_z0.argtypes = []
    lib.rgbdslam_b200_depth_cov_z0.restype = C.c_double
    lib.rgbdslam_b200_brute_force_orb.argtypes = [vp, C.c_int, vp, C.c_int, vp, vp]
    lib.rgbdslam_b200_node_create_from_features.argtypes = [C.c_int32, vp, vp, C.c_int, C.POINTER(u64)]
    lib.rgbdslam_b200_node_num_features.argtypes = [u64, C.POINTER(C.c_int)]
    lib.rgbdslam_b200_node_download.argtypes = [u64, vp, vp]
    lib.rgbdslam_b200_node_destroy.argtypes = [u64]
    lib.rgbdslam_b200_match_pairs.argtypes = [vp, vp, C.c_int, u64, i64, vp, vp, vp]
    lib.rgbdslam_b200_match_pairs_host.argtypes = [vp, vp, vp, vp, vp, vp, vp, vp, C.c_int, u64, i64, vp, vp, vp]
    lib.rgbdslam_b200_match_pairs_submit.argtypes = [C.c_int, vp, vp, C.c_int, u64, i64, vp, vp, vp]
    lib.rgbdslam_b200_match_pairs_host_submit.argtypes = [C.c_int, vp, vp, vp, vp, vp, vp, vp, vp, C.c_int, u64, i64, vp, vp, vp]
    lib.rgbdslam_b200_match_pairs_wait.argtypes = [C.c_int]
    lib.rgbdslam_b200_set_hamming_path.argtypes = [C.c_int]
    lib.rgbdslam_b200_set_sift_matcher.argtypes = [C.c_int]
    lib.rgbdslam_b200_node_set_keypoints.argtypes = [u64, vp]
    lib.rgbdslam_b200_node_set_depth.argtypes = [u64, vp, C.c_int, C.c_int, vp]
    lib.rgbdslam_b200_observation_likelihood.argtypes = [u64, u64, vp, vp]
    lib.rgbdslam_b200_detector_create.argtypes = [C.POINTER(u64)]
    lib.rgbdslam_b200_detector_destroy.argtypes = [u64]
    lib.rgbdslam_b200_detector_thresholds.argtypes = [u64, vp, C.c_int]
    lib.rgbdslam_b200_orb_detect.argtypes = [u64, vp, vp, C.c_int, C.c_int, vp, C.c_int, C.POINTER(C.c_int)]
    lib.rgbdslam_b200_orb_compute.argtypes = [vp, C.c_int, C.c_int, vp, C.c_int, vp, vp, C.POINTER(C.c_int)]
    lib.rgbdslam_b200_nodes_create.argtypes = [u64, C.c_int, vp, vp, vp, C.c_int, C.c_int, vp, vp, vp, vp]
    lib.rgbdslam_b200_nodes_create_ex.argtypes = [u64, C.c_int, vp, vp, vp, C.c_int, C.c_int, vp, vp, C.c_int, vp, vp]
    lib.rgbdslam_b200_nodes_create_sharded.argtypes = [u64, u64, C.c_int, vp, vp, vp, C.c_int, C.c_int, vp, vp, C.c_int, vp, vp]
    lib.rgbdslam_b200_nodes_create_resized.argtypes = [u64, C.c_int, vp, vp, C.c_int, C.c_int, vp, C.c_int, C.c_int, vp, vp, C.c_int,
                                                       vp, vp]
    lib.rgbdslam_b200_nodes_create_sharded_resized.argtypes = [u64, u64, C.c_int, vp, vp, C.c_int, C.c_int, vp, C.c_int, C.c_int, vp,
                                                               vp, C.c_int, vp, vp]
    lib.rgbdslam_b200_node_download_keypoints.argtypes = [u64, vp]
    lib.rgbdslam_b200_node_download_cloud.argtypes = [u64, C.c_int, vp, C.POINTER(C.c_int), C.POINTER(C.c_int)]
    lib.rgbdslam_b200_render_cloud.argtypes = [C.c_int, vp, vp, C.c_double, C.c_int, C.c_int, vp, i64, C.POINTER(i64), vp]
    lib.rgbdslam_b200_reduce_clouds.argtypes = [C.c_int, vp, C.c_double, vp]
    lib.rgbdslam_b200_transform_clouds.argtypes = [C.c_int, vp, vp]
    lib.rgbdslam_b200_icp_align.argtypes = [C.c_int, vp, vp, C.c_int, vp]
    lib.rgbdslam_b200_icp_align_ex.argtypes = [C.c_int, vp, vp, C.c_int, C.c_int, vp]
    lib.rgbdslam_b200_octomap_default_params.argtypes = [C.POINTER(OctomapParams)]
    lib.rgbdslam_b200_octomap_default_params.restype = None
    lib.rgbdslam_b200_octomap_create.argtypes = [C.POINTER(OctomapParams), C.POINTER(u64)]
    lib.rgbdslam_b200_octomap_insert.argtypes = [u64, C.c_int, vp, vp, C.c_double]
    lib.rgbdslam_b200_octomap_write.argtypes = [u64, vp, i64, C.POINTER(i64)]
    lib.rgbdslam_b200_octomap_stats.argtypes = [u64, C.POINTER(i64), C.POINTER(i64)]
    lib.rgbdslam_b200_octomap_clear.argtypes = [u64]
    lib.rgbdslam_b200_octomap_destroy.argtypes = [u64]
    lib.rgbdslam_b200_node_clear_cloud.argtypes = [u64]
    lib.rgbdslam_b200_octomap_filter_clouds.argtypes = [u64, C.c_int, vp, vp, C.c_double, vp]
    lib.rgbdslam_b200_orb_debug_plane.argtypes = [C.c_int, C.c_int, C.c_int, vp, C.c_int, C.POINTER(C.c_int), C.POINTER(C.c_int)]
    lib.rgbdslam_b200_orb_debug_candidates.argtypes = [C.c_int, vp, vp, C.c_int, C.POINTER(C.c_int), C.POINTER(C.c_int)]
    lib.rgbdslam_b200_node_create_from_sift.argtypes = [C.c_int32, vp, vp, C.c_int, C.POINTER(u64)]
    lib.rgbdslam_b200_knn2_l2.argtypes = [vp, C.c_int, vp, C.c_int, vp, vp]
    lib.rgbdslam_b200_comm_unique_id.argtypes = [vp]
    lib.rgbdslam_b200_comm_init.argtypes = [C.c_int, C.c_int, vp, C.POINTER(u64)]
    lib.rgbdslam_b200_comm_destroy.argtypes = [u64]
    lib.rgbdslam_b200_allgather_edges.argtypes = [u64, vp, C.c_int, vp]
    lib.rgbdslam_b200_allgather_slot_edges.argtypes = [u64, C.c_int, C.c_int, vp]
    lib.rgbdslam_b200_posegraph_optimize.argtypes = [C.c_int, vp, vp, C.c_int, vp, vp, vp, C.c_double, C.c_double,
                                                     C.POINTER(C.c_double), C.POINTER(C.c_int), C.POINTER(C.c_int)]
    lib.rgbdslam_b200_posegraph_reserve.argtypes = [C.c_int, C.c_int]
    lib.rgbdslam_b200_graph_from_pairs.argtypes = [C.c_int, C.c_int, vp, vp, C.c_double, vp, vp, vp, vp, vp, C.POINTER(C.c_int), C.POINTER(C.c_int)]
    lib.rgbdslam_b200_posegraph_chi2.argtypes = [C.c_int, vp, C.c_int, vp, vp, vp, C.c_double, C.POINTER(C.c_double), vp]
    lib.rgbdslam_b200_landmark_ba.argtypes = [C.c_int, vp, vp, C.c_int, vp, C.c_int, vp, vp, vp, vp, vp, C.c_int, vp, vp, vp, C.c_int,
                                              C.c_double, C.POINTER(C.c_double), C.POINTER(C.c_double), C.POINTER(C.c_int),
                                              C.POINTER(C.c_int)]
    lib.rgbdslam_b200_last_timing.argtypes = [C.POINTER(C.c_float), C.POINTER(C.c_float)]
    lib.rgbdslam_b200_slot_stage_times.argtypes = [C.c_int, vp]
    lib.rgbdslam_b200_timeline_epoch.argtypes = []
    lib.rgbdslam_b200_slot_timeline.argtypes = [C.c_int, vp]
    lib.rgbdslam_b200_last_timing_slot.argtypes = [C.c_int, C.POINTER(C.c_float), C.POINTER(C.c_float)]
    for name in declared_symbols():
        fn = getattr(lib, name)  # AttributeError if the .so does not export a declared symbol
        if fn.restype is C.c_int and name not in ("rgbdslam_b200_default_params",):
            fn.restype = C.c_int
    if path is None:
        _lib = lib
    return lib


def graph_from_pairs(pairs: np.ndarray, results: np.ndarray, n_frames: int, dt: float = 1.0 / 30.0) -> dict:
    """rgbdslam_b200_graph_from_pairs (host glue, runs without a GPU): same dict as pipeline.build_graph."""
    lib = load_library()
    pairs = np.ascontiguousarray(pairs, np.int32).reshape(-1, 2)
    results = np.ascontiguousarray(results, PAIR_RESULT_DTYPE)
    cap = len(pairs) + n_frames
    poses = np.zeros((n_frames, 7)); fixed = np.zeros(n_frames, np.uint8)
    ij = np.zeros((cap, 2), np.int32); meas = np.zeros((cap, 7)); info = np.zeros((cap, 36))
    ne, nc = C.c_int(), C.c_int()
    rc = lib.rgbdslam_b200_graph_from_pairs(n_frames, len(pairs), _ptr(pairs), _ptr(results), dt, _ptr(poses), _ptr(fixed), _ptr(ij),
                                            _ptr(meas), _ptr(info), C.byref(ne), C.byref(nc))
    if rc != 0:
        raise B200Error(f"rgbdslam_b200 error {rc}: {lib.rgbdslam_b200_last_error().decode()}")
    n = ne.value
    return dict(init=poses, fixed=fixed, ij=ij[:n].copy(), meas=meas[:n].copy(), info=info[:n].copy(), n_valid_edges=n - nc.value,
                n_const_edges=nc.value)


def default_params() -> Params:
    p = Params()
    load_library().rgbdslam_b200_default_params(C.byref(p))
    return p


def _ptr(a):
    if a is None:
        return None
    if isinstance(a, np.ndarray):
        assert a.flags.c_contiguous
        return a.ctypes.data
    if hasattr(a, "data_ptr"):  # torch tensor (pinned host memory for the e2e path)
        assert a.is_contiguous()
        return a.data_ptr()
    raise TypeError(type(a))


class Frontend:
    """Host-side mirror of the reference's front-end interface for this path.

    ``Frontend.match_node_pairs`` == ``Node::matchNodePair`` (node.cpp:1305) for a batch of pairs,
    ``Frontend.brute_force_search_orb`` == ``bruteForceSearchORB`` (features.cpp:168) per query row.
    """

    def __init__(self, device: int = 0, params: Params | None = None):
        self.lib = load_library()
        self.params = params if params is not None else default_params()
        self._check(self.lib.rgbdslam_b200_init(device, C.byref(self.params)))
        self._nodes: list[int] = []

    # -- helpers -----------------------------------------------------------
    def _check(self, rc: int):
        if rc != 0:
            raise B200Error(f"rgbdslam_b200 error {rc}: {self.lib.rgbdslam_b200_last_error().decode()}")

    def set_stream(self, stream_ptr: int | None):
        self._check(self.lib.rgbdslam_b200_set_stream(stream_ptr))

    def set_hamming_path(self, path: int):
        """1 = wgmma int8 tensor-core GEMM (default), 0 = SIMT popcount."""
        self._check(self.lib.rgbdslam_b200_set_hamming_path(path))

    def set_sift_matcher(self, matcher: int):
        """0 = exact 2-NN ratio matcher (FLANN branch), 1 = SiftGPU matcher; applies to SIFT nodes created afterwards"""
        self._check(self.lib.rgbdslam_b200_set_sift_matcher(matcher))

    def synchronize(self):
        self._check(self.lib.rgbdslam_b200_synchronize())

    @property
    def launch_count(self) -> int:
        return int(self.lib.rgbdslam_b200_launch_count())

    @property
    def depth_cov_z0(self) -> float:
        return float(self.lib.rgbdslam_b200_depth_cov_z0())

    def stage_times(self, slot: int = 0) -> dict:
        t = np.zeros(6, np.float32)
        self._check(self.lib.rgbdslam_b200_slot_stage_times(slot, _ptr(t)))
        return dict(zip(("h2d", "expand", "hamming", "select_ransac", "d2h", "total"), (float(v) for v in t)))

    def timeline_epoch(self) -> None:
        self._check(self.lib.rgbdslam_b200_timeline_epoch())

    def slot_timeline(self, slot: int) -> np.ndarray:
        """device times (ms since timeline_epoch) of submit, h2d done, expand done, match start, match end, ransac end, d2h done"""
        t = np.zeros(7, np.float32)
        self._check(self.lib.rgbdslam_b200_slot_timeline(slot, _ptr(t)))
        return t

    def last_timing(self, slot: int = 0) -> tuple[float, float]:
        a, b = C.c_float(), C.c_float()
        self._check(self.lib.rgbdslam_b200_last_timing_slot(slot, C.byref(a), C.byref(b)))
        return a.value, b.value

    # -- bruteForceSearchORB ------------------------------------------------
    def brute_force_search_orb(self, q: np.ndarray, t: np.ndarray):
        q = np.ascontiguousarray(q, dtype=np.uint8).reshape(-1, 32)
        t = np.ascontiguousarray(t, dtype=np.uint8).reshape(-1, 32)
        idx = np.empty(len(q), np.int32)
        hd = np.empty(len(q), np.int32)
        self._check(self.lib.rgbdslam_b200_brute_force_orb(_ptr(q), len(q), _ptr(t), len(t), _ptr(idx), _ptr(hd)))
        return hd, idx

    # -- nodes ----------------------------------------------------------------
    def node_from_features(self, node_id: int, desc: np.ndarray, xyz1: np.ndarray) -> int:
        desc = np.ascontiguousarray(desc, dtype=np.uint8).reshape(-1, 32)
        xyz1 = np.ascontiguousarray(xyz1, dtype=np.float32).reshape(-1, 4)
        assert len(desc) == len(xyz1)
        h = C.c_uint64()
        self._check(self.lib.rgbdslam_b200_node_create_from_features(node_id, _ptr(desc), _ptr(xyz1), len(desc), C.byref(h)))
        self._nodes.append(h.value)
        return h.value

    def node_from_sift(self, node_id: int, desc128: np.ndarray, xyz1: np.ndarray) -> int:
        desc128 = np.ascontiguousarray(desc128, dtype=np.float32).reshape(-1, 128)
        xyz1 = np.ascontiguousarray(xyz1, dtype=np.float32).reshape(-1, 4)
        h = C.c_uint64()
        self._check(self.lib.rgbdslam_b200_node_create_from_sift(node_id, _ptr(desc128), _ptr(xyz1), len(desc128), C.byref(h)))
        self._nodes.append(h.value)
        return h.value

    def knn2_l2(self, q: np.ndarray, t: np.ndarray):
        q = np.ascontiguousarray(q, np.float32).reshape(-1, 128)
        t = np.ascontiguousarray(t, np.float32).reshape(-1, 128)
        idx = np.zeros((len(q), 2), np.int32)
        d = np.zeros((len(q), 2), np.float32)
        self._check(self.lib.rgbdslam_b200_knn2_l2(_ptr(q), len(q), _ptr(t), len(t), _ptr(idx), _ptr(d)))
        return idx, d

    def node_set_keypoints(self, h: int, kp: np.ndarray):
        """kp: KEYPOINT_DTYPE array (only pt.x / pt.y are used) with one entry per feature of the node"""
        k = np.ascontiguousarray(kp, dtype=KEYPOINT_DTYPE)
        if len(k) != self.node_num_features(h):
            raise ValueError("one keypoint per feature")
        self._check(self.lib.rgbdslam_b200_node_set_keypoints(C.c_uint64(int(h)), _ptr(k)))

    def node_set_depth(self, h: int, depth_m: np.ndarray, K4):
        d = np.ascontiguousarray(depth_m, np.float32)
        k = np.ascontiguousarray(K4, np.float32)
        self._check(self.lib.rgbdslam_b200_node_set_depth(C.c_uint64(int(h)), _ptr(d), d.shape[1], d.shape[0], _ptr(k)))

    def observation_likelihood(self, newer: int, older: int, T4x4) -> np.ndarray:
        """pairwiseObservationLikelihood for an explicit 4x4 transformation (newer -> older): inlier, outlier, occluded, all"""
        T = np.ascontiguousarray(np.asarray(T4x4, np.float32).T)  # column-major Matrix4f
        out = np.zeros(4, np.uint32)
        self._check(self.lib.rgbdslam_b200_observation_likelihood(C.c_uint64(int(newer)), C.c_uint64(int(older)), _ptr(T), _ptr(out)))
        return out

    def node_num_features(self, h: int) -> int:
        n = C.c_int()
        self._check(self.lib.rgbdslam_b200_node_num_features(h, C.byref(n)))
        return n.value

    def node_download(self, h: int):
        n = self.node_num_features(h)
        desc = np.empty((n, 32), np.uint8)
        xyz = np.empty((n, 4), np.float32)
        self._check(self.lib.rgbdslam_b200_node_download(h, _ptr(desc), _ptr(xyz)))
        return desc, xyz

    def node_destroy(self, h: int):
        self._check(self.lib.rgbdslam_b200_node_destroy(h))
        if h in self._nodes:
            self._nodes.remove(h)

    # -- matchNodePair ----------------------------------------------------------
    def _alloc_out(self, npairs, want_matches):
        res = np.zeros(npairs, PAIR_RESULT_DTYPE)
        mm = self.params.max_matches
        allm = np.zeros((npairs, mm), DMATCH_DTYPE) if want_matches else None
        inl = np.zeros((npairs, mm), DMATCH_DTYPE) if want_matches else None
        return res, allm, inl

    def match_node_pairs(self, newer: list[int], older: list[int], seed: int = 0, first_pair_index: int = 0,
                         want_matches: bool = True, out=None):
        npairs = len(newer)
        a = np.asarray(newer, dtype=np.uint64)
        b = np.asarray(older, dtype=np.uint64)
        res, allm, inl = out if out is not None else self._alloc_out(npairs, want_matches)
        self._check(self.lib.rgbdslam_b200_match_pairs(_ptr(a), _ptr(b), npairs, seed, first_pair_index,
                                                       _ptr(res), _ptr(allm), _ptr(inl)))
        return res, allm, inl

    def submit_node_pairs(self, slot: int, newer_arr: np.ndarray, older_arr: np.ndarray, out, seed: int = 0,
                          first_pair_index: int = 0):
        """Asynchronous match_node_pairs on pipeline slot `slot`; newer_arr / older_arr: uint64 handle arrays that stay
        alive until wait_slot(); out = (results, all_matches | None, inlier_matches | None) host arrays."""
        res, allm, inl = out
        self._check(self.lib.rgbdslam_b200_match_pairs_submit(slot, _ptr(newer_arr), _ptr(older_arr), len(newer_arr), seed,
                                                              first_pair_index, _ptr(res), _ptr(allm), _ptr(inl)))

    def submit_pairs_host(self, slot: int, desc_newer, xyz_newer, n_newer, desc_older, xyz_older, n_older, id_newer, id_older,
                          out, seed: int = 0, first_pair_index: int = 0):
        res, allm, inl = out
        self._check(self.lib.rgbdslam_b200_match_pairs_host_submit(
            slot, _ptr(desc_newer), _ptr(xyz_newer), _ptr(n_newer), _ptr(desc_older), _ptr(xyz_older), _ptr(n_older),
            _ptr(id_newer), _ptr(id_older), len(n_newer), seed, first_pair_index, _ptr(res), _ptr(allm), _ptr(inl)))

    def wait_slot(self, slot: int):
        self._check(self.lib.rgbdslam_b200_match_pairs_wait(slot))

    def match_pairs_host(self, desc_newer, xyz_newer, n_newer, desc_older, xyz_older, n_older, id_newer=None,
                         id_older=None, seed: int = 0, first_pair_index: int = 0, want_matches: bool = True, out=None):
        """Host feature buffers in (numpy or pinned torch tensors), host results out."""
        n_newer = np.ascontiguousarray(n_newer, dtype=np.int32)
        n_older = np.ascontiguousarray(n_older, dtype=np.int32)
        npairs = len(n_newer)
        idn = None if id_newer is None else np.ascontiguousarray(id_newer, dtype=np.int32)
        ido = None if id_older is None else np.ascontiguousarray(id_older, dtype=np.int32)
        res, allm, inl = out if out is not None else self._alloc_out(npairs, want_matches)
        self._check(self.lib.rgbdslam_b200_match_pairs_host(
            _ptr(desc_newer), _ptr(xyz_newer), _ptr(n_newer), _ptr(desc_older), _ptr(xyz_older), _ptr(n_older),
            _ptr(idn), _ptr(ido), npairs, seed, first_pair_index, _ptr(res), _ptr(allm), _ptr(inl)))
        return res, allm, inl

    # -- Node construction from images (node.cpp:101-240) -------------------------------
    def detector_create(self) -> int:
        h = C.c_uint64()
        self._check(self.lib.rgbdslam_b200_detector_create(C.byref(h)))
        return h.value

    def detector_destroy(self, det: int):
        self._check(self.lib.rgbdslam_b200_detector_destroy(det))

    def detector_thresholds(self, det: int, values=None) -> np.ndarray:
        t = np.zeros(16, np.float64) if values is None else np.ascontiguousarray(values, np.float64)
        self._check(self.lib.rgbdslam_b200_detector_thresholds(det, _ptr(t), 0 if values is None else 1))
        return t

    def orb_detect(self, det: int, gray: np.ndarray, mask: np.ndarray | None, capacity: int = 4096):
        gray = np.ascontiguousarray(gray, np.uint8)
        mask = None if mask is None else np.ascontiguousarray(mask, np.uint8)
        out = np.zeros(capacity, KEYPOINT_DTYPE)
        n = C.c_int()
        self._check(self.lib.rgbdslam_b200_orb_detect(det, _ptr(gray), _ptr(mask), gray.shape[1], gray.shape[0], _ptr(out),
                                                      capacity, C.byref(n)))
        return out[:min(n.value, capacity)]

    def orb_compute(self, gray: np.ndarray, kps: np.ndarray):
        gray = np.ascontiguousarray(gray, np.uint8)
        kps = np.ascontiguousarray(kps, KEYPOINT_DTYPE)
        out = np.zeros(max(len(kps), 1), KEYPOINT_DTYPE)
        desc = np.zeros((max(len(kps), 1), 32), np.uint8)
        n = C.c_int()
        self._check(self.lib.rgbdslam_b200_orb_compute(_ptr(gray), gray.shape[1], gray.shape[0], _ptr(kps), len(kps), _ptr(out),
                                                       _ptr(desc), C.byref(n)))
        return out[:n.value], desc[:n.value]

    def nodes_create(self, det: int, gray, depth, mask, K4, ids=None, mask_from_depth: bool = False, mask_from_cloud: bool = False,
                     keep_cloud: bool = False, bayer: bool = False, store_cloud: bool = False, encoding_rgb: bool = False):
        """gray [F,H,W] u8 or [F,H,W,3] colour (channel 0 = R), depth [F,H,W] f32 metres or u16 millimetres, or an organised
        cloud [F,H,W,8] (PointXYZRGB) / [F,H,W,4] (PointXYZ) f32 for the point-cloud constructor, mask [F,H,W] u8 or None ->
        (handles, n_features).  numpy arrays or pinned torch tensors (copied from asynchronously).  mask_from_depth /
        mask_from_cloud: derive the detection mask on the device (depthToCV8UC1 of the float or 16-bit depth /
        calculateDepthMask).  K4 may be None for cloud input.  keep_cloud (cloud input): the nodes keep their cloud for the
        environment measurement model, which projects into K4 (the reference's depth_camera_fx / fy / cx / cy; None = all
        zero).  bayer: gray [F,H,W] holds bayer_grbg8 mosaics, debayered on the device.  store_cloud: every node keeps its
        colour cloud (node_cloud, render_cloud); encoding_rgb: channel 0 of the visual is red (the reference default reads it
        as blue, encoding_bgr)."""
        depth_u16 = _is_u16(depth)
        if isinstance(gray, np.ndarray):
            gray = np.ascontiguousarray(gray, np.uint8)
            depth = np.ascontiguousarray(depth, np.uint16 if depth_u16 else np.float32)
            mask = None if mask is None else np.ascontiguousarray(mask, np.uint8)
        flags = node_input_flags(gray.shape, depth.shape, mask_from_depth, mask_from_cloud, keep_cloud, depth_u16, bayer, store_cloud,
                                 encoding_rgb)
        F, H, W = gray.shape[:3]
        K4 = None if K4 is None else np.ascontiguousarray(K4, np.float32)
        ids = None if ids is None else np.ascontiguousarray(ids, np.int32)
        handles = np.zeros(F, np.uint64)
        nf = np.zeros(F, np.int32)
        no_mask = mask_from_depth or mask_from_cloud
        self._check(self.lib.rgbdslam_b200_nodes_create_ex(det, F, _ptr(gray), _ptr(depth), _ptr(None if no_mask else mask), W, H,
                                                           _ptr(K4), _ptr(ids), flags, _ptr(handles), _ptr(nf)))
        self._nodes += [int(h) for h in handles]
        return [int(h) for h in handles], nf

    def nodes_create_sharded(self, det: int, comm: int, total_frames: int, gray, depth, mask, K4, ids=None,
                             mask_from_depth: bool = False, mask_from_cloud: bool = False, bayer: bool = False):
        """Frame-sharded nodes_create: gray / depth / mask hold THIS rank's frames (sharding.frame_shard); returns handles and
        feature counts of ALL total_frames nodes (every rank ends up holding every node).  Shapes and the depth dtype select
        the input as in nodes_create."""
        depth_u16 = _is_u16(depth)
        if isinstance(gray, np.ndarray):
            gray = np.ascontiguousarray(gray, np.uint8)
            depth = np.ascontiguousarray(depth, np.uint16 if depth_u16 else np.float32)
            mask = None if mask is None else np.ascontiguousarray(mask, np.uint8)
        flags = node_input_flags(gray.shape, depth.shape, mask_from_depth, mask_from_cloud, depth_u16=depth_u16, bayer=bayer)
        H, W = gray.shape[1:3]
        K4 = None if K4 is None else np.ascontiguousarray(K4, np.float32)
        ids = None if ids is None else np.ascontiguousarray(ids, np.int32)
        handles = np.zeros(total_frames, np.uint64)
        nf = np.zeros(total_frames, np.int32)
        own = gray.shape[0] > 0
        self._check(self.lib.rgbdslam_b200_nodes_create_sharded(
            det, C.c_uint64(comm), total_frames, _ptr(gray) if own else None, _ptr(depth) if own else None,
            _ptr(None if (mask_from_depth or mask_from_cloud or not own) else mask), W, H, _ptr(K4), _ptr(ids), flags, _ptr(handles),
            _ptr(nf)))
        self._nodes += [int(h) for h in handles]
        return [int(h) for h in handles], nf

    @staticmethod
    def _depth_image_inputs(gray, depth, mask):
        depth_u16 = _is_u16(depth)
        if isinstance(gray, np.ndarray):
            gray = np.ascontiguousarray(gray, np.uint8)
            depth = np.ascontiguousarray(depth, np.uint16 if depth_u16 else np.float32)
            mask = None if mask is None else np.ascontiguousarray(mask, np.uint8)
        return gray, depth, mask, depth_u16

    def nodes_create_resized(self, det: int, gray, depth, mask, K4, ids=None, mask_from_depth: bool = False, bayer: bool = False,
                             store_cloud: bool = False, encoding_rgb: bool = False):
        """nodes_create for a depth image of another size than the visual (include/rgbdslam_b200/depth_resize.h): gray [F,H,W]
        u8 or [F,H,W,3] colour, depth [F,dh,dw] f32 metres or u16 millimetres, resized on the device to H x W as the listener's
        cv::resize(INTER_NEAREST) does; mask [F,H,W] u8 or None; K4 the visual camera's.  The nodes equal nodes_create's on
        cv2.resize(depth, (W, H), interpolation=cv2.INTER_NEAREST).  Raises ValueError for cloud-shaped depth or another frame
        count."""
        gray, depth, mask, depth_u16 = self._depth_image_inputs(gray, depth, mask)
        flags = resized_input_flags(gray.shape, depth.shape, mask_from_depth=mask_from_depth, depth_u16=depth_u16, bayer=bayer,
                                    store_cloud=store_cloud, encoding_rgb=encoding_rgb)
        F, H, W = gray.shape[:3]
        dh, dw = depth.shape[1:3]
        K4 = None if K4 is None else np.ascontiguousarray(K4, np.float32)
        ids = None if ids is None else np.ascontiguousarray(ids, np.int32)
        handles = np.zeros(F, np.uint64)
        nf = np.zeros(F, np.int32)
        self._check(self.lib.rgbdslam_b200_nodes_create_resized(det, F, _ptr(gray), _ptr(depth), dw, dh,
                                                                _ptr(None if mask_from_depth else mask), W, H, _ptr(K4), _ptr(ids),
                                                                flags, _ptr(handles), _ptr(nf)))
        self._nodes += [int(h) for h in handles]
        return [int(h) for h in handles], nf

    def nodes_create_sharded_resized(self, det: int, comm: int, total_frames: int, gray, depth, mask, K4, ids=None,
                                     mask_from_depth: bool = False, bayer: bool = False):
        """nodes_create_sharded for depth images of another size than the visual: gray / depth / mask hold THIS rank's frames,
        depth [F,dh,dw] as in nodes_create_resized; returns handles and feature counts of ALL total_frames nodes."""
        gray, depth, mask, depth_u16 = self._depth_image_inputs(gray, depth, mask)
        flags = resized_input_flags(gray.shape, depth.shape, mask_from_depth=mask_from_depth, depth_u16=depth_u16, bayer=bayer)
        H, W = gray.shape[1:3]
        dh, dw = depth.shape[1:3]
        K4 = None if K4 is None else np.ascontiguousarray(K4, np.float32)
        ids = None if ids is None else np.ascontiguousarray(ids, np.int32)
        handles = np.zeros(total_frames, np.uint64)
        nf = np.zeros(total_frames, np.int32)
        own = gray.shape[0] > 0
        self._check(self.lib.rgbdslam_b200_nodes_create_sharded_resized(
            det, C.c_uint64(comm), total_frames, _ptr(gray) if own else None, _ptr(depth) if own else None, dw, dh,
            _ptr(None if (mask_from_depth or not own) else mask), W, H, _ptr(K4), _ptr(ids), flags, _ptr(handles), _ptr(nf)))
        self._nodes += [int(h) for h in handles]
        return [int(h) for h in handles], nf

    def orb_debug_plane(self, which: int, cell: int, level: int) -> np.ndarray:
        w, h = C.c_int(), C.c_int()
        self._check(self.lib.rgbdslam_b200_orb_debug_plane(which, cell, level, None, 0, C.byref(w), C.byref(h)))
        buf = np.zeros((h.value, w.value), np.uint8)
        self._check(self.lib.rgbdslam_b200_orb_debug_plane(which, cell, level, _ptr(buf), buf.size, C.byref(w), C.byref(h)))
        return buf

    def orb_debug_candidates(self, cell: int):
        dt = np.dtype([("x", "<u2"), ("y", "<u2"), ("level", "u1"), ("score", "u1"), ("pad", "<u2")])
        cand = np.zeros(12288, dt)
        resp = np.zeros(12288, np.float32)
        n, thr = C.c_int(), C.c_int()
        self._check(self.lib.rgbdslam_b200_orb_debug_candidates(cell, _ptr(cand), _ptr(resp), 12288, C.byref(n), C.byref(thr)))
        m = min(n.value, 12288)
        return cand[:m], resp[:m], thr.value

    def node_keypoints(self, h: int) -> np.ndarray:
        out = np.zeros(self.node_num_features(h), KEYPOINT_DTYPE)
        self._check(self.lib.rgbdslam_b200_node_download_keypoints(h, _ptr(out)))
        return out

    # -- stored clouds and the registered map ---------------------------------------------
    def node_cloud(self, h: int, point_bytes: int = 32) -> np.ndarray:
        """Node::pc_col of a node built with store_cloud: (H, W) records of POINT32_DTYPE or POINT16_DTYPE"""
        w, hh = C.c_int(), C.c_int()
        self._check(self.lib.rgbdslam_b200_node_download_cloud(C.c_uint64(int(h)), point_bytes, None, C.byref(w), C.byref(hh)))
        out = np.zeros((hh.value, w.value), POINT32_DTYPE if point_bytes == 32 else POINT16_DTYPE)
        self._check(self.lib.rgbdslam_b200_node_download_cloud(C.c_uint64(int(h)), point_bytes, _ptr(out), C.byref(w), C.byref(hh)))
        return out

    def render_cloud(self, nodes, transforms12, maximum_depth: float = float("inf"), preserve_raster: bool = False,
                     point_bytes: int = 32, out=None, count_only: bool = False):
        """transformAndAppendPointCloud of the nodes in order (transforms12: (n, 3, 4) float64, node -> map).  Returns
        (records, used16) -- used16 (n, 4, 4) the float matrices applied -- or the record count with count_only.  out: an
        optional host array (numpy or pinned torch uint8) large enough for the records."""
        hs = np.ascontiguousarray(np.asarray(nodes, np.uint64))
        T = np.ascontiguousarray(np.asarray(transforms12, np.float64).reshape(len(hs), 12))
        n = C.c_int64()
        if count_only:
            self._check(self.lib.rgbdslam_b200_render_cloud(len(hs), _ptr(hs), _ptr(T), maximum_depth, int(preserve_raster), point_bytes,
                                                            None, 0, C.byref(n), None))
            return n.value
        used = np.zeros((len(hs), 16), np.float32)
        if out is None:
            self._check(self.lib.rgbdslam_b200_render_cloud(len(hs), _ptr(hs), _ptr(T), maximum_depth, int(preserve_raster), point_bytes,
                                                            None, 0, C.byref(n), None))
            out = np.zeros(n.value, POINT32_DTYPE if point_bytes == 32 else POINT16_DTYPE)
        cap = (out.numel() * out.element_size() if hasattr(out, "numel") else out.nbytes) // point_bytes
        self._check(self.lib.rgbdslam_b200_render_cloud(len(hs), _ptr(hs), _ptr(T), maximum_depth, int(preserve_raster), point_bytes,
                                                        _ptr(out), cap, C.byref(n), _ptr(used)))
        return (out[:n.value] if isinstance(out, np.ndarray) and out.dtype.itemsize == point_bytes else out), \
            used.reshape(-1, 4, 4).transpose(0, 2, 1)

    def reduce_clouds(self, nodes, voxelfilter_size: float) -> np.ndarray:
        """Node::reducePointCloud(voxelfilter_size) of the nodes' stored clouds on the device: each becomes one centroid per
        occupied voxel, a cloud of width n and height 1 for node_cloud / render_cloud.  Returns the new point counts (-1: the leaf size is too
        small for that node's cloud, which stays as it is)."""
        hs = np.ascontiguousarray(np.asarray(nodes, np.uint64))
        counts = np.zeros(len(hs), np.int32)
        self._check(self.lib.rgbdslam_b200_reduce_clouds(len(hs), _ptr(hs), float(voxelfilter_size), _ptr(counts)))
        return counts

    def transform_clouds(self, nodes, transforms12):
        """pcl::transformPointCloud of the nodes' stored clouds in place on the device (transform_individual_clouds):
        transforms12 (n, 3, 4) float64, each cast to float; points with a non-finite coordinate stay.  The nodes keep the
        transformed clouds for node_cloud, render_cloud, reduce_clouds and the OctoMap calls."""
        hs = np.ascontiguousarray(np.asarray(nodes, np.uint64).reshape(-1))
        T = np.ascontiguousarray(np.asarray(transforms12, np.float64).reshape(len(hs), 12))
        self._check(self.lib.rgbdslam_b200_transform_clouds(len(hs), _ptr(hs), _ptr(T)))

    def icp_align(self, source_handles, target_handles, max_cloud_size: int = 10000, method: str = "icp") -> np.ndarray:
        """icpAlignment(filterCloud(source), filterCloud(target), Identity) of the nodes' stored clouds, pair by pair, on the
        device (the ICP fallback of matchNodePair).  method is icp_method: "icp" (IterativeClosestPoint) or "icp_nl"
        (IterativeClosestPointNonLinear).  Returns ICP_RESULT_DTYPE records; T (column-major, as ransac_trafo) maps the
        source cloud onto the target cloud and is the identity unless converged."""
        if method not in ICP_METHODS:
            raise ValueError(f"icp method must be one of {sorted(ICP_METHODS)}, not {method!r}")
        s = np.ascontiguousarray(np.asarray(source_handles, np.uint64).reshape(-1))
        t = np.ascontiguousarray(np.asarray(target_handles, np.uint64).reshape(-1))
        if len(s) != len(t):
            raise ValueError("one target per source")
        out = np.zeros(len(s), ICP_RESULT_DTYPE)
        self._check(self.lib.rgbdslam_b200_icp_align_ex(len(s), _ptr(s), _ptr(t), int(max_cloud_size), ICP_METHODS[method],
                                                         _ptr(out)))
        return out

    # -- the colour OctoMap ----------------------------------------------------------------
    def octomap_create(self, resolution: float = 0.05, prob_hit: float = 0.9, prob_miss: float = 0.4, clamping_min: float = 0.001,
                       clamping_max: float = 0.999) -> int:
        """An empty colour OctoMap on the device (ColorOctomapServer::reset with these parameters)."""
        p = OctomapParams(resolution, prob_hit, prob_miss, clamping_min, clamping_max)
        h = C.c_uint64()
        self._check(self.lib.rgbdslam_b200_octomap_create(C.byref(p), C.byref(h)))
        return h.value

    def octomap_insert(self, octomap: int, nodes, transforms12, max_range: float = float("inf")):
        """insertCloudCallback of the nodes' stored clouds in order; transforms12: (n, 3, 4) float32 node -> map, e.g.
        octomap_pose of each estimate; max_range is maximum_depth (< 0 or inf: none)."""
        hs = np.ascontiguousarray(np.asarray(nodes, np.uint64).reshape(-1))
        T = np.ascontiguousarray(np.asarray(transforms12, np.float32).reshape(len(hs), 12))
        self._check(self.lib.rgbdslam_b200_octomap_insert(C.c_uint64(octomap), len(hs), _ptr(hs), _ptr(T), float(max_range)))

    def octomap_write(self, octomap: int) -> bytes:
        """The .ot file (ColorOcTree::write) as bytes."""
        n = C.c_int64()
        self._check(self.lib.rgbdslam_b200_octomap_write(C.c_uint64(octomap), None, 0, C.byref(n)))
        buf = np.zeros(n.value, np.uint8)
        self._check(self.lib.rgbdslam_b200_octomap_write(C.c_uint64(octomap), _ptr(buf), n.value, C.byref(n)))
        return buf.tobytes()

    def octomap_stats(self, octomap: int) -> tuple[int, int]:
        """(tree nodes with the root, leaves)"""
        a, b = C.c_int64(), C.c_int64()
        self._check(self.lib.rgbdslam_b200_octomap_stats(C.c_uint64(octomap), C.byref(a), C.byref(b)))
        return a.value, b.value

    def octomap_clear(self, octomap: int):
        self._check(self.lib.rgbdslam_b200_octomap_clear(C.c_uint64(octomap)))

    def octomap_destroy(self, octomap: int):
        self._check(self.lib.rgbdslam_b200_octomap_destroy(C.c_uint64(octomap)))

    def octomap_filter_clouds(self, octomap: int, nodes, sensor7, threshold: float = 0.9) -> np.ndarray:
        """ColorOctomapServer::occupancyFilter of the nodes' stored clouds against the map, in place (occupancyFilterClouds).
        sensor7: (n, 7) float32 per node qx qy qz qw ox oy oz -- cloud_sensor_pose of its estimate, or 0 0 0 1 0 0 0 for a
        cloud updateCloudOrigin never saw; threshold is occupancy_filter_threshold.  Returns the new point counts."""
        hs = np.ascontiguousarray(np.asarray(nodes, np.uint64).reshape(-1))
        S = np.ascontiguousarray(np.asarray(sensor7, np.float32).reshape(len(hs), 7))
        counts = np.zeros(len(hs), np.int32)
        self._check(self.lib.rgbdslam_b200_octomap_filter_clouds(C.c_uint64(octomap), len(hs), _ptr(hs), _ptr(S), float(threshold),
                                                                 _ptr(counts)))
        return counts

    def node_clear_cloud(self, h: int):
        """Node::clearPointCloud: the node drops its stored cloud"""
        self._check(self.lib.rgbdslam_b200_node_clear_cloud(C.c_uint64(int(h))))

    # -- multi-GPU exchange -------------------------------------------------------------
    def comm_unique_id(self) -> np.ndarray:
        uid = np.zeros(128, np.uint8)
        self._check(self.lib.rgbdslam_b200_comm_unique_id(_ptr(uid)))
        return uid

    def comm_init(self, rank: int, world: int, uid: np.ndarray) -> int:
        h = C.c_uint64()
        uid = np.ascontiguousarray(uid, np.uint8)
        self._check(self.lib.rgbdslam_b200_comm_init(rank, world, _ptr(uid), C.byref(h)))
        return h.value

    def comm_destroy(self, comm: int):
        self._check(self.lib.rgbdslam_b200_comm_destroy(comm))

    def allgather_edges(self, comm: int, local: np.ndarray, world: int, out: np.ndarray | None = None) -> np.ndarray:
        local = np.ascontiguousarray(local, PAIR_RESULT_DTYPE)
        if out is None:
            out = np.zeros(world * len(local), PAIR_RESULT_DTYPE)
        self._check(self.lib.rgbdslam_b200_allgather_edges(comm, _ptr(local), len(local), _ptr(out)))
        return out

    # -- GraphManager::optimizeGraph ----------------------------------------------
    def allgather_slot_edges(self, comm: int, slot: int, n_per_rank: int, out: np.ndarray):
        """all-gather of the slot's in-flight edge records into `out` (host, world * n_per_rank records); wait_slot() completes it"""
        self._check(self.lib.rgbdslam_b200_allgather_slot_edges(C.c_uint64(comm), slot, n_per_rank, _ptr(out)))

    def optimize_graph(self, poses, fixed, ij, meas, info, stop: float = 0.01, huber_delta: float = 1.0):
        """== GraphManager::optimizeGraph (graph_manager.cpp:900).  Returns (poses, chi2, lm_iters, cg_iters)."""
        x = np.array(poses, np.float64, order="C")
        fixed = np.ascontiguousarray(fixed, np.uint8)
        ij = np.ascontiguousarray(ij, np.int32)
        meas = np.ascontiguousarray(meas, np.float64)
        info = np.ascontiguousarray(info, np.float64)
        chi2, it, cg = C.c_double(), C.c_int(), C.c_int()
        self._check(self.lib.rgbdslam_b200_posegraph_optimize(len(x), _ptr(x), _ptr(fixed), len(ij), _ptr(ij), _ptr(meas),
                                                              _ptr(info), stop, huber_delta, C.byref(chi2), C.byref(it), C.byref(cg)))
        return x, chi2.value, it.value, cg.value

    def landmark_ba(self, poses, fixed, points, obs_cam, obs_point, obs_uvd, obs_info3, K4, ij=None, meas=None, info=None,
                    iterations: int = 10, huber_delta: float = 1.0):
        """Camera + landmark bundle adjustment (the reference's DO_FEATURE_OPTIMIZATION graph, landmark.cpp:97-187).
        Returns (poses, points, chi2_before, chi2_after, lm_iterations, pcg_iterations)."""
        x = np.array(poses, np.float64, order="C")
        pts = np.array(points, np.float64, order="C").reshape(-1, 3)
        fixed = np.ascontiguousarray(fixed, np.uint8)
        oc = np.ascontiguousarray(obs_cam, np.int32)
        op = np.ascontiguousarray(obs_point, np.int32)
        uvd = np.ascontiguousarray(obs_uvd, np.float64).reshape(-1, 3)
        w3 = np.ascontiguousarray(obs_info3, np.float64).reshape(-1, 3)
        K = np.ascontiguousarray(K4, np.float64)
        ne = 0 if ij is None else len(ij)
        ij_ = None if ne == 0 else np.ascontiguousarray(ij, np.int32)
        meas_ = None if ne == 0 else np.ascontiguousarray(meas, np.float64)
        info_ = None if ne == 0 else np.ascontiguousarray(info, np.float64)
        c0, c1, it, cg = C.c_double(), C.c_double(), C.c_int(), C.c_int()
        self._check(self.lib.rgbdslam_b200_landmark_ba(len(x), _ptr(x), _ptr(fixed), len(pts), _ptr(pts), len(oc), _ptr(oc), _ptr(op),
                                                       _ptr(uvd), _ptr(w3), _ptr(K), ne, _ptr(ij_), _ptr(meas_), _ptr(info_), iterations,
                                                       huber_delta, C.byref(c0), C.byref(c1), C.byref(it), C.byref(cg)))
        return x, pts, c0.value, c1.value, it.value, cg.value

    def posegraph_reserve(self, nv: int, ne: int):
        self._check(self.lib.rgbdslam_b200_posegraph_reserve(nv, ne))

    def graph_chi2(self, poses, ij, meas, info, huber_delta: float = 1.0, per_edge: bool = False):
        x = np.ascontiguousarray(poses, np.float64)
        ij = np.ascontiguousarray(ij, np.int32)
        meas = np.ascontiguousarray(meas, np.float64)
        info = np.ascontiguousarray(info, np.float64)
        chi2 = C.c_double()
        pe = np.zeros(len(ij), np.float64) if per_edge else None
        self._check(self.lib.rgbdslam_b200_posegraph_chi2(len(x), _ptr(x), len(ij), _ptr(ij), _ptr(meas), _ptr(info),
                                                          huber_delta, C.byref(chi2), _ptr(pe)))
        return (chi2.value, pe) if per_edge else chi2.value

    def close(self):
        for h in list(self._nodes):
            self.lib.rgbdslam_b200_node_destroy(h)
        self._nodes.clear()
