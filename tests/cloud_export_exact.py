"""numpy restatement of the reference's per-node exports, next to tests/map_cloud_exact.py (whose cloud dicts and tf helpers it
uses):
- transform_cloud   pcl::transformPointCloud(*pc_col, *pc_col, m) (PCL 1.7), the transform_individual_clouds step of
                    saveIndividualCloudsToFile (graph_mgr_io.cpp:372-374)
- world_to_points   its pose without transform_individual_clouds (graph_mgr_io.cpp:56-90, 384-396), tf and ground truth absent
- sensor_pose       the sensor orientation / origin either branch writes, and pose_text / viewpoint, their text
- feature_locations the float transform of saveAllFeaturesToFile (graph_mgr_io.cpp:445-497), and cv2_features_yaml, the file
                    OpenCV's FileStorage writes of them
Every float operation is one numpy float32 operation, so nothing is contracted.
"""
import numpy as np

import map_cloud_exact as mx

F32 = np.float32


def transform_cloud(pc, T12):
    """pc (a map_cloud_exact cloud dict) after transformPointCloud by the 3 x 4 double T12 cast to float: a point with a
    non-finite x, y or z stays, every other becomes ((m0 x + m1 y) + m2 z) + m3 per row.  Colour, data[3] and raster stay."""
    M = mx.transform_as_matrix(T12)
    x, y, z = (np.asarray(pc[k], F32) for k in ("x", "y", "z"))
    fin = np.isfinite(x) & np.isfinite(y) & np.isfinite(z)
    with np.errstate(all="ignore"):
        t = [(((M[r, 0] * x) + (M[r, 1] * y)) + (M[r, 2] * z)) + M[r, 3] for r in range(3)]
    out = dict(pc)
    for k, c, tc in zip("xyz", (x, y, z), t):
        out[k] = np.where(fin, tc, c).astype(F32)
    return out


def from_records(rec, w, h):
    """a cloud dict of 32-byte records (node_download_cloud): data[3] of a 32-byte record carries no colour, so w16 is not kept"""
    r = np.asarray(rec).reshape(-1)
    return dict(x=r["x"].copy(), y=r["y"].copy(), z=r["z"].copy(), rgb=r["rgb"].copy(), w16=r["w"].copy(), w=w, h=h)


def tf_inverse(A):
    """tf::Transform::inverse: (R^T, R^T (-t)), each entry (a0 b0 + a1 b1) + a2 b2"""
    R, m = A[:, :3].T, -A[:, 3]
    t = np.array([(R[r, 0] * m[0] + R[r, 1] * m[1]) + R[r, 2] * m[2] for r in range(3)])
    return np.concatenate([R, t[:, None]], 1)


def world_to_points(M):
    """(init_base_pose_ * base2points * M * base2points.inverse()) * base2points with identity init_base_pose_ and base2points,
    every product formed; M is eigenTransf2TF(estimate), row-major 3 x 4 double"""
    I = np.concatenate([np.eye(3), np.zeros((3, 1))], 1)
    w2b = mx.tf_mul(mx.tf_mul(mx.tf_mul(I, I), np.asarray(M, np.float64)), tf_inverse(I))
    return mx.tf_mul(w2b, I)


def tf_get_rotation(M):
    """tf::Matrix3x3::getRotation (x, y, z, w) in double"""
    tr = (M[0, 0] + M[1, 1]) + M[2, 2]
    g = np.zeros(4)
    if tr > 0.0:
        s = np.sqrt(tr + 1.0)
        g[3] = s * 0.5
        s = 0.5 / s
        g[0], g[1], g[2] = (M[2, 1] - M[1, 2]) * s, (M[0, 2] - M[2, 0]) * s, (M[1, 0] - M[0, 1]) * s
    else:
        i = (2 if M[1, 1] < M[2, 2] else 1) if M[0, 0] < M[1, 1] else (2 if M[0, 0] < M[2, 2] else 0)
        j, k = (i + 1) % 3, (i + 2) % 3
        s = np.sqrt(((M[i, i] - M[j, j]) - M[k, k]) + 1.0)
        g[i] = s * 0.5
        s = 0.5 / s
        g[3] = (M[k, j] - M[j, k]) * s
        g[j] = (M[j, i] + M[i, j]) * s
        g[k] = (M[k, i] + M[i, k]) * s
    return g


def quatf_to_rotation_matrix(q):
    """Eigen's Quaternionf::toRotationMatrix of q (x, y, z, w, float32)"""
    x, y, z, w = (F32(v) for v in q)
    tx, ty, tz = F32(2) * x, F32(2) * y, F32(2) * z
    twx, twy, twz, txx, txy, txz = tx * w, ty * w, tz * w, tx * x, ty * x, tz * x
    tyy, tyz, tzz = ty * y, tz * y, tz * z
    one = F32(1)
    return np.array([[one - (tyy + tzz), txy - twz, txz + twy], [txy + twz, one - (txx + tzz), tyz - twx],
                     [txz - twy, tyz + twx, one - (txx + tyy)]], F32)


def sensor_pose(M=None):
    """(q (x, y, z, w), o) float32 of the pose written: transform_individual_clouds (M None) the reference's Quaternionf(0, 0, 0, 1)
    -- w = 0, z = 1 -- at origin 0; otherwise world_to_points(M)'s getRotation and origin cast to float"""
    if M is None:
        return np.array([0, 0, 1, 0], F32), np.zeros(3, F32)
    W = world_to_points(M)
    return tf_get_rotation(W).astype(F32), W[:, 3].astype(F32)


def pose_text(q, o):
    """the .txt of saveIndividualCloudsToFile: rows "R R R o " of toRotationMatrix, then "0 0 0 1\\n", floats as '%g'"""
    R = quatf_to_rotation_matrix(q)
    return "".join("%g %g %g %g " % (R[i, 0], R[i, 1], R[i, 2], o[i]) for i in range(3)) + "0 0 0 1\n"


def viewpoint(q, o):
    """the PCD VIEWPOINT line's values: ox oy oz qw qx qy qz as '%g'"""
    return " ".join("%g" % v for v in (o[0], o[1], o[2], q[3], q[0], q[1], q[2]))


def feature_locations(T12, xyz):
    """world2rgbMat * (x, y, z, 1) in float, world2rgbMat the double 3 x 4 cast to float: ((c0 x + c1 y) + c2 z) + c3"""
    M = mx.transform_as_matrix(T12)
    p = np.asarray(xyz, F32).reshape(-1, 3)
    with np.errstate(all="ignore"):
        return np.stack([(((M[r, 0] * p[:, 0]) + (M[r, 1] * p[:, 1])) + (M[r, 2] * p[:, 2])) + M[r, 3] for r in range(3)], 1).astype(F32)


def cv2_features_yaml(path, locations, descriptors):
    """the file cv2.FileStorage writes of saveAllFeaturesToFile's calls: Feature_Locations, one flow map {x, y, z} per row
    (each float forwarded as a double), then Feature_Descriptors, an (n, 32) uint8 matrix"""
    import cv2
    fs = cv2.FileStorage(str(path), cv2.FileStorage_WRITE)
    fs.startWriteStruct("Feature_Locations", cv2.FileNode_SEQ)
    for x, y, z in np.asarray(locations, F32).reshape(-1, 3):
        fs.startWriteStruct("", cv2.FileNode_MAP | cv2.FileNode_FLOW)
        fs.write("x", float(x))
        fs.write("y", float(y))
        fs.write("z", float(z))
        fs.endWriteStruct()
    fs.endWriteStruct()
    fs.write("Feature_Descriptors", np.ascontiguousarray(descriptors, np.uint8).reshape(-1, 32))
    fs.release()
    return open(path, "rb").read()
