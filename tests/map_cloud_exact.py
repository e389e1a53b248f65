"""numpy restatement of the reference's colour clouds and registered map, and the ctypes wrapper of its C oracle
(tests/map_cloud_oracle.c):
- create_cloud   createXYZRGBPointCloud (misc.cpp:467-556) of a depth image and its visual, the Node's pc_col
- cloud_points   pc_col of the point-cloud constructor (node.cpp:261): the cloud as stored with its colour word
- render         transformAndAppendPointCloud (misc.cpp:183-238) of several clouds, node order then raster order
- world2cam      the double composition of GraphManager::saveAllCloudsToFile (graph_mgr_io.cpp:526-541):
                 cam2rgb * eigenTransf2TF(pose), as the C++ shim forms it
A cloud is a dict of flat arrays x, y, z (float32), rgb (the colour word, uint32) and w16 (data[3] of a 16-byte PointXYZ
record: the colour word, except point 0 of a depth-image cloud, 1.0f), plus its raster w, h.  Every float operation is one
numpy float32 operation, so nothing is contracted; R p sums (r0 p0 + r1 p1) + r2 p2 (DESIGN.md 4.12).
"""
import ctypes as C
import functools
import subprocess
import tempfile
from pathlib import Path

import numpy as np

HERE = Path(__file__).resolve().parent
F32 = np.float32
ONE_F = np.uint32(0x3F800000)
POINT32 = np.dtype([("x", "<f4"), ("y", "<f4"), ("z", "<f4"), ("w", "<u4"), ("rgb", "<u4"), ("pad", "<u4", (3,))])
POINT16 = np.dtype([("x", "<f4"), ("y", "<f4"), ("z", "<f4"), ("w", "<u4")])


def colour_words(visual, bgr=True):
    """The packed b, g, r, a word of every pixel: a grey visual gives R = G = B; channel 0 is blue with encoding_bgr and red
    without it; alpha 0."""
    v = np.asarray(visual, np.uint32)
    if v.ndim == 2:
        return v | (v << 8) | (v << 16)
    c0, c1, c2 = v[..., 0], v[..., 1], v[..., 2]
    return (c0 | (c1 << 8) | (c2 << 16)) if bgr else (c2 | (c1 << 8) | (c0 << 16))


def create_cloud(depth, visual, K4, step=2, scaling=1.0, min_depth=0.1, bgr=True):
    """createXYZRGBPointCloud for a skip step that divides the image: point (rx, ry) is pixel (rx * step, ry * step)."""
    depth = np.asarray(depth, F32)
    H, W = depth.shape
    assert H % step == 0 and W % step == 0
    fx, fy, cx, cy = (F32(k) for k in K4)
    fxinv, fyinv = F32(1.0 / np.float64(fx)), F32(1.0 / np.float64(fy))
    v, u = np.mgrid[0:H:step, 0:W:step]
    uf, vf = u.astype(F32).ravel(), v.astype(F32).ravel()
    with np.errstate(all="ignore"):
        Z = (depth[::step, ::step].astype(np.float64) * np.float64(scaling)).astype(F32).ravel()
        valid = Z >= F32(min_depth)
        x = np.where(valid, ((uf - cx) * Z) * fxinv, (uf - cx) * fxinv).astype(F32)
        y = np.where(valid, ((vf - cy) * Z) * fyinv, (vf - cy) * fyinv).astype(F32)
    z = np.where(valid, Z, F32(np.nan)).astype(F32)
    rgb = colour_words(np.asarray(visual)[::step, ::step], bgr).reshape(-1).astype(np.uint32)
    rgb[0] = 0  # color_idx 0 fails `color_idx > 0`: point 0 keeps the default colour
    w16 = rgb.copy()
    w16[0] = ONE_F
    return dict(x=x, y=y, z=z, rgb=rgb, w16=w16, w=W // step, h=H // step)


def cloud_points(cloud):
    """pc_col of the point-cloud constructor: (H, W, 8) PointXYZRGB (colour at float 4) or (H, W, 4) PointXYZ (data[3])."""
    c = np.ascontiguousarray(cloud, F32)
    H, W, stride = c.shape
    rgb = c[..., 4 if stride == 8 else 3].view(np.uint32).ravel().copy()
    return dict(x=c[..., 0].ravel().copy(), y=c[..., 1].ravel().copy(), z=c[..., 2].ravel().copy(), rgb=rgb, w16=rgb.copy(), w=W,
                h=H)


def records(x, y, z, rgb, w16, point_bytes):
    out = np.zeros(len(x), POINT32 if point_bytes == 32 else POINT16)
    out["x"], out["y"], out["z"] = x, y, z
    if point_bytes == 32:
        out["w"] = ONE_F
        out["rgb"] = rgb
    else:
        out["w"] = w16
    return out


def organised(pc, point_bytes=32):
    """the cloud as node_download_cloud returns it: (h, w) records"""
    return records(pc["x"], pc["y"], pc["z"], pc["rgb"], pc["w16"], point_bytes).reshape(pc["h"], pc["w"])


def transform_as_matrix(T12):
    """pcl_ros::transformAsMatrix: the double 3 x 4 cast entry by entry to float"""
    return np.asarray(T12, np.float64).reshape(3, 4).astype(F32)


def render(pcs, transforms12, maximum_depth=np.inf, preserve=False, point_bytes=32):
    """transformAndAppendPointCloud of every cloud in order."""
    md = F32(maximum_depth)
    parts = []
    for pc, T in zip(pcs, transforms12):
        M = transform_as_matrix(T)
        x, y, z = pc["x"], pc["y"], pc["z"]
        with np.errstate(all="ignore"):
            far = (((x * x) + (y * y)) + (z * z)) > md * md if md >= 0 else np.zeros(len(x), bool)
            nanp = np.isnan(x) | np.isnan(y) | np.isnan(z)
            t = [(((M[r, 0] * x) + (M[r, 1] * y)) + (M[r, 2] * z)) + M[r, 3] for r in range(3)]
        o = [np.where(far, F32(np.nan), np.where(nanp, c, tc)).astype(F32) for c, tc in zip((x, y, z), t)]
        keep = np.ones(len(x), bool) if preserve else ~far & ~nanp
        parts.append(records(o[0][keep], o[1][keep], o[2][keep], pc["rgb"][keep], pc["w16"][keep], point_bytes))
    return np.concatenate(parts) if parts else np.zeros(0, POINT32 if point_bytes == 32 else POINT16)


# ---- the double composition of saveAllCloudsToFile ------------------------------------------------------------------------

def quat_from_rpy(roll, pitch, yaw):
    """tf::createQuaternionFromRPY -> tf::Quaternion::setRPY (x, y, z, w)"""
    hy, hp, hr = yaw * 0.5, pitch * 0.5, roll * 0.5
    cy, sy, cp, sp, cr, sr = np.cos(hy), np.sin(hy), np.cos(hp), np.sin(hp), np.cos(hr), np.sin(hr)
    return np.array([sr * cp * cy - cr * sp * sy, cr * sp * cy + sr * cp * sy, cr * cp * sy - sr * sp * cy, cr * cp * cy + sr * sp * sy])


def quat_from_matrix(R):
    """Eigen's Quaternion(Matrix3d) (x, y, z, w)"""
    t = R[0, 0] + R[1, 1] + R[2, 2]
    if t > 0:
        s = np.sqrt(t + 1.0)
        w = 0.5 * s
        s = 0.5 / s
        return np.array([(R[2, 1] - R[1, 2]) * s, (R[0, 2] - R[2, 0]) * s, (R[1, 0] - R[0, 1]) * s, w])
    i = 0
    if R[1, 1] > R[0, 0]:
        i = 1
    if R[2, 2] > R[i, i]:
        i = 2
    j, k = (i + 1) % 3, (i + 2) % 3
    s = np.sqrt(R[i, i] - R[j, j] - R[k, k] + 1.0)
    q = np.zeros(4)
    q[i] = 0.5 * s
    s = 0.5 / s
    q[3] = (R[k, j] - R[j, k]) * s
    q[j] = (R[j, i] + R[i, j]) * s
    q[k] = (R[k, i] + R[i, k]) * s
    return q


def matrix_from_quat(q):
    """tf::Matrix3x3::setRotation"""
    x, y, z, w = q
    d = x * x + y * y + z * z + w * w
    s = 2.0 / d
    xs, ys, zs = x * s, y * s, z * s
    wx, wy, wz = w * xs, w * ys, w * zs
    xx, xy, xz = x * xs, x * ys, x * zs
    yy, yz, zz = y * ys, y * zs, z * zs
    return np.array([[1.0 - (yy + zz), xy - wz, xz + wy], [xy + wz, 1.0 - (xx + zz), yz - wx], [xz - wy, yz + wx, 1.0 - (xx + yy)]])


def tf_mul(A, B):
    """tf::Transform * tf::Transform: (R_a R_b, R_a t_b + t_a), each entry a tf::tdotx-style sum (a0 b0 + a1 b1) + a2 b2"""
    Ra, ta, Rb, tb = A[:, :3], A[:, 3], B[:, :3], B[:, 3]
    R = np.array([[(Ra[r, 0] * Rb[0, c] + Ra[r, 1] * Rb[1, c]) + Ra[r, 2] * Rb[2, c] for c in range(3)] for r in range(3)])
    t = np.array([((Ra[r, 0] * tb[0] + Ra[r, 1] * tb[1]) + Ra[r, 2] * tb[2]) + ta[r] for r in range(3)])
    return np.concatenate([R, t[:, None]], 1)


def world2cam(pose4x4):
    """cam2rgb * eigenTransf2TF(pose) in double, row-major 3 x 4: cam2rgb = (createQuaternionFromRPY(-1.57, 0, -1.57),
    (0, -0.04, 0)); eigenTransf2TF takes the pose's rotation through Eigen's quaternion and tf's quaternion -> matrix."""
    P = np.asarray(pose4x4, np.float64)
    cam2rgb = np.concatenate([matrix_from_quat(quat_from_rpy(-1.57, 0.0, -1.57)), np.array([[0.0], [-0.04], [0.0]])], 1)
    pose = np.concatenate([matrix_from_quat(quat_from_matrix(P[:3, :3])), P[:3, 3:4]], 1)
    return tf_mul(cam2rgb, pose)


# ---- the C oracle ----------------------------------------------------------------------------------------------------------

@functools.lru_cache(maxsize=None)
def _oracle_lib() -> C.CDLL:
    """tests/map_cloud_oracle.c built into a temporary directory (the source tree may be read-only)."""
    out = Path(tempfile.mkdtemp(prefix="map_cloud_oracle_")) / "libmap_cloud_oracle.so"
    subprocess.run(["gcc", "-O2", "-fPIC", "-shared", "-ffp-contract=off", "-Wall", "-o", str(out), str(HERE / "map_cloud_oracle.c"),
                    "-lm"], check=True, capture_output=True)
    lib = C.CDLL(str(out))
    lib.map_create_cloud.restype = None
    lib.map_transform_append.restype = C.c_long
    return lib


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


def oracle_create_cloud(depth, visual, K4, step=2, scaling=1.0, min_depth=0.1, bgr=True, point_bytes=32):
    """the C oracle of create_cloud: (h, w) records"""
    d = np.ascontiguousarray(depth, F32)
    vis = np.ascontiguousarray(visual, np.uint8)
    H, W = d.shape
    ch = 1 if vis.ndim == 2 else 3
    K = np.ascontiguousarray(K4, F32)
    out = np.zeros((H // step) * (W // step), POINT32 if point_bytes == 32 else POINT16)
    _oracle_lib().map_create_cloud(_p(d), _p(vis), C.c_int(W), C.c_int(H), C.c_int(ch), _p(K), C.c_int(step), C.c_double(scaling),
                                   C.c_float(min_depth), C.c_int(int(bgr)), C.c_int(point_bytes), _p(out))
    return out.reshape(H // step, W // step)


def oracle_render(organised_clouds, transforms12, maximum_depth=np.inf, preserve=False):
    """the C oracle of render on 32-byte organised clouds"""
    lib = _oracle_lib()
    parts = []
    for pc, T in zip(organised_clouds, transforms12):
        src = np.ascontiguousarray(pc.reshape(-1))
        out = np.zeros(len(src), POINT32)
        T = np.ascontiguousarray(T, np.float64).reshape(12)
        n = lib.map_transform_append(_p(src), C.c_long(len(src)), _p(T), C.c_float(maximum_depth), C.c_int(int(preserve)), _p(out))
        parts.append(out[:n])
    return np.concatenate(parts)
