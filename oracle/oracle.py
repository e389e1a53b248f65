"""ctypes wrapper of the C oracle (oracle/liboracle.so) -- TEST INFRASTRUCTURE, not product code.

Only tests/, bench.py (cpu_baseline / --impl reference) and __graft_entry__.smoke() import this.
"""
from __future__ import annotations

import ctypes as C
import subprocess
from pathlib import Path

import numpy as np

HERE = Path(__file__).resolve().parent

DMATCH_DTYPE = np.dtype([("queryIdx", "<i4"), ("trainIdx", "<i4"), ("imgIdx", "<i4"), ("distance", "<f4")])
RESULT_DTYPE = np.dtype([
    ("id1", "<i4"), ("id2", "<i4"), ("n_all_matches", "<i4"), ("n_inliers", "<i4"), ("rmse", "<f4"),
    ("valid_iterations", "<i4"), ("ransac_trafo", "<f4", (16,)), ("info_scale", "<f8"), ("used_identity", "<i4"),
    ("real_iterations", "<i4"),
])


class OParams(C.Structure):
    _fields_ = [("min_matches", C.c_int32), ("max_matches", C.c_int32), ("ransac_iterations", C.c_int32),
                ("pad_", C.c_int32), ("max_dist_for_inliers", C.c_double), ("sigma_depth", C.c_double),
                ("depth_cov_z0", C.c_double)]


def build(force: bool = False) -> Path:
    out = HERE / "liboracle.so"
    srcs = sorted(HERE.glob("*.c"))
    if force or not out.exists() or out.stat().st_mtime < max(s.stat().st_mtime for s in srcs + [HERE / "Makefile"]):
        subprocess.run(["make", "-C", str(HERE), "all"], check=True, capture_output=True)
    return out


_lib = None


def lib() -> C.CDLL:
    global _lib
    if _lib is None:
        _lib = C.CDLL(str(build()))
        _lib.oracle_rand31.restype = C.c_uint32
        _lib.oracle_rand31.argtypes = [C.c_uint64, C.c_uint64, C.c_uint32, C.c_uint32]
        _lib.oracle_match_distance.restype = C.c_float
        _lib.oracle_match_distance.argtypes = [C.c_int, C.c_uint32]
        _lib.oracle_error_function2.restype = C.c_double
    return _lib


def ref_lib():
    """The reference's own bruteForceSearchORB, compiled from /root/reference (None if not built)."""
    p = HERE / "_ref" / "libref_features.so"
    if not p.exists():
        return None
    return C.CDLL(str(p))


def make_params(min_matches=20, max_matches=300, ransac_iterations=200, max_dist_for_inliers=3.0, sigma_depth=0.01,
                depth_cov_z0=-1.0) -> OParams:
    return OParams(min_matches, max_matches, ransac_iterations, 0, max_dist_for_inliers, sigma_depth, depth_cov_z0)


def _p(a):
    return None if a is None else a.ctypes.data_as(C.c_void_p)


def brute_force_orb(q: np.ndarray, t: np.ndarray):
    q = np.ascontiguousarray(q, np.uint8).reshape(-1, 32)
    t = np.ascontiguousarray(t, np.uint8).reshape(-1, 32)
    idx = np.empty(len(q), np.int32)
    hd = np.empty(len(q), np.int32)
    lib().oracle_brute_force_orb_batch(_p(q), C.c_int(len(q)), _p(t), C.c_int(len(t)), _p(idx), _p(hd))
    return hd, idx


def ref_brute_force_orb(q: np.ndarray, t: np.ndarray):
    """Calls the REFERENCE function int bruteForceSearchORB(const uint64_t*, const uint64_t*, const unsigned&, int&)."""
    rl = ref_lib()
    fn = getattr(rl, "_Z19bruteForceSearchORBPKmS0_RKjRi")
    fn.restype = C.c_int
    q = np.ascontiguousarray(q, np.uint8).reshape(-1, 32)
    t = np.ascontiguousarray(t, np.uint8).reshape(-1, 32)
    idx = np.empty(len(q), np.int32)
    hd = np.empty(len(q), np.int32)
    size = C.c_uint(len(t))
    for i in range(len(q)):
        r = C.c_int(-7)
        hd[i] = fn(C.c_void_p(q[i].ctypes.data), _p(t), C.byref(size), C.byref(r))
        idx[i] = r.value
    return hd, idx


def feature_matching_orb(q, t, max_matches, seed, pair):
    q = np.ascontiguousarray(q, np.uint8).reshape(-1, 32)
    t = np.ascontiguousarray(t, np.uint8).reshape(-1, 32)
    out = np.zeros(max(len(q), 1), DMATCH_DTYPE)
    fn = lib().oracle_feature_matching_orb
    fn.restype = C.c_int
    n = fn(_p(q), C.c_int(len(q)), _p(t), C.c_int(len(t)), C.c_int(max_matches), C.c_uint64(seed), C.c_uint64(pair), _p(out))
    return out[:n]


def match_pairs(params: OParams, desc_newer, xyz_newer, n_newer, desc_older, xyz_older, n_older, id_newer=None,
                id_older=None, seed=0, first_pair_index=0, threads=1, want_matches=True):
    n_newer = np.ascontiguousarray(n_newer, np.int32)
    n_older = np.ascontiguousarray(n_older, np.int32)
    npairs = len(n_newer)
    res = np.zeros(npairs, RESULT_DTYPE)
    allm = np.zeros((npairs, params.max_matches), DMATCH_DTYPE) if want_matches else None
    inl = np.zeros((npairs, params.max_matches), DMATCH_DTYPE) if want_matches else None
    idn = None if id_newer is None else np.ascontiguousarray(id_newer, np.int32)
    ido = None if id_older is None else np.ascontiguousarray(id_older, np.int32)
    d1 = np.ascontiguousarray(desc_newer, np.uint8)
    x1 = np.ascontiguousarray(xyz_newer, np.float32)
    d2 = np.ascontiguousarray(desc_older, np.uint8)
    x2 = np.ascontiguousarray(xyz_older, np.float32)
    lib().oracle_match_pairs(C.byref(params), _p(d1), _p(x1), _p(n_newer), _p(d2), _p(x2), _p(n_older), _p(idn), _p(ido),
                             C.c_int(npairs), C.c_uint64(seed), C.c_int64(first_pair_index), _p(res), _p(allm), _p(inl),
                             C.c_int(threads))
    return res, allm, inl


def get_transform_from_matches(xyz_newer, xyz_older, matches):
    x1 = np.ascontiguousarray(xyz_newer, np.float32)
    x2 = np.ascontiguousarray(xyz_older, np.float32)
    m = np.ascontiguousarray(matches)
    T = np.zeros(16, np.float32)
    lib().oracle_get_transform_from_matches(_p(x1), _p(x2), _p(m), None, C.c_int(len(m)), _p(T))
    return T.reshape(4, 4).T.copy()  # column-major -> numpy row/col


def error_function2(params: OParams, x1, x2, T4x4):
    a = np.ascontiguousarray(x1, np.float32)
    b = np.ascontiguousarray(x2, np.float32)
    Tc = np.ascontiguousarray(np.asarray(T4x4, np.float64).T.reshape(-1))  # column-major
    return lib().oracle_error_function2(C.byref(params), _p(a), _p(b), _p(Tc))


def first_depth_z0(params: OParams, allm_row, n_all, xyz_newer, xyz_older):
    """z of the first correspondence errorFunction2 would see for this pair (misc2.h:30-35 latch emulation)."""
    if n_all <= params.min_matches:
        return 0.0
    for m in allm_row[:n_all]:
        zf, zt = xyz_newer[m["queryIdx"], 2], xyz_older[m["trainIdx"], 2]
        if zf == 0 or zt == 0 or np.isnan(zf) or np.isnan(zt):
            continue
        return float(zf)
    return 0.0


# ---- pose graph ------------------------------------------------------------------------------------
def edge_se3(xi, xj, z, want_jac=True):
    xi = np.ascontiguousarray(xi, np.float64); xj = np.ascontiguousarray(xj, np.float64); z = np.ascontiguousarray(z, np.float64)
    e = np.zeros(6); Ji = np.zeros(36); Jj = np.zeros(36)
    lib().oracle_edge_se3(_p(xi), _p(xj), _p(z), _p(e), _p(Ji) if want_jac else None, _p(Jj) if want_jac else None)
    return e, Ji.reshape(6, 6), Jj.reshape(6, 6)


def vertex_oplus(x, d):
    x = np.array(x, np.float64); d = np.ascontiguousarray(d, np.float64)
    lib().oracle_vertex_oplus(_p(x), _p(d))
    return x


def posegraph_optimize(poses, fixed, ij, meas, info, stop=0.01, huber_delta=1.0):
    """== GraphManager::optimizeGraph (graph_manager.cpp:900-1066); returns (poses, chi2, lm_iterations, cg_iterations)."""
    x = np.array(poses, np.float64, order="C")
    fixed = np.ascontiguousarray(fixed, np.uint8); ij = np.ascontiguousarray(ij, np.int32)
    meas = np.ascontiguousarray(meas, np.float64); info = np.ascontiguousarray(info, np.float64)
    it = C.c_int(0); cg = C.c_int(0)
    fn = lib().oracle_posegraph_optimize
    fn.restype = C.c_double
    chi2 = fn(C.c_int(len(x)), _p(x), _p(fixed), C.c_int(len(ij)), _p(ij), _p(meas), _p(info), C.c_double(stop),
              C.c_double(huber_delta), C.byref(it), C.byref(cg))
    return x, chi2, it.value, cg.value


def posegraph_chi2(poses, ij, meas, info, huber_delta=1.0):
    x = np.ascontiguousarray(poses, np.float64); ij = np.ascontiguousarray(ij, np.int32)
    meas = np.ascontiguousarray(meas, np.float64); info = np.ascontiguousarray(info, np.float64)
    rob = C.c_double(0)
    fn = lib().oracle_posegraph_chi2
    fn.restype = C.c_double
    chi2 = fn(C.c_int(len(x)), _p(x), C.c_int(len(ij)), _p(ij), _p(meas), _p(info), C.c_double(huber_delta), C.byref(rob))
    return chi2, rob.value


# ---- pairwise g2o refinement (refine_oracle.c; SURVEY.md 8a row a16) ---------------------------------------------

def get_transform_from_matches_g2o(params: OParams, xyz_newer, kp_newer, xyz_older, kp_older, matches, sel, T4x4, iterations):
    """getTransformFromMatchesG2O (transformation_estimation.cpp:126-170).  kp_*: (n, 2) pixel coordinates;
    T4x4: float 4x4 initial estimate (row-major numpy view of the Matrix4f); returns the refined float 4x4."""
    x1 = np.ascontiguousarray(xyz_newer, np.float32); x2 = np.ascontiguousarray(xyz_older, np.float32)
    k1 = np.ascontiguousarray(kp_newer, np.float32).reshape(-1, 2); k2 = np.ascontiguousarray(kp_older, np.float32).reshape(-1, 2)
    m = np.ascontiguousarray(matches, DMATCH_DTYPE)
    s = np.ascontiguousarray(sel, np.int32)
    T = np.array(np.asarray(T4x4, np.float32).T, order="C")  # column-major storage; a copy: the call writes the result into it
    lib().oracle_get_transform_from_matches_g2o(C.byref(params), _p(x1), _p(k1), _p(x2), _p(k2), _p(m), _p(s), C.c_int(len(s)), _p(T),
                                                C.c_int(int(iterations)))
    return T.T.copy()


def refine_g2o(params: OParams, iterations, xyz_newer, kp_newer, xyz_older, kp_older, matches, T4x4, rmse, inl_mask, valid_iterations=0):
    """node.cpp:1225-1268 on top of a RANSAC result.  inl_mask: uint8 per match.  Returns (T, rmse, inl_mask, n_inl, valid_it)."""
    x1 = np.ascontiguousarray(xyz_newer, np.float32); x2 = np.ascontiguousarray(xyz_older, np.float32)
    k1 = np.ascontiguousarray(kp_newer, np.float32).reshape(-1, 2); k2 = np.ascontiguousarray(kp_older, np.float32).reshape(-1, 2)
    m = np.ascontiguousarray(matches, DMATCH_DTYPE)
    T = np.array(np.asarray(T4x4, np.float32).T, order="C")  # a copy: the call writes the result into it
    inl = np.ascontiguousarray(inl_mask, np.uint8).copy()
    r = C.c_float(float(rmse)); n = C.c_int(int(inl.sum())); vi = C.c_int(int(valid_iterations))
    lib().oracle_refine_g2o(C.byref(params), C.c_int(int(iterations)), _p(x1), _p(k1), _p(x2), _p(k2), _p(m), C.c_int(len(m)), _p(T),
                            C.byref(r), _p(inl), C.byref(n), C.byref(vi))
    return T.T.copy(), float(r.value), inl, int(n.value), int(vi.value)


# ---- environment measurement model (emm_oracle.c; SURVEY.md 8f rank 3) --------------------------------------------

def create_cloud_z(depth, step=2, scaling=1.0, min_depth=0.1):
    d = np.ascontiguousarray(depth, np.float32)
    h, w = d.shape
    out = np.zeros(((h + step - 1) // step, (w + step - 1) // step), np.float32)
    lib().oracle_create_cloud_z(_p(d), C.c_int(w), C.c_int(h), C.c_int(step), C.c_float(scaling), C.c_float(min_depth), _p(out))
    return out


def pairwise_observation(params: OParams, T4x4, newer_z, newerK, older_z, olderK, cloud_step=2, skip_step=8):
    """pairwiseObservationLikelihood (node.cpp:1520-1554): returns uint32[4] = inlier, outlier, occluded, all points."""
    T = np.ascontiguousarray(np.asarray(T4x4, np.float32).T)
    nz = np.ascontiguousarray(newer_z, np.float32); oz = np.ascontiguousarray(older_z, np.float32)
    nk = np.ascontiguousarray(newerK, np.float32); ok = np.ascontiguousarray(olderK, np.float32)
    out = np.zeros(4, np.uint32)
    lib().oracle_pairwise_observation(C.byref(params), _p(T), _p(nz), C.c_int(nz.shape[1]), C.c_int(nz.shape[0]), _p(nk), _p(oz),
                                      C.c_int(oz.shape[1]), C.c_int(oz.shape[0]), _p(ok), C.c_int(cloud_step), C.c_int(skip_step), _p(out))
    return out


def observation_criterion_met(inliers, outliers, occluded, obs_thresh):
    q = C.c_double(0.0)
    ok = lib().oracle_observation_criterion_met(C.c_uint32(int(inliers)), C.c_uint32(int(outliers)),
                                                C.c_uint32(int(inliers + outliers + occluded)), C.c_double(obs_thresh), C.byref(q))
    return bool(ok), q.value
