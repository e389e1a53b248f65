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
        ("use_feature_min_depth_", C.c_uint8), ("allow_features_without_depth_", C.c_uint8), ("reserved_", C.c_uint8 * 2),
    ]


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
assert PAIR_RESULT_DTYPE.itemsize == C.sizeof(PairResult) == 120
assert DMATCH_DTYPE.itemsize == C.sizeof(DMatch) == 16
assert KEYPOINT_DTYPE.itemsize == C.sizeof(KeyPoint) == 28

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
    lib.rgbdslam_b200_node_download_keypoints.argtypes = [u64, vp]
    lib.rgbdslam_b200_orb_debug_detect_path.argtypes = [C.c_int]
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

    def nodes_create(self, det: int, gray, depth, mask, K4, ids=None, mask_from_depth: bool = False):
        """gray [F,H,W] u8, depth [F,H,W] f32, mask [F,H,W] u8 or None -> (handles, n_features).  numpy arrays or pinned torch
        tensors (copied from asynchronously).  mask_from_depth: derive the detection mask on the device (depthToCV8UC1)."""
        if isinstance(gray, np.ndarray):
            gray = np.ascontiguousarray(gray, np.uint8)
            depth = np.ascontiguousarray(depth, np.float32)
            mask = None if mask is None else np.ascontiguousarray(mask, np.uint8)
        F, H, W = gray.shape
        K4 = np.ascontiguousarray(K4, np.float32)
        ids = None if ids is None else np.ascontiguousarray(ids, np.int32)
        handles = np.zeros(F, np.uint64)
        nf = np.zeros(F, np.int32)
        self._check(self.lib.rgbdslam_b200_nodes_create_ex(det, F, _ptr(gray), _ptr(depth), _ptr(None if mask_from_depth else mask), W, H,
                                                           _ptr(K4), _ptr(ids), 1 if mask_from_depth else 0, _ptr(handles), _ptr(nf)))
        self._nodes += [int(h) for h in handles]
        return [int(h) for h in handles], nf

    def nodes_create_sharded(self, det: int, comm: int, total_frames: int, gray, depth, mask, K4, ids=None,
                             mask_from_depth: bool = False):
        """Frame-sharded nodes_create: gray / depth / mask hold THIS rank's frames (sharding.frame_shard); returns handles and
        feature counts of ALL total_frames nodes (every rank ends up holding every node)."""
        if isinstance(gray, np.ndarray):
            gray = np.ascontiguousarray(gray, np.uint8)
            depth = np.ascontiguousarray(depth, np.float32)
            mask = None if mask is None else np.ascontiguousarray(mask, np.uint8)
        _, H, W = gray.shape
        K4 = np.ascontiguousarray(K4, np.float32)
        ids = None if ids is None else np.ascontiguousarray(ids, np.int32)
        handles = np.zeros(total_frames, np.uint64)
        nf = np.zeros(total_frames, np.int32)
        own = gray.shape[0] > 0
        self._check(self.lib.rgbdslam_b200_nodes_create_sharded(
            det, C.c_uint64(comm), total_frames, _ptr(gray) if own else None, _ptr(depth) if own else None,
            _ptr(None if (mask_from_depth or not own) else mask), W, H, _ptr(K4), _ptr(ids), 1 if mask_from_depth else 0, _ptr(handles), _ptr(nf)))
        self._nodes += [int(h) for h in handles]
        return [int(h) for h in handles], nf

    def orb_debug_detect_path(self, unfused: bool):
        self._check(self.lib.rgbdslam_b200_orb_debug_detect_path(1 if unfused else 0))

    def orb_debug_plane(self, which: int, cell: int, level: int) -> np.ndarray:
        buf = np.zeros(1024 * 1024, np.uint8)
        w, h = C.c_int(), C.c_int()
        self._check(self.lib.rgbdslam_b200_orb_debug_plane(which, cell, level, _ptr(buf), buf.size, C.byref(w), C.byref(h)))
        return buf[: w.value * h.value].reshape(h.value, w.value).copy()

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
