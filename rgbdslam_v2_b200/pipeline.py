"""Offline mirror of the reference's back-end glue around the hot path (host logic, numpy only):

  candidate_pairs   the candidate set of GraphManager::nodeComparisons (graph_manager.cpp:516-526) in the offline
                    formulation of SURVEY.md 8e: (predecessor_candidates - 1) = 3 sequential predecessors, 4 sliding-window
                    neighbours, 4 uniform-random earlier frames (no Dijkstra feedback)
  build_graph       how nodeComparisons / addEdgeToG2O turn MatchingResults into vertices and edges
                    (graph_manager.cpp:550-583, 636-655, 811-898): vertex estimate = v1 * T of the accepted edge with the most
                    inliers, constant-position identity edge (information I / dt) when the predecessor was not matched
  run_sequence      frames -> nodes -> pair matching -> graph -> optimizeGraph -> trajectory
The compute steps go through a backend object (the CUDA Frontend in the product; tests plug in the CPU oracle)."""
from __future__ import annotations

import numpy as np

from .synth import pose_compose


def rot_to_quat(R: np.ndarray) -> np.ndarray:
    """Eigen::Quaternion(Matrix3) (Shepperd's method), returns (x, y, z, w)."""
    R = np.asarray(R, np.float64)
    t = np.trace(R)
    if t > 0:
        s = np.sqrt(t + 1.0) * 2
        q = np.array([(R[2, 1] - R[1, 2]) / s, (R[0, 2] - R[2, 0]) / s, (R[1, 0] - R[0, 1]) / s, 0.25 * s])
    else:
        i = int(np.argmax(np.diag(R)))
        j, k = (i + 1) % 3, (i + 2) % 3
        s = np.sqrt(R[i, i] - R[j, j] - R[k, k] + 1.0) * 2
        q = np.zeros(4)
        q[i] = 0.25 * s
        q[j] = (R[j, i] + R[i, j]) / s
        q[k] = (R[k, i] + R[i, k]) / s
        q[3] = (R[k, j] - R[j, k]) / s
    return q / np.linalg.norm(q)


def mat_to_pose7(T: np.ndarray) -> np.ndarray:
    T = np.asarray(T, np.float64)
    return np.concatenate([T[:3, 3], rot_to_quat(T[:3, :3])])


def quat_to_rot(q):
    x, y, z, w = q / np.linalg.norm(q)
    return np.array([[1 - 2 * (y * y + z * z), 2 * (x * y - z * w), 2 * (x * z + y * w)],
                     [2 * (x * y + z * w), 1 - 2 * (x * x + z * z), 2 * (y * z - x * w)],
                     [2 * (x * z - y * w), 2 * (y * z + x * w), 1 - 2 * (x * x + y * y)]])


def pose7_to_mat(p):
    T = np.eye(4)
    T[:3, :3] = quat_to_rot(np.asarray(p[3:], np.float64))
    T[:3, 3] = p[:3]
    return T


def candidate_pairs(n_frames: int, seed: int = 0, seq: int = 3, window: int = 4, sampled: int = 4):
    """[(newer, older)] in processing order (per new frame: predecessors first)."""
    rng = np.random.default_rng(seed)
    pairs = []
    for k in range(1, n_frames):
        cand = [k - d for d in range(1, seq + 1) if k - d >= 0]
        cand += [k - d for d in range(seq + 1, seq + window + 1) if k - d >= 0]
        lo = k - (seq + window) - 1
        if lo >= 0:
            pool = np.arange(0, lo + 1)
            cand += sorted(rng.choice(pool, size=min(sampled, len(pool)), replace=False).tolist(), reverse=True)
        pairs += [(k, c) for c in cand]
    return pairs


def build_graph(pairs, results, n_frames: int, dt: float = 1.0 / 30.0):
    """results: structured array (id1, id2, n_inliers, ransac_trafo [16, column-major], info_scale) aligned with pairs.
    Returns dict(init [n,7], fixed, ij, meas, info, n_valid_edges, n_const_edges)."""
    poses = np.zeros((n_frames, 7))
    poses[:, 6] = 1.0
    ij, meas, info = [], [], []
    by_new = {}
    for (newer, older), r in zip(pairs, results):
        by_new.setdefault(newer, []).append((older, r))
    n_const = 0
    for k in range(1, n_frames):
        best_inl = 0
        have_vertex = False
        predecessor_matched = False
        for older, r in by_new.get(k, []):
            if r["id1"] < 0:
                continue
            T = np.asarray(r["ransac_trafo"], np.float64).reshape(4, 4).T  # edge.transform = final_trafo.cast<double>()
            z = mat_to_pose7(T)
            set_estimate = int(r["n_inliers"]) > best_inl
            if not have_vertex or set_estimate:  # addEdgeToG2O: new vertex = v1 * T, or setEstimate when more inliers
                poses[k] = pose_compose(poses[older], z)
                have_vertex = True
            if int(r["n_inliers"]) > best_inl:
                best_inl = int(r["n_inliers"])
            ij.append((older, k)); meas.append(z); info.append(np.eye(6).reshape(-1) * float(r["info_scale"]))
            if older == k - 1:
                predecessor_matched = True
        if not predecessor_matched:  # constant position assumption (graph_manager.cpp:636-655), time delta < 0.1 s
            z = np.array([0, 0, 0, 0, 0, 0, 1.0])
            poses[k] = pose_compose(poses[k - 1], z)  # addEdgeToG2O(..., set_estimate = true)
            ij.append((k - 1, k)); meas.append(z); info.append(np.eye(6).reshape(-1) / dt)
            n_const += 1
    fixed = np.zeros(n_frames, np.uint8)
    fixed[0] = 1  # pose_relative_to = first (graph_manager.cpp:933-936)
    return dict(init=poses, fixed=fixed, ij=np.array(ij, np.int32).reshape(-1, 2), meas=np.array(meas).reshape(-1, 7),
                info=np.array(info).reshape(-1, 36), n_valid_edges=len(ij) - n_const, n_const_edges=n_const)


def run_sequence(backend, gray, depth, mask, K4, seed: int = 0, stop: float = 0.01):
    """backend: .construct_nodes(gray, depth, mask, K4) -> nodes; .match(nodes, pairs, seed) -> results;
    .optimize(graph, stop) -> (poses, chi2).  Returns dict(traj [n,7], graph, results, chi2)."""
    n = len(gray)
    nodes = backend.construct_nodes(gray, depth, mask, K4)
    pairs = candidate_pairs(n, seed)
    results = backend.match(nodes, pairs, seed)
    graph = build_graph(pairs, results, n)
    traj, chi2 = backend.optimize(graph, stop)
    return dict(traj=traj, graph=graph, results=results, chi2=chi2, pairs=pairs)


def build_graph_fast(pairs: np.ndarray, results, n_frames: int, dt: float = 1.0 / 30.0):
    """build_graph for long sequences: same vertices / edges / order, the per-edge work vectorised (22 k pairs in C4).
    pairs: int array [P,2] (newer, older) grouped by newer frame in processing order."""
    pairs = np.asarray(pairs, np.int64).reshape(-1, 2)
    valid = np.asarray(results["id1"]) >= 0
    T = np.asarray(results["ransac_trafo"], np.float64).reshape(-1, 4, 4).transpose(0, 2, 1)  # column-major -> row-major
    z = np.zeros((len(pairs), 7))
    for i in np.nonzero(valid)[0]:
        z[i] = mat_to_pose7(T[i])
    inl = np.asarray(results["n_inliers"]).astype(np.int64)
    scale = np.asarray(results["info_scale"], np.float64)
    poses = np.zeros((n_frames, 7)); poses[:, 6] = 1.0
    ij, meas, info_scale = [], [], []
    n_const = 0
    ident = np.array([0, 0, 0, 0, 0, 0, 1.0])
    # pairs of frame k are contiguous
    starts = np.searchsorted(pairs[:, 0], np.arange(n_frames + 1))
    for k in range(1, n_frames):
        lo, hi = starts[k], starts[k + 1]
        idx = lo + np.nonzero(valid[lo:hi])[0]
        pred = False
        if len(idx):
            best = idx[np.argmax(inl[idx])]  # first maximum: later edges only override with strictly more inliers
            poses[k] = pose_compose(poses[pairs[best, 1]], z[best])
            for i in idx:
                ij.append((pairs[i, 1], k)); meas.append(z[i]); info_scale.append(scale[i])
            pred = bool((pairs[idx, 1] == k - 1).any())
        if not pred:
            poses[k] = pose_compose(poses[k - 1], ident)
            ij.append((k - 1, k)); meas.append(ident); info_scale.append(1.0 / dt)
            n_const += 1
    fixed = np.zeros(n_frames, np.uint8); fixed[0] = 1
    info = np.zeros((len(ij), 36)); info[:, ::7] = np.asarray(info_scale)[:, None]
    return dict(init=poses, fixed=fixed, ij=np.array(ij, np.int32).reshape(-1, 2), meas=np.array(meas).reshape(-1, 7), info=info,
                n_valid_edges=len(ij) - n_const, n_const_edges=n_const)


def match_pairs_pipelined(fe, handles, pairs: np.ndarray, seed: int, first_pair_index: int = 0, batch: int = 256, depth: int = 5,
                          out: np.ndarray | None = None):
    """Node::matchNodePair for a long pair list: batches of `batch` pairs kept in flight on `depth` pipeline slots
    (rgbdslam_b200_match_pairs_submit / _wait).  pairs: [P,2] (newer, older) indices into `handles`; the RNG key of pair i
    is first_pair_index + i, so a sharded list reproduces the single-process results.  Returns the edge records."""
    from ._capi import PAIR_RESULT_DTYPE
    pairs = np.asarray(pairs, np.int64).reshape(-1, 2)
    n = len(pairs)
    res = out if out is not None else np.zeros(n, PAIR_RESULT_DTYPE)
    h = np.asarray(handles, np.uint64)
    newer = np.ascontiguousarray(h[pairs[:, 0]]); older = np.ascontiguousarray(h[pairs[:, 1]])
    nb = (n + batch - 1) // batch
    for b in range(nb):
        slot = 1 + b % depth
        if b >= depth:
            fe.wait_slot(slot)
        i0, i1 = b * batch, min(n, (b + 1) * batch)
        fe.submit_node_pairs(slot, newer[i0:i1], older[i0:i1], (res[i0:i1], None, None), seed=seed,
                             first_pair_index=first_pair_index + i0)
    for b in range(max(0, nb - depth), nb):
        fe.wait_slot(1 + b % depth)
    return res


class GpuBackend:
    """The product path: every compute step is a C-ABI call into the CUDA library."""

    def __init__(self, frontend):
        self.fe = frontend
        self.det = frontend.detector_create()

    def construct_nodes(self, gray, depth, mask, K4):
        handles, _ = self.fe.nodes_create(self.det, gray, depth, mask, K4, ids=np.arange(len(gray), dtype=np.int32))
        return handles

    def match(self, nodes, pairs, seed):
        newer = [nodes[a] for a, _ in pairs]
        older = [nodes[b] for _, b in pairs]
        res, _, _ = self.fe.match_node_pairs(newer, older, seed=seed, want_matches=False)
        return res

    def n_features(self, handle) -> int:
        return self.fe.node_num_features(handle)

    def match_one_to_many(self, node, olds, seed, first_pair_index=None):
        """The comparisons of one new node as ONE batched call (graph_manager.cpp:548); RNG keys = first_pair_index + k,
        by default 64 * node id + k."""
        first = 64 * node.id if first_pair_index is None else first_pair_index
        res, _, _ = self.fe.match_node_pairs([node.handle] * len(olds), [o.handle for o in olds], seed=seed,
                                             first_pair_index=first, want_matches=False)
        return res

    def optimize(self, graph, stop):
        x, chi2, _, _ = self.fe.optimize_graph(graph["init"], graph["fixed"], graph["ij"], graph["meas"], graph["info"], stop=stop)
        return x, chi2


# ---------------------------------------------------------------------------------------------------
# Batch evaluation back-end (SURVEY.md 8f rank 1): prune / re-optimise / trajectory export.

def prune_edges(graph: dict, per_edge_chi2: np.ndarray, thresh: float) -> int:
    """GraphManager::pruneEdgesWithErrorAbove (graph_manager.cpp:1106-1246), in place on `graph`.
    For every ACTIVE edge with chi2 > thresh: measurement := identity; non-consecutive edges are removed from the
    active set when both end vertices have more than one incident edge, else their information becomes 1e-100 * I;
    consecutive edges get information I.  Returns the number of edges over the threshold."""
    ij, n = graph["ij"], len(graph["ij"])
    active = graph.setdefault("active", np.ones(n, bool))
    # v->edges().size(): every edge ever added to the optimizer counts (removal only leaves the active set)
    deg = np.bincount(ij.reshape(-1), minlength=len(graph["init"]))
    ident = np.array([0, 0, 0, 0, 0, 0, 1.0])
    counter = 0
    for k in np.nonzero(active)[0]:
        if per_edge_chi2[k] > thresh:
            counter += 1
            graph["meas"][k] = ident
            a, b = ij[k]
            if abs(int(a) - int(b)) != 1:
                if deg[a] > 1 and deg[b] > 1:
                    active[k] = False
                else:
                    graph["info"][k] = np.eye(6).reshape(-1) * 1e-100
            else:
                graph["info"][k] = np.eye(6).reshape(-1)
    return counter


def active_view(graph: dict) -> dict:
    a = graph.get("active")
    if a is None:
        return graph
    return dict(graph, ij=np.ascontiguousarray(graph["ij"][a]), meas=np.ascontiguousarray(graph["meas"][a]),
                info=np.ascontiguousarray(graph["info"][a]))


def evaluation_sequence(backend, graph: dict, stop: float = 0.01):
    """OpenNIListener::evaluation (openni_listener.cpp:431-466): optimise, then prune at chi2 5 / 1 / 0.25, each
    followed by optimizeGraph(-100) (= the parameter's stop rule) or a single iteration when nothing was pruned.
    backend needs .optimize(graph, stop) and .edge_chi2(poses, graph).  Returns the trajectories of levels 1..4."""
    g = dict(graph, meas=graph["meas"].copy(), info=graph["info"].copy())
    levels = []
    x, chi2 = backend.optimize(active_view(g), stop)
    g["init"] = x
    levels.append((x.copy(), chi2, 0))
    for thr in (5.0, 1.0, 0.25):
        full = backend.edge_chi2(x, g)
        n = prune_edges(g, full, thr)
        x, chi2 = backend.optimize(active_view(g), stop if n > 0 else 1.0)
        g["init"] = x
        levels.append((x.copy(), chi2, n))
    return levels


def save_trajectory(path: str, poses7: np.ndarray, stamps: np.ndarray):
    """TUM trajectory format written by logTransform (misc.cpp:90-93): timestamp tx ty tz qx qy qz qw, fixed notation."""
    with open(path, "w") as f:
        f.write("# TF Coordinate Frame ID: (data: )\n")
        for t, p in zip(stamps, poses7):
            f.write("%f %f %f %f %f %f %f %f\n" % (t, *p))


def _gpu_edge_chi2(self, poses, graph):
    _, pe = self.fe.graph_chi2(poses, graph["ij"], graph["meas"], graph["info"], per_edge=True)
    return pe


GpuBackend.edge_chi2 = _gpu_edge_chi2
