"""TEST INFRASTRUCTURE (host-logic oracle): Python twin of the product's C++ shim include/rgbdslam_b200/graph_manager.hpp,
used by tests/ to drive the online front with either backend (CUDA library or CPU oracle).  The product implementation of
this logic is the C++ shim; nothing in rgbdslam_v2_b200/ imports this module.

Host-side mirror of the reference's ONLINE graph front (SURVEY.md 8a row a18 / 8f rank 2): which old nodes a new
node is compared with, which MatchingResults become edges, keyframes, the constant-position fallback, and when the
optimiser runs.  Pure host logic (numpy); every compute step is a backend call -- the CUDA library in the product
(`pipeline.GpuBackend`: the <= 12 comparisons of one new node are ONE `rgbdslam_b200_match_pairs` batch, the
counterpart of `QtConcurrent::blockingMapped(nodes_to_comp, &Node::matchNodePair)`, graph_manager.cpp:548).

Reference map (src/graph_manager.cpp unless noted):
  GraphManager.add_node                      addNode :681-782, firstNode :361-409
  GraphManager.node_comparisons              nodeComparisons :421-658
  GraphManager.potential_edge_targets        getPotentialEdgeTargetsWithDijkstra :204-324
  GraphManager.add_edge                      addEdgeToG2O :811-898
  GraphManager.add_keyframe                  addKeyframe :784-809
  is_big_trafo / is_small_trafo / trafo_size misc.cpp:272-315
  GraphManager.graph_arrays                  fixationOfVertices :911-937 on the persistent fixed flags (:381, :889-892,
                                             :1031-1036)
The reference draws from the global rand(); here every draw comes from the library's counter-based generator keyed
by (seed, new node id), so a run is reproducible (parity on the selected sets is therefore statistical).
g2o's HyperDijkstra is not under /root/reference; its published behaviour is restated in `_geodesic_ball`.

Every decision, every estimate and every optimiser input equals the C++ shim's bit for bit: the pose algebra
(`pose_from_matrix`, `compose`, `inverse`) is the shim's, operation for operation.  Where the shim departs from the
reference on purpose, so does this twin:
  - the feature gate reads `n_features`, the node's feature count; the reference reads the 2-D keypoint count, which
    equals the 3-D count for every node the Node constructor builds;
  - the new node is never its own geodesic candidate (the reference can draw it and compare it with itself);
  - the initial comparison (min_translation_meter / min_rotation_degree > 0) is keyed 64 id + 63, a pair index the
    batched comparisons (64 id + k, k < 12) never take;
  - the constant-position time delta is floored at 1 ms;
  - an optimisation without any fixed vertex fixes its first vertex (the PCG needs an anchor; g2o's damped LM has none).
`records` keeps, per add_node call, what the shim's trace reports: the return value, the candidates, the edges added,
keyframes, earliest_loop_closure_node, the estimates, and the input and output of every optimisation."""
from __future__ import annotations

import inspect
import math

from dataclasses import dataclass, field

import numpy as np

_M64 = (1 << 64) - 1


def _mix64(x: int) -> int:
    x = (x + 0x9E3779B97F4A7C15) & _M64
    x = ((x ^ (x >> 30)) * 0xBF58476D1CE4E5B9) & _M64
    x = ((x ^ (x >> 27)) * 0x94D049BB133111EB) & _M64
    return x ^ (x >> 31)


class _Rand:
    """rand() stand-in: the splitmix64 counter generator of the CUDA library / oracle (stream 0xC0 = candidate selection)."""

    def __init__(self, seed: int, node_id: int):
        self.key = _mix64((seed & _M64) ^ _mix64(node_id & _M64))
        self.ctr = 0

    def __call__(self) -> int:
        v = _mix64(self.key ^ ((0xC0 << 32) | self.ctr)) >> 33
        self.ctr += 1
        return v


def _quat_to_rot(q) -> list:
    """graph_manager.hpp quatToRot: row-major 3 x 3 of the normalised quaternion (x, y, z, w)."""
    n = math.sqrt(q[0] * q[0] + q[1] * q[1] + q[2] * q[2] + q[3] * q[3])
    x, y, z, w = q[0] / n, q[1] / n, q[2] / n, q[3] / n
    return [1 - 2 * (y * y + z * z), 2 * (x * y - z * w), 2 * (x * z + y * w),
            2 * (x * y + z * w), 1 - 2 * (x * x + z * z), 2 * (y * z - x * w),
            2 * (x * z - y * w), 2 * (y * z + x * w), 1 - 2 * (x * x + y * y)]


def _rot_to_quat(R) -> list:
    """graph_manager.hpp rotToQuat: Eigen::Quaternion(Matrix3), normalised."""
    q = [0.0] * 4
    tr = R[0] + R[4] + R[8]
    if tr > 0:
        s = math.sqrt(tr + 1.0)
        q[3] = 0.5 * s
        s = 0.5 / s
        q[0] = (R[7] - R[5]) * s; q[1] = (R[2] - R[6]) * s; q[2] = (R[3] - R[1]) * s
    else:
        i = 0
        if R[4] > R[0]:
            i = 1
        if R[8] > R[4 * i]:
            i = 2
        j = (i + 1) % 3
        k = (j + 1) % 3
        s = math.sqrt(R[4 * i] - R[4 * j] - R[4 * k] + 1.0)
        q[i] = 0.5 * s
        s = 0.5 / s
        q[3] = (R[3 * k + j] - R[3 * j + k]) * s
        q[j] = (R[3 * j + i] + R[3 * i + j]) * s
        q[k] = (R[3 * k + i] + R[3 * i + k]) * s
    n = math.sqrt(q[0] * q[0] + q[1] * q[1] + q[2] * q[2] + q[3] * q[3])
    return [v / n for v in q]


def pose_from_matrix(T) -> np.ndarray:
    """graph_manager.hpp poseFromIsometry: (t, q) of a row-major 4 x 4."""
    T = np.asarray(T, np.float64)
    R = [float(T[r, c]) for r in range(3) for c in range(3)]
    return np.array([float(T[0, 3]), float(T[1, 3]), float(T[2, 3])] + _rot_to_quat(R))


def compose(a, b) -> np.ndarray:
    """graph_manager.hpp compose: a * b of two 7-vectors."""
    a = [float(v) for v in a]; b = [float(v) for v in b]
    Ra, Rb = _quat_to_rot(a[3:]), _quat_to_rot(b[3:])
    R = [Ra[3 * r] * Rb[c] + Ra[3 * r + 1] * Rb[3 + c] + Ra[3 * r + 2] * Rb[6 + c] for r in range(3) for c in range(3)]
    t = [a[r] + Ra[3 * r] * b[0] + Ra[3 * r + 1] * b[1] + Ra[3 * r + 2] * b[2] for r in range(3)]
    return np.array(t + _rot_to_quat(R))


def inverse(a) -> np.ndarray:
    """graph_manager.hpp inverse of a 7-vector."""
    a = [float(v) for v in a]
    R = _quat_to_rot(a[3:])
    t = [-(R[r] * a[0] + R[3 + r] * a[1] + R[6 + r] * a[2]) for r in range(3)]
    return np.array(t + [-a[3], -a[4], -a[5], a[6]])


_IDENTITY7 = (0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 1.0)


@dataclass
class Params:
    """The ParameterServer entries this logic reads (defaults: parameter_server.cpp:85-123)."""
    min_matches: int = 20
    predecessor_candidates: int = 4
    neighbor_candidates: int = 4
    min_sampled_candidates: int = 4
    geodesic_depth: int = 3
    min_translation_meter: float = 0.0
    min_rotation_degree: float = 0.0
    max_translation_meter: float = 1e10
    max_rotation_degree: float = 360.0
    keep_all_nodes: bool = False
    keep_good_nodes: bool = False
    optimizer_skip_step: int = 1
    optimizer_iterations: float = 0.01
    odom_frame_name: str = ""
    max_connections: int = -1   # node.cpp:1310-1312: > 0 stops comparing once the node has that many accepted transformations
    pose_relative_to: str = "first"  # fixationOfVertices strategy: first / previous / largest_loop / inaffected


def trafo_size(T: np.ndarray):
    """misc.cpp:272-276: rotation angle about the axis (degrees) and translation norm (graph_manager.hpp trafoSize)."""
    T = np.asarray(T, np.float64)
    c = (float(T[0, 0]) + float(T[1, 1]) + float(T[2, 2]) - 1) / 2
    angle = math.acos(c) * 180.0 / math.pi if -1.0 <= c <= 1.0 else math.nan  # acos(>1) = NaN like the reference
    x, y, z = float(T[0, 3]), float(T[1, 3]), float(T[2, 3])
    return angle, math.sqrt(x * x + y * y + z * z)


def is_big_trafo(T: np.ndarray, p: Params) -> bool:
    angle, dist = trafo_size(T)
    return dist > p.min_translation_meter or angle > p.min_rotation_degree  # misc.cpp:278-283 (NaN compares false)


def is_small_trafo(T: np.ndarray, seconds: float, p: Params) -> bool:
    if seconds <= 0.0:
        return True  # misc.cpp:304-307
    angle, dist = trafo_size(T)
    return dist / seconds < p.max_translation_meter and angle / seconds < p.max_rotation_degree


@dataclass
class GraphNode:
    id: int
    handle: object            # what the backend needs to match this node (device handle / feature arrays)
    n_features: int
    stamp: float
    vertex: bool = False      # has a vertex in the optimiser (vertex id == node id here)
    matchable: bool = True
    valid_tf_estimate: bool = True


@dataclass
class GraphManager:
    backend: object
    params: Params = field(default_factory=Params)
    seed: int = 0

    def __post_init__(self):
        self.nodes: dict[int, GraphNode] = {}
        self.poses: dict[int, np.ndarray] = {}            # vertex estimates (7-vectors)
        self.edges: list[tuple[int, int]] = []            # (id1 = older, id2 = newer)
        self.meas: list[np.ndarray] = []
        self.info: list[np.ndarray] = []
        self.adj: dict[int, set[int]] = {}
        self.keyframe_ids: list[int] = []
        self.curr_best = dict(id1=-1, n_inliers=0)
        self.loop_closure_edges = self.sequential_edges = 0
        self.n_const_edges = 0
        self.last_chi2 = None
        self.comparisons: list[tuple[int, list[int]]] = []  # (new id, compared-with ids) for inspection / tests
        self.earliest_loop_closure_node = 0
        # vertices with setFixed(true): the first one (:381); "inaffected" frees both ends of every new edge (:889-892); the
        # end of an optimisation fixes ("inaffected") or frees (every other strategy) them all (:1031-1036)
        self.fixed_ids: set[int] = set()
        self.records: list[dict] = []   # one per add_node call, see the module docstring
        self._optimizations: list[dict] = []

    def _reset(self):
        """resetGraph, as far as this twin keeps state (the comparison and optimisation logs stay)."""
        self.nodes.clear(); self.poses.clear(); self.edges.clear(); self.meas.clear(); self.info.clear(); self.adj.clear()
        self.keyframe_ids.clear(); self.fixed_ids.clear()
        self.curr_best = dict(id1=-1, n_inliers=0)
        self.loop_closure_edges = self.sequential_edges = self.n_const_edges = 0
        self.earliest_loop_closure_node = 0

    # ---- graph_manager.cpp:361-409
    def _first_node(self, node: GraphNode):
        node.id = len(self.nodes)
        self.nodes[node.id] = node
        node.vertex = True
        self.poses[node.id] = np.array(_IDENTITY7)  # init_base_pose_ = identity without ground truth
        self.fixed_ids.add(node.id)                 # reference_pose->setFixed(true) (:381)
        self.adj[node.id] = set()
        self.add_keyframe(node.id)

    def add_keyframe(self, node_id: int):
        self.keyframe_ids.append(node_id)

    # ---- graph_manager.cpp:811-898
    def add_edge(self, id1: int, id2: int, T: np.ndarray, info: np.ndarray, large_edge: bool, set_estimate: bool) -> bool:
        n1, n2 = self.nodes.get(id1), self._pending if id2 == self._pending.id else self.nodes.get(id2)
        v1, v2 = n1 is not None and n1.vertex, n2 is not None and n2.vertex
        if (not v1 or not v2) and not large_edge:
            return False  # :828-833 edge to a new vertex is too short
        if not v1 and not v2:
            return False
        z = pose_from_matrix(T)
        if not v2:
            n2.vertex = True
            self.poses[id2] = compose(self.poses[id1], z)  # :860
            self.adj.setdefault(id2, set())
        elif not v1:  # ":850 unexpected by the programmer"
            n1.vertex = True
            self.poses[id1] = compose(self.poses[id2], inverse(z))
            self.adj.setdefault(id1, set())
        elif set_estimate:
            self.poses[id2] = compose(self.poses[id1], z)  # :866
        self.edges.append((id1, id2)); self.meas.append(z); self.info.append(np.asarray(info, np.float64).reshape(36))
        self.adj[id1].add(id2); self.adj[id2].add(id1)
        if abs(id1 - id2) > self.params.predecessor_candidates:
            self.loop_closure_edges += 1  # :882-886
        else:
            self.sequential_edges += 1
        if self.params.pose_relative_to == "inaffected":  # :889-892
            self.fixed_ids.discard(id1); self.fixed_ids.discard(id2)
        elif self.params.pose_relative_to == "largest_loop":  # :893-896: only this strategy lowers it
            self.earliest_loop_closure_node = min(self.earliest_loop_closure_node, id1, id2)
        return True

    # ---- g2o::HyperDijkstra::shortestPaths(v, UniformCostFunction, maxDistance) + visited()
    def _geodesic_ball(self, source: int, max_distance: float) -> set[int]:
        """Vertices g2o marks visited: the source plus every vertex whose hop count d satisfies d < maxDistance
        (hyper_dijkstra.cpp relaxes z only `if (zDistance + conditioner < known && zDistance < maxDistance)`)."""
        dist = {source: 0}
        frontier = [source]
        while frontier:
            nxt = []
            for u in frontier:
                for z in self.adj.get(u, ()):
                    d = dist[u] + 1
                    if z not in dist and d < max_distance:
                        dist[z] = d
                        nxt.append(z)
            frontier = nxt
        return set(dist)

    # ---- graph_manager.cpp:204-324
    def potential_edge_targets(self, rand: _Rand, sequential: int, geodesic: int, sampled: int, predecessor_id: int = -1,
                               include_predecessor: bool = False) -> list[int]:
        ids: list[int] = []
        n_graph = len(self.nodes)
        if predecessor_id < 0:
            predecessor_id = n_graph - 1
        n_vertices = sum(1 for n in self.nodes.values() if n.vertex)
        if n_vertices <= sequential + geodesic + sampled or n_vertices <= 1:  # :213-220 fewer nodes than targets: take all
            sequential = sequential + geodesic + sampled
            geodesic = sampled = 0
            predecessor_id = n_graph - 1
        if sequential > 0:
            i = 1
            while i < sequential + 1 and predecessor_id - i >= 0:  # :222-228
                ids.append(predecessor_id - i)
                i += 1
        if geodesic > 0:
            weights: dict[int, int] = {}
            for vid in sorted(self._geodesic_ball(predecessor_id, self.params.geodesic_depth)):  # std::map iterates by id
                if vid == self._pending.id:
                    continue  # the new node itself (the reference can draw it: a comparison of the node with itself)
                if not self.nodes[vid].matchable:
                    continue
                if vid < predecessor_id - sequential or (predecessor_id < vid <= n_graph - 1):  # :264
                    weights[vid] = abs(predecessor_id - vid)  # far-away neighbours are more likely
            total = sum(weights.values())
            while len(ids) < sequential + geodesic and weights:  # :273-293
                pick = rand() % total
                acc = 0
                for vid in sorted(weights):
                    acc += weights[vid]
                    if acc > pick:
                        ids.insert(0, vid)
                        total -= weights.pop(vid)
                        break
        if sampled > 0:
            pool = [k for k in self.keyframe_ids if k not in ids and self.nodes[k].matchable]  # :299-304
            while len(ids) < geodesic + sampled + sequential and pool:  # :307-314
                i = rand() % len(pool)
                ids.insert(0, pool[i])
                pool[i] = pool[-1]
                pool.pop()
        if include_predecessor:
            ids.append(predecessor_id)
        return ids

    def _match(self, node: GraphNode, olds: list, first_pair_index: int | None = None):
        """backend.match_one_to_many: the pairs (node, olds[k]) keyed first_pair_index + k, by default 64 id + k.  A backend
        whose match_one_to_many takes no first_pair_index (one whose results do not depend on the key) is always called with
        the default."""
        fn = self.backend.match_one_to_many
        if first_pair_index is None or "first_pair_index" not in inspect.signature(fn).parameters:
            return fn(node, olds, self.seed)
        return fn(node, olds, self.seed, first_pair_index=first_pair_index)

    # ---- graph_manager.cpp:421-658
    def node_comparisons(self, node: GraphNode) -> tuple[bool, bool]:
        """Returns (found_match, edge_to_keyframe)."""
        p = self.params
        if node.n_features < p.min_matches and not p.keep_all_nodes:
            return False, False
        node.id = len(self.nodes)
        self._pending = node
        self.earliest_loop_closure_node = node.id  # :444
        rand = _Rand(self.seed, node.id)
        n_edges_before = len(self.edges)
        edge_to_keyframe = False
        seq_prev = max(self.nodes)
        prev_best = -1  # `MatchingResult mr; int prev_best = mr.edge.id1;` -- always -1 (:452-453)
        self.curr_best = dict(id1=-1, n_inliers=0)
        predecessor_matched = False
        accepted = 0  # Node::initial_node_matches_ (node.cpp:1417): every transformation matchNodePair found for this node

        if p.min_translation_meter > 0.0 or p.min_rotation_degree > 0.0:  # initial comparison :458-513
            prev = self.nodes[len(self.nodes) - 1]
            r = self._match(node, [prev], 64 * node.id + 63)[0]
            if r["id1"] >= 0:
                accepted += 1
                T = np.asarray(r["ransac_trafo"], np.float64).reshape(4, 4).T
                dt = node.stamp - prev.stamp
                if not is_big_trafo(T, p) or not is_small_trafo(T, dt, p):
                    self.curr_best = dict(id1=int(r["id1"]), n_inliers=int(r["n_inliers"]))
                    return False, False
                if not self.add_edge(prev.id, node.id, T, np.eye(6) * float(r["info_scale"]), True, True):
                    return False, False
                self.nodes[node.id] = node
                edge_to_keyframe = prev.id in self.keyframe_ids
                prev.valid_tf_estimate = True
                self.curr_best = dict(id1=prev.id, n_inliers=int(r["n_inliers"]))
                predecessor_matched = True

        seq_cand, geod_cand, samp_cand = p.predecessor_candidates - 1, p.neighbor_candidates, p.min_sampled_candidates
        if predecessor_matched:
            targets = self.potential_edge_targets(rand, seq_cand, geod_cand, samp_cand, self.curr_best["id1"])
        else:
            targets = self.potential_edge_targets(rand, seq_cand, geod_cand, samp_cand, seq_prev, True)
        if prev_best >= 0 and prev_best not in targets:
            targets.append(prev_best)
        self.comparisons.append((node.id, list(targets)))

        results = self._match(node, [self.nodes[t] for t in targets]) if targets else []
        for t, r in zip(targets, results):  # :550-583 (result order == candidate order)
            if p.max_connections > 0 and accepted > p.max_connections:
                continue  # "enough is enough": matchNodePair returns an empty result (node.cpp:1310-1312)
            if r["id1"] < 0:
                continue
            accepted += 1
            T = np.asarray(r["ransac_trafo"], np.float64).reshape(4, 4).T
            dt = node.stamp - self.nodes[t].stamp
            more = int(r["n_inliers"]) > self.curr_best["n_inliers"]
            if is_small_trafo(T, dt, p) and self.add_edge(t, node.id, T, np.eye(6) * float(r["info_scale"]), is_big_trafo(T, p), more):
                self.nodes[node.id] = node
                if t == node.id - 1:
                    predecessor_matched = True
                self.nodes[t].valid_tf_estimate = True
                if more:
                    self.curr_best = dict(id1=t, n_inliers=int(r["n_inliers"]))
                if t in self.keyframe_ids:
                    edge_to_keyframe = True

        found_trafo = len(self.edges) != n_edges_before
        valid_odometry = bool(p.odom_frame_name)
        keep_anyway = p.keep_all_nodes or (node.n_features > p.min_matches and p.keep_good_nodes)
        dt_prev = abs(node.stamp - self.nodes[seq_prev].stamp)
        if (not found_trafo and valid_odometry) or (not found_trafo and keep_anyway) or (not predecessor_matched and dt_prev < 0.1):
            # constant position assumption :636-655 (information I / dt)
            self.add_edge(seq_prev, node.id, np.eye(4), np.eye(6) / max(dt_prev, 1e-3), True, True)  # :647, floored at 1 ms
            self.nodes[node.id] = node
            node.valid_tf_estimate = False
            self.curr_best = dict(id1=seq_prev, n_inliers=0)
            self.n_const_edges += 1
        return len(self.edges) > n_edges_before, edge_to_keyframe

    # ---- graph_manager.cpp:681-782
    def add_node(self, handle, n_features: int, stamp: float) -> bool:
        n_targets, n_edges = len(self.comparisons), len(self.edges)
        self._optimizations = []
        node = GraphNode(-1, handle, int(n_features), float(stamp))
        ret = self._add_node(node)
        reset = len(self.edges) < n_edges
        self.records.append(dict(
            ret=ret, id=node.id, n_features=node.n_features, targets=self.comparisons[-1][1] if len(self.comparisons) > n_targets else None,
            edges=[(a, b, self.meas[k], self.info[k]) for k, (a, b) in enumerate(self.edges) if reset or k >= n_edges],
            keyframe_ids=list(self.keyframe_ids), earliest=self.earliest_loop_closure_node,
            estimates={k: v.copy() for k, v in self.poses.items()}, optimizations=self._optimizations))
        return ret

    def _add_node(self, node: GraphNode) -> bool:
        if node.n_features < self.params.min_matches:
            return False
        if not self.nodes:
            self._first_node(node)
            return True
        found, edge_to_kf = self.node_comparisons(node)
        if found:
            self.nodes[node.id] = node
            if not edge_to_kf and self.earliest_loop_closure_node > self.keyframe_ids[-1]:  # :731
                self.add_keyframe(node.id - 1)  # the previous node is still localised w.r.t. a keyframe (:732)
            n_vertices = sum(1 for n in self.nodes.values() if n.vertex)
            if self.params.optimizer_skip_step > 0 and n_vertices % self.params.optimizer_skip_step == 0:
                self.optimize()
        elif len(self.nodes) == 1 and node.n_features > self.nodes[0].n_features:
            # only one node so far and it has fewer features: the new node replaces it (:762-769)
            self._reset()
            self._first_node(node)
            return True
        return found

    def fixation_of_vertices(self, ids: list[int], fixed: np.ndarray):
        """fixationOfVertices (graph_manager.cpp:911-937) on the persistent flags in `fixed`, in place; "inaffected" leaves
        them as they are.  An optimisation without any fixed vertex fixes its first one."""
        strategy = self.params.pose_relative_to
        if strategy == "previous" and len(self.nodes) > 2:
            fixed[:] = 0
            fixed[ids.index(self.nodes[len(self.nodes) - 2].id)] = 1
        elif strategy == "largest_loop":
            fixed[:] = [1 if k < self.earliest_loop_closure_node else 0 for k in ids]
        elif strategy == "first":
            fixed[:] = 0
            fixed[ids.index(self.nodes[0].id)] = 1
        if len(fixed) and not fixed.any():
            fixed[0] = 1

    def graph_arrays(self) -> dict:
        """What optimizeGraph hands the solver: vertices in id order, fixed flags after fixationOfVertices, edges in order."""
        ids = sorted(k for k, n in self.nodes.items() if n.vertex)
        index = {k: i for i, k in enumerate(ids)}
        fixed = np.array([1 if k in self.fixed_ids else 0 for k in ids], np.uint8)
        self.fixation_of_vertices(ids, fixed)
        return dict(init=np.stack([self.poses[k] for k in ids]), fixed=fixed, ids=np.array(ids),
                    ij=np.array([(index[a], index[b]) for a, b in self.edges], np.int32).reshape(-1, 2),
                    meas=np.array(self.meas).reshape(-1, 7), info=np.array(self.info).reshape(-1, 36))

    def optimize(self, stop: float | None = None) -> float:
        """optimizeGraph: LM over all camera-camera edges; estimates are written back to the vertices."""
        g = self.graph_arrays()
        if len(g["ij"]) == 0:
            return 0.0
        x, chi2 = self.backend.optimize(g, self.params.optimizer_iterations if stop is None else stop)
        for k, pose in zip(g["ids"], x):
            self.poses[int(k)] = np.array(pose, np.float64)
        self.fixed_ids = set(int(k) for k in g["ids"]) if self.params.pose_relative_to == "inaffected" else set()  # :1031-1036
        self.last_chi2 = chi2
        self._optimizations.append(dict(g, x=np.array(x, np.float64), chi2=chi2))
        return chi2

    def trajectory(self) -> tuple[np.ndarray, np.ndarray]:
        ids = sorted(k for k, n in self.nodes.items() if n.vertex)
        return np.array(ids), np.stack([self.poses[k] for k in ids])


def run_online(backend, gray, depth, mask, K4, stamps=None, seed: int = 0, params: Params | None = None):
    """Drive a live sequence the way OpenNIListener does (openni_listener.cpp:779-813): one Node per frame, addNode in
    arrival order.  backend: .construct_nodes, .n_features(handle), .match_one_to_many(node, olds, seed[, first_pair_index]),
    .optimize."""
    n = len(gray)
    stamps = np.arange(n) / 30.0 if stamps is None else np.asarray(stamps, np.float64)
    gm = GraphManager(backend, params or Params(), seed)
    handles = backend.construct_nodes(gray, depth, mask, K4)
    for k in range(n):
        gm.add_node(handles[k], backend.n_features(handles[k]), stamps[k])
    return gm
