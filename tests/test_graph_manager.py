"""Online graph front (graph_manager.cpp:204-324, 421-658, 681-782) restated in rgbdslam_v2_b200/graph_manager.py:
host logic only, driven here by a scripted backend (no GPU)."""
import numpy as np
import pytest

from oracle import graph_manager_oracle as G
from rgbdslam_v2_b200._capi import PAIR_RESULT_DTYPE
from rgbdslam_v2_b200.pipeline import pose7_to_mat, mat_to_pose7


class ScriptedBackend:
    """Ground-truth relative transforms; `visible(new, old)` decides which comparisons succeed."""

    def __init__(self, poses, visible):
        self.poses, self.visible, self.calls = poses, visible, []

    def match_one_to_many(self, node, olds, seed):
        self.calls.append((node.id, [o.id for o in olds]))
        res = np.zeros(len(olds), PAIR_RESULT_DTYPE)
        for k, o in enumerate(olds):
            if self.visible(node.id, o.id):
                T = np.linalg.inv(self.poses[o.id]) @ self.poses[node.id]  # pose of the newer camera in the older one's frame
                res[k]["id1"], res[k]["id2"] = o.id, node.id
                res[k]["n_inliers"] = 100 - min(abs(node.id - o.id), 50)
                res[k]["ransac_trafo"] = T.T.reshape(-1).astype(np.float32)
                res[k]["info_scale"] = 1e4
            else:
                res[k]["id1"] = res[k]["id2"] = -1
        return res

    def optimize(self, graph, stop):
        return graph["init"], 0.0


def _line(n, step=0.05):
    poses = []
    for k in range(n):
        T = np.eye(4); T[0, 3] = step * k
        poses.append(T)
    return poses


def _run(n, visible, **kw):
    poses = _line(n)
    be = ScriptedBackend(poses, visible)
    gm = G.GraphManager(be, G.Params(**kw), seed=3)
    for k in range(n):
        gm.add_node(k, 500, k / 30.0)
    return gm, be, poses


def test_few_nodes_compare_with_all_predecessors():
    gm, be, _ = _run(8, lambda a, b: True)
    # while camera_vertices <= 3 + 4 + 4 every earlier node is a sequential target, predecessor appended last (:213-220, :316)
    for new, olds in be.calls:
        assert sorted(olds) == list(range(new)) and olds[-1] == new - 1
    assert len(gm.edges) == sum(range(8)) and gm.n_const_edges == 0


def test_candidate_budget_and_classes():
    n = 60
    gm, be, _ = _run(n, lambda a, b: abs(a - b) <= 3 or (a % 10 == 0 and b % 10 == 0))
    for new, olds in be.calls[15:]:
        assert len(olds) == len(set(olds))
        assert len(olds) <= 3 + 4 + 4 + 1                          # (:516-526) + the predecessor
        assert olds[-1] == new - 1                                 # include_predecessor, compared first (list is walked backwards)
        seq = [o for o in olds if new - 1 - 3 <= o < new - 1]
        assert seq == [new - 2, new - 3, new - 4]                  # sequential targets right before the predecessor
        rest = [o for o in olds if o < new - 4]
        assert all(0 <= o < new - 4 for o in rest)
    # sampled candidates only come from keyframes, geodesic ones from the <3-hop ball around the predecessor
    assert set(gm.keyframe_ids) <= set(range(n)) and gm.keyframe_ids[0] == 0


def test_geodesic_ball_is_strictly_inside_max_distance():
    gm, _, _ = _run(12, lambda a, b: abs(a - b) == 1)             # a chain
    assert gm._geodesic_ball(6, 3) == {4, 5, 6, 7, 8}             # hop count < 3
    assert gm._geodesic_ball(0, 1) == {0}


def test_constant_position_edge_when_predecessor_is_lost():
    lost = {20}
    gm, be, poses = _run(21, lambda a, b: a not in lost and abs(a - b) <= 3)
    assert gm.n_const_edges == 1
    k = gm.edges.index((19, 20))
    assert np.allclose(gm.meas[k], [0, 0, 0, 0, 0, 0, 1]) and np.allclose(gm.info[k].reshape(6, 6), np.eye(6) * 30.0)  # I / dt
    assert not gm.nodes[20].valid_tf_estimate  # until a later node links to it (:571)
    assert np.allclose(gm.poses[20], gm.poses[19])


def test_vertex_estimate_follows_the_edge_with_most_inliers():
    gm, be, poses = _run(20, lambda a, b: abs(a - b) <= 3)
    ids, traj = gm.trajectory()
    assert list(ids) == list(range(20))
    for k in ids:
        assert np.allclose(pose7_to_mat(traj[k])[:3, 3], poses[k][:3, 3], atol=1e-6)
    assert gm.sequential_edges == len(gm.edges) and gm.loop_closure_edges == 0


def test_keyframe_added_when_no_edge_reaches_one():
    # only the direct predecessor is ever matched: node k has no edge to keyframe 0 once k >= 2 -> keyframes trail the head
    gm, _, _ = _run(12, lambda a, b: a - b == 1)
    assert gm.keyframe_ids[:3] == [0, 1, 2] and gm.keyframe_ids == sorted(set(gm.keyframe_ids))


def test_motion_gates():
    p = G.Params(min_translation_meter=0.1, min_rotation_degree=5.0, max_translation_meter=2.0, max_rotation_degree=90.0)
    T = np.eye(4); T[0, 3] = 0.05
    assert not G.is_big_trafo(T, p) and G.is_small_trafo(T, 1 / 30.0, p)
    T[0, 3] = 0.2
    assert G.is_big_trafo(T, p) and not G.is_small_trafo(T, 1 / 30.0, p) and G.is_small_trafo(T, 0.0, p)
    c, s = np.cos(np.radians(10)), np.sin(np.radians(10))
    R = np.eye(4); R[:2, :2] = [[c, -s], [s, c]]
    assert G.trafo_size(R)[0] == pytest.approx(10.0) and G.is_big_trafo(R, p)
    # with min_translation > 0 a frame that barely moved is not added as a node (:470-485)
    poses = _line(6, step=0.01)
    be = ScriptedBackend(poses, lambda a, b: True)
    gm = G.GraphManager(be, G.Params(min_translation_meter=0.1), seed=0)
    added = [gm.add_node(k, 500, k / 30.0) for k in range(6)]
    assert added == [True, False, False, False, False, False]


def test_too_few_features_is_skipped():
    gm, _, _ = _run(3, lambda a, b: True)
    assert gm.add_node(99, 5, 1.0) is False and len(gm.nodes) == 3


def test_max_connections_stops_further_comparisons():
    # every comparison succeeds; with max_connections = 2 a node keeps 3 matched edges (the 4th comparison finds the counter at
    # 3 > 2 and returns empty, node.cpp:1310-1312).  The predecessor is the LAST candidate, so it is among the skipped ones
    # and the node also gets the constant-position edge (graph_manager.cpp:636-655) -- the reference does the same.
    gm, be, _ = _run(12, lambda a, b: True, max_connections=2)
    ident = np.array([0, 0, 0, 0, 0, 0, 1.0])
    matched = {}
    for (a, b), z in zip(gm.edges, gm.meas):
        if not np.allclose(z, ident):
            matched[b] = matched.get(b, 0) + 1
    assert max(matched.values()) == 3 and matched[11] == 3 and gm.n_const_edges > 0
    gm2, _, _ = _run(12, lambda a, b: True)
    assert max(np.bincount([b for _, b in gm2.edges])) > 4 and gm2.n_const_edges == 0


def _run_strategy(n, visible, strategy, **kw):
    return _run(n, visible, pose_relative_to=strategy, **kw)[0]


def test_fixation_first_and_previous():
    # fixationOfVertices (graph_manager.cpp:918-936): "first" fixes node 0, "previous" the node before the newest
    for strategy, expect in [("first", lambda n: 0), ("previous", lambda n: n - 2 if n > 2 else 0)]:
        gm = _run_strategy(10, lambda a, b: abs(a - b) <= 2, strategy)
        for rec in gm.records[1:]:
            (o,) = rec["optimizations"]
            n = len(o["ids"])
            assert list(np.nonzero(o["fixed"])[0]) == [expect(n)], (strategy, n, o["fixed"])


def test_fixation_largest_loop_follows_the_earliest_loop_closure_node():
    # the loop closure 9 -> 2 lowers earliest_loop_closure_node_ to 2 (:893-896): vertices 0 and 1 are fixed in that
    # optimisation (:922-931); without a loop closure the earliest node is the new one and everything before it is fixed
    gm = _run_strategy(12, lambda a, b: a - b == 1 or (a, b) == (9, 2), "largest_loop")
    rec = gm.records[9]
    assert rec["earliest"] == 2 and list(rec["optimizations"][0]["fixed"]) == [1, 1] + [0] * 8
    rec = gm.records[10]
    assert rec["earliest"] == 9 and list(rec["optimizations"][0]["fixed"]) == [1] * 9 + [0, 0]
    # "first" leaves earliest_loop_closure_node_ at the new node's id
    gm = _run_strategy(12, lambda a, b: a - b == 1 or (a, b) == (9, 2), "first")
    assert [r["earliest"] for r in gm.records[1:]] == list(range(1, 12))


def test_fixation_inaffected_frees_the_ends_of_new_edges():
    # after an optimisation every vertex is fixed (:1031-1033); the edges of the next node free both their ends (:889-892)
    gm = _run_strategy(9, lambda a, b: a - b in (1, 3), "inaffected")
    for k in range(5, 9):
        (o,) = gm.records[k]["optimizations"]
        freed = {k, k - 1, k - 3}
        assert list(o["fixed"]) == [0 if v in freed else 1 for v in o["ids"]], (k, o["fixed"])
    assert gm.fixed_ids == set(range(9))
    # the first optimisation frees vertex 0 too: nothing is fixed, so the first vertex anchors the solve
    assert list(gm.records[1]["optimizations"][0]["fixed"]) == [1, 0]


def test_keyframe_rule_reads_earliest_loop_closure_node():
    # node 10 matches 9 and 3, neither a keyframe (keyframes 0, 2, 4, 6, 8): with "first" the earliest loop closure node is
    # node 10 itself, newer than the last keyframe, so 9 becomes one (:731-732); with "largest_loop" the edge to 3 lowers it
    # below keyframe 8 and no keyframe is added
    def visible(a, b):
        return b in (9, 3) if a == 10 else a - b in (1, 2)
    for strategy, last in [("first", 9), ("largest_loop", 8)]:
        gm = _run_strategy(11, visible, strategy)
        assert gm.keyframe_ids[:5] == [0, 2, 4, 6, 8] and gm.keyframe_ids[-1] == last, (strategy, gm.keyframe_ids)


def test_first_node_is_replaced_by_a_richer_one():
    # addNode (:762-769): no match with the only node, which has fewer features -> resetGraph + firstNode(new node).  The
    # constant-position edge (frames < 0.1 s apart) counts as a match, so the frames here are 0.5 s apart.
    be = ScriptedBackend(_line(4), lambda a, b: False)
    gm = G.GraphManager(be, G.Params(), seed=0)
    assert gm.add_node("a", 30, 0.0) and gm.add_node("b", 500, 0.5)
    assert list(gm.nodes) == [0] and gm.nodes[0].handle == "b" and gm.keyframe_ids == [0] and gm.fixed_ids == {0}
    assert gm.records[1]["ret"] and gm.records[1]["id"] == 0 and gm.records[1]["edges"] == []
    assert not gm.add_node("c", 400, 1.0)  # fewer features than the first node: not added, no replacement
    assert list(gm.nodes) == [0] and gm.nodes[0].handle == "b"
    # 1/30 s apart the constant-position edge keeps the new node: no replacement
    gm = G.GraphManager(ScriptedBackend(_line(4), lambda a, b: False), G.Params(), seed=0)
    assert gm.add_node("a", 30, 0.0) and gm.add_node("b", 500, 1 / 30)
    assert list(gm.nodes) == [0, 1] and gm.n_const_edges == 1


class KeyedBackend(ScriptedBackend):
    """records the generator key of each call's first pair, resolved as pipeline.GpuBackend resolves it"""

    def match_one_to_many(self, node, olds, seed, first_pair_index=None):
        self.keys.append((node.id, len(olds), 64 * node.id if first_pair_index is None else first_pair_index))
        return super().match_one_to_many(node, olds, seed)


def test_initial_comparison_key_self_candidates_and_max_connections():
    poses = _line(30)
    be = KeyedBackend(poses, lambda a, b: abs(a - b) <= 3)
    be.keys = []
    gm = G.GraphManager(be, G.Params(min_translation_meter=0.01, max_connections=1), seed=3)
    for k in range(30):
        gm.add_node(k, 500, k / 30.0)
    # the initial comparison is keyed 64 id + 63, the batch 64 id + k (nodeComparisons, graph_manager.hpp)
    initial = [(i, f) for i, n, f in be.keys if n == 1 and f % 64 == 63]
    assert len(initial) == 29 and all(f == 64 * i + 63 for i, f in initial)
    assert all(f == 64 * i for i, n, f in be.keys if f % 64 != 63)
    # the new node is never its own candidate (the geodesic ball around the matched predecessor holds it)
    assert all(new not in olds for new, olds in be.calls)
    # max_connections counts the initial comparison's transformation (node.cpp:1310-1312, :1417): with 1, the initial edge
    # and one more
    ident = np.array([0, 0, 0, 0, 0, 0, 1.0])
    per_node = np.bincount([b for (a, b), z in zip(gm.edges, gm.meas) if not np.allclose(z, ident)])
    assert (per_node[1:] == 2).all(), per_node
