"""GPU parity tests of the pose-graph solve (GraphManager::optimizeGraph) vs the CPU oracle."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def fe(built):
    from rgbdslam_v2_b200 import Frontend
    f = Frontend(0)
    yield f
    f.close()


def test_chi2_and_per_edge_chi2(fe, oracle_mod):
    from rgbdslam_v2_b200 import synth
    g = synth.make_pose_graph(300, 1500, seed=2, outlier_frac=0.03)
    chi, pe = fe.graph_chi2(g["init"], g["ij"], g["meas"], g["info"], per_edge=True)
    ochi, orob = oracle_mod.posegraph_chi2(g["init"], g["ij"], g["meas"], g["info"])
    assert chi == pytest.approx(ochi, rel=1e-10)
    assert pe.sum() == pytest.approx(ochi, rel=1e-10)
    e = oracle_mod.edge_se3(g["init"][g["ij"][7, 0]], g["init"][g["ij"][7, 1]], g["meas"][7], False)[0]
    assert pe[7] == pytest.approx(e @ g["info"][7].reshape(6, 6) @ e, rel=1e-9)


@pytest.mark.parametrize("nv,ne,stop,seed", [(200, 1000, 0.01, 1), (500, 3000, 0.01, 4), (500, 3000, 20.0, 4),
                                             (64, 63, 0.01, 7), (400, 2500, 1e-4, 9)])
def test_optimize_vs_oracle(fe, oracle_mod, nv, ne, stop, seed):
    from rgbdslam_v2_b200 import synth
    g = synth.make_pose_graph(nv, ne, seed=seed)
    x, chi2, it, cg = fe.optimize_graph(g["init"], g["fixed"], g["ij"], g["meas"], g["info"], stop=stop)
    ox, ochi2, oit, ocg = oracle_mod.posegraph_optimize(g["init"], g["fixed"], g["ij"], g["meas"], g["info"], stop=stop)
    c0, _ = oracle_mod.posegraph_chi2(g["init"], g["ij"], g["meas"], g["info"])
    assert chi2 < c0 or ne == nv - 1
    # tolerance: converged chi2 within 1e-6 relative, poses within 1e-6 m / 1e-6 (same LM/PCG, different summation order)
    assert chi2 == pytest.approx(ochi2, rel=1e-6, abs=1e-9)
    assert abs(it - oit) <= 2  # the final 'nothing left to do' iteration (PCG starts below tolerance) is borderline
    assert np.abs(x[:, :3] - ox[:, :3]).max() < 1e-6
    sgn = np.sign((x[:, 3:] * ox[:, 3:]).sum(1))[:, None]
    assert np.abs(x[:, 3:] - sgn * ox[:, 3:]).max() < 1e-6
    assert np.array_equal(x[0], g["init"][0])  # fixed vertex (graph_manager.cpp:911-937 "first")
    # the returned chi2 is the chi2 of the returned poses
    assert fe.graph_chi2(x, g["ij"], g["meas"], g["info"]) == pytest.approx(chi2, rel=1e-9)


def test_huber_outliers_and_ate(fe, oracle_mod):
    from rgbdslam_v2_b200 import synth
    g = synth.make_pose_graph(600, 3600, seed=11, outlier_frac=0.05)
    x, chi2, it, cg = fe.optimize_graph(g["init"], g["fixed"], g["ij"], g["meas"], g["info"], stop=0.01)
    ox, ochi2, oit, _ = oracle_mod.posegraph_optimize(g["init"], g["fixed"], g["ij"], g["meas"], g["info"], stop=0.01)
    ate, oate = synth.ate_rmse(x[:, :3], g["gt"][:, :3]), synth.ate_rmse(ox[:, :3], g["gt"][:, :3])
    assert abs(ate - oate) < 1e-3  # north star: trajectory ATE RMSE within 1 mm of the reference
    assert synth.ate_rmse(x[:, :3], ox[:, :3]) < 1e-3
    assert ate < 0.05 and chi2 == pytest.approx(ochi2, rel=1e-4)


def test_several_fixed_vertices_and_multi_edges(fe, oracle_mod):
    from rgbdslam_v2_b200 import synth
    g = synth.make_pose_graph(120, 500, seed=13)
    g["fixed"][[0, 40, 80]] = 1
    g["init"][[40, 80]] = g["gt"][[40, 80]]
    ij = np.concatenate([g["ij"], g["ij"][:50]])  # duplicate edges between the same vertices are separate constraints
    meas = np.concatenate([g["meas"], g["meas"][:50]]); info = np.concatenate([g["info"], g["info"][:50]])
    x, chi2, it, _ = fe.optimize_graph(g["init"], g["fixed"], ij, meas, info, stop=0.001)
    ox, ochi2, oit, _ = oracle_mod.posegraph_optimize(g["init"], g["fixed"], ij, meas, info, stop=0.001)
    assert np.array_equal(x[[0, 40, 80]], g["init"][[0, 40, 80]])
    assert chi2 == pytest.approx(ochi2, rel=1e-6) and np.abs(x[:, :3] - ox[:, :3]).max() < 1e-6


def test_c5_size_properties(fe, oracle_mod):
    """BASELINE config C5: 5000 vertices / 30 000 edges."""
    from rgbdslam_v2_b200 import synth
    g = synth.make_pose_graph(5000, 30000, seed=0)
    c0 = fe.graph_chi2(g["init"], g["ij"], g["meas"], g["info"])
    x, chi2, it, cg = fe.optimize_graph(g["init"], g["fixed"], g["ij"], g["meas"], g["info"], stop=0.01)
    assert chi2 < 1e-3 * c0 and it >= 5 and cg > 0
    assert np.array_equal(x[0], g["init"][0])
    assert np.abs(np.linalg.norm(x[:, 3:], axis=1) - 1).max() < 1e-12
    ate0, ate = synth.ate_rmse(g["init"][:, :3], g["gt"][:, :3]), synth.ate_rmse(x[:, :3], g["gt"][:, :3])
    assert ate < 0.05 and ate < 0.05 * ate0
    # the CPU oracle stops at the same point of the same stop rule (graph_manager.cpp:1006-1014)
    ox, ochi2, oit, _ = oracle_mod.posegraph_optimize(g["init"], g["fixed"], g["ij"], g["meas"], g["info"], stop=0.01)
    assert abs(ate - synth.ate_rmse(ox[:, :3], g["gt"][:, :3])) < 1e-3 and synth.ate_rmse(x[:, :3], ox[:, :3]) < 1e-3
    assert chi2 == pytest.approx(ochi2, rel=1e-4) and abs(it - oit) <= 2
    # idempotence: optimising the optimum again changes nothing measurable
    x2, chi2b, _, _ = fe.optimize_graph(x, g["fixed"], g["ij"], g["meas"], g["info"], stop=0.01)
    assert chi2b <= chi2 * (1 + 1e-9) and np.abs(x2[:, :3] - x[:, :3]).max() < 1e-4


def _hub_graph(nv, seed):
    """a chain with one hub vertex connected to every other vertex (degree nv - 1: more incidences than one CTA of the resident
    solver can keep in shared memory) plus a few random loop closures"""
    from rgbdslam_v2_b200 import synth
    g = synth.make_pose_graph(nv, nv - 1, seed=seed)  # odometry chain only
    rng = np.random.default_rng(seed)
    gt = g["gt"]
    hub = 3
    ij, meas = [list(e) for e in g["ij"]], [m for m in g["meas"]]
    others = [v for v in range(nv) if v != hub and abs(v - hub) > 1]
    pairs = [(hub, v) if k % 2 == 0 else (v, hub) for k, v in enumerate(others)]  # the hub in both roles of an edge
    pairs += [tuple(rng.choice(nv, 2, replace=False)) for _ in range(nv // 2)]
    for i, j in pairs:
        rel = synth.pose_compose(synth.pose_inverse(gt[i]), gt[j])
        d = np.concatenate([rng.normal(0, 0.005, 3), rng.normal(0, 0.002, 3)])
        rel = synth.pose_compose(rel, np.concatenate([d, [np.sqrt(1 - d[3:] @ d[3:])]]))
        ij.append([int(i), int(j)]); meas.append(rel)
    ne = len(ij)
    info = np.tile((np.eye(6) * 200.0).reshape(1, 36), (ne, 1))
    return dict(init=g["init"], fixed=g["fixed"], ij=np.array(ij, np.int32), meas=np.array(meas), info=info, gt=gt)


def test_resident_solver_matches_general_kernel_on_hub_graph(fe, monkeypatch):
    """700 vertices on one CTA per SM (132 on an H100 SXM: 6 per CTA); the hub's incidences exceed the 568 a CTA stages in
    shared memory, so the resident kernel takes its global-memory path for the tail -- same solution as the general kernel
    (RB200_PG_RESIDENT=0)"""
    g = _hub_graph(700, seed=5)
    monkeypatch.setenv("RB200_PG_RESIDENT", "1")
    x1, c1, it1, cg1 = fe.optimize_graph(g["init"], g["fixed"], g["ij"], g["meas"], g["info"], stop=0.01)
    monkeypatch.setenv("RB200_PG_RESIDENT", "0")
    x0, c0, it0, cg0 = fe.optimize_graph(g["init"], g["fixed"], g["ij"], g["meas"], g["info"], stop=0.01)
    assert c1 == pytest.approx(c0, rel=1e-7)
    assert abs(it1 - it0) <= 2
    assert np.abs(x1[:, :3] - x0[:, :3]).max() < 1e-6
    sgn = np.sign((x1[:, 3:] * x0[:, 3:]).sum(1))[:, None]
    assert np.abs(x1[:, 3:] - sgn * x0[:, 3:]).max() < 1e-6
    from rgbdslam_v2_b200 import synth
    assert synth.ate_rmse(x1[:, :3], g["gt"][:, :3]) < 0.02


def test_edge_vertex_index_out_of_range_is_rejected_before_any_launch(fe):
    """an edge vertex index < 0 or >= the vertex count raises in optimize_graph, graph_chi2 and landmark_ba, launches nothing and
    leaves nothing behind: the same valid calls give the same results before and after"""
    from rgbdslam_v2_b200 import B200Error, synth
    g = synth.make_pose_graph(60, 200, seed=8)
    d = synth.make_ba_problem(n_cams=5, n_points=40, seed=3)

    def valid():
        x, chi2, it, cg = fe.optimize_graph(g["init"], g["fixed"], g["ij"], g["meas"], g["info"], stop=0.01)
        c0, pe = fe.graph_chi2(g["init"], g["ij"], g["meas"], g["info"], per_edge=True)
        ba = fe.landmark_ba(d["poses"], d["fixed"], d["points"], d["obs_cam"], d["obs_point"], d["obs_uvd"], d["obs_info3"], d["K4"],
                            ij=d["ij"], meas=d["meas"], info=d["info"], iterations=4)
        return (x, chi2, it, cg, c0, pe) + tuple(ba)

    before = valid()
    assert before[2] >= 1 and before[-2] >= 1
    n0 = fe.launch_count
    for k, bad in [(0, len(g["init"])), (1, -1), (1, 10**6)]:
        ij = g["ij"].copy(); ij[len(ij) // 2, k] = bad
        with pytest.raises(B200Error):
            fe.optimize_graph(g["init"], g["fixed"], ij, g["meas"], g["info"], stop=0.01)
        with pytest.raises(B200Error):
            fe.graph_chi2(g["init"], ij, g["meas"], g["info"], per_edge=True)
        bij = d["ij"].copy(); bij[-1, k] = len(d["poses"]) if bad >= 0 else bad
        with pytest.raises(B200Error):
            fe.landmark_ba(d["poses"], d["fixed"], d["points"], d["obs_cam"], d["obs_point"], d["obs_uvd"], d["obs_info3"], d["K4"],
                           ij=bij, meas=d["meas"], info=d["info"], iterations=4)
    assert fe.launch_count == n0
    after = valid()
    for a, b in zip(before, after):
        assert np.array_equal(a, b)


def test_reserve_then_solve(fe):
    from rgbdslam_v2_b200 import synth
    fe.posegraph_reserve(3000, 40000)
    g = synth.make_pose_graph(150, 600, seed=3)
    x, chi2, it, cg = fe.optimize_graph(g["init"], g["fixed"], g["ij"], g["meas"], g["info"], stop=0.01)
    assert np.isfinite(chi2) and it >= 1
