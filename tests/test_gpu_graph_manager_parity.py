"""The C++ GraphManager shim (include/rgbdslam_b200/graph_manager.hpp) against its Python twin (oracle/graph_manager_oracle.py),
decision for decision, on rendered sequences: tests/cpp/test_graph_manager_trace.cpp builds one Node per frame and calls addNode
in arrival order, the twin runs `run_online` on `pipeline.GpuBackend` with the same frames, seed and parameters.  Both call the
same library on the same nodes, so return values, candidate lists, edges with their measurements and information matrices,
keyframes, vertex estimates and every optimiser input are compared bit for bit; the solver's output is held to the float64
oracle at the bar of test_gpu_posegraph.py.  pruneEdgesWithErrorAbove is held to a numpy restatement."""
import subprocess
import time
from pathlib import Path

import numpy as np
import pytest

from oracle import graph_manager_oracle as G

pytestmark = pytest.mark.gpu

ROOT = Path(__file__).resolve().parent.parent
SEED = 9
MAX_KEYPOINTS = 600
STRATEGIES = ["first", "previous", "largest_loop", "inaffected"]
# the sequence: 30 frames forward along synth.trajectory(240), then back over 20 of them (revisits: geodesic and sampled
# candidates, loop closures); frame 40 shows uniform noise: it has features but matches nothing
INDEX = list(range(0, 30)) + list(range(28, 8, -1))
JUMP = 40


def _noise(seed):
    from rgbdslam_v2_b200 import synth
    return np.random.default_rng(seed).integers(0, 256, (synth.H, synth.W)).astype(np.uint8)


@pytest.fixture(scope="module")
def exe(built, tmp_path_factory):
    out = tmp_path_factory.mktemp("trace") / "test_graph_manager_trace"
    libdir = ROOT / "rgbdslam_v2_b200"
    subprocess.run(["g++", "-std=c++17", "-O2", "-Wall", f"-I{ROOT / 'include'}", str(ROOT / "tests/cpp/test_graph_manager_trace.cpp"),
                    "-o", str(out), f"-L{libdir}", "-lrgbdslam_b200", f"-Wl,-rpath,{libdir}"], check=True)
    return out


@pytest.fixture(scope="module")
def fe(built):
    from rgbdslam_v2_b200 import Frontend
    from rgbdslam_v2_b200._capi import default_params
    p = default_params(); p.depth_cov_z0 = 2.0; p.max_keypoints = MAX_KEYPOINTS
    f = Frontend(0, p)
    yield f
    f.close()


@pytest.fixture(scope="module")
def frames(built):
    from oracle import orb_oracle
    from rgbdslam_v2_b200 import synth
    gray, depth = synth.render_frames_torch(synth.trajectory(240)[INDEX], "cuda:0")
    gray, depth = gray.cpu().numpy(), depth.cpu().numpy()
    gray[JUMP] = _noise(JUMP)
    mask = np.stack([orb_oracle.depth_to_mask(d) for d in depth])
    return gray, depth, mask, np.arange(len(gray)) / 30.0


def _few_features(frames):
    """frame 0 shows noise, detected only in a 96 x 96 window, 0.5 s before frame 1: it matches nothing and has fewer features
    than frame 1, which replaces it; frame 20 is uniform grey (no features: not added)."""
    gray, depth, mask, stamps = (a.copy() for a in frames)
    gray[0] = _noise(0)
    window = mask[0, 200:296, 280:376].copy()
    mask[0] = 0
    mask[0, 200:296, 280:376] = window
    gray[20] = 128
    stamps[1:] += 0.5
    return gray, depth, mask, stamps


def _write_frames(path, gray, depth, mask, stamps):
    from rgbdslam_v2_b200 import synth
    F, H, W = gray.shape
    with open(path, "wb") as f:
        np.array([F, W, H], np.int64).tofile(f)
        np.array([synth.FX, synth.FY, synth.CX, synth.CY], np.float64).tofile(f)
        np.asarray(stamps, np.float64).tofile(f)
        np.ascontiguousarray(gray, np.uint8).tofile(f)
        np.ascontiguousarray(depth, np.float32).tofile(f)
        np.ascontiguousarray(mask, np.uint8).tofile(f)


def _write_params(path, p: G.Params, extra=(), thresholds=()):
    v = [SEED, 2.0, MAX_KEYPOINTS, p.min_matches, p.predecessor_candidates, p.neighbor_candidates, p.min_sampled_candidates,
         p.geodesic_depth, p.min_translation_meter, p.min_rotation_degree, p.max_translation_meter, p.max_rotation_degree,
         p.keep_all_nodes, p.keep_good_nodes, p.optimizer_skip_step, p.optimizer_iterations, 1.0, bool(p.odom_frame_name),
         STRATEGIES.index(p.pose_relative_to), p.max_connections, len(extra)]
    for a, b, T, scale in extra:
        v += [a, b] + list(np.asarray(T, np.float64).T.reshape(16)) + [scale]
    v += [len(thresholds)] + list(thresholds)
    np.array(v, np.float64).tofile(path)


class _Reader:
    def __init__(self, path):
        self.v, self.at = np.fromfile(path, np.float64), 0

    def take(self, n=None):
        if n is None:
            self.at += 1
            return self.v[self.at - 1]
        self.at += n
        return self.v[self.at - n:self.at]

    def int(self):
        return int(self.take())

    def ints(self, n):
        return [int(x) for x in self.take(n)]

    def edges(self):
        out = []
        for _ in range(self.int()):
            a, b = self.int(), self.int()
            out.append((a, b, self.take(7).copy(), self.take(36).copy()))
        return out

    def opts(self):
        out = []
        for _ in range(self.int()):
            nv = self.int()
            ids = np.array(self.ints(nv)); fixed = np.array(self.ints(nv), np.uint8); init = self.take(7 * nv).reshape(nv, 7)
            ne = self.int()
            ij = np.array(self.ints(2 * ne), np.int32).reshape(ne, 2)
            meas, info = self.take(7 * ne).reshape(ne, 7), self.take(36 * ne).reshape(ne, 36)
            x = self.take(7 * nv).reshape(nv, 7)
            out.append(dict(ids=ids, fixed=fixed, init=init, ij=ij, meas=meas, info=info, x=x, chi2=self.take()))
        return out


def _parse(path, n_frames):
    r = _Reader(path)
    records = []
    for k in range(n_frames):
        assert r.int() == 1 and r.int() == k
        rec = dict(ret=bool(r.int()), id=r.int(), n2d=r.int(), n3d=r.int())
        nt = r.int()
        rec["targets"] = None if nt < 0 else r.ints(nt)
        rec["edges"] = r.edges()
        rec["keyframe_ids"] = r.ints(r.int())
        rec["earliest"] = r.int()
        rec["estimates"] = {}
        for _ in range(r.int()):
            i = r.int()
            rec["estimates"][i] = r.take(7).copy()
        rec["optimizations"] = r.opts()
        records.append(rec)
    assert r.int() == 2
    extra = r.ints(r.int())
    prunes = []
    while r.at < len(r.v):
        assert r.int() == 3
        thr = r.take(); nv = r.int()
        ids = r.ints(nv); poses = r.take(7 * nv).reshape(nv, 7)

        def state():
            ne = r.int()
            return np.array(r.ints(ne), bool), r.edges()
        before = state()
        pruned = r.int()
        after = state()
        prunes.append(dict(thr=thr, ids=ids, poses=poses, before=before, pruned=pruned, after=after, opts=r.opts()))
    return records, extra, prunes


def _same(a, b) -> bool:
    a, b = np.ascontiguousarray(a, np.float64), np.ascontiguousarray(b, np.float64)
    return a.shape == b.shape and a.tobytes() == b.tobytes()


def _check_solve(oracle_mod, o, stop, where):
    """the solver's output on the shim's arrays: the float64 oracle's, at the bar of test_gpu_posegraph.py"""
    ox, ochi2, _, _ = oracle_mod.posegraph_optimize(o["init"], o["fixed"], o["ij"], o["meas"], o["info"], stop=stop)
    assert o["chi2"] == pytest.approx(ochi2, rel=1e-6, abs=1e-9), where
    assert np.abs(o["x"][:, :3] - ox[:, :3]).max() < 1e-6, where
    sgn = np.sign((o["x"][:, 3:] * ox[:, 3:]).sum(1))[:, None]
    assert np.abs(o["x"][:, 3:] - sgn * ox[:, 3:]).max() < 1e-6, where
    assert np.array_equal(o["x"][o["fixed"] == 1], o["init"][o["fixed"] == 1]), where


def _expected_fixed(strategy, o, rec, prev_ids, n_nodes):
    """the reference's flags at this optimisation (graph_manager.cpp:381, :889-892, :911-937, :1031-1036) + the shim's anchor"""
    ids = list(o["ids"])
    if strategy == "first":
        f = [1 if k == 0 else 0 for k in ids]
    elif strategy == "previous":
        f = [1 if k == n_nodes - 2 else 0 for k in ids] if n_nodes > 2 else [1 if k == 0 else 0 for k in ids]
    elif strategy == "largest_loop":
        f = [1 if k < rec["earliest"] else 0 for k in ids]
    else:  # inaffected: fixed after the previous optimisation (the first vertex before any), freed by every edge added since
        touched = {v for e in rec["_since"] for v in e[:2]}
        f = [1 if (k in prev_ids and k not in touched) else 0 for k in ids]
    if not any(f):
        f[0] = 1
    return np.array(f, np.uint8)


def _compare(records, gm, oracle_mod, stop=0.01):
    strategy = gm.params.pose_relative_to
    assert len(records) == len(gm.records)
    n_opt = 0
    prev_ids, since = {0}, []  # "inaffected": fixed flags as the last optimisation left them, edges added since
    for k, (c, t) in enumerate(zip(records, gm.records)):
        where = f"frame {k}"
        assert c["n2d"] == c["n3d"] == t["n_features"], where  # the feature gate: 2-D count == 3-D count == n_features
        assert c["ret"] == t["ret"], where
        if c["ret"]:
            assert c["id"] == t["id"], where
        assert c["targets"] == t["targets"], where
        assert len(c["edges"]) == len(t["edges"]), where
        for (a, b, z, i), (ta, tb, tz, ti) in zip(c["edges"], t["edges"]):
            assert (a, b) == (ta, tb) and _same(z, tz) and _same(i, ti), (where, a, b)
        assert c["keyframe_ids"] == t["keyframe_ids"], where
        assert c["earliest"] == t["earliest"], where
        assert sorted(c["estimates"]) == sorted(t["estimates"]), where
        for i in c["estimates"]:
            assert _same(c["estimates"][i], t["estimates"][i]), (where, i)
        assert len(c["optimizations"]) == len(t["optimizations"]), where
        if c["ret"] and len(c["estimates"]) == 1:
            prev_ids, since = {c["id"]}, []  # (re)started graph: the first vertex is fixed
        since += c["edges"]
        for o, to in zip(c["optimizations"], t["optimizations"]):
            assert np.array_equal(o["ids"], to["ids"]) and np.array_equal(o["ij"], to["ij"]), where
            assert np.array_equal(o["fixed"], to["fixed"]), where
            for key in ("init", "meas", "info", "x"):
                assert _same(o[key], to[key]), (where, key)
            n_nodes = len(c["estimates"])
            c["_since"] = since
            assert np.array_equal(o["fixed"], _expected_fixed(strategy, o, c, prev_ids, n_nodes)), (where, o["fixed"])
            _check_solve(oracle_mod, o, stop, where)
            prev_ids, since = set(o["ids"].tolist()), []
            n_opt += 1
    return n_opt


def _run(exe, tmp_path, fe, frames, params: G.Params, extra=(), thresholds=()):
    from rgbdslam_v2_b200 import pipeline, synth
    gray, depth, mask, stamps = frames
    fpath, ppath, opath = tmp_path / "frames.bin", tmp_path / "params.bin", tmp_path / "trace.bin"
    _write_frames(fpath, gray, depth, mask, stamps)
    _write_params(ppath, params, extra, thresholds)
    r = subprocess.run([str(exe), str(fpath), str(ppath), str(opath)], capture_output=True, text=True)
    assert r.returncode == 0, r.stdout + r.stderr
    records, extra_ok, prunes = _parse(opath, len(gray))
    K4 = (synth.FX, synth.FY, synth.CX, synth.CY)
    gm = G.run_online(pipeline.GpuBackend(fe), gray, depth, mask, K4, stamps, seed=SEED, params=params)
    return records, gm, extra_ok, prunes


CASES = {
    "default": dict(),
    "min_translation": dict(min_translation_meter=0.03, min_rotation_degree=5.0),  # ~2.7 cm per frame: every other one
    "max_connections_1": dict(max_connections=1),
    "max_connections_3": dict(max_connections=3),
    "keep_good_nodes": dict(keep_good_nodes=True),
    "skip_step_3": dict(optimizer_skip_step=3),
    "previous": dict(pose_relative_to="previous"),
    "largest_loop": dict(pose_relative_to="largest_loop"),
    "inaffected": dict(pose_relative_to="inaffected"),
    "few_features": dict(),
    "min_translation_max_connections_1": dict(min_translation_meter=0.03, min_rotation_degree=5.0, max_connections=1),
}


@pytest.mark.parametrize("case", list(CASES))
def test_shim_and_twin_decide_alike(exe, fe, frames, oracle_mod, tmp_path, case):
    t0 = time.perf_counter()
    fr = frames
    if case == "few_features":
        fr = _few_features(frames)
    elif case == "keep_good_nodes":  # 0.2 s between frames: a node without any transformation keeps no constant-position edge
        fr = frames[:3] + (np.arange(len(frames[0])) * 0.2,)
    params = G.Params(**CASES[case])
    records, gm, _, _ = _run(exe, tmp_path, fe, fr, params)
    n_opt = _compare(records, gm, oracle_mod)
    added = [r["ret"] for r in records]
    edges = [e for r in records for e in r["edges"]]
    # each case reaches the decisions it is there for
    assert n_opt > 0 and sum(added) >= 10, (case, n_opt, sum(added))
    if case == "default":
        assert all(added) and any(abs(a - b) > params.predecessor_candidates for a, b, _, _ in edges)  # loop closures
        assert any(t < r["id"] - 5 for r in records[12:] for t in r["targets"] or [])  # geodesic or sampled candidates
        assert len(records[-1]["keyframe_ids"]) > 1
    if case.startswith("min_translation"):
        assert not all(added[1:])  # frames that moved too little are not added
    if case == "keep_good_nodes":  # the noise frame has no transformation: kept with a constant-position edge, information I / 0.2
        (a, b, z, i), = records[JUMP]["edges"]
        assert records[JUMP]["ret"] and (a, b) == (JUMP - 1, JUMP) and _same(z, [0, 0, 0, 0, 0, 0, 1.0])
        assert _same(i, (np.eye(6) / abs(fr[3][JUMP] - fr[3][JUMP - 1])).reshape(36))
    if case == "few_features":
        assert records[1]["ret"] and records[1]["id"] == 0 and records[1]["keyframe_ids"] == [0]  # frame 1 replaced frame 0
        assert records[0]["ret"] and records[0]["n2d"] < records[1]["n2d"] and not records[20]["ret"]
    if case == "skip_step_3":
        assert all(len(o["ids"]) % 3 == 0 for r in records for o in r["optimizations"])
    if case == "largest_loop":
        assert any(r["earliest"] < r["id"] - params.predecessor_candidates for r in records if r["ret"])
    print(f"{case}: {sum(added)} nodes, {len(edges)} edges, {n_opt} optimisations, {time.perf_counter() - t0:.1f} s")


def _prune_restated(prune, oracle_mod):
    """pruneEdgesWithErrorAbove (graph_manager.cpp:1106-1246) in numpy on the per-edge chi2 of the float64 oracle.  Returns the
    expected (active, meas, info) of every edge, the edges whose chi2 lies within 1e-9 relative of the threshold, and the count."""
    active, edges = prune["before"]
    thr = float(np.float32(prune["thr"]))
    index = {k: i for i, k in enumerate(prune["ids"])}
    deg = {}
    for a, b, _, _ in edges:
        deg[a] = deg.get(a, 0) + 1; deg[b] = deg.get(b, 0) + 1
    act, meas, info = active.copy(), [e[2].copy() for e in edges], [e[3].copy() for e in edges]
    near, counter = set(), 0
    for e, (a, b, z, inf) in enumerate(edges):
        if not active[e]:
            continue
        ij = np.array([[index[a], index[b]]], np.int32)
        chi2, _ = oracle_mod.posegraph_chi2(prune["poses"], ij, z[None], inf[None])
        if abs(chi2 - thr) <= 1e-9 * thr:
            near.add(e)
        if not chi2 > thr:
            continue
        counter += 1
        meas[e] = np.array([0, 0, 0, 0, 0, 0, 1.0])
        if abs(a - b) != 1:
            if deg[a] > 1 and deg[b] > 1:
                act[e] = False
                continue
            info[e] = (np.eye(6) * 1e-100).reshape(36)
        else:
            info[e] = np.eye(6).reshape(36)
    return act, meas, info, near, counter


def test_prune_edges_with_error_above(exe, fe, frames, oracle_mod, tmp_path):
    """planted wrong loop closures on the final graph, then pruneEdgesWithErrorAbove(5 / 1 / 0.25), each followed by
    optimizeGraph (openni_listener.cpp:431-466)"""
    from rgbdslam_v2_b200 import synth
    rng = np.random.default_rng(4)
    extra = []
    for a, b in [(3, 45), (8, 38), (12, 47), (20, 21), (0, 33)]:
        T = np.eye(4)
        T[:3, :3] = synth.random_rigid(rng, 0.5, 20.0)[:3, :3]
        T[:3, 3] = rng.normal(0, 0.3, 3)
        extra.append((a, b, T, 1e3))
    records, gm, extra_ok, prunes = _run(exe, tmp_path, fe, frames, G.Params(), extra, (5.0, 1.0, 0.25))
    _compare(records, gm, oracle_mod)
    assert extra_ok == [1] * len(extra)
    n_near = 0
    for prune in prunes:
        act, meas, info, near, counter = _prune_restated(prune, oracle_mod)
        got_active, got_edges = prune["after"]
        n_near += len(near)
        for e, (a, b, z, i) in enumerate(got_edges):
            if e in near:
                continue
            assert got_active[e] == act[e] and _same(z, meas[e]) and _same(i, info[e]), (prune["thr"], e, a, b)
        assert counter - len(near) <= prune["pruned"] <= counter + len(near), prune["thr"]
        for o in prune["opts"]:
            _check_solve(oracle_mod, o, 0.01, f"after pruning at {prune['thr']}")
    assert prunes[0]["pruned"] >= len(extra)  # every planted edge is over 5
    assert not all(prunes[0]["after"][0])     # and non-consecutive ones between well-connected vertices leave the active set
    print(f"pruning: {[p['pruned'] for p in prunes]} edges over 5 / 1 / 0.25, {n_near} within 1e-9 of a threshold")
