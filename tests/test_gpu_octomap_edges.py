"""GPU tests of the colour OctoMap and the occupancy filter at the rules' edges (DESIGN.md 4.14, 4.15): every planted case of
tests/octomap_planted.py gives the oracle's .ot bytes and stats in one call, one call per node, one batch per node and the
case's own split; the filter cases keep the oracle's records with any chunking; 16 384 and 16 385 scans in one call, across
the batch limit of kOctMaxScans, equal the oracle."""
import time

import numpy as np
import pytest

import node_helpers as nh
import octomap_exact as ox
import octomap_planted as op
from test_octomap_oracle_cpu import leaves

pytestmark = pytest.mark.gpu

MODES = ["one-call", "per-node", "node-batches", "split"]


@pytest.fixture(scope="module")
def fe(built):
    from rgbdslam_v2_b200 import Frontend
    f = Frontend(0, nh.params(0, adjuster_max_iterations=0))  # the ungridded detector: 144 x 144 frames
    yield f
    f.close()


def _nodes(fe, scans, chunk=1024):
    """one point-cloud node per scan, with its stored cloud"""
    det = fe.detector_create()
    hs = []
    for k in range(0, len(scans), chunk):
        part = scans[k:k + chunk]
        grey = np.full((len(part), op.H, op.W), 128, np.uint8)
        h, _ = fe.nodes_create(det, grey, op.clouds(part), None, None, store_cloud=True)
        hs += list(h)
    fe.detector_destroy(det)
    return hs


@pytest.fixture(scope="module")
def case_nodes(fe):
    made = {}

    def get(name):
        if name not in made:
            made[name] = _nodes(fe, op.CASES[name].scans)
        return made[name]

    yield get
    for hs in made.values():
        nh.destroy(fe, hs)


@pytest.fixture(scope="module")
def expected():
    made = {}

    def get(name):
        if name not in made:
            m = op.oracle(op.CASES[name])
            made[name] = (m.write(), m.stats())
        return made[name]

    return get


def _splits(case, mode):
    n = len(case.scans)
    if mode == "per-node":
        return [1] * n
    if mode == "split":
        return case.calls or [n // 2, n - n // 2]
    return [n]


def _device(fe, case, hs, splits):
    om = fe.octomap_create(**case.params)
    T = op.transforms(case.scans)
    k = 0
    for s in splits:
        fe.octomap_insert(om, hs[k:k + s], T[k:k + s], op.device_max_range(case))
        k += s
    out = fe.octomap_write(om), fe.octomap_stats(om)
    fe.octomap_destroy(om)
    return out


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("name", sorted(op.CASES))
def test_planted_case_equals_the_oracle(fe, case_nodes, expected, monkeypatch, name, mode):
    case = op.CASES[name]
    if mode == "node-batches":
        monkeypatch.setenv("RB200_OCT_BATCH_ENTRIES", "1")  # every node is its own batch
    data, st = _device(fe, case, case_nodes(name), _splits(case, mode))
    ref, ref_st = expected(name)
    assert st == ref_st
    assert data == ref


@pytest.mark.parametrize("chunk", [None, "1"], ids=["default-chunks", "one-point-chunks"])
@pytest.mark.parametrize("res", [1.0, 0.05])
def test_planted_filter_cases_equal_the_oracle(fe, monkeypatch, res, chunk):
    if chunk:
        monkeypatch.setenv("RB200_OCF_CHUNK_POINTS", chunk)
    mc = op.filter_map(res)
    m = op.filter_oracle(res)
    hs = _nodes(fe, mc.scans)
    om = fe.octomap_create(**mc.params)
    fe.octomap_insert(om, hs, op.transforms(mc.scans))
    assert fe.octomap_write(om) == m.write()
    nh.destroy(fe, hs)
    for name, f in op.filter_cases(res, leaves(m.write())).items():
        for thr in f.thresholds:
            fh = _nodes(fe, [op.scan(np.zeros(3, np.float32), f.pts)])
            r32, r16 = fe.node_cloud(fh[0], 32).reshape(-1), fe.node_cloud(fh[0], 16).reshape(-1)
            keep = m.occupancy_filter(np.stack([r32["x"], r32["y"], r32["z"]], 1), f.sensor7[:4], f.sensor7[4:], thr)
            counts = fe.octomap_filter_clouds(om, fh, f.sensor7[None], thr)
            g32, g16 = fe.node_cloud(fh[0], 32).reshape(-1), fe.node_cloud(fh[0], 16).reshape(-1)
            assert counts[0] == keep.sum(), (name, thr)
            assert g32.tobytes() == r32[keep].tobytes() and g16.tobytes() == r16[keep].tobytes(), (name, thr)
            nh.destroy(fe, fh)
    fe.octomap_destroy(om)


# ---- the scan limit --------------------------------------------------------------------------------------------------------

LIMIT = 1 << 14  # kOctMaxScans


def _limit_scans(n):
    """every scan from one origin: two of three hit (2, 0, 0) with their own colour, the third frees it on a longer ray;
    every scan colours (0, 2, 0); the last one also hits a cell of its own (0, 0, 4 + n % 2)"""
    A = np.array([0.5, 0.5, 0.5], np.float32)
    out = []
    for i in range(n):
        pts = [(2.5, 0.5, 0.5) if i % 3 != 2 else (6.5, 0.5, 0.5), (0.5, 2.5, 0.5)]
        if i == n - 1:
            pts.append((0.5, 0.5, 4.5 + n % 2))
        rgb = [(i * 0x9E3779B1 >> 8) & 0xFEFEFE, (i * 0x85EBCA6B >> 8) & 0xFEFEFE, 0x123456]
        out.append(op.scan(A, np.asarray(pts, np.float32), rgb[:len(pts)]))
    return out


@pytest.fixture(scope="module")
def limit_runs():
    """the oracle's bytes after LIMIT and LIMIT + 1 scans (the last scan of each run differs)"""
    refs = {}
    for n in (LIMIT, LIMIT + 1):
        case = op.Case(f"limit-{n}", 1.0, _limit_scans(n))
        m = op.oracle(case)
        refs[n] = (case, m.write(), m.stats())
    return refs


@pytest.mark.parametrize("n", [LIMIT, LIMIT + 1])
def test_scan_limit_batches_equal_the_oracle(fe, limit_runs, n):
    case, ref, ref_st = limit_runs[n]
    t0 = time.perf_counter()
    hs = _nodes(fe, case.scans)
    t1 = time.perf_counter()
    data, st = _device(fe, case, hs, [n])
    t2 = time.perf_counter()
    nh.destroy(fe, hs)
    print(f"{n} scans: nodes {t1 - t0:.2f} s, insert + write {t2 - t1:.2f} s")
    assert st == ref_st and data == ref
    lv = leaves(ref)
    assert (32768, 32768, 32772 + n % 2) in lv and lv[(32770, 32768, 32768)][1] != (255, 255, 255)
