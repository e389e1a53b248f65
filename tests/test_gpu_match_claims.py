"""The ORB match kernel's CTAs claim work items from a per-slot ticket counter that every launch leaves where the next launch
on that slot expects it.  Several slots in flight at once, each launching several times with more items than SMs and ragged
pairs, must all give the best matches of the SIMT path."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu

SIZES = [(1000, 1000), (257, 129), (5, 1), (130, 2), (3, 600), (1000, 128), (999, 1025), (1, 1), (64, 4096), (4096, 64)]


@pytest.fixture(scope="module")
def fe(built):
    from rgbdslam_v2_b200 import Frontend
    from rgbdslam_v2_b200._capi import default_params
    p = default_params()
    p.depth_cov_z0 = 2.0
    f = Frontend(0, p)
    yield f
    f.close()


def _batch(fe, rng, n_pairs, id0):
    newer, older = [], []
    for i in range(n_pairs):
        nq, nt = SIZES[(i + id0) % len(SIZES)]
        q = rng.integers(0, 256, (nq, 32), dtype=np.uint8)
        t = rng.integers(0, 256, (nt, 32), dtype=np.uint8)
        k = min(nq, nt) // 2
        if k:
            q[:k] = t[rng.permutation(nt)[:k]] ^ (rng.random((k, 32)) < 0.05).astype(np.uint8)
        xq = np.concatenate([rng.uniform(0.5, 3, (nq, 3)), np.ones((nq, 1))], 1).astype(np.float32)
        xt = np.concatenate([rng.uniform(0.5, 3, (nt, 3)), np.ones((nt, 1))], 1).astype(np.float32)
        newer.append(fe.node_from_features(id0 + 2 * i + 1, q, xq))
        older.append(fe.node_from_features(id0 + 2 * i, t, xt))
    return np.array(newer, np.uint64), np.array(older, np.uint64)


def test_claim_counter_across_launches_and_concurrent_slots(fe):
    rng = np.random.default_rng(2024)
    slots = (1, 2, 3)
    # 50 ragged pairs = 175 work items per launch, more than the 132 SMs of an H100
    batches = [_batch(fe, rng, 50, 1000 * (j + 1)) for j in range(len(slots))]
    try:
        fe.set_hamming_path(0)
        ref = [fe.match_node_pairs(n, o, seed=9) for n, o in batches]
    finally:
        fe.set_hamming_path(1)
    for rnd in range(3):
        outs = [fe._alloc_out(len(n), True) for n, _ in batches]
        for slot, (n, o), out in zip(slots, batches, outs):
            fe.submit_node_pairs(slot, n, o, out, seed=9)
        # the synchronous entry points share slot 0's counter with match_pairs: launch there too while the others run
        r0 = fe.match_node_pairs(*batches[rnd % len(batches)], seed=9)
        for slot in slots:
            fe.wait_slot(slot)
        for j, ((res, allm, _), (rres, rallm, _)) in enumerate(zip(outs + [r0], ref + [ref[rnd % len(batches)]])):
            assert np.array_equal(res["n_all_matches"], rres["n_all_matches"]), (rnd, j)
            for i in range(len(res)):
                n = int(res["n_all_matches"][i])
                for f in ("queryIdx", "trainIdx", "distance"):
                    assert np.array_equal(allm[i, :n][f], rallm[i, :n][f]), (rnd, j, i, f)
    for n, o in batches:
        for h in list(n) + list(o):
            fe.node_destroy(int(h))
