"""CPU twin of rgbdslam_v2_b200.pipeline.GpuBackend built on the oracle -- TEST INFRASTRUCTURE (used by tests/ and by the
CPU-baseline / parity legs of bench.py), never by the product path."""
import numpy as np


class OracleBackend:
    """cv2 ORB + reference glue (oracle/orb_oracle.py), C oracle for matching / RANSAC and the pose graph."""

    def __init__(self, oracle_mod, max_keypoints):
        from oracle import orb_oracle
        self.o, self.orb = oracle_mod, orb_oracle
        self.st = orb_oracle.DetectorState()
        self.K = max_keypoints

    def construct_nodes(self, gray, depth, mask, K4):
        return [self.orb.node_construct(g, d, m, K4, self.st, max_keypoints=self.K) for g, d, m in zip(gray, depth, mask)]

    def match(self, nodes, pairs, seed):
        prm = self.o.make_params(depth_cov_z0=2.0)
        dn = np.concatenate([nodes[a][1] for a, _ in pairs]); xn = np.concatenate([nodes[a][2] for a, _ in pairs])
        do = np.concatenate([nodes[b][1] for _, b in pairs]); xo = np.concatenate([nodes[b][2] for _, b in pairs])
        nn = [len(nodes[a][1]) for a, _ in pairs]; no = [len(nodes[b][1]) for _, b in pairs]
        res, _, _ = self.o.match_pairs(prm, dn, xn, nn, do, xo, no, [a for a, _ in pairs], [b for _, b in pairs], seed=seed,
                                       threads=8, want_matches=False)
        return res

    def n_features(self, handle):
        return len(handle[1])

    def match_one_to_many(self, node, olds, seed, first_pair_index=None):
        prm = self.o.make_params(depth_cov_z0=2.0)
        new = node.handle
        dn = np.concatenate([new[1]] * len(olds)); xn = np.concatenate([new[2]] * len(olds))
        do = np.concatenate([o.handle[1] for o in olds]); xo = np.concatenate([o.handle[2] for o in olds])
        res, _, _ = self.o.match_pairs(prm, dn, xn, [len(new[1])] * len(olds), do, xo, [len(o.handle[1]) for o in olds],
                                       [node.id] * len(olds), [o.id for o in olds], seed=seed,
                                       first_pair_index=64 * node.id if first_pair_index is None else first_pair_index,
                                       threads=8, want_matches=False)
        return res

    def optimize(self, graph, stop):
        x, chi2, _, _ = self.o.posegraph_optimize(graph["init"], graph["fixed"], graph["ij"], graph["meas"], graph["info"], stop=stop)
        return x, chi2

    def edge_chi2(self, poses, graph):
        out = np.zeros(len(graph["ij"]))
        for k, (i, j) in enumerate(graph["ij"]):
            e = self.o.edge_se3(poses[i], poses[j], graph["meas"][k], False)[0]
            out[k] = e @ graph["info"][k].reshape(6, 6) @ e
        return out
