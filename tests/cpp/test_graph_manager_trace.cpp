// Trace of the GraphManager shim (include/rgbdslam_b200/graph_manager.hpp) on a rendered sequence, for a bit-exact comparison
// with its Python twin (oracle/graph_manager_oracle.py) in tests/test_gpu_graph_manager_parity.py.
//   test_graph_manager_trace FRAMES PARAMS OUT
// FRAMES: int64 F, W, H; float64 fx, fy, cx, cy; float64 stamps[F]; uint8 grey[F][H][W]; float32 depth[F][H][W] (metres);
//         uint8 detection mask[F][H][W]
// PARAMS: float64 values, in this order: seed, depth_cov_z0, max_keypoints, the GraphManager::Params fields (min_matches,
//         predecessor_candidates, neighbor_candidates, min_sampled_candidates, geodesic_depth, min_translation_meter,
//         min_rotation_degree, max_translation_meter, max_rotation_degree, keep_all_nodes, keep_good_nodes, optimizer_skip_step,
//         optimizer_iterations, huber_delta, valid_odometry, pose_relative_to as 0 first / 1 previous / 2 largest_loop /
//         3 inaffected), Node::max_connections; n extra edges, each id1, id2, its 4 x 4 transform (column-major) and information
//         scale, added to the final graph with addEdgeToG2O; n pruning thresholds, each pruneEdgesWithErrorAbove + optimizeGraph.
// OUT: float64 values (ids and counts are exact), one record per addNode call (tag 1), then the extra edges (tag 2), then one
//      record per threshold (tag 3); the layout is what write_* below append, read back by the test.
// Each frame is one Node of the raw-image constructor, addNode in arrival order.  Exit code 77 without a GPU.
#include <cstdio>
#include <fstream>
#include <string>
#include <vector>

#include "rgbdslam_b200/graph_manager.hpp"

using namespace rgbdslam_b200;

namespace {

struct Out {
  std::vector<double> v;
  void put(double x) { v.push_back(x); }
  void put(const double* p, size_t n) { v.insert(v.end(), p, p + n); }
};

// optimizeGraph observed: the arrays gather + fixationOfVertices hand the solver, and the estimates it returns
struct TraceGraphManager : GraphManager {
  std::vector<std::vector<double>> opts;
  double optimizeGraph(double break_criterion = -1.0, bool nonthreaded = false) override {
    std::vector<int> ids;
    std::vector<double> poses, meas, info;
    std::vector<uint8_t> fixed;
    std::vector<int32_t> ij;
    gather(ids, poses, fixed, ij, meas, info);
    if (ij.empty()) return GraphManager::optimizeGraph(break_criterion, nonthreaded);
    fixationOfVertices(ids, fixed);
    const double chi2 = GraphManager::optimizeGraph(break_criterion, nonthreaded);
    Out o;
    o.put((double)ids.size());
    for (int id : ids) o.put(id);
    for (uint8_t f : fixed) o.put(f);
    o.put(poses.data(), poses.size());
    o.put((double)(ij.size() / 2));
    for (int32_t k : ij) o.put(k);
    o.put(meas.data(), meas.size());
    o.put(info.data(), info.size());
    for (int id : ids) o.put(estimates_.at(id).v, 7);
    o.put(chi2);
    opts.push_back(o.v);
    return chi2;
  }
  void write_opts(Out& o) {
    o.put((double)opts.size());
    for (auto& r : opts) o.put(r.data(), r.size());
    opts.clear();
  }
  void write_edges(Out& o, size_t from) {
    o.put((double)(edges_.size() - from));
    for (size_t e = from; e < edges_.size(); e++) {
      o.put(edges_[e].first);
      o.put(edges_[e].second);
      o.put(meas_[e].v, 7);
      o.put(info_[e].m, 36);
    }
  }
};

template <class T>
void read(std::ifstream& f, T* p, size_t n) {
  f.read(reinterpret_cast<char*>(p), (std::streamsize)(n * sizeof(T)));
  if (!f) throw std::runtime_error("short input file");
}

}  // namespace

int main(int argc, char** argv) {
  if (argc != 4) {
    std::fprintf(stderr, "usage: %s FRAMES PARAMS OUT\n", argv[0]);
    return 2;
  }
  std::ifstream ff(argv[1], std::ios::binary), pf(argv[2], std::ios::binary);
  int64_t dims[3];
  read(ff, dims, 3);
  const int F = (int)dims[0], W = (int)dims[1], H = (int)dims[2];
  const size_t px = (size_t)W * H;
  double K[4];
  read(ff, K, 4);
  std::vector<double> stamps(F);
  read(ff, stamps.data(), F);
  std::vector<uint8_t> grey(F * px), mask(F * px);
  std::vector<float> depth(F * px);
  read(ff, grey.data(), grey.size());
  read(ff, depth.data(), depth.size());
  read(ff, mask.data(), mask.size());
  std::vector<double> prm;
  for (double x; pf.read(reinterpret_cast<char*>(&x), sizeof x);) prm.push_back(x);
  size_t at = 0;
  auto next = [&]() {
    if (at >= prm.size()) throw std::runtime_error("short parameter file");
    return prm[at++];
  };

  rgbdslam_b200_params lp;
  rgbdslam_b200_default_params(&lp);
  const uint64_t seed = (uint64_t)next();
  lp.depth_cov_z0 = next();
  lp.max_keypoints = (int32_t)next();
  if (rgbdslam_b200_init(0, &lp) != 0) {
    std::printf("init failed (expected without a GPU): %s\n", rgbdslam_b200_last_error());
    return 77;
  }
  int rc = 0;
  {
    TraceGraphManager gm;
    gm.seed = seed;
    GraphManager::Params& p = gm.params;
    p.min_matches = (int)next(); p.predecessor_candidates = (int)next(); p.neighbor_candidates = (int)next();
    p.min_sampled_candidates = (int)next(); p.geodesic_depth = (int)next();
    p.min_translation_meter = next(); p.min_rotation_degree = next(); p.max_translation_meter = next(); p.max_rotation_degree = next();
    p.keep_all_nodes = next() != 0; p.keep_good_nodes = next() != 0; p.optimizer_skip_step = (int)next();
    p.optimizer_iterations = next(); p.huber_delta = next(); p.valid_odometry = next() != 0;
    static const char* strategies[] = {"first", "previous", "largest_loop", "inaffected"};
    p.pose_relative_to = strategies[(int)next()];
    Node::max_connections() = (int)next();

    std::vector<int> targets;
    bool compared = false;
    gm.on_edge_targets_ = [&](const std::vector<int>& t) { targets = t; compared = true; };
    uint64_t detector = 0;
    check(rgbdslam_b200_detector_create(&detector), "detector_create");
    const float K4[4] = {(float)K[0], (float)K[1], (float)K[2], (float)K[3]};
    Out o;
    for (int k = 0; k < F; k++) {
      Node* n = new Node(&grey[k * px], &depth[k * px], &mask[k * px], W, H, K4, k, detector, stamps[k]);
      const size_t n2d = n->feature_locations_2d_.size(), n3d = n->feature_locations_3d_.size();
      size_t edges_before = gm.edges_.size();
      compared = false;
      const bool added = gm.addNode(n);
      if (gm.edges_.size() < edges_before) edges_before = 0;  // the first node was replaced (resetGraph)
      o.put(1); o.put(k); o.put(added ? 1 : 0); o.put(added ? n->id_ : -1); o.put((double)n2d); o.put((double)n3d);
      o.put(compared ? (double)targets.size() : -1.0);
      if (compared) for (int t : targets) o.put(t);
      gm.write_edges(o, edges_before);
      o.put((double)gm.keyframe_ids_.size());
      for (int id : gm.keyframe_ids_) o.put(id);
      o.put(gm.earliest_loop_closure_node_);
      o.put((double)gm.estimates_.size());
      for (auto& kv : gm.estimates_) { o.put(kv.first); o.put(kv.second.v, 7); }
      gm.write_opts(o);
      if (!added) delete n;
    }
    const int n_extra = (int)next();
    o.put(2); o.put(n_extra);
    for (int e = 0; e < n_extra; e++) {
      LoadedEdge3D edge;
      edge.id1 = (int)next(); edge.id2 = (int)next();
      for (int i = 0; i < 16; i++) edge.transform.m[i] = next();
      const double scale = next();
      std::memset(&edge.informationMatrix, 0, sizeof(edge.informationMatrix));
      for (int i = 0; i < 6; i++) edge.informationMatrix.m[7 * i] = scale;
      const bool ok = gm.graph_.count(edge.id1) && gm.graph_.count(edge.id2) &&
                      gm.addEdgeToG2O(edge, gm.graph_[edge.id1], gm.graph_[edge.id2], false, false);
      o.put(ok ? 1 : 0);
    }
    const int n_thresh = (int)next();
    for (int t = 0; t < n_thresh; t++) {
      const double thresh = next();
      std::vector<int> ids;
      std::vector<double> poses, meas, info;
      std::vector<uint8_t> fixed;
      std::vector<int32_t> ij;
      std::vector<size_t> which;
      gm.gather(ids, poses, fixed, ij, meas, info, &which);
      o.put(3); o.put(thresh);
      o.put((double)ids.size());
      for (int id : ids) o.put(id);
      o.put(poses.data(), poses.size());
      auto write_state = [&]() {  // every edge ever added: active flag, ids, measurement, information
        o.put((double)gm.edges_.size());
        for (size_t e = 0; e < gm.edges_.size(); e++) o.put(gm.active_[e] ? 1 : 0);
        gm.write_edges(o, 0);
      };
      write_state();
      o.put(gm.pruneEdgesWithErrorAbove((float)thresh));
      write_state();
      gm.optimizeGraph();
      gm.write_opts(o);
    }
    check(rgbdslam_b200_detector_destroy(detector), "detector_destroy");
    std::FILE* f = std::fopen(argv[3], "wb");
    if (!f || std::fwrite(o.v.data(), sizeof(double), o.v.size(), f) != o.v.size()) rc = 1;
    if (f && std::fclose(f) != 0) rc = 1;
    std::printf("%d frames, %zu nodes, %zu edges, %zu keyframes\n", F, gm.graph_.size(), gm.edges_.size(), gm.keyframe_ids_.size());
  }
  rgbdslam_b200_shutdown();
  return rc;
}
