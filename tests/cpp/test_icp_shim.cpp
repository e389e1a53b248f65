// The ICP fallback through the shim (Node::pcl_icp(), USE_PCL_ICP in the reference) and its icp_method (Node::icp_method(),
// icp.cpp:50-58).  RANSAC is made to fail with a tiny max_dist_for_inliers.  Input (argv[1]): int32 W, H, F, F grey images
// (W x H bytes), F float depth images (W x H floats).  Prints "ICP SHIM OK" when every check holds.  (CPU: compile + link;
// GPU: run.)
#include <cmath>
#include <cstdio>
#include <cstring>
#include <memory>
#include <string>
#include <vector>

#include "rgbdslam_b200/graph_manager.hpp"

using namespace rgbdslam_b200;

static int ok = 1;
#define CHECK(c)                                              \
  do {                                                        \
    if (!(c)) {                                               \
      std::printf("check failed line %d: %s\n", __LINE__, #c); \
      ok = 0;                                                 \
    }                                                         \
  } while (0)

static bool zero_info(const MatchingResult& m) {
  for (double v : m.edge.informationMatrix.m)
    if (v != 0.0) return false;
  return true;
}

// the edge of an ICP result as matchNodePair fills it
static bool is_icp_edge(const MatchingResult& mr, const rgbdslam_b200_icp_result& ir, int id1, int id2) {
  bool tr = true;
  for (int k = 0; k < 16; k++) tr &= mr.edge.transform.m[k] == (double)ir.T[k];
  return tr && mr.edge.id1 == id1 && mr.edge.id2 == id2 && !std::memcmp(mr.icp_trafo.m, ir.T, sizeof(ir.T)) &&
         !std::memcmp(mr.final_trafo.m, ir.T, sizeof(ir.T));
}

static bool same(const MatchingResult& a, const MatchingResult& b) {
  return a.edge.id1 == b.edge.id1 && a.edge.id2 == b.edge.id2 && !std::memcmp(&a.edge.transform, &b.edge.transform, sizeof(a.edge.transform)) &&
         !std::memcmp(&a.edge.informationMatrix, &b.edge.informationMatrix, sizeof(a.edge.informationMatrix)) && a.rmse == b.rmse &&
         !std::memcmp(&a.ransac_trafo, &b.ransac_trafo, sizeof(Matrix4f)) && !std::memcmp(&a.final_trafo, &b.final_trafo, sizeof(Matrix4f)) &&
         !std::memcmp(&a.icp_trafo, &b.icp_trafo, sizeof(Matrix4f)) && a.all_matches.size() == b.all_matches.size() &&
         a.inlier_matches.size() == b.inlier_matches.size() && a.inlier_points == b.inlier_points && a.all_points == b.all_points;
}

int main(int argc, char** argv) {
  if (argc != 2) return 2;
  rgbdslam_b200_params p;
  rgbdslam_b200_default_params(&p);
  p.depth_cov_z0 = 2.0;
  p.max_dist_for_inliers = 1e-9;  // no hypothesis finds inliers: RANSAC fails on every pair with enough matches
  if (rgbdslam_b200_init(0, &p) != 0) {
    std::printf("init failed (expected without a GPU): %s\n", rgbdslam_b200_last_error());
    return 77;
  }
  FILE* f = std::fopen(argv[1], "rb");
  int32_t dims[3];
  if (!f || std::fread(dims, 4, 3, f) != 3) return 2;
  const int W = dims[0], H = dims[1], F = dims[2];
  std::vector<uint8_t> gray((size_t)F * W * H);
  std::vector<float> depth((size_t)F * W * H);
  if (std::fread(gray.data(), 1, gray.size(), f) != gray.size() || std::fread(depth.data(), 4, depth.size(), f) != depth.size()) return 2;
  std::fclose(f);
  {
    Ptr<Feature2D> det(createDetector("ORB"));
    Ptr<DescriptorExtractor> ext = createDescriptorExtractor("ORB");
    CameraInfoConstPtr cam(new CameraInfo());
    auto make = [&](int frame, int id) {
      Mat visual(H, W, RB_8UC1, gray.data() + (size_t)frame * W * H);
      Mat d(H, W, RB_32FC1, depth.data() + (size_t)frame * W * H);
      myHeader hdr;
      hdr.seq = frame;
      hdr.stamp = frame / 30.0;
      std::unique_ptr<Node> n(new Node(visual, d, Mat(), cam, hdr, det, ext));
      n->id_ = id;
      return n;
    };
    // ---- off: the results of the plain RANSAC path ----
    Node::pcl_icp() = false;
    std::unique_ptr<Node> a0 = make(0, 0), a1 = make(1, 1);
    {
      rgbdslam_b200_pair_result r;
      std::vector<DMatch> all(p.max_matches), inl(p.max_matches);
      uint64_t hn = a1->handle(), ho = a0->handle();
      check(rgbdslam_b200_match_pairs(&hn, &ho, 1, 3, 0, &r, all.data(), inl.data()), "match_pairs");
      const MatchingResult direct = to_matching_result(r, all.data(), inl.data());
      const MatchingResult mr = a1->matchNodePair(a0.get(), 3, 0);
      CHECK(r.id1 < 0 && r.n_all_matches >= p.min_matches && r.info_scale == 0.0);
      CHECK(same(mr, direct) && mr.edge.id1 == -1 && a1->initial_node_matches_ == 0);
      // a node built with pcl_icp() off has no cloud: turning the fallback on later leaves its pairs without an edge
      Node::pcl_icp() = true;
      CHECK(a1->matchNodePair(a0.get(), 3, 0).edge.id1 == -1 && a1->initial_node_matches_ == 0);
    }
    // ---- on ----
    Node::pcl_icp() = true;
    std::unique_ptr<Node> n0 = make(0, 0), n1 = make(1, 1), n2 = make(2, 2), n3 = make(3, 3);
    {
      const MatchingResult mr = n1->matchNodePair(n0.get(), 3, 0);
      rgbdslam_b200_icp_result ir;
      uint64_t src = n0->handle(), tgt = n1->handle();  // the older cloud onto the newer one
      check(rgbdslam_b200_icp_align(1, &src, &tgt, Node::gicp_max_cloud_size(), &ir), "icp_align");
      CHECK(mr.edge.id1 == 0 && mr.edge.id2 == 1 && n1->initial_node_matches_ == 1 && ir.converged == 1);
      CHECK(!std::memcmp(mr.icp_trafo.m, ir.T, sizeof(ir.T)) && !std::memcmp(mr.final_trafo.m, ir.T, sizeof(ir.T)));
      bool tr = true;
      for (int k = 0; k < 16; k++) tr &= mr.edge.transform.m[k] == (double)ir.T[k];
      CHECK(tr && zero_info(mr) && mr.all_matches.size() >= (size_t)p.min_matches);
      // the reference's direction: the ICP edge maps older points into the newer frame, so the x translation of the camera
      // (moving along the trajectory) appears with the opposite sign of a RANSAC edge's; here: not the identity
      CHECK(std::fabs(ir.T[12]) + std::fabs(ir.T[13]) + std::fabs(ir.T[14]) > 1e-4);
      std::printf("icp edge 0->1: iterations %d criterion %d correspondences %d t = (%g %g %g)\n", ir.iterations, ir.criterion,
                  ir.n_correspondences, ir.T[12], ir.T[13], ir.T[14]);
    }
    // icp_method: "icp_nl" gives rgbdslam_b200_icp_align_ex(..., ICP_NL)'s edge; "gicp" or an unknown name the "icp" edge
    {
      CHECK(Node::icp_method() == "icp");
      uint64_t src = n0->handle(), tgt = n1->handle();
      rgbdslam_b200_icp_result icp, icp_nl, plain;
      check(rgbdslam_b200_icp_align_ex(1, &src, &tgt, Node::gicp_max_cloud_size(), RGBDSLAM_B200_ICP_METHOD_ICP, &icp), "icp");
      check(rgbdslam_b200_icp_align_ex(1, &src, &tgt, Node::gicp_max_cloud_size(), RGBDSLAM_B200_ICP_METHOD_ICP_NL, &icp_nl),
            "icp_nl");
      check(rgbdslam_b200_icp_align(1, &src, &tgt, Node::gicp_max_cloud_size(), &plain), "icp_align");
      CHECK(!std::memcmp(&plain, &icp, sizeof(icp)) && icp_nl.converged == 1);
      std::printf("icp: iterations %d criterion %d; icp_nl: iterations %d criterion %d\n", icp.iterations, icp.criterion,
                  icp_nl.iterations, icp_nl.criterion);
      const char* names[] = {"icp_nl", "icp", "gicp", "no_such_method"};
      for (const char* name : names) {
        Node::icp_method() = name;
        std::unique_ptr<Node> n = make(1, 1);
        const MatchingResult mr = n->matchNodePair(n0.get(), 3, 0);
        const bool nl = std::string(name) == "icp_nl";
        CHECK(is_icp_edge(mr, nl ? icp_nl : icp, 0, 1) && n->initial_node_matches_ == 1);
        if (!is_icp_edge(mr, nl ? icp_nl : icp, 0, 1)) std::printf("  method %s\n", name);
      }
      Node::icp_method() = "icp";
    }
    // non-adjacent: no ICP
    CHECK(n3->matchNodePair(n0.get(), 3, 0).edge.id1 == -1 && n3->initial_node_matches_ == 0);
    // fewer than min_matches feature matches (a blank frame has no features, but a cloud): no ICP
    {
      std::vector<uint8_t> blank((size_t)W * H, 0);
      Mat visual(H, W, RB_8UC1, blank.data());
      Mat d(H, W, RB_32FC1, depth.data() + (size_t)2 * W * H);
      myHeader hdr;
      Node few(visual, d, Mat(), cam, hdr, det, ext);
      few.id_ = 2;
      const MatchingResult mr = n3->matchNodePair(&few, 3, 0);
      CHECK(mr.edge.id1 == -1 && (int)mr.all_matches.size() < p.min_matches && n3->initial_node_matches_ == 0);
    }
    // max_connections, in order: three adjacent candidates, at most max_connections + 1 accepted before the limit binds
    {
      Node::max_connections() = 1;
      std::unique_ptr<Node> b = make(2, 2);
      std::vector<const Node*> olds = {n1.get(), n2.get(), n1.get()};
      const std::vector<MatchingResult> v = Node::matchNodePairs(b.get(), olds, 3, 0);
      CHECK(v[0].edge.id1 == 1 && v[1].edge.id1 == 2 && v[2].edge.id1 == -1 && b->initial_node_matches_ == 2);
      b->initial_node_matches_ = 0;  // the same comparisons one call at a time, as the reference's loop makes them
      for (size_t k = 0; k < olds.size(); k++) CHECK(same(v[k], b->matchNodePair(olds[k], 3, (int64_t)k)));
      CHECK(b->initial_node_matches_ == 2);
      Node::max_connections() = -1;
    }
    // the online GraphManager with the fallback
    {
      GraphManager gm;
      gm.seed = 5;
      for (int i = 0; i < F; i++) {
        std::unique_ptr<Node> n = make(i, -1);
        n->id_ = -1;
        Node* raw = n.release();
        if (!gm.addNode(raw)) delete raw;
      }
      gm.optimizeGraph();
      int finite = 1;
      for (auto& kv : gm.graph_) {
        double t[12];
        gm.mapTransform(kv.second->vertex_id_, t);
        for (double x : t) finite &= std::isfinite(x);
      }
      CHECK(finite && gm.graph_.size() >= (size_t)F / 2);
      std::printf("graph nodes %zu\n", gm.graph_.size());
    }
  }
  rgbdslam_b200_shutdown();
  std::printf(ok ? "ICP SHIM OK\n" : "ICP SHIM FAILED\n");
  return ok ? 0 : 1;
}
