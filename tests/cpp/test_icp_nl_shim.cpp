// icp_method through the shim (Node::icp_method(), icp.cpp:50-58).  RANSAC is made to fail with a tiny max_dist_for_inliers,
// so the adjacent pair takes the ICP edge.  With "icp_nl" the edge is rgbdslam_b200_icp_align_ex(..., ICP_NL)'s; with "gicp"
// or an unknown name it is the "icp" edge.  Input (argv[1]): int32 W, H, F, F grey images (W x H bytes), F float depth images
// (W x H floats).  Prints "ICP_NL SHIM OK" when every check holds.  (CPU: compile + link; GPU: run.)
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

// the edge of an ICP result as matchNodePair fills it
static bool is_icp_edge(const MatchingResult& mr, const rgbdslam_b200_icp_result& ir, int id1, int id2) {
  bool tr = true;
  for (int k = 0; k < 16; k++) tr &= mr.edge.transform.m[k] == (double)ir.T[k];
  return tr && mr.edge.id1 == id1 && mr.edge.id2 == id2 && !std::memcmp(mr.icp_trafo.m, ir.T, sizeof(ir.T)) &&
         !std::memcmp(mr.final_trafo.m, ir.T, sizeof(ir.T));
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
    Node::pcl_icp() = true;
    CHECK(Node::icp_method() == "icp");
    std::unique_ptr<Node> n0 = make(0, 0);
    uint64_t src = n0->handle();
    rgbdslam_b200_icp_result icp, icp_nl;
    std::unique_ptr<Node> probe = make(1, 1);
    uint64_t tgt = probe->handle();
    check(rgbdslam_b200_icp_align_ex(1, &src, &tgt, Node::gicp_max_cloud_size(), RGBDSLAM_B200_ICP_METHOD_ICP, &icp), "icp");
    check(rgbdslam_b200_icp_align_ex(1, &src, &tgt, Node::gicp_max_cloud_size(), RGBDSLAM_B200_ICP_METHOD_ICP_NL, &icp_nl),
          "icp_nl");
    rgbdslam_b200_icp_result plain;
    check(rgbdslam_b200_icp_align(1, &src, &tgt, Node::gicp_max_cloud_size(), &plain), "icp_align");
    CHECK(!std::memcmp(&plain, &icp, sizeof(icp)) && icp_nl.converged == 1);
    std::printf("icp: iterations %d criterion %d; icp_nl: iterations %d criterion %d\n", icp.iterations, icp.criterion,
                icp_nl.iterations, icp_nl.criterion);
    const char* names[] = {"icp_nl", "icp", "gicp", "no_such_method"};
    for (const char* name : names) {
      Node::icp_method() = name;
      std::unique_ptr<Node> n1 = make(1, 1);
      const MatchingResult mr = n1->matchNodePair(n0.get(), 3, 0);
      const bool nl = std::string(name) == "icp_nl";
      CHECK(is_icp_edge(mr, nl ? icp_nl : icp, 0, 1) && n1->initial_node_matches_ == 1);
      if (!is_icp_edge(mr, nl ? icp_nl : icp, 0, 1)) std::printf("  method %s\n", name);
    }
    Node::icp_method() = "icp";
  }
  rgbdslam_b200_shutdown();
  std::printf(ok ? "ICP_NL SHIM OK\n" : "ICP_NL SHIM FAILED\n");
  return ok ? 0 : 1;
}
