// The voxel filter through the shim: image Nodes built with Node::store_pointclouds(), added to the online GraphManager,
// GraphManager::saveAllClouds, then GraphManager::reducePointClouds and saveAllClouds again.  Input (argv[1]): int32 W, H, F,
// F grey images (W x H bytes), F float depth images (W x H floats).  Writes the raw map to argv[2] + "_raw.pcd", the reduced
// one to argv[2] + "_reduced.pcd" and the 32-byte render_cloud records of the reduced nodes under mapTransform to argv[3].
// (CPU: compile + link; GPU: run.)
#include <cstdio>
#include <string>
#include <vector>

#include "rgbdslam_b200/graph_manager.hpp"

using namespace rgbdslam_b200;

int main(int argc, char** argv) {
  if (argc != 4) return 2;
  rgbdslam_b200_params p;
  rgbdslam_b200_default_params(&p);
  p.depth_cov_z0 = 2.0;
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
  int ok = 1;
  {
    Node::store_pointclouds() = true;
    GraphManager gm;
    gm.seed = 5;
    Ptr<Feature2D> detector_(createDetector("ORB"));
    Ptr<DescriptorExtractor> extractor_ = createDescriptorExtractor("ORB");
    CameraInfoConstPtr cam_info(new CameraInfo());
    for (int i = 0; i < F; i++) {
      Mat visual(H, W, RB_8UC1, gray.data() + (size_t)i * W * H);
      Mat d(H, W, RB_32FC1, depth.data() + (size_t)i * W * H);
      myHeader hdr;
      hdr.seq = i;
      hdr.stamp = i / 30.0;
      Node* n = new Node(visual, d, Mat(), cam_info, hdr, detector_, extractor_);
      if (!gm.addNode(n)) delete n;
    }
    gm.optimizeGraph();
    const std::string base = argv[2];
    const size_t raw = gm.saveAllClouds(base + "_raw.pcd");
    Node* first = gm.graph_.begin()->second;
    // an invalid voxelfilter_size warns and changes nothing (node.cpp:1457-1459)
    ok &= gm.reducePointClouds() == 0;  // the default, -1
    first->reducePointCloud(-1.0);
    first->reducePointCloud(0.0);
    ok &= first->pointCloud()->width == (uint32_t)W / 2 && first->pointCloud()->height == (uint32_t)H / 2;
    // one node on its own, then the whole graph (the first node a second time)
    first->reducePointCloud(0.02);
    const uint32_t first_points = first->pointCloud()->width;
    ok &= first->pointCloud()->height == 1 && first_points > 0 && first_points < (uint32_t)(W / 2 * H / 2);
    GraphManager::voxelfilter_size() = 0.05;
    ok &= gm.reducePointClouds() == gm.graph_.size();
    ok &= first->pointCloud()->width < first_points;
    const size_t reduced = gm.saveAllClouds(base + "_reduced.pcd");
    std::vector<uint64_t> handles;
    std::vector<double> T;
    for (auto& kv : gm.graph_) {
      const Node* n = kv.second;
      ok &= n->pointCloud()->height == 1;
      if (!n->valid_tf_estimate_) continue;
      double t[12];
      gm.mapTransform(n->vertex_id_, t);
      handles.push_back(n->handle());
      T.insert(T.end(), t, t + 12);
    }
    int64_t count = 0;
    check(rgbdslam_b200_render_cloud((int)handles.size(), handles.data(), T.data(), GraphManager::maximum_depth(), 0, 32, nullptr, 0,
                                     &count, nullptr),
          "render_cloud");
    std::vector<PointXYZRGB> pts((size_t)count);
    check(rgbdslam_b200_render_cloud((int)handles.size(), handles.data(), T.data(), GraphManager::maximum_depth(), 0, 32, pts.data(),
                                     count, &count, nullptr),
          "render_cloud");
    FILE* o = std::fopen(argv[3], "wb");
    ok &= o && std::fwrite(pts.data(), sizeof(PointXYZRGB), pts.size(), o) == pts.size();
    if (o) std::fclose(o);
    ok &= reduced == pts.size() && reduced > 0 && reduced < raw && gm.graph_.size() >= (size_t)F / 2;
    std::printf("nodes %zu raw %zu reduced %zu\n", gm.graph_.size(), raw, reduced);
  }
  rgbdslam_b200_shutdown();
  std::printf(ok ? "VOXEL SHIM OK\n" : "VOXEL SHIM FAILED\n");
  return ok ? 0 : 1;
}
