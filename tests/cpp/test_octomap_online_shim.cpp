// The reference's online OctoMap (octomap_online_creation) and occupancyFilterClouds against the shim.
//   test_octomap_online_shim frames.bin outdir: image Nodes built with Node::store_pointclouds() are added to a GraphManager with
//     octomap_online_creation on, and octomap_clear_raycasted_clouds too when the file outdir/clear exists.  After each
//     addNode it prints "ADDED frame added [newest_id optimised valid_tf T[12 hex]]": the newest node, whether addNode ran
//     optimizeGraph, its valid_tf_estimate_ and the transform it renders with.  Then saveOctomap(outdir/online.ot); per node its
//     cloud (32-byte records) to outdir/before_<id>.bin and "SENSOR id q[4] o[3] hex" (the sensor pose its cloud holds);
//     occupancyFilterClouds() with occupancy_filter_threshold 3e4; per node "CLOUD id 0|1" (1: it has a stored cloud) and
//     its cloud to outdir/after_<id>.bin.  Input: int32 W, H, F, F grey images (W x H bytes), F float depth images.
#include <cstdio>
#include <fstream>
#include <string>
#include <vector>

#include "rgbdslam_b200/graph_manager.hpp"

using namespace rgbdslam_b200;

static void print_hex(const float* v, int n) {
  for (int k = 0; k < n; k++) {
    uint32_t u;
    std::memcpy(&u, &v[k], 4);
    std::printf(" %08x", u);
  }
}

static void dump(const Node* n, const std::string& path) {
  int w = 0, h = 0;
  if (rgbdslam_b200_node_download_cloud(n->handle(), 32, nullptr, &w, &h) != 0) return;
  std::vector<PointXYZRGB> pts((size_t)w * h);
  if (!pts.empty()) check(rgbdslam_b200_node_download_cloud(n->handle(), 32, pts.data(), &w, &h), "node_download_cloud");
  FILE* o = std::fopen(path.c_str(), "wb");
  if (!o) return;
  std::fwrite(pts.data(), sizeof(PointXYZRGB), pts.size(), o);
  std::fclose(o);
}

int main(int argc, char** argv) {
  if (argc != 3) return 2;
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
  const std::string out = argv[2];
  const bool clear = (bool)std::ifstream(out + "/clear");
  int ok = 1;
  {
    Node::store_pointclouds() = true;
    GraphManager::octomap_online_creation() = true;
    GraphManager::octomap_clear_raycasted_clouds() = clear;
    GraphManager::occupancy_filter_threshold() = 3e4;
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
      const bool added = gm.addNode(n);
      std::printf("ADDED %d %d", i, (int)added);
      if (added) {
        const Node* newest = gm.graph_.at((int)gm.graph_.size() - 1);
        const bool optimised = gm.graph_.size() == 1 ||
                               (gm.params.optimizer_skip_step > 0 && (int)gm.estimates_.size() % gm.params.optimizer_skip_step == 0);
        std::printf(" %d %d %d", newest->id_, (int)optimised, (int)newest->valid_tf_estimate_);
        if (gm.estimates_.count(newest->vertex_id_)) {
          float T[12];
          gm.octomapTransform(newest->vertex_id_, T);
          print_hex(T, 12);
        }
      } else {
        delete n;
      }
      std::printf("\n");
    }
    gm.saveOctomap(out + "/online.ot");
    for (auto& kv : gm.graph_) {
      dump(kv.second, out + "/before_" + std::to_string(kv.first) + ".bin");
      std::printf("SENSOR %d", kv.first);
      print_hex(kv.second->cloud_sensor_pose_, 7);
      std::printf("\n");
    }
    gm.occupancyFilterClouds();
    for (auto& kv : gm.graph_) {
      int w = 0, h = 0;
      const int rc = rgbdslam_b200_node_download_cloud(kv.second->handle(), 32, nullptr, &w, &h);
      std::printf("CLOUD %d %d\n", kv.first, rc == 0 ? 1 : 0);
      dump(kv.second, out + "/after_" + std::to_string(kv.first) + ".bin");
    }
    ok &= gm.graph_.size() >= (size_t)F / 2;
  }
  rgbdslam_b200_shutdown();
  std::printf(ok ? "ONLINE SHIM OK\n" : "ONLINE SHIM FAILED\n");
  return ok ? 0 : 1;
}
