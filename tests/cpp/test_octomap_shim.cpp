// The reference's OctoMap path against the shim.
//   test_octomap_shim pose: reads lines of 12 doubles (row-major rotation R, translation t) from stdin and prints the 12
//     float bits (hex) of octomapPose(R, t) per line.  Needs no GPU.
//   test_octomap_shim frames.bin outdir: image Nodes built with Node::store_pointclouds(), added to the online GraphManager,
//     optimised, then GraphManager::saveOctomap twice: (1) octomap_autosave_step 3, no clear flags, into outdir/a.ot -- every
//     write is also copied to outdir/a_<k>.ot --, and writeOctomap(outdir/a_again.ot); the nodes' clouds are dumped as
//     32-byte records to outdir/cloud_<id>.bin; (2) both clear flags, into outdir/b.ot (writes copied to outdir/b_<k>.ot),
//     then writeOctomap(outdir/b_after.ot).  Prints "NODE id selected R[9] t[3] T[12 hex]" per node and "CLEARED id 0|1"
//     (1: the node has no stored cloud any more) after (2).  Input: int32 W, H, F, F grey images (W x H bytes), F float depth images (W x H floats).
#include <cstdio>
#include <iostream>
#include <stdexcept>
#include <string>
#include <vector>

#include "rgbdslam_b200/graph_manager.hpp"

using namespace rgbdslam_b200;

struct RecordingGraphManager : GraphManager {
  std::string prefix;
  mutable int writes = 0;
  void writeOctomap(const std::string& filename) const override {
    GraphManager::writeOctomap(filename);
    if (!prefix.empty()) GraphManager::writeOctomap(prefix + "_" + std::to_string(++writes) + ".ot");
  }
};

static void print_bits(const float* T) {
  for (int k = 0; k < 12; k++) {
    uint32_t u;
    std::memcpy(&u, &T[k], 4);
    std::printf(" %08x", u);
  }
}

int main(int argc, char** argv) {
  if (argc == 2 && std::string(argv[1]) == "pose") {
    double v[12];
    while (std::cin >> v[0]) {
      for (int k = 1; k < 12; k++) std::cin >> v[k];
      float T[12];
      octomapPose(v, v + 9, T);
      print_bits(T);
      std::printf("\n");
    }
    return 0;
  }
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
  int ok = 1;
  {
    Node::store_pointclouds() = true;
    RecordingGraphManager gm;
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
    for (auto& kv : gm.graph_) {
      const Node* n = kv.second;
      const bool sel = gm.updateCloudOrigin(n);
      std::printf("NODE %d %d", n->id_, (int)sel);
      if (sel) {
        const double* e = gm.estimates_.at(n->vertex_id_).v;
        double R[9];
        quatToRot(e + 3, R);
        for (int k = 0; k < 9; k++) std::printf(" %.17g", R[k]);
        for (int k = 0; k < 3; k++) std::printf(" %.17g", e[k]);
        float T[12];
        gm.octomapTransform(n->vertex_id_, T);
        print_bits(T);
        pointcloud_type::Ptr pc = n->pointCloud();
        FILE* o = std::fopen((out + "/cloud_" + std::to_string(n->id_) + ".bin").c_str(), "wb");
        ok &= o && std::fwrite(pc->points.data(), sizeof(point_type), pc->points.size(), o) == pc->points.size();
        if (o) std::fclose(o);
      }
      std::printf("\n");
    }
    GraphManager::octomap_autosave_step() = 3;
    gm.prefix = out + "/a";
    gm.saveOctomap(out + "/a.ot");
    std::printf("WRITES a %d\n", gm.writes);
    gm.prefix.clear();
    gm.writeOctomap(out + "/a_again.ot");
    GraphManager::octomap_clear_after_save() = true;
    GraphManager::octomap_clear_raycasted_clouds() = true;
    gm.prefix = out + "/b";
    gm.writes = 0;
    gm.saveOctomap(out + "/b.ot");
    std::printf("WRITES b %d\n", gm.writes);
    gm.prefix.clear();
    gm.writeOctomap(out + "/b_after.ot");
    for (auto& kv : gm.graph_) {  // a cleared node has no stored cloud left: node_download_cloud refuses it
      int w = 0, h = 0;
      const int rc = rgbdslam_b200_node_download_cloud(kv.second->handle(), 32, nullptr, &w, &h);
      std::printf("CLEARED %d %d\n", kv.second->id_, rc == RGBDSLAM_B200_ERR_STATE ? 1 : 0);
    }
    ok &= gm.graph_.size() >= (size_t)F / 2;
  }
  rgbdslam_b200_shutdown();
  std::printf(ok ? "OCTOMAP SHIM OK\n" : "OCTOMAP SHIM FAILED\n");
  return ok ? 0 : 1;
}
