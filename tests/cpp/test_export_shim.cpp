// The reference's per-node exports against the shim: GraphManager::saveIndividualClouds in both transform_individual_clouds
// modes and GraphManager::saveAllFeatures.
//   test_export_shim frames.bin outdir: image Nodes built with Node::store_pointclouds() are added to a GraphManager, which is
//     optimised; node 1 then loses its valid estimate ("INVALIDATED 1") and the newest valid node its cloud ("CLEARED id").
//     Per node it prints
//     "NODE id valid has_estimate iso[12] tf[12] map[12]" (%.17g: the estimate as a 3 x 4, eigenTransf2TF of it and
//     mapTransform), writes its cloud's 32-byte records to outdir/before_<id>.bin ("CLOUD id w h") and its features to
//     outdir/features_<id>.bin (int32 n, n x 4 float locations, n x 32 descriptor bytes).  Then saveIndividualClouds
//     (outdir/plain), "SENSOR plain id q[4] o[3]" (hex) per node; with transform_individual_clouds saveIndividualClouds
//     (outdir/xf1), the clouds to outdir/xf1_<id>.bin, "SENSOR xf1 ..."; again (outdir/xf2, outdir/xf2_<id>.bin); then
//     saveAllFeatures(outdir/features.yml).  "SAVED name n" gives each call's return value.  Input: int32 W, H, F, F grey
//     images (W x H bytes), F float depth images.
#include <cstdio>
#include <stdexcept>
#include <string>
#include <vector>

#include "rgbdslam_b200/graph_manager.hpp"

using namespace rgbdslam_b200;

static bool dump_cloud(const Node* n, const std::string& path, int* w, int* h) {
  if (rgbdslam_b200_node_download_cloud(n->handle(), 32, nullptr, w, h) != 0) return false;
  std::vector<PointXYZRGB> pts((size_t)*w * *h);
  if (!pts.empty()) check(rgbdslam_b200_node_download_cloud(n->handle(), 32, pts.data(), w, h), "node_download_cloud");
  FILE* o = std::fopen(path.c_str(), "wb");
  if (!o) return false;
  std::fwrite(pts.data(), sizeof(PointXYZRGB), pts.size(), o);
  std::fclose(o);
  return true;
}

static void print_sensor(const GraphManager& gm, const char* name) {
  for (auto& kv : gm.graph_) {
    std::printf("SENSOR %s %d", name, kv.first);
    for (int k = 0; k < 7; k++) {
      uint32_t u;
      std::memcpy(&u, &kv.second->cloud_sensor_pose_[k], 4);
      std::printf(" %08x", u);
    }
    std::printf("\n");
  }
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
  int ok = 1;
  try {
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
    // node 1 loses its valid estimate: skipped by saveIndividualClouds, its locations by saveAllFeatures
    gm.graph_.at(1)->valid_tf_estimate_ = false;
    std::printf("INVALIDATED 1\n");
    for (auto it = gm.graph_.rbegin(); it != gm.graph_.rend(); ++it)
      if (it->second->valid_tf_estimate_) {
        it->second->clearPointCloud();
        std::printf("CLEARED %d\n", it->first);
        break;
      }
    for (auto& kv : gm.graph_) {
      const Node* n = kv.second;
      const bool est = gm.estimates_.count(n->vertex_id_) != 0;
      std::printf("NODE %d %d %d", n->id_, (int)n->valid_tf_estimate_, (int)est);
      if (est) {
        const Pose7& e = gm.estimates_.at(n->vertex_id_);
        double R[9], tf[12], map[12];
        quatToRot(e.v + 3, R);
        const double iso[12] = {R[0], R[1], R[2], e.v[0], R[3], R[4], R[5], e.v[1], R[6], R[7], R[8], e.v[2]};
        gm.eigenTransf2TF(n->vertex_id_, tf);
        gm.mapTransform(n->vertex_id_, map);
        for (const double* m : {iso, (const double*)tf, (const double*)map})
          for (int k = 0; k < 12; k++) std::printf(" %.17g", m[k]);
      }
      std::printf("\n");
      int w = 0, h = 0;
      if (dump_cloud(n, out + "/before_" + std::to_string(n->id_) + ".bin", &w, &h)) std::printf("CLOUD %d %d %d\n", n->id_, w, h);
      FILE* o = std::fopen((out + "/features_" + std::to_string(n->id_) + ".bin").c_str(), "wb");
      const int32_t nf = (int32_t)n->feature_locations_3d_.size();
      ok &= o && n->feature_descriptors_.size() == (size_t)nf * 32;
      if (!o) continue;
      std::fwrite(&nf, 4, 1, o);
      std::fwrite(n->feature_locations_3d_.data(), 16, nf, o);
      std::fwrite(n->feature_descriptors_.data(), 1, n->feature_descriptors_.size(), o);
      std::fclose(o);
    }
    std::printf("SAVED plain %zu\n", gm.saveIndividualClouds(out + "/plain"));
    print_sensor(gm, "plain");
    GraphManager::transform_individual_clouds() = true;
    for (const char* name : {"xf1", "xf2"}) {
      std::printf("SAVED %s %zu\n", name, gm.saveIndividualClouds(out + "/" + name));
      for (auto& kv : gm.graph_) {
        int w = 0, h = 0;
        dump_cloud(kv.second, out + "/" + name + "_" + std::to_string(kv.first) + ".bin", &w, &h);
      }
      print_sensor(gm, name);
    }
    GraphManager::transform_individual_clouds() = false;
    std::printf("SAVED features %zu\n", gm.saveAllFeatures(out + "/features.yml"));
    try {
      gm.saveAllFeatures(out + "/features.xml");
      ok = 0;
    } catch (const std::invalid_argument&) {
    }
    GraphManager empty;
    try {
      empty.saveAllFeatures(out + "/empty.yml");
      ok = 0;
    } catch (const std::runtime_error&) {
    }
    ok &= gm.graph_.size() >= (size_t)F / 2;
  } catch (const std::exception& e) {
    std::printf("ERROR %s\n", e.what());
    ok = 0;
  }
  rgbdslam_b200_shutdown();
  std::printf(ok ? "EXPORT SHIM OK\n" : "EXPORT SHIM FAILED\n");
  return ok ? 0 : 1;
}
