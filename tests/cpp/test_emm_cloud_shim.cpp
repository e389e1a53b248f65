// The reference's point-cloud call site against the shim with the environment measurement model on (observability_threshold
// > 0): new Node(visual_img, detector_, extractor_, point_cloud) keeps the cloud, and matchNodePair reports the model's
// counts.  Input (argv[1]): int32 W, H, F, float K[4] (depth_camera_fx, fy, cx, cy), F grey images (W x H bytes), F
// organised PointXYZRGB clouds (W x H x 8 floats).  Prints one line per pair, "PAIR newer older edge.id1 inlier outlier
// occluded all T[16]" (ransac_trafo, column-major), for the test to compare with its restatement.  (CPU: compile + link;
// GPU: run.)
#include <cstdio>
#include <memory>
#include <vector>

#include "rgbdslam_b200/node.hpp"

using namespace rgbdslam_b200;

int main(int argc, char** argv) {
  if (argc != 2) return 2;
  rgbdslam_b200_params p;
  rgbdslam_b200_default_params(&p);
  p.depth_cov_z0 = 2.0;
  p.observability_threshold = 0.3;
  if (rgbdslam_b200_init(0, &p) != 0) {
    std::printf("init failed (expected without a GPU): %s\n", rgbdslam_b200_last_error());
    return 77;
  }
  FILE* f = std::fopen(argv[1], "rb");
  int32_t dims[3];
  float K[4];
  if (!f || std::fread(dims, 4, 3, f) != 3 || std::fread(K, 4, 4, f) != 4) return 2;
  const int W = dims[0], H = dims[1], F = dims[2];
  std::vector<std::vector<uint8_t>> gray(F, std::vector<uint8_t>((size_t)W * H));
  for (auto& g : gray)
    if (std::fread(g.data(), 1, g.size(), f) != g.size()) return 2;
  std::vector<pointcloud_type::Ptr> clouds;
  for (int i = 0; i < F; i++) {
    pointcloud_type::Ptr c(new pointcloud_type());
    c->width = W;
    c->height = H;
    c->points.resize((size_t)W * H);
    if (std::fread(c->points.data(), sizeof(point_type), c->points.size(), f) != c->points.size()) return 2;
    clouds.push_back(c);
  }
  std::fclose(f);
  int judged = 0;
  {
    for (int k = 0; k < 4; k++) Node::depth_camera_intrinsics()[k] = K[k];
    Ptr<Feature2D> detector_(createDetector("ORB"));
    Ptr<DescriptorExtractor> extractor_ = createDescriptorExtractor("ORB");
    std::vector<std::unique_ptr<Node>> nodes;
    for (int i = 0; i < F; i++) {
      Mat visual_img(H, W, RB_8UC1, gray[i].data());
      nodes.emplace_back(new Node(visual_img, detector_, extractor_, clouds[i]));
      nodes.back()->id_ = i;  // GraphManager::addNode
    }
    for (int i = 1; i < F; i++)
      for (int j = 0; j < i; j++) {
        const MatchingResult mr = nodes[i]->matchNodePair(nodes[j].get(), 4, 0);
        std::printf("PAIR %d %d %d %u %u %u %u", i, j, mr.edge.id1, mr.inlier_points, mr.outlier_points, mr.occluded_points,
                    mr.all_points);
        for (int k = 0; k < 16; k++) std::printf(" %.9g", mr.ransac_trafo.m[k]);
        std::printf("\n");
        judged += mr.all_points > 0;  // the model runs on the pairs RANSAC accepts
      }
  }
  rgbdslam_b200_shutdown();
  const int ok = judged > 0;
  std::printf(ok ? "EMM CLOUD SHIM OK\n" : "EMM CLOUD SHIM FAILED\n");
  return ok ? 0 : 1;
}
