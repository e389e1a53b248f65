// The reference's FAST call sites against the shim: createDetector("FAST") with feature_detector_type FAST (openni_listener.cpp:130),
// the reference-shaped Node constructor, detect() / compute() (CPU: compile + link; GPU: run).
#include <cstdio>
#include <stdexcept>
#include <vector>

#include "rgbdslam_b200/node.hpp"

using namespace rgbdslam_b200;

static uint64_t s = 88172645463325252ull;
static uint32_t rnd() { s ^= s << 13; s ^= s >> 7; s ^= s << 17; return (uint32_t)(s >> 32); }

int main() {
  rgbdslam_b200_params p;
  rgbdslam_b200_default_params(&p);
  p.depth_cov_z0 = 2.0;
  p.feature_detector_type = RGBDSLAM_B200_DETECTOR_FAST;
  if (rgbdslam_b200_init(0, &p) != 0) {
    std::printf("init failed (expected without a GPU): %s\n", rgbdslam_b200_last_error());
    return 77;
  }
  int ok = 1;
  {
    Ptr<Feature2D> detector_(createDetector("FAST"));
    Ptr<DescriptorExtractor> extractor_ = createDescriptorExtractor("ORB");
    const int W = 640, H = 480;
    std::vector<uint8_t> img((size_t)W * H), msk((size_t)W * H, 255);
    std::vector<float> dep((size_t)W * H, 2.0f);
    for (int y = 0; y < H; y++)
      for (int x = 0; x < W; x++) img[(size_t)y * W + x] = (uint8_t)(((x / 9 + y / 7) % 2) * 140 + (rnd() % 60));
    Mat visual(H, W, RB_8UC1, img.data()), depth(H, W, RB_32FC1, dep.data()), detection_mask(H, W, RB_8UC1, msk.data());
    CameraInfoConstPtr cam_info(new CameraInfo());
    myHeader depth_header;
    depth_header.stamp = 3.25;
    Node* n = new Node(visual, depth, detection_mask, cam_info, depth_header, detector_, extractor_);
    const size_t nf = n->feature_locations_2d_.size();
    std::printf("Node(visual, depth, mask, cam_info, header, FAST detector, extractor): %zu features\n", nf);
    ok = ok && nf > 100 && nf <= 600 && nf == n->feature_locations_3d_.size() && n->feature_descriptors_.size() == 32 * nf &&
         n->stamp_ == 3.25;
    for (const KeyPoint& k : n->feature_locations_2d_)
      ok = ok && k.size == 7.f && k.angle == -1.f && k.octave == 0 && k.response >= 2.f && k.x == (float)(int)k.x;
    std::vector<KeyPoint> kps;
    detector_->detect(visual, kps, detection_mask);
    std::vector<uint8_t> desc;
    const size_t n_det = kps.size();
    extractor_->compute(visual, kps, desc);
    std::printf("detect: %zu keypoints, compute kept %zu\n", n_det, kps.size());
    ok = ok && n_det > 100 && kps.size() <= n_det && desc.size() == 32 * kps.size();
    for (const KeyPoint& k : kps) ok = ok && k.angle == -1.f;
    delete n;
    bool threw = false;  // the name must agree with the parameter
    try { createDetector("ORB"); } catch (const std::invalid_argument& e) { threw = std::string(e.what()).find("feature_detector_type") != std::string::npos; }
    ok = ok && threw;
    threw = false;
    try { createDetector("SURF"); } catch (const std::invalid_argument&) { threw = true; }
    ok = ok && threw;
  }
  p.feature_detector_type = RGBDSLAM_B200_DETECTOR_ORB;
  ok = ok && rgbdslam_b200_init(0, &p) == 0;
  bool threw = false;
  try { createDetector("FAST"); } catch (const std::invalid_argument&) { threw = true; }
  Feature2D* orb = createDetector("ORB");
  ok = ok && threw && orb != nullptr;
  delete orb;
  rgbdslam_b200_shutdown();
  std::printf(ok ? "FAST SHIM OK\n" : "FAST SHIM FAILED\n");
  return ok ? 0 : 1;
}
