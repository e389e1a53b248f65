// The reference's depth-image call site with the listener's raw 16UC1 depth (openni_listener.cpp:633-659) against the shim:
// Node(visual, CV_16UC1 depth, mask, ...) equals Node(visual, CV_32FC1 depth, mask, ...) built on the listener's conversions
// -- depth.convertTo(CV_32FC1, 0.001) and, when no mask is given, depthToCV8UC1's convertTo(CV_8UC1, 0.05, -25) -- with a
// grey and a colour visual and a strided 16-bit Mat (CPU: compile + link; GPU: run).
#include <algorithm>
#include <cmath>
#include <cstdio>
#include <cstring>
#include <stdexcept>
#include <vector>

#include "rgbdslam_b200/node.hpp"

using namespace rgbdslam_b200;

static uint64_t s = 88172645463325252ull;
static uint32_t rnd() { s ^= s << 13; s ^= s >> 7; s ^= s << 17; return (uint32_t)(s >> 32); }

static bool same(const Node& a, const Node& b) {
  const size_t n = a.feature_locations_2d_.size();
  return n > 100 && n == b.feature_locations_2d_.size() &&
         std::memcmp(a.feature_locations_2d_.data(), b.feature_locations_2d_.data(), n * sizeof(KeyPoint)) == 0 &&
         std::memcmp(a.feature_locations_3d_.data(), b.feature_locations_3d_.data(), n * sizeof(Vector4f)) == 0 &&
         a.feature_descriptors_ == b.feature_descriptors_;
}

int main() {
  rgbdslam_b200_params p;
  rgbdslam_b200_default_params(&p);
  p.depth_cov_z0 = 2.0;
  if (rgbdslam_b200_init(0, &p) != 0) {
    std::printf("init failed (expected without a GPU): %s\n", rgbdslam_b200_last_error());
    return 77;
  }
  int ok = 1;
  {
    const int W = 640, H = 480, S = W + 7;  // the 16-bit image is stored with a row stride of S pixels
    std::vector<uint8_t> gray((size_t)W * H), rgb((size_t)W * H * 3), given((size_t)W * H);
    std::vector<uint16_t> raw((size_t)S * H, 0);
    std::vector<float> metres((size_t)W * H);
    std::vector<uint8_t> mask((size_t)W * H);
    for (int y = 0; y < H; y++)
      for (int x = 0; x < W; x++) {
        const size_t i = (size_t)y * W + x;
        const uint8_t v = (uint8_t)(((x / 9 + y / 7) % 2) * 140 + (rnd() % 60));
        gray[i] = v;
        rgb[3 * i] = v;
        rgb[3 * i + 1] = (uint8_t)(255 - v);
        rgb[3 * i + 2] = (uint8_t)(v / 2);
        given[i] = (x / 80 + y / 60) % 3 ? 255 : 0;
        uint16_t d = (uint16_t)(1500 + 2 * x + y);
        if ((x / 40 + y / 40) % 7 == 0) d = 0;                   // holes
        if (x > 400 && y > 300) d = (uint16_t)(300 + x - 400);   // a near patch across the 510 mm edge
        raw[(size_t)y * S + x] = d;
        metres[i] = (float)d * 0.001f;
        mask[i] = (uint8_t)std::min(std::max((int)std::lrintf(std::fmaf((float)d, 0.05f, -25.f)), 0), 255);
      }
    CameraInfoConstPtr cam_info(new CameraInfo());
    Mat depth16(raw.data(), H, W, (size_t)S * 2, RB_16UC1), depth32(H, W, RB_32FC1, metres.data());
    Mat mono8(H, W, RB_8UC1, mask.data()), given8(H, W, RB_8UC1, given.data());
    int cases = 0;
    for (int colour = 0; colour < 2; colour++) {
      Mat visual = colour ? Mat(H, W, RB_8UC3, rgb.data()) : Mat(H, W, RB_8UC1, gray.data());
      for (int with_mask = 0; with_mask < 2; with_mask++) {
        Ptr<Feature2D> da(createDetector("ORB")), db(createDetector("ORB"));
        Ptr<DescriptorExtractor> ex = createDescriptorExtractor("ORB");
        Node a(visual, depth16, with_mask ? given8 : Mat(), cam_info, myHeader(), da, ex);
        Node b(visual, depth32, with_mask ? given8 : mono8, cam_info, myHeader(), db, ex);
        const bool eq = same(a, b);
        std::printf("colour %d, mask %s: %zu features, %s\n", colour, with_mask ? "given" : "from depth",
                    a.feature_locations_2d_.size(), eq ? "equal" : "DIFFERENT");
        ok = ok && eq;
        cases++;
      }
    }
    ok = ok && cases == 4;
    try {  // refused: a 16-bit depth of another size
      Ptr<Feature2D> d(createDetector("ORB"));
      Mat small(raw.data(), H / 2, W / 2, (size_t)S * 2, RB_16UC1);
      Node bad(Mat(H, W, RB_8UC1, gray.data()), small, Mat(), cam_info, myHeader(), d, createDescriptorExtractor("ORB"));
      ok = 0;
    } catch (const std::invalid_argument&) {
    }
  }
  rgbdslam_b200_shutdown();
  std::printf(ok ? "RAW SHIM OK\n" : "RAW SHIM FAILED\n");
  return ok ? 0 : 1;
}
