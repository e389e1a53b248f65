// The listener's depth-image handling against the shim: listenerNode(visual, depth of another size, ...) equals the Node
// constructor on the depth the listener hands over -- cv::resize(depth, visual.size(), INTER_NEAREST) (openni_listener.cpp:
// 651-656), restated here with cv2's double index rule -- and depthToCV8UC1's mono8 mask of it (:659).  Two pairs: a 1280 x 1024
// colour visual with a 640 x 480 CV_16UC1 depth, and a 640 x 480 grey visual with a 320 x 240 CV_32FC1 depth stored with a row
// stride (CPU: compile + link; GPU: run).
#include <algorithm>
#include <cmath>
#include <cstdio>
#include <cstring>
#include <memory>
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

// cv2 4.13's resizeNN source index of destination index x for n destination and dn source pixels
static int nn_index(int x, int n, int dn) { return std::min((int)std::floor(x * (1.0 / ((double)n / dn))), dn - 1); }

template <class T>
static std::vector<T> host_resize(const T* src, size_t step_px, int dw, int dh, int w, int h) {
  std::vector<T> out((size_t)w * h);
  for (int y = 0; y < h; y++)
    for (int x = 0; x < w; x++) out[(size_t)y * w + x] = src[(size_t)nn_index(y, h, dh) * step_px + nn_index(x, w, dw)];
  return out;
}

// one visual / depth pair: listenerNode against Node(visual, resized depth, mono8 mask) with a fresh detector each
static bool run_pair(int W, int H, bool colour, int DW, int DH, bool u16) {
  const int S = DW + 5;  // the depth is stored with a row stride of S pixels
  std::vector<uint8_t> gray((size_t)W * H), rgb((size_t)W * H * 3);
  for (int y = 0; y < H; y++)
    for (int x = 0; x < W; x++) {
      const size_t i = (size_t)y * W + x;
      const uint8_t v = (uint8_t)(((x / 9 + y / 7) % 2) * 140 + (rnd() % 60));
      gray[i] = v;
      rgb[3 * i] = v;
      rgb[3 * i + 1] = (uint8_t)(255 - v);
      rgb[3 * i + 2] = (uint8_t)(v / 2);
    }
  std::vector<uint16_t> raw((size_t)S * DH, 0);
  std::vector<float> metres((size_t)S * DH, 0.f);
  for (int y = 0; y < DH; y++)
    for (int x = 0; x < DW; x++) {
      uint16_t d = (uint16_t)(1500 + 3 * x + 2 * y);
      if ((x / 20 + y / 20) % 7 == 0) d = 0;                          // holes
      if (x > DW * 2 / 3 && y > DH * 2 / 3) d = (uint16_t)(300 + x % 400);  // a near patch across the 510 mm edge
      raw[(size_t)y * S + x] = d;
      metres[(size_t)y * S + x] = d ? (float)d * 0.001f : NAN;
    }
  // what the listener hands to the Node: the resized depth and depthToCV8UC1 of it (misc.cpp:414-425)
  std::vector<uint16_t> raw_r = host_resize(raw.data(), S, DW, DH, W, H);
  std::vector<float> metres_r = host_resize(metres.data(), S, DW, DH, W, H);
  std::vector<uint8_t> mono8((size_t)W * H);
  for (size_t i = 0; i < mono8.size(); i++) {
    if (u16) {
      mono8[i] = (uint8_t)std::min(std::max((int)std::lrintf(std::fmaf((float)raw_r[i], 0.05f, -25.f)), 0), 255);
    } else {
      const float v = metres_r[i] * 100.f;
      mono8[i] = (v == v && v < 2147483648.f && std::lrintf(v) >= 1) ? (uint8_t)std::min(std::lrintf(v), 255L) : 0;
    }
  }
  CameraInfo* c = new CameraInfo();
  c->K[0] = 525.0 * W / 640;
  c->K[4] = 525.0 * H / 480;
  c->K[2] = W / 2.0 - 0.5;
  c->K[5] = H / 2.0 - 0.5;
  CameraInfoConstPtr cam_info(c);
  Mat visual = colour ? Mat(H, W, RB_8UC3, rgb.data()) : Mat(H, W, RB_8UC1, gray.data());
  Mat depth = u16 ? Mat(raw.data(), DH, DW, (size_t)S * 2, RB_16UC1) : Mat(metres.data(), DH, DW, (size_t)S * 4, RB_32FC1);
  Mat depth_r = u16 ? Mat(H, W, RB_16UC1, raw_r.data()) : Mat(H, W, RB_32FC1, metres_r.data());
  Ptr<Feature2D> da(createDetector("ORB")), db(createDetector("ORB"));
  Ptr<DescriptorExtractor> ex = createDescriptorExtractor("ORB");
  myHeader hdr;
  hdr.seq = 17;
  hdr.stamp = 2.5;
  std::unique_ptr<Node> a(listenerNode(visual, depth, cam_info, hdr, da, ex));
  Node b(visual, depth_r, Mat(H, W, RB_8UC1, mono8.data()), cam_info, hdr, db, ex);
  const bool eq = same(*a, b) && a->seq_id_ == 17 && a->stamp_ == 2.5;
  std::printf("visual %dx%d %s, depth %dx%d %s: %zu features, %s\n", W, H, colour ? "CV_8UC3" : "CV_8UC1", DW, DH,
              u16 ? "CV_16UC1" : "CV_32FC1", a->feature_locations_2d_.size(), eq ? "equal" : "DIFFERENT");
  return eq;
}

int main() {
  rgbdslam_b200_params p;
  rgbdslam_b200_default_params(&p);
  p.depth_cov_z0 = 2.0;
  if (rgbdslam_b200_init(0, &p) != 0) {
    std::printf("init failed (expected without a GPU): %s\n", rgbdslam_b200_last_error());
    return 77;
  }
  int ok = run_pair(1280, 1024, true, 640, 480, true);
  ok = run_pair(640, 480, false, 320, 240, false) && ok;
  rgbdslam_b200_shutdown();
  std::printf(ok ? "RESIZE SHIM OK\n" : "RESIZE SHIM FAILED\n");
  return ok ? 0 : 1;
}
