// The reference's point-cloud call site against the shim: new Node(visual_img, detector_, extractor_, point_cloud,
// depth_mono8_img) (openni_listener.cpp:754) with a colour image and a PointXYZRGB cloud, then the same with PointXYZ, and the
// arguments the constructor refuses (CPU: compile + link; GPU: run).
#include <cmath>
#include <cstdio>
#include <stdexcept>
#include <vector>

#include "rgbdslam_b200/node.hpp"

using namespace rgbdslam_b200;

static uint64_t s = 88172645463325252ull;
static uint32_t rnd() { s ^= s << 13; s ^= s >> 7; s ^= s << 17; return (uint32_t)(s >> 32); }

template <class PointT>
static typename PointCloud<PointT>::Ptr make_cloud(int W, int H) {
  typename PointCloud<PointT>::Ptr c(new PointCloud<PointT>());
  c->width = W;
  c->height = H;
  c->points.resize((size_t)W * H);
  c->header.stamp = 7.5;
  for (int y = 0; y < H; y++)
    for (int x = 0; x < W; x++) {
      PointT& p = c->points[(size_t)y * W + x];
      const float z = 2.f + 0.001f * x;
      p.x = (x - 319.5f) * z / 525.f;
      p.y = (y - 239.5f) * z / 525.f;
      p.z = (x / 40 + y / 40) % 7 == 0 ? NAN : z;  // holes
      p.data_w = 1.f;
    }
  return c;
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
    Ptr<Feature2D> detector_(createDetector("ORB"));
    Ptr<DescriptorExtractor> extractor_ = createDescriptorExtractor("ORB");
    const int W = 640, H = 480;
    std::vector<uint8_t> img((size_t)W * H * 3), msk((size_t)W * H, 255);
    for (int y = 0; y < H; y++)
      for (int x = 0; x < W; x++) {
        const uint8_t v = (uint8_t)(((x / 9 + y / 7) % 2) * 140 + (rnd() % 60));
        uint8_t* px = &img[((size_t)y * W + x) * 3];
        px[0] = v;
        px[1] = (uint8_t)(255 - v);
        px[2] = (uint8_t)(v / 2);
      }
    Mat visual_img(H, W, RB_8UC3, img.data()), depth_mono8_img(H, W, RB_8UC1, msk.data());
    pointcloud_type::Ptr point_cloud = make_cloud<PointXYZRGB>(W, H);
    Node* n = new Node(visual_img, detector_, extractor_, point_cloud, depth_mono8_img);
    const size_t nf = n->feature_locations_2d_.size();
    std::printf("Node(visual CV_8UC3, detector, extractor, PointXYZRGB cloud, mask): %zu features\n", nf);
    ok = ok && nf > 100 && nf <= 600 && nf == n->feature_locations_3d_.size() && n->feature_descriptors_.size() == 32 * nf &&
         n->stamp_ == 7.5 && n->id_ == -1;
    for (size_t i = 0; i < nf; i++) {  // each point is the cloud's, at the keypoint's truncated position
      const KeyPoint& k = n->feature_locations_2d_[i];
      const PointXYZRGB& q = point_cloud->points[(size_t)(int)k.y * W + (int)k.x];
      const Vector4f& v = n->feature_locations_3d_[i];
      ok = ok && v.x == q.x && v.y == q.y && v.z == q.z && v.w == 1.f;
    }
    delete n;
    PointCloud<PointXYZ>::Ptr xyz = make_cloud<PointXYZ>(W, H);
    Node n2(visual_img, detector_, extractor_, xyz);
    std::printf("Node(visual CV_8UC3, detector, extractor, PointXYZ cloud): %zu features\n", n2.feature_locations_2d_.size());
    ok = ok && n2.feature_locations_2d_.size() > 100 && n2.feature_locations_3d_.size() == n2.feature_locations_2d_.size();
    // refused: an unorganised cloud, a cloud of another size, a mask of another size
    int refused = 0;
    PointCloud<PointXYZ>::Ptr flat(new PointCloud<PointXYZ>());
    flat->width = W * H;
    flat->height = 1;
    flat->points = xyz->points;
    try { Node bad(visual_img, detector_, extractor_, flat); } catch (const std::invalid_argument&) { refused++; }
    PointCloud<PointXYZ>::Ptr small = make_cloud<PointXYZ>(W / 2, H / 2);
    try { Node bad(visual_img, detector_, extractor_, small); } catch (const std::invalid_argument&) { refused++; }
    Mat small_mask(H / 2, W / 2, RB_8UC1, msk.data());
    try { Node bad(visual_img, detector_, extractor_, xyz, small_mask); } catch (const std::invalid_argument&) { refused++; }
    ok = ok && refused == 3;
    // the depth-image constructor takes a colour image too
    std::vector<float> dep((size_t)W * H, 2.0f);
    Mat depth(H, W, RB_32FC1, dep.data());
    CameraInfoConstPtr cam_info(new CameraInfo());
    Node n3(visual_img, depth, depth_mono8_img, cam_info, myHeader(), detector_, extractor_);
    ok = ok && n3.feature_locations_2d_.size() > 100;
  }
  rgbdslam_b200_shutdown();
  std::printf(ok ? "CLOUD SHIM OK\n" : "CLOUD SHIM FAILED\n");
  return ok ? 0 : 1;
}
