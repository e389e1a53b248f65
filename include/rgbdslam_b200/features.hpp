// features.hpp -- header-only shim of the reference's detector / extractor factory surface over the C ABI (SURVEY.md 8b):
//   cv::Feature2D* createDetector(const std::string& detectorType)                         src/features.h:9-10, features.cpp:63-113
//   cv::Ptr<cv::DescriptorExtractor> createDescriptorExtractor(std::string descriptorType)  src/features.h:11-14, features.cpp:115-161
//   detector->detect(gray, keypoints, mask)  /  extractor->compute(gray, keypoints, descriptors)   node.cpp:160,202
// held by OpenNIListener as `cv::Ptr<cv::Feature2D> detector_; cv::Ptr<cv::DescriptorExtractor> extractor_;`
// (openni_listener.h:195-196, created openni_listener.cpp:130-132) and handed to every Node constructor, so the detector's
// adaptive per-cell thresholds live across frames.
//
// OpenCV is not a dependency of this header: `Mat` is the (data, rows, cols, step, type) view of a cv::Mat header -- a
// maintainer with OpenCV passes `Mat(m.data, m.rows, m.cols, m.step, m.type())` or adds the one-line converting constructor
// shown in INTEGRATION.md.  Two detectors are built -- the two a stock OpenCV build gives the reference: ORB (its default
// and its fallback for every non-free type, features.cpp:79-88,139-149) and FAST (DetectorAdjuster("FAST", 20),
// feature_adjuster.cpp:88-91) -- both under the same dynamic + grid wrappers; the extractor is always ORB.  The library's
// parameter feature_detector_type (rgbdslam_b200_params, parameter_server.cpp:80) decides which detector
// createDetector makes, as the ParameterServer value does in openni_listener.cpp:130; asking for a type that disagrees
// with it, or for SURF / SIFT, throws instead of silently substituting another detector.
#pragma once
#include <cstdint>
#include <memory>
#include <stdexcept>
#include <string>
#include <vector>

#include "../rgbdslam_b200.h"

namespace rgbdslam_b200 {

typedef rgbdslam_b200_keypoint KeyPoint;  // == cv::KeyPoint (7 x 4 B)

enum { RB_8UC1 = 0, RB_16UC1 = 2, RB_32FC1 = 5, RB_8UC3 = 16 };  // == CV_8UC1, CV_16UC1, CV_32FC1, CV_8UC3

inline int channels_of(int t) { return t == RB_8UC3 ? 3 : 1; }
inline size_t pixel_bytes(int t) { return t == RB_32FC1 ? 4 : t == RB_16UC1 ? 2 : (size_t)channels_of(t); }

struct Mat {  // non-owning view with cv::Mat's field names
  unsigned char* data = nullptr;
  int rows = 0, cols = 0;
  size_t step = 0;  // bytes per row
  int type_ = RB_8UC1;
  Mat() {}
  Mat(void* d, int r, int c, size_t s, int t) : data((unsigned char*)d), rows(r), cols(c), step(s), type_(t) {}
  Mat(int r, int c, int t, void* d) : data((unsigned char*)d), rows(r), cols(c), step((size_t)c * pixel_bytes(t)), type_(t) {}
  int type() const { return type_; }
  int channels() const { return channels_of(type_); }
  bool empty() const { return data == nullptr || rows == 0 || cols == 0; }
  bool isContinuous() const { return step == (size_t)cols * pixel_bytes(type_); }
};

namespace detail {
inline void check_rc(int rc, const char* what) {
  if (rc != 0) throw std::runtime_error(std::string(what) + ": " + rgbdslam_b200_last_error());
}
// contiguous copy of a strided image (the C ABI takes w * h packed pixels)
template <class T>
inline const T* packed(const Mat& m, std::vector<T>& tmp) {
  if (m.isContinuous()) return reinterpret_cast<const T*>(m.data);
  const size_t row = (size_t)m.cols * m.channels();
  tmp.resize((size_t)m.rows * row);
  for (int r = 0; r < m.rows; r++)
    std::copy(reinterpret_cast<const T*>(m.data + r * m.step), reinterpret_cast<const T*>(m.data + r * m.step) + row,
              tmp.begin() + (size_t)r * row);
  return tmp.data();
}
}  // namespace detail

// cv::Feature2D as far as the reference uses it (node.cpp:160,202).  One class serves as detector and as extractor, like
// cv::ORB does; the detector owns the persistent threshold state and its type (rgbdslam_b200_detector_create).
class Feature2D {
 public:
  explicit Feature2D(bool is_detector) : handle_(0) {
    if (is_detector) detail::check_rc(rgbdslam_b200_detector_create(&handle_), "detector_create");
  }
  virtual ~Feature2D() {
    if (handle_) rgbdslam_b200_detector_destroy(handle_);
  }
  Feature2D(const Feature2D&) = delete;
  Feature2D& operator=(const Feature2D&) = delete;

  // detector->detect(gray_img, feature_locations_2d_, detection_mask)  (node.cpp:160)
  void detect(const Mat& image, std::vector<KeyPoint>& keypoints, const Mat& mask = Mat()) {
    if (!handle_) throw std::runtime_error("detect() on an object created by createDescriptorExtractor");
    if (image.type() != RB_8UC1 || (!mask.empty() && (mask.type() != RB_8UC1 || mask.rows != image.rows || mask.cols != image.cols)))
      throw std::invalid_argument("detect: image and mask must be CV_8UC1 of the same size");
    std::vector<uint8_t> ti, tm;
    const uint8_t* g = detail::packed<uint8_t>(image, ti);
    const uint8_t* m = mask.empty() ? nullptr : detail::packed<uint8_t>(mask, tm);
    keypoints.resize(4096);
    int n = 0;
    detail::check_rc(rgbdslam_b200_orb_detect(handle_, g, m, image.cols, image.rows, keypoints.data(), (int)keypoints.size(), &n),
                     "orb_detect");
    keypoints.resize((size_t)(n < 4096 ? n : 4096));
  }

  // extractor->compute(gray_img, feature_locations_2d_, feature_descriptors_)  (node.cpp:202): keypoints too close to the
  // border are removed and the rest re-ordered by octave, as cv::ORB does; descriptors: keypoints.size() x 32 bytes
  void compute(const Mat& image, std::vector<KeyPoint>& keypoints, std::vector<uint8_t>& descriptors) {
    if (image.type() != RB_8UC1) throw std::invalid_argument("compute: image must be CV_8UC1");
    std::vector<uint8_t> ti;
    const uint8_t* g = detail::packed<uint8_t>(image, ti);
    std::vector<KeyPoint> out(keypoints.size() ? keypoints.size() : 1);
    descriptors.assign((keypoints.size() ? keypoints.size() : 1) * 32, 0);
    int n = 0;
    detail::check_rc(rgbdslam_b200_orb_compute(g, image.cols, image.rows, keypoints.data(), (int)keypoints.size(), out.data(),
                                               descriptors.data(), &n),
                     "orb_compute");
    out.resize((size_t)n);
    descriptors.resize((size_t)n * 32);
    keypoints.swap(out);
  }

  uint64_t handle() const { return handle_; }  // rgbdslam_b200 detector handle (0 for a pure extractor)

 private:
  uint64_t handle_;
};
typedef Feature2D DescriptorExtractor;  // cv::DescriptorExtractor is a typedef of cv::Feature2D since OpenCV 3
template <class T>
using Ptr = std::shared_ptr<T>;  // cv::Ptr

// features.cpp:63-113.  The grid / dynamic wrappers are part of the detector here (detector_grid_resolution,
// adjuster_max_iterations and max_keypoints are read from the library's parameters like the reference reads its
// ParameterServer): the grid adjuster, the whole-frame adjuster (detector_grid_resolution <= 1) or, with
// adjuster_max_iterations <= 0, the bare DetectorAdjuster on the whole frame at a fixed threshold, as the reference
// chooses.  "ORB" and "FAST" need the library's feature_detector_type to name the same detector.  "SIFTGPU"
// returns NULL like the reference (:69-71).
inline Feature2D* createDetector(const std::string& detectorType) {
  if (detectorType == "SIFTGPU") return nullptr;
  if (detectorType != "ORB" && detectorType != "FAST")
    throw std::invalid_argument("createDetector(\"" + detectorType +
                                "\"): only ORB and FAST are built (SURF / SIFT adjusters: features.cpp:72-83 are not)");
  rgbdslam_b200_params p;  // before rgbdslam_b200_init the library makes ORB detectors (rgbdslam_b200_detector_create)
  const bool fast = rgbdslam_b200_get_params(&p) == 0 && p.feature_detector_type == RGBDSLAM_B200_DETECTOR_FAST;
  const char* configured = fast ? "FAST" : "ORB";
  if (detectorType != configured)
    throw std::invalid_argument("createDetector(\"" + detectorType + "\"): the library's parameter feature_detector_type is " +
                                configured + " (set rgbdslam_b200_params.feature_detector_type before rgbdslam_b200_init)");
  return new Feature2D(true);
}

// features.cpp:115-161
inline Ptr<DescriptorExtractor> createDescriptorExtractor(const std::string& descriptorType) {
  if (descriptorType != "ORB" && descriptorType != "SIFTGPU")  // SIFTGPU -> ORB fallback, features.cpp:153-156
    throw std::invalid_argument("createDescriptorExtractor(\"" + descriptorType + "\"): only ORB is built");
  return Ptr<DescriptorExtractor>(new Feature2D(false));
}

// sensor_msgs::CameraInfo as far as the Node constructor reads it (node.cpp:913-916: K[0], K[4], K[2], K[5]) and the
// depth header (myHeader: seq, stamp, frame_id -- src/header.h)
struct CameraInfo {
  double K[9] = {525.0, 0, 319.5, 0, 525.0, 239.5, 0, 0, 1};
};
typedef std::shared_ptr<const CameraInfo> CameraInfoConstPtr;
struct myHeader {
  uint32_t seq = 0;
  double stamp = 0.0;  // ros::Time as seconds
  std::string frame_id;
};

}  // namespace rgbdslam_b200
