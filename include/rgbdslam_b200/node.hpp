// node.hpp -- header-only C++ shim that keeps the reference's call sites compiling against the C ABI.
//
// Mirrors, for the frame-pair hot path only:
//   LoadedEdge3D                 src/edge.h:24-32
//   MatchingResult               src/matching_result.h:24-46
//   Node (feature members, matchNodePair, featureMatching-free ctor from features)   src/node.h:64-178
//   the two image constructors (depth image node.cpp:101-240, point cloud :252-369) and pcl::PointCloud / PointXYZ[RGB]
//   listenerNode: the listener's depth-image handling and Node construction (openni_listener.cpp:633-659, 779)
//   bruteForceSearchORB          src/features.h:13, src/features.cpp:168-182
// The reference types Eigen::Matrix4f / Eigen::Isometry3d / cv::DMatch / cv::KeyPoint are replaced by
// layout-compatible PODs (column-major float[16] etc.) so this header has no third-party dependency; a
// maintainer who has Eigen/OpenCV maps them with Eigen::Map / reinterpret_cast (see INTEGRATION.md).
#pragma once
#include <cstdint>
#include <cstdio>
#include <cstring>
#include <memory>
#include <stdexcept>
#include <type_traits>
#include <string>
#include <vector>

#include "../rgbdslam_b200.h"
#include "cloud_transform.h"
#include "depth_resize.h"
#include "icp.h"
#include "map.h"
#include "octomap.h"
#include "voxel.h"
#include "features.hpp"

namespace rgbdslam_b200 {

struct Matrix4f {  // == Eigen::Matrix4f storage (column-major)
  float m[16];
  static Matrix4f Identity() {
    Matrix4f r;
    for (int i = 0; i < 16; i++) r.m[i] = (i % 5 == 0) ? 1.f : 0.f;
    return r;
  }
  float operator()(int row, int col) const { return m[4 * col + row]; }
};
struct Isometry3d {  // == Eigen::Isometry3d storage (4x4 column-major double)
  double m[16];
};
struct Matrix6d {
  double m[36];
};
struct Vector4f {
  float x, y, z, w;
};

// pcl::PointXYZ / pcl::PointXYZRGB as an organised cloud stores them (x, y, z at byte offsets 0, 4, 8; PointXYZRGB's colour
// packed b, g, r, a at offset 16) and pcl::PointCloud<PointT> as far as the point-cloud Node constructor reads it.  The
// reference's point_type is PointXYZRGB, or PointXYZ with RGB_IS_4TH_DIM (parameter_server.h:33-42).
struct alignas(16) PointXYZ {
  float x, y, z, data_w;
};
struct alignas(16) PointXYZRGB {
  float x, y, z, data_w;
  uint8_t b, g, r, a;
  float data_c[3];
};
static_assert(sizeof(PointXYZ) == 16 && sizeof(PointXYZRGB) == 32, "layout of pcl::PointXYZ / pcl::PointXYZRGB");
template <class PointT>
struct PointCloud {
  typedef std::shared_ptr<PointCloud<PointT>> Ptr;
  typedef std::shared_ptr<const PointCloud<PointT>> ConstPtr;
  myHeader header;
  std::vector<PointT> points;  // row-major, width x height
  uint32_t width = 0, height = 0;
  bool is_dense = false;
  bool isOrganized() const { return height > 1; }
};
typedef PointXYZRGB point_type;  // the reference's default point_type
typedef PointCloud<point_type> pointcloud_type;
typedef rgbdslam_b200_dmatch DMatch;  // == cv::DMatch  (KeyPoint: features.hpp)

struct LoadedEdge3D {  // src/edge.h:24-32
  int id1, id2;
  Isometry3d transform;
  Matrix6d informationMatrix;
};

class MatchingResult {  // src/matching_result.h:24-46
 public:
  MatchingResult()
      : rmse(0.0), ransac_trafo(Matrix4f::Identity()), final_trafo(Matrix4f::Identity()), icp_trafo(Matrix4f::Identity()),
        inlier_points(0), outlier_points(0), occluded_points(0), all_points(0) {
    edge.id1 = edge.id2 = -1;
    std::memset(&edge.transform, 0, sizeof(edge.transform));
    std::memset(&edge.informationMatrix, 0, sizeof(edge.informationMatrix));
  }
  std::vector<DMatch> inlier_matches;
  std::vector<DMatch> all_matches;
  LoadedEdge3D edge;
  float rmse;
  Matrix4f ransac_trafo, final_trafo, icp_trafo;
  unsigned int inlier_points, outlier_points, occluded_points, all_points;
};

inline void check(int rc, const char* what) {
  if (rc != 0) throw std::runtime_error(std::string(what) + ": " + rgbdslam_b200_last_error());
}

// Fill a MatchingResult from the flat ABI record (what node.cpp:1334-1339 does with the RANSAC output).
inline MatchingResult to_matching_result(const rgbdslam_b200_pair_result& r, const DMatch* all, const DMatch* inl) {
  MatchingResult mr;
  mr.all_matches.assign(all, all + r.n_all_matches);
  mr.inlier_matches.assign(inl, inl + r.n_inliers);
  mr.rmse = r.rmse;
  std::memcpy(mr.ransac_trafo.m, r.ransac_trafo, sizeof(r.ransac_trafo));
  mr.edge.id1 = r.id1;
  mr.edge.id2 = r.id2;
  mr.inlier_points = r.inlier_points;  // environment measurement model (node.cpp:1551-1554), 0 when it is off
  mr.outlier_points = r.outlier_points;
  mr.occluded_points = r.occluded_points;
  mr.all_points = r.all_points;
  if (r.id1 >= 0) {
    mr.final_trafo = mr.ransac_trafo;                                               // node.cpp:1334
    for (int i = 0; i < 16; i++) mr.edge.transform.m[i] = (double)r.ransac_trafo[i];  // node.cpp:1339
    for (int i = 0; i < 6; i++) mr.edge.informationMatrix.m[7 * i] = r.info_scale;    // node.cpp:1335
  }
  return mr;
}

class Node {  // src/node.h: the members the hot path reads + matchNodePair
 public:
  int id_ = -1, seq_id_ = -1, vertex_id_ = -1;
  double stamp_ = 0.0;           // header_.stamp in seconds
  bool matchable_ = true, valid_tf_estimate_ = true;  // node.h:160,178
  mutable int initial_node_matches_ = 0;              // node.h:207: accepted transformations of this node (max_connections)
  // pc_col->sensor_orientation_ (qx qy qz qw) and sensor_origin_ (ox oy oz): PCL's default until GraphManager::updateCloudOrigin
  // records the estimate (graph_mgr_io.cpp:232-233); occupancyFilterClouds applies it.  Mutable like the cloud header it is.
  mutable float cloud_sensor_pose_[7] = {0, 0, 0, 1, 0, 0, 0};
  std::vector<KeyPoint> feature_locations_2d_;  // node.h:167
  std::vector<Vector4f> feature_locations_3d_;  // node.h:174
  std::vector<uint8_t> feature_descriptors_;    // N x 32 (cv::Mat CV_8U rows), node.h:169

  Node() {}
  // The reference's constructor, argument for argument (node.h:64-70, call site openni_listener.cpp:779):
  //   Node(visual, depth, detection_mask, cam_info, depth_header, detector, extractor)
  // visual CV_8UC1 or CV_8UC3 (converted as cvtColor(CV_RGB2GRAY): channel 0 weighted as R), depth CV_32FC1 metres (NaN =
  // invalid), detection_mask CV_8UC1 non-zero at potential keypoint locations
  // (node.h:61-63).  depth may also be the listener's raw CV_16UC1 millimetres (0 = invalid), converted on the device as
  // noCloudCallback does (openni_listener.cpp:633-659; RGBDSLAM_B200_DEPTH_U16); there the listener always derives the mask
  // with depthToCV8UC1, so an empty detection_mask means that mask (MASK_FROM_DEPTH) and a given one is used as given.
  // detector / extractor: createDetector / createDescriptorExtractor (features.hpp); the whole constructor
  // -- detect, removeDepthless, retainBest, compute, projectTo3D -- runs as one rgbdslam_b200_nodes_create call, the
  // extractor argument only documents the pairing (ORB or FAST keypoints, ORB descriptors).  id_ stays -1 until
  // GraphManager::addNode assigns it.  Frames of up to 4095 px per side (the limits of rgbdslam_b200_nodes_create; above
  // 1023 px the detector grid must be >= 2 and round(1.5 * max_keypoints / cells) < 606).
  Node(const Mat& visual, const Mat& depth, const Mat& detection_mask, const CameraInfoConstPtr& cam_info, myHeader depth_header,
       Ptr<Feature2D> detector, Ptr<DescriptorExtractor> extractor)
      : stamp_(depth_header.stamp) {
    if (!detector || !detector->handle()) throw std::invalid_argument("Node: detector must come from createDetector(\"ORB\" or \"FAST\")");
    if (!extractor) throw std::invalid_argument("Node: null extractor");
    const bool u16 = depth.type() == RB_16UC1;
    if ((visual.type() != RB_8UC1 && visual.type() != RB_8UC3) || (depth.type() != RB_32FC1 && !u16) || depth.rows != visual.rows ||
        depth.cols != visual.cols)
      throw std::invalid_argument("Node: visual must be CV_8UC1 or CV_8UC3 and depth CV_32FC1 or CV_16UC1 of the same size");
    seq_id_ = (int)depth_header.seq;
    std::vector<uint8_t> tg, tm;
    std::vector<float> td;
    std::vector<uint16_t> tr;
    const uint8_t* g = detail::packed<uint8_t>(visual, tg);
    const float* d = u16 ? reinterpret_cast<const float*>(detail::packed<uint16_t>(depth, tr)) : detail::packed<float>(depth, td);
    const uint8_t* m = detection_mask.empty() ? nullptr : detail::packed<uint8_t>(detection_mask, tm);
    const CameraInfo ci = cam_info ? *cam_info : CameraInfo();
    const float K4[4] = {(float)ci.K[0], (float)ci.K[4], (float)ci.K[2], (float)ci.K[5]};  // node.cpp:913-916
    construct(g, d, m, visual.cols, visual.rows, K4, detector->handle(), image_flags(visual, u16, u16 && !m));
  }
  // The reference's point-cloud constructor, argument for argument (node.h:74-78, call site openni_listener.cpp:754):
  //   Node(visual, detector, extractor, point_cloud, detection_mask)
  // visual CV_8UC1 or CV_8UC3 (converted as cvtColor(CV_RGB2GRAY): channel 0 weighted as R), point_cloud an organised cloud of
  // the same size as visual, detection_mask empty or of the same size.  detect, projectTo3D (the first max_keypoints keypoints
  // whose cloud point at the truncated position has no NaN coordinate, the point as stored) and compute run as one
  // rgbdslam_b200_nodes_create_ex call; each 3-D point stays with its keypoint through compute() (see rgbdslam_b200.h).
  // With the environment measurement model on (observability_threshold > 0) the node keeps its cloud (pc_col, node.cpp:261;
  // RGBDSLAM_B200_KEEP_CLOUD), which the model projects into depth_camera_intrinsics(); matchNodePair then reports its counts.
  template <class PointT>
  Node(const Mat& visual, Ptr<Feature2D> detector, Ptr<DescriptorExtractor> extractor, std::shared_ptr<PointCloud<PointT>> point_cloud,
       const Mat& detection_mask = Mat()) {
    static_assert(std::is_same<PointT, PointXYZRGB>::value || std::is_same<PointT, PointXYZ>::value,
                  "Node: the point cloud must hold PointXYZRGB or PointXYZ");
    if (!detector || !detector->handle()) throw std::invalid_argument("Node: detector must come from createDetector(\"ORB\" or \"FAST\")");
    if (!extractor) throw std::invalid_argument("Node: null extractor");
    if (!point_cloud || !point_cloud->isOrganized() || point_cloud->points.size() != (size_t)point_cloud->width * point_cloud->height)
      throw std::invalid_argument("Node: the point cloud must be organised (height > 1, width x height points)");
    if (visual.type() != RB_8UC1 && visual.type() != RB_8UC3) throw std::invalid_argument("Node: visual must be CV_8UC1 or CV_8UC3");
    if ((int)point_cloud->width != visual.cols || (int)point_cloud->height != visual.rows ||
        (!detection_mask.empty() && (detection_mask.type() != RB_8UC1 || detection_mask.rows != visual.rows ||
                                     detection_mask.cols != visual.cols)))
      throw std::invalid_argument("Node: visual, point cloud and detection_mask (CV_8UC1) must have the same size");
    stamp_ = point_cloud->header.stamp;  // timestamp_(point_cloud->header.stamp)
    std::vector<uint8_t> tg, tm;
    const uint8_t* g = detail::packed<uint8_t>(visual, tg);
    const uint8_t* m = detection_mask.empty() ? nullptr : detail::packed<uint8_t>(detection_mask, tm);
    rgbdslam_b200_params prm;
    const bool emm = rgbdslam_b200_get_params(&prm) == 0 && prm.observability_threshold > 0.0;
    const int flags = (visual.type() == RB_8UC3 ? RGBDSLAM_B200_VISUAL_RGB : 0) |
                      (std::is_same<PointT, PointXYZRGB>::value ? RGBDSLAM_B200_CLOUD_XYZRGB : RGBDSLAM_B200_CLOUD_XYZ) |
                      (emm || pcl_icp() ? RGBDSLAM_B200_KEEP_CLOUD : 0) | (store_pointclouds() ? RGBDSLAM_B200_STORE_CLOUD : 0);
    construct(g, reinterpret_cast<const float*>(point_cloud->points.data()), m, visual.cols, visual.rows,
              emm ? depth_camera_intrinsics() : nullptr, detector->handle(), flags);
  }
  // Node(visual, depth, detection_mask, cam_info, depth_header, detector, extractor) (node.cpp:101-240): detect, filter,
  // describe, back-project on the device; the public feature members are filled from the result.  `detector` is the handle of
  // rgbdslam_b200_detector_create -- the counterpart of the detector_ / extractor_ pair OpenNIListener keeps
  // (openni_listener.cpp:130-132), whose adaptive per-cell thresholds live across frames.
  Node(const uint8_t* gray, const float* depth_m, const uint8_t* detection_mask, int w, int h, const float K4[4], int id,
       uint64_t detector, double stamp = 0.0)
      : id_(id), stamp_(stamp) {
    construct(gray, depth_m, detection_mask, w, h, K4, detector);
  }
  // Construct from already extracted features (what the reference ctor node.cpp:101-240 leaves behind).
  Node(int id, const std::vector<uint8_t>& desc, const std::vector<Vector4f>& xyz) : id_(id) {
    feature_descriptors_ = desc;
    feature_locations_3d_ = xyz;
    upload();
  }
  ~Node() {  // Node::~Node (node.cpp:371)
    if (handle_) rgbdslam_b200_node_destroy(handle_);
  }
  Node(const Node&) = delete;
  Node& operator=(const Node&) = delete;

  // the nodes_create flags of a depth-image Node: the visual's channels, the depth's type, the mask derived from the depth, and
  // the stored cloud of store_pointclouds() / pcl_icp()
  static int image_flags(const Mat& visual, bool depth_u16, bool mask_from_depth) {
    return (visual.type() == RB_8UC3 ? RGBDSLAM_B200_VISUAL_RGB : 0) | (depth_u16 ? RGBDSLAM_B200_DEPTH_U16 : 0) |
           (mask_from_depth ? RGBDSLAM_B200_MASK_FROM_DEPTH : 0) |
           (store_pointclouds() || pcl_icp() ? RGBDSLAM_B200_STORE_CLOUD | (encoding_bgr() ? 0 : RGBDSLAM_B200_ENCODING_RGB) : 0);
  }
  // flags: rgbdslam_b200_nodes_create_ex's (colour visual, point cloud in place of the depth image)
  void construct(const uint8_t* gray, const float* depth_m, const uint8_t* detection_mask, int w, int h, const float K4[4],
                 uint64_t detector, int flags = 0) {
    int32_t n = 0, id32 = id_ < 0 ? 0 : id_;
    check(rgbdslam_b200_nodes_create_ex(detector, 1, gray, depth_m, detection_mask, w, h, K4, &id32, flags, &handle_, &n),
          "nodes_create");
    download_features(n);
  }
  // the same for a depth image of depth_w x depth_h pixels, resized to w x h on the device (rgbdslam_b200_nodes_create_resized)
  void construct_resized(const uint8_t* gray, const void* depth, int depth_w, int depth_h, const uint8_t* detection_mask, int w,
                         int h, const float K4[4], uint64_t detector, int flags) {
    int32_t n = 0, id32 = id_ < 0 ? 0 : id_;
    check(rgbdslam_b200_nodes_create_resized(detector, 1, gray, depth, depth_w, depth_h, detection_mask, w, h, K4, &id32, flags,
                                             &handle_, &n),
          "nodes_create_resized");
    download_features(n);
  }
  // the public feature members from the node's n features on the device
  void download_features(int n) {
    feature_locations_2d_.resize(n);
    feature_locations_3d_.resize(n);
    feature_descriptors_.resize((size_t)n * 32);
    if (n > 0) {
      check(rgbdslam_b200_node_download_keypoints(handle_, feature_locations_2d_.data()), "node_download_keypoints");
      check(rgbdslam_b200_node_download(handle_, feature_descriptors_.data(), reinterpret_cast<float*>(feature_locations_3d_.data())),
            "node_download");
    }
  }

  void upload() {
    if (handle_) rgbdslam_b200_node_destroy(handle_);
    handle_ = 0;
    // the device copy only needs a non-negative id (negative ids in a result mean "no transformation"); the ids of the
    // MatchingResult come from the host objects, which addNode may renumber (graph_manager.cpp:434)
    check(rgbdslam_b200_node_create_from_features(id_ < 0 ? 0 : id_, feature_descriptors_.data(),
                                                  reinterpret_cast<const float*>(feature_locations_3d_.data()),
                                                  (int)feature_locations_3d_.size(), &handle_),
          "node_create_from_features");
  }
  uint64_t handle() const { return handle_; }

  // MatchingResult Node::matchNodePair(const Node* older_node)  (node.cpp:1305).  Never throws on a failed
  // match: failure is edge.id1 == edge.id2 == -1 (node.cpp:1420), as in the reference.
  MatchingResult matchNodePair(const Node* older_node, uint64_t seed = 0, int64_t pair_index = 0) const {
    std::vector<MatchingResult> v = matchNodePairs(this, std::vector<const Node*>(1, older_node), seed, pair_index);
    return v[0];
  }

  // The QtConcurrent::blockingMapped(nodes_to_comp, bind(&Node::matchNodePair, new_node, _1)) fan-out of
  // graph_manager.cpp:548 as ONE batched launch.
  static std::vector<MatchingResult> matchNodePairs(const Node* newer, const std::vector<const Node*>& older,
                                                    uint64_t seed = 0, int64_t first_pair_index = 0) {
    const int n = (int)older.size();
    std::vector<MatchingResult> out(n);
    if (n == 0) return out;
    // the match arrays of the C ABI hold params.max_matches entries per pair: ask the library, never assume the default
    rgbdslam_b200_params prm;
    if (rgbdslam_b200_get_params(&prm) != 0) return out;  // not initialised: invalid edges, matchNodePair never throws
    const int mm = prm.max_matches;
    std::vector<uint64_t> a(n, newer->handle_), b(n);
    for (int i = 0; i < n; i++) b[i] = older[i]->handle_;
    std::vector<rgbdslam_b200_pair_result> res(n);
    std::vector<DMatch> all((size_t)n * mm), inl((size_t)n * mm);
    int rc = rgbdslam_b200_match_pairs(a.data(), b.data(), n, seed, first_pair_index, res.data(), all.data(), inl.data());
    if (rc != 0) return out;  // invalid edges (-1,-1): matchNodePair never throws (node.cpp:1308,1424)
    // With pcl_icp() a pair that had min_matches feature matches but no RANSAC transformation (info_scale stays 0 then; a pair
    // the measurement model rejected has one) between adjacent nodes takes the ICP edge (node.cpp:1356-1377).  ICP always
    // accepts, so the pairs that reach it before max_connections binds are known before it runs: one icp_align call serves
    // them all.  Should that call fail, those pairs keep no edge, as without the fallback.
    std::vector<char> icp(n, 0);
    std::vector<rgbdslam_b200_icp_result> icp_res(n);
    if (pcl_icp()) {
      std::vector<uint64_t> src, tgt;
      std::vector<int> at;
      int accepted = newer->initial_node_matches_;
      for (int i = 0; i < n; i++) {
        if (max_connections() > 0 && accepted > max_connections()) break;
        if (res[i].id1 >= 0) {
          ++accepted;
        } else if (res[i].n_all_matches >= prm.min_matches && res[i].info_scale == 0.0 && newer->id_ - older[i]->id_ <= 1) {
          ++accepted;
          at.push_back(i);
          src.push_back(older[i]->handle_);  // the older cloud is the source, the newer one the target (node.cpp:1364)
          tgt.push_back(newer->handle_);
        }
      }
      std::vector<rgbdslam_b200_icp_result> r(at.size());
      // icp_method (icp.cpp:50-58): "icp_nl" is IterativeClosestPointNonLinear; any other name, "gicp" included, is "icp"
      const int method = icp_method() == "icp_nl" ? RGBDSLAM_B200_ICP_METHOD_ICP_NL : RGBDSLAM_B200_ICP_METHOD_ICP;
      if (!at.empty() &&
          rgbdslam_b200_icp_align_ex((int)at.size(), src.data(), tgt.data(), gicp_max_cloud_size(), method, r.data()) == 0)
        for (size_t k = 0; k < at.size(); k++) {
          icp[at[k]] = 1;
          icp_res[at[k]] = r[k];
        }
    }
    for (int i = 0; i < n; i++) {
      // "enough is enough" (node.cpp:1310-1312), in the order the reference's sequential loop would meet the candidates:
      // once the node has more than max_connections accepted transformations the remaining comparisons return empty
      if (max_connections() > 0 && newer->initial_node_matches_ > max_connections()) continue;
      out[i] = to_matching_result(res[i], &all[(size_t)i * mm], &inl[(size_t)i * mm]);
      if (icp[i]) {  // node.cpp:1358-1375; edge.informationMatrix is left as it is, zero here (uninitialised in the reference)
        std::memcpy(out[i].icp_trafo.m, icp_res[i].T, sizeof(icp_res[i].T));
        out[i].final_trafo = out[i].icp_trafo;
        for (int k = 0; k < 16; k++) out[i].edge.transform.m[k] = (double)icp_res[i].T[k];
      }
      if (res[i].id1 >= 0 || icp[i]) {  // node.cpp:1337-1338: edge.id1 = older_node->id_, edge.id2 = this->id_
        out[i].edge.id1 = older[i]->id_;
        out[i].edge.id2 = newer->id_;
        ++newer->initial_node_matches_;  // node.cpp:1417
      }
    }
    return out;
  }

  // USE_PCL_ICP, the reference's compile-time switch (CMakeLists.txt:20, off there too): the ICP fallback of matchNodePair for
  // adjacent nodes whose RANSAC failed (rgbdslam_b200_icp_align).  Read when a Node is constructed (the node then keeps its
  // cloud: the image constructor adds STORE_CLOUD, the cloud constructor KEEP_CLOUD) and in matchNodePair.  The ICP edge maps
  // the older cloud onto the newer one, the inverse direction of a RANSAC edge, as in the reference; its information matrix is
  // zero.  gicp_max_cloud_size (parameter_server.cpp:111): filterCloud's point budget per cloud.
  static bool& pcl_icp() {
    static bool v = false;
    return v;
  }
  static int& gicp_max_cloud_size() {
    static int v = 10000;
    return v;
  }
  // icp_method (parameter_server.cpp:110): "icp" (IterativeClosestPoint) or "icp_nl" (IterativeClosestPointNonLinear); any
  // other name takes "icp", as icp.cpp:55-57 does.  Read in matchNodePair.
  static std::string& icp_method() {
    static std::string v = "icp";
    return v;
  }

  // parameters store_pointclouds / encoding_bgr (parameter_server.cpp), read when an image Node is constructed.  With
  // store_pointclouds the node keeps pc_col (createXYZRGBPointCloud, node.cpp:126-131; the input cloud, :261) on the device
  // for pointCloud() and GraphManager::saveAllClouds.  Unlike the reference, whose default is true, it defaults to false here,
  // so that a node costs no cloud memory (614 kB per 640 x 480 frame) unless the map is wanted.  encoding_bgr (default true,
  // as in the reference) reads channel 0 of a three-channel visual as blue.
  static bool& store_pointclouds() {
    static bool v = false;
    return v;
  }
  static bool& encoding_bgr() {
    static bool v = true;
    return v;
  }
  // Node::pc_col: the node's organised colour cloud, downloaded from the device (rgbdslam_b200_node_download_cloud); the
  // node must have been built with store_pointclouds().
  pointcloud_type::Ptr pointCloud() const {
    int w = 0, h = 0;
    check(rgbdslam_b200_node_download_cloud(handle_, (int)sizeof(point_type), nullptr, &w, &h), "node_download_cloud");
    pointcloud_type::Ptr pc = std::make_shared<pointcloud_type>();
    pc->points.resize((size_t)w * h);
    pc->width = (uint32_t)w;
    pc->height = (uint32_t)h;
    if (w > 0 && h > 0)
      check(rgbdslam_b200_node_download_cloud(handle_, (int)sizeof(point_type), pc->points.data(), &w, &h), "node_download_cloud");
    return pc;
  }

  // Node::reducePointCloud (node.cpp:1448-1460): pc_col becomes its voxel grid of leaf size vfs on the device
  // (rgbdslam_b200_reduce_clouds), so pointCloud() afterwards is the n x 1 cloud of centroids.  vfs <= 0 warns and changes
  // nothing, like the reference; a NaN or infinite vfs throws.  When the leaf size is too small for the cloud (PCL's
  // "Leaf size is too small" warning) the cloud also stays as it is.
  void reducePointCloud(double vfs) {
    if (vfs <= 0.0) {
      std::fprintf(stderr, "Point Clouds can't be reduced because of invalid voxelfilter_size\n");
      return;
    }
    check(rgbdslam_b200_reduce_clouds(1, &handle_, vfs, nullptr), "reduce_clouds");
  }

  // Node::clearPointCloud (octomap_clear_raycasted_clouds): the node drops pc_col on the device
  // (rgbdslam_b200_node_clear_cloud); pointCloud() afterwards is empty.
  void clearPointCloud() { check(rgbdslam_b200_node_clear_cloud(handle_), "node_clear_cloud"); }

  static int& max_connections() {  // parameter max_connections (parameter_server.cpp:104), -1 = unlimited
    static int v = -1;
    return v;
  }
  // parameters depth_camera_fx, depth_camera_fy, depth_camera_cx, depth_camera_cy (parameter_server.cpp:42-45), default 0:
  // the camera the environment measurement model projects kept point clouds into (misc.cpp:56-63).  Read when a point-cloud
  // Node is constructed.  All zero, as in the reference with the parameters unset, projects every finite point to pixel (0, 0).
  static float* depth_camera_intrinsics() {
    static float v[4] = {0.f, 0.f, 0.f, 0.f};
    return v;
  }

 private:
  uint64_t handle_ = 0;
};

// OpenNIListener::noCloudCallback's image handling (openni_listener.cpp:633-659) and noCloudCameraCallback's
// new Node(visual, depth, depth_mono8_img_, cam_info, depth_header, detector, extractor) (:779) in one call.  visual CV_8UC1 or
// CV_8UC3 as for the Node constructor; depth CV_32FC1 metres or the raw CV_16UC1 millimetres, of any size up to 4095 px per side.
// A depth of another size than the visual is resized to the visual's size as the listener does, cv::resize(depth, depth,
// visual.size(), 0, 0, INTER_NEAREST) (:651-656), on the device (rgbdslam_b200/depth_resize.h); the 16-bit depth is converted
// as the Node constructor converts it.  The detection mask is depthToCV8UC1 of that depth (:659; RGBDSLAM_B200_MASK_FROM_DEPTH),
// which the listener always builds.  cam_info is the visual camera's.  store_pointclouds(), pcl_icp() and encoding_bgr() apply
// as in the constructor.  The caller owns the returned Node.  The Node constructor itself keeps refusing a depth of another size:
// in the reference the resize is the listener's step, not the Node's.
inline Node* listenerNode(const Mat& visual, const Mat& depth, const CameraInfoConstPtr& cam_info, myHeader depth_header,
                          Ptr<Feature2D> detector, Ptr<DescriptorExtractor> extractor) {
  if (!detector || !detector->handle()) throw std::invalid_argument("listenerNode: detector must come from createDetector(\"ORB\" or \"FAST\")");
  if (!extractor) throw std::invalid_argument("listenerNode: null extractor");
  const bool u16 = depth.type() == RB_16UC1;
  if ((visual.type() != RB_8UC1 && visual.type() != RB_8UC3) || (depth.type() != RB_32FC1 && !u16) || depth.empty())
    throw std::invalid_argument("listenerNode: visual must be CV_8UC1 or CV_8UC3 and depth CV_32FC1 or CV_16UC1");
  std::unique_ptr<Node> node(new Node());
  node->stamp_ = depth_header.stamp;
  node->seq_id_ = (int)depth_header.seq;
  std::vector<uint8_t> tg;
  std::vector<float> td;
  std::vector<uint16_t> tr;
  const uint8_t* g = detail::packed<uint8_t>(visual, tg);
  const void* d = u16 ? static_cast<const void*>(detail::packed<uint16_t>(depth, tr)) : detail::packed<float>(depth, td);
  const CameraInfo ci = cam_info ? *cam_info : CameraInfo();
  const float K4[4] = {(float)ci.K[0], (float)ci.K[4], (float)ci.K[2], (float)ci.K[5]};  // node.cpp:913-916
  node->construct_resized(g, d, depth.cols, depth.rows, nullptr, visual.cols, visual.rows, K4, detector->handle(),
                          Node::image_flags(visual, u16, true));
  return node.release();
}

}  // namespace rgbdslam_b200

// int bruteForceSearchORB(const uint64_t* v, const uint64_t* search_array, const unsigned int& size, int& result_index)
// -- src/features.h:13.  Single-query form kept for source compatibility; batch callers should use
// rgbdslam_b200_brute_force_orb directly (one launch for all query rows).
inline int bruteForceSearchORB(const uint64_t* v, const uint64_t* search_array, const unsigned int& size, int& result_index) {
  int32_t idx = -1, hd = 257;
  if (rgbdslam_b200_brute_force_orb(v, 1, search_array, (int)size, &idx, &hd) != 0)
    throw std::runtime_error(rgbdslam_b200_last_error());
  result_index = idx;
  return hd;
}
