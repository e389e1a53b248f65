// graph_manager.hpp -- header-only C++ shim of the reference's GraphManager call surface over the C ABI (SURVEY.md 8b):
//   bool   GraphManager::addNode(Node*)                                  src/graph_manager.cpp:681-782 (firstNode :361-409)
//   bool   nodeComparisons(Node*, ...)                                   :421-658   (the <= 12 comparisons = ONE batched call)
//   QList<int> getPotentialEdgeTargetsWithDijkstra(...)                  :204-324
//   bool   addEdgeToG2O(const LoadedEdge3D&, Node*, Node*, bool, bool)   :811-898
//   double optimizeGraph(double break_criterion = -1, bool nonthreaded)  :900-1066  -> rgbdslam_b200_posegraph_optimize
//   unsigned pruneEdgesWithErrorAbove(float)                             :1106-1246 -> rgbdslam_b200_posegraph_chi2
//   void   saveTrajectory(filename)                                      graph_mgr_io.cpp:615-677 / logTransform misc.cpp:90-93
//   void   saveAllClouds(filename)  == saveAllCloudsToFile               graph_mgr_io.cpp:502-583 -> rgbdslam_b200_render_cloud
//   size_t reducePointClouds()      == reducePointCloud for every node   graph_manager.cpp:1310-1319 -> rgbdslam_b200_reduce_clouds
//   void   saveOctomap(filename)    == saveOctomapImpl                   graph_mgr_io.cpp:253-310 -> rgbdslam_b200_octomap_*
//   void   renderToOctomap(Node*), writeOctomap(filename)              graph_mgr_io.cpp:312-329
//   void   occupancyFilterClouds()                                      graph_manager.cpp:1372-1381 -> rgbdslam_b200_octomap_filter_clouds
//   size_t saveIndividualClouds(basename) == saveIndividualCloudsToFile graph_mgr_io.cpp:330-433 -> rgbdslam_b200_transform_clouds
//   size_t saveAllFeatures(filename) == saveAllFeaturesToFile           graph_mgr_io.cpp:445-497 (export_text.hpp, host only)
// Host logic only; every compute step is a C-ABI call.  The reference draws from the global rand(); here every draw comes
// from the library's counter-based generator keyed by (seed, node id).  g2o's HyperDijkstra (not under /root/reference) is
// restated in geodesicBall().  oracle/graph_manager_oracle.py is the Python twin of this file, decision for decision; where
// this file departs from the reference on purpose it says so: the 3-D feature count of nodes without 2-D keypoints (addNode),
// the new node never being its own geodesic candidate (getPotentialEdgeTargetsWithDijkstra), the initial comparison's
// generator key (nodeComparisons), the 1 ms floor of the constant-position time delta and the anchor of an optimisation
// without a fixed vertex (fixationOfVertices).
#pragma once
#include <algorithm>
#include <cctype>
#include <cmath>
#include <cstdio>
#include <functional>
#include <map>
#include <set>
#include <stdexcept>
#include <string>

#include "export_text.hpp"
#include "node.hpp"

namespace rgbdslam_b200 {

struct Pose7 {  // t (x, y, z) + unit quaternion (x, y, z, w): VertexSE3 estimate / EdgeSE3 measurement
  double v[7];
  static Pose7 Identity() { return Pose7{{0, 0, 0, 0, 0, 0, 1}}; }
};

inline void quatToRot(const double* q, double R[9]) {
  const double n = std::sqrt(q[0] * q[0] + q[1] * q[1] + q[2] * q[2] + q[3] * q[3]);
  const double x = q[0] / n, y = q[1] / n, z = q[2] / n, w = q[3] / n;
  R[0] = 1 - 2 * (y * y + z * z); R[1] = 2 * (x * y - z * w);     R[2] = 2 * (x * z + y * w);
  R[3] = 2 * (x * y + z * w);     R[4] = 1 - 2 * (x * x + z * z); R[5] = 2 * (y * z - x * w);
  R[6] = 2 * (x * z - y * w);     R[7] = 2 * (y * z + x * w);     R[8] = 1 - 2 * (x * x + y * y);
}
inline void rotToQuat(const double R[9], double* q) {  // Eigen::Quaternion(Matrix3), normalised
  const double tr = R[0] + R[4] + R[8];
  if (tr > 0) {
    double s = std::sqrt(tr + 1.0);
    q[3] = 0.5 * s;
    s = 0.5 / s;
    q[0] = (R[7] - R[5]) * s; q[1] = (R[2] - R[6]) * s; q[2] = (R[3] - R[1]) * s;
  } else {
    int i = 0;
    if (R[4] > R[0]) i = 1;
    if (R[8] > R[4 * i]) i = 2;
    const int j = (i + 1) % 3, k = (j + 1) % 3;
    double s = std::sqrt(R[4 * i] - R[4 * j] - R[4 * k] + 1.0);
    q[i] = 0.5 * s;
    s = 0.5 / s;
    q[3] = (R[3 * k + j] - R[3 * j + k]) * s;
    q[j] = (R[3 * j + i] + R[3 * i + j]) * s;
    q[k] = (R[3 * k + i] + R[3 * i + k]) * s;
  }
  const double n = std::sqrt(q[0] * q[0] + q[1] * q[1] + q[2] * q[2] + q[3] * q[3]);
  for (int a = 0; a < 4; a++) q[a] /= n;
}
// What updateCloudOrigin stores in a node's cloud for an estimate with rotation R (row-major, double) and translation t:
// sensor_orientation_ q (x, y, z, w), R cast to float as an Eigen Quaternionf (Eigen's trace -- its unrolled reduction
// m00 + (m11 + m22) -- and largest-diagonal algorithm, in float), and sensor_origin_ o, t as float.
// rgbdslam_v2_b200._capi.cloud_sensor_pose is the same step in numpy.
inline void cloudSensorPose(const double R[9], const double t[3], float q[4], float o[3]) {
  float r[9];
  for (int i = 0; i < 9; i++) r[i] = (float)R[i];
  const float tr = r[0] + (r[4] + r[8]);
  if (tr > 0.0f) {
    float s = std::sqrt(tr + 1.0f);
    q[3] = 0.5f * s;
    s = 0.5f / s;
    q[0] = (r[7] - r[5]) * s; q[1] = (r[2] - r[6]) * s; q[2] = (r[3] - r[1]) * s;
  } else {
    int i = 0;
    if (r[4] > r[0]) i = 1;
    if (r[8] > r[4 * i]) i = 2;
    const int j = (i + 1) % 3, k = (j + 1) % 3;
    float s = std::sqrt(r[4 * i] - r[4 * j] - r[4 * k] + 1.0f);
    q[i] = 0.5f * s;
    s = 0.5f / s;
    q[3] = (r[3 * k + j] - r[3 * j + k]) * s;
    q[j] = (r[3 * j + i] + r[3 * i + j]) * s;
    q[k] = (r[3 * k + i] + r[3 * i + k]) * s;
  }
  for (int i = 0; i < 3; i++) o[i] = (float)t[i];
}
// tf and Eigen conversions, on row-major 3 x 4 transforms (rotation | origin):
// tf::Matrix3x3::setRotation(tf::Quaternion(x, y, z, w)) in double, into the rotation part of M
inline void tfSetRotation(const double* q, double M[12]) {
  const double x = q[0], y = q[1], z = q[2], w = q[3];
  const double d = x * x + y * y + z * z + w * w, s = 2.0 / d;
  const double xs = x * s, ys = y * s, zs = z * s, wx = w * xs, wy = w * ys, wz = w * zs;
  const double xx = x * xs, xy = x * ys, xz = x * zs, yy = y * ys, yz = y * zs, zz = z * zs;
  M[0] = 1.0 - (yy + zz), M[1] = xy - wz, M[2] = xz + wy;
  M[4] = xy + wz, M[5] = 1.0 - (xx + zz), M[6] = yz - wx;
  M[8] = xz - wy, M[9] = yz + wx, M[10] = 1.0 - (xx + yy);
}
// tf::Matrix3x3::getRotation of the rotation part of M (tf's branch and tie rule): g (x, y, z, w)
inline void tfGetRotation(const double M[12], double g[4]) {
  const double mt = M[0] + M[5] + M[10];
  if (mt > 0.0) {
    double s = std::sqrt(mt + 1.0);
    g[3] = s * 0.5;
    s = 0.5 / s;
    g[0] = (M[9] - M[6]) * s; g[1] = (M[2] - M[8]) * s; g[2] = (M[4] - M[1]) * s;
  } else {
    const int i = M[0] < M[5] ? (M[5] < M[10] ? 2 : 1) : (M[0] < M[10] ? 2 : 0);
    const int j = (i + 1) % 3, k = (i + 2) % 3;
    double s = std::sqrt(M[5 * i] - M[5 * j] - M[5 * k] + 1.0);
    g[i] = s * 0.5;
    s = 0.5 / s;
    g[3] = (M[4 * k + j] - M[4 * j + k]) * s;
    g[j] = (M[4 * j + i] + M[4 * i + j]) * s;
    g[k] = (M[4 * k + i] + M[4 * i + k]) * s;
  }
}
// Eigen's Quaternionf::toRotationMatrix of q (x, y, z, w), into the rotation part of T
inline void quatfToRotationMatrix(const float q[4], float T[12]) {
  const float fx = q[0], fy = q[1], fz = q[2], fw = q[3];
  const float tx = 2.0f * fx, ty = 2.0f * fy, tz = 2.0f * fz;
  const float twx = tx * fw, twy = ty * fw, twz = tz * fw, txx = tx * fx, txy = ty * fx, txz = tz * fx;
  const float tyy = ty * fy, tyz = tz * fy, tzz = tz * fz;
  T[0] = 1.0f - (tyy + tzz), T[1] = txy - twz, T[2] = txz + twy;
  T[4] = txy + twz, T[5] = 1.0f - (txx + tzz), T[6] = tyz - twx;
  T[8] = txz - twy, T[9] = tyz + twx, T[10] = 1.0f - (txx + tyy);
}
// tf::Transform * tf::Transform: (Ra Rb, Ra tb + ta), every entry a sum (a0 b0 + a1 b1) + a2 b2
inline void tfMul(const double A[12], const double B[12], double T[12]) {
  for (int r = 0; r < 3; r++) {
    for (int c = 0; c < 3; c++) T[4 * r + c] = (A[4 * r] * B[c] + A[4 * r + 1] * B[4 + c]) + A[4 * r + 2] * B[8 + c];
    T[4 * r + 3] = ((A[4 * r] * B[3] + A[4 * r + 1] * B[7]) + A[4 * r + 2] * B[11]) + A[4 * r + 3];
  }
}
// tf::Transform::inverse: (R^T, R^T (-t)), -t negating every component (a zero origin becomes -0)
inline void tfInverse(const double A[12], double T[12]) {
  const double m[3] = {-A[3], -A[7], -A[11]};
  for (int r = 0; r < 3; r++) {
    for (int c = 0; c < 3; c++) T[4 * r + c] = A[4 * c + r];
    T[4 * r + 3] = (A[r] * m[0] + A[4 + r] * m[1]) + A[8 + r] * m[2];
  }
}

// The float 3 x 4 (row-major, node -> map) saveOctomap applies to a node whose estimate has rotation R (row-major, double)
// and translation t: cloudSensorPose, then insertCloudCallback widens the quaternion to a tf::Quaternion,
// tf::Matrix3x3::setRotation builds the basis in double, pcl_ros::transformPointCloud takes it back with getRotation (tf's
// branch and tie rule), narrows it to a Quaternionf and applies toRotationMatrix (float).  The ray origin is the translation
// column.  rgbdslam_v2_b200._capi.octomap_pose is the same chain in numpy.
inline void octomapPose(const double R[9], const double t[3], float T[12]) {
  float q[4], o[3];  // q: x, y, z, w
  cloudSensorPose(R, t, q, o);
  const double qd[4] = {q[0], q[1], q[2], q[3]};
  double M[12], g[4];
  tfSetRotation(qd, M);
  tfGetRotation(M, g);
  const float gf[4] = {(float)g[0], (float)g[1], (float)g[2], (float)g[3]};
  quatfToRotationMatrix(gf, T);
  T[3] = o[0], T[7] = o[1], T[11] = o[2];
}

inline Pose7 poseFromIsometry(const Isometry3d& T) {  // column-major 4x4
  double R[9];
  for (int r = 0; r < 3; r++)
    for (int c = 0; c < 3; c++) R[3 * r + c] = T.m[4 * c + r];
  Pose7 p;
  p.v[0] = T.m[12]; p.v[1] = T.m[13]; p.v[2] = T.m[14];
  rotToQuat(R, p.v + 3);
  return p;
}
inline Pose7 compose(const Pose7& a, const Pose7& b) {  // a * b
  double Ra[9], Rb[9], R[9];
  quatToRot(a.v + 3, Ra);
  quatToRot(b.v + 3, Rb);
  for (int r = 0; r < 3; r++)
    for (int c = 0; c < 3; c++) R[3 * r + c] = Ra[3 * r] * Rb[c] + Ra[3 * r + 1] * Rb[3 + c] + Ra[3 * r + 2] * Rb[6 + c];
  Pose7 p;
  for (int r = 0; r < 3; r++) p.v[r] = a.v[r] + Ra[3 * r] * b.v[0] + Ra[3 * r + 1] * b.v[1] + Ra[3 * r + 2] * b.v[2];
  rotToQuat(R, p.v + 3);
  return p;
}
inline Pose7 inverse(const Pose7& a) {
  double R[9];
  quatToRot(a.v + 3, R);
  Pose7 p;
  for (int r = 0; r < 3; r++) p.v[r] = -(R[r] * a.v[0] + R[3 + r] * a.v[1] + R[6 + r] * a.v[2]);
  p.v[3] = -a.v[3]; p.v[4] = -a.v[4]; p.v[5] = -a.v[5]; p.v[6] = a.v[6];
  return p;
}

// misc.cpp:272-315
inline void trafoSize(const Isometry3d& t, double& angle, double& dist) {
  angle = std::acos((t.m[0] + t.m[5] + t.m[10] - 1) / 2) * 180.0 / M_PI;
  dist = std::sqrt(t.m[12] * t.m[12] + t.m[13] * t.m[13] + t.m[14] * t.m[14]);
}

class GraphManager {
 public:
  struct Params {  // the ParameterServer entries this logic reads (parameter_server.cpp:85-123)
    int min_matches = 20, predecessor_candidates = 4, neighbor_candidates = 4, min_sampled_candidates = 4, geodesic_depth = 3;
    double min_translation_meter = 0.0, min_rotation_degree = 0.0, max_translation_meter = 1e10, max_rotation_degree = 360.0;
    bool keep_all_nodes = false, keep_good_nodes = false;
    int optimizer_skip_step = 1;
    double optimizer_iterations = 0.01, huber_delta = 1.0;
    bool valid_odometry = false;  // !odom_frame_name.empty()
    // fixationOfVertices strategy (graph_manager.cpp:911-937, parameter_server.cpp:118): "first" (default), "previous",
    // "largest_loop", "inaffected" (the reference's benchmark setting, test/test_settings.launch:94)
    std::string pose_relative_to = "first";
  };
  Params params;
  uint64_t seed = 0;

  std::map<int, Node*> graph_;                 // graph_manager.h:156 (owned after addNode, like the reference)
  std::vector<int> keyframe_ids_;
  std::vector<std::pair<int, int>> edges_;     // (id1 = older, id2 = newer) of cam_cam_edges_
  std::vector<Pose7> meas_;
  std::vector<Matrix6d> info_;
  std::vector<bool> active_;                   // false: removed by pruneEdgesWithErrorAbove
  std::map<int, Pose7> estimates_;             // VertexSE3 estimates by node id (vertex id == node id here)
  MatchingResult curr_best_result_;
  unsigned loop_closures_edges = 0, sequential_edges = 0;
  double last_chi2 = 0.0;
  int earliest_loop_closure_node_ = 0;         // graph_manager.h:356
  // vertices with setFixed(true): firstNode fixes the first one (:381), "inaffected" frees both ends of every new edge (:889-892),
  // the end of optimizeGraph fixes ("inaffected") or frees (every other strategy) them all (:1031-1036)
  std::set<int> fixed_ids_;
  // optional observer: nodeComparisons passes it the candidate ids in the order getPotentialEdgeTargetsWithDijkstra returned them
  std::function<void(const std::vector<int>&)> on_edge_targets_;

  virtual ~GraphManager() {
    for (auto& kv : graph_) delete kv.second;
    if (octomap_) rgbdslam_b200_octomap_destroy(octomap_);
  }

  bool isBigTrafo(const Isometry3d& t) const {
    double a, d;
    trafoSize(t, a, d);
    return d > params.min_translation_meter || a > params.min_rotation_degree;
  }
  bool isSmallTrafo(const Isometry3d& t, double seconds) const {
    if (seconds <= 0.0) return true;
    double a, d;
    trafoSize(t, a, d);
    return d / seconds < params.max_translation_meter && a / seconds < params.max_rotation_degree;
  }

  // ---- graph_manager.cpp:681-782
  bool addNode(Node* new_node) {
    // the reference gates on feature_locations_2d_ only (:687); nodes built from bare features (no 2-D keypoints) fall back
    // to their 3-D feature count
    const size_t nfeat = new_node->feature_locations_2d_.empty() ? new_node->feature_locations_3d_.size()
                                                                 : new_node->feature_locations_2d_.size();
    if ((int)nfeat < params.min_matches) return false;
    if (graph_.empty()) {
      firstNode(new_node);
      return true;
    }
    bool edge_to_last_keyframe_found = false;
    const bool found_match = nodeComparisons(new_node, edge_to_last_keyframe_found);
    if (found_match) {
      graph_[new_node->id_] = new_node;
      if (!edge_to_last_keyframe_found && earliest_loop_closure_node_ > keyframe_ids_.back())  // :731
        keyframe_ids_.push_back(new_node->id_ - 1);
      if (params.optimizer_skip_step > 0 && (int)estimates_.size() % params.optimizer_skip_step == 0) optimizeGraph();
    } else if (graph_.size() == 1) {
      // only one node so far and it has fewer features: the new node replaces it (:760-767)
      Node* first = graph_.begin()->second;
      const size_t nfirst = first->feature_locations_2d_.empty() ? first->feature_locations_3d_.size() : first->feature_locations_2d_.size();
      if (nfeat > nfirst) {
        resetGraph();
        firstNode(new_node);
        return true;
      }
    }
    return found_match;
  }

  void resetGraph() {  // GraphManager::resetGraph as far as this shim keeps state
    for (auto& kv : graph_) delete kv.second;
    graph_.clear(); keyframe_ids_.clear(); edges_.clear(); meas_.clear(); info_.clear(); active_.clear(); estimates_.clear();
    adj_.clear(); fixed_ids_.clear();
    curr_best_result_ = MatchingResult();
    loop_closures_edges = sequential_edges = 0;
    earliest_loop_closure_node_ = 0;
  }

  // ---- graph_manager.cpp:204-324
  std::vector<int> getPotentialEdgeTargetsWithDijkstra(const Node* new_node, int sequential_targets, int geodesic_targets,
                                                       int sampled_targets, int predecessor_id = -1, bool include_predecessor = false) {
    Rand rnd(seed, (uint64_t)new_node->id_);
    std::vector<int> ids;  // QList: push_front == insert at begin
    const int gsize = (int)graph_.size();
    if (predecessor_id < 0) predecessor_id = gsize - 1;
    if ((int)estimates_.size() <= sequential_targets + geodesic_targets + sampled_targets || estimates_.size() <= 1) {
      sequential_targets += geodesic_targets + sampled_targets;
      geodesic_targets = sampled_targets = 0;
      predecessor_id = gsize - 1;
    }
    for (int i = 1; i < sequential_targets + 1 && predecessor_id - i >= 0; i++) ids.push_back(predecessor_id - i);
    if (geodesic_targets > 0) {
      std::map<int, int> weights;
      int sum = 0;
      for (int vid : geodesicBall(predecessor_id, params.geodesic_depth)) {
        if (vid == new_node->id_) continue;  // (the reference can pick the new node itself here: a self-edge)
        if (!graph_.at(vid)->matchable_) continue;
        if (vid < predecessor_id - sequential_targets || (vid > predecessor_id && vid <= gsize - 1)) {
          weights[vid] = std::abs(predecessor_id - vid);
          sum += weights[vid];
        }
      }
      while ((int)ids.size() < sequential_targets + geodesic_targets && !weights.empty()) {
        const int pick = (int)(rnd() % (uint32_t)sum);
        int acc = 0;
        for (auto it = weights.begin(); it != weights.end(); ++it) {
          acc += it->second;
          if (acc > pick) {
            ids.insert(ids.begin(), it->first);
            sum -= it->second;
            weights.erase(it);
            break;
          }
        }
      }
    }
    if (sampled_targets > 0) {
      std::vector<int> pool;
      for (int k : keyframe_ids_)
        if (std::find(ids.begin(), ids.end(), k) == ids.end() && graph_.at(k)->matchable_) pool.push_back(k);
      while ((int)ids.size() < geodesic_targets + sampled_targets + sequential_targets && !pool.empty()) {
        const int i = (int)(rnd() % (uint32_t)pool.size());
        ids.insert(ids.begin(), pool[i]);
        pool[i] = pool.back();
        pool.pop_back();
      }
    }
    if (include_predecessor) ids.push_back(predecessor_id);
    return ids;
  }

  // ---- graph_manager.cpp:811-898
  bool addEdgeToG2O(const LoadedEdge3D& edge, Node* n1, Node* n2, bool largeEdge, bool set_estimate) {
    if (edge.id1 == edge.id2) return false;
    const bool v1 = estimates_.count(n1->id_) != 0, v2 = estimates_.count(n2->id_) != 0;
    if ((!v1 || !v2) && !largeEdge) return false;
    if (!v1 && !v2) return false;
    const Pose7 z = poseFromIsometry(edge.transform);
    if (!v1 && v2) {
      estimates_[n1->id_] = compose(estimates_[n2->id_], inverse(z));
      n1->vertex_id_ = n1->id_;
    } else if (!v2 && v1) {
      estimates_[n2->id_] = compose(estimates_[n1->id_], z);
      n2->vertex_id_ = n2->id_;
    } else if (set_estimate) {
      estimates_[n2->id_] = compose(estimates_[n1->id_], z);
    }
    edges_.push_back(std::make_pair(edge.id1, edge.id2));
    meas_.push_back(z);
    info_.push_back(edge.informationMatrix);
    active_.push_back(true);
    adj_[edge.id1].insert(edge.id2);
    adj_[edge.id2].insert(edge.id1);
    if (std::abs(edge.id1 - edge.id2) > params.predecessor_candidates) loop_closures_edges++;
    else sequential_edges++;
    if (params.pose_relative_to == "inaffected") {  // :889-892
      fixed_ids_.erase(edge.id1);
      fixed_ids_.erase(edge.id2);
    } else if (params.pose_relative_to == "largest_loop") {  // :893-896: only this strategy lowers it
      earliest_loop_closure_node_ = std::min(earliest_loop_closure_node_, std::min(edge.id1, edge.id2));
    }
    return true;
  }

  // ---- graph_manager.cpp:900-1066.  break_criterion: >= 1 iterations, (0, 1) relative chi2 improvement, < 0 the parameter.
  // Virtual so that a caller can observe every optimisation, those addNode runs included.
  virtual double optimizeGraph(double break_criterion = -1.0, bool /*nonthreaded*/ = false) {
    std::vector<int> ids;
    std::vector<double> poses, meas, info;
    std::vector<uint8_t> fixed;
    std::vector<int32_t> ij;
    gather(ids, poses, fixed, ij, meas, info);
    if (ij.empty()) {
      renderNewestOnline();
      return 0.0;
    }
    fixationOfVertices(ids, fixed);
    const double stop = break_criterion > 0.0 ? break_criterion : params.optimizer_iterations;  // :942
    double chi2 = 0;
    int it = 0, cg = 0;
    check(rgbdslam_b200_posegraph_optimize((int)ids.size(), poses.data(), fixed.data(), (int)ij.size() / 2, ij.data(), meas.data(),
                                           info.data(), stop, params.huber_delta, &chi2, &it, &cg),
          "posegraph_optimize");
    for (size_t k = 0; k < ids.size(); k++) std::memcpy(estimates_[ids[k]].v, &poses[7 * k], sizeof(double) * 7);
    // after the optimisation (:1031-1037): "inaffected" leaves every camera vertex fixed -- only vertices added afterwards are
    // free in the next run --, every other strategy un-fixes them all
    fixed_ids_.clear();
    if (params.pose_relative_to == "inaffected") fixed_ids_.insert(ids.begin(), ids.end());
    last_chi2 = chi2;
    renderNewestOnline();
    return chi2;
  }

  // fixationOfVertices (graph_manager.cpp:911-937).  `fixed` comes in with the persistent flags (fixed_ids_, see there).
  // "inaffected" has no branch there: the flags stay as the previous optimisation and the edges added since left them; its
  // Dijkstra-selected vertex subset (:969-977) is overridden by the second initializeOptimization(cam_cam_edges_) (:989-992),
  // so all edges are always active.
  void fixationOfVertices(const std::vector<int>& ids, std::vector<uint8_t>& fixed) const {
    const std::string& strategy = params.pose_relative_to;
    auto index_of = [&](int id) { return (int)(std::lower_bound(ids.begin(), ids.end(), id) - ids.begin()); };
    if (strategy == "previous" && graph_.size() > 2) {
      std::fill(fixed.begin(), fixed.end(), 0);
      fixed[index_of(graph_.at((int)graph_.size() - 2)->id_)] = 1;
    } else if (strategy == "largest_loop") {
      for (size_t k = 0; k < ids.size(); k++) fixed[k] = ids[k] < earliest_loop_closure_node_ ? 1 : 0;
    } else if (strategy == "first") {
      std::fill(fixed.begin(), fixed.end(), 0);
      fixed[index_of(graph_.at(0)->id_)] = 1;
    }
    // an optimisation without any fixed vertex has a gauge freedom; g2o then fixes nothing either, but its damped LM
    // still runs -- the PCG here needs one anchor
    if (std::find(fixed.begin(), fixed.end(), 1) == fixed.end() && !fixed.empty()) fixed[0] = 1;
  }

  // The optimiser's input: the vertices in id order with their estimates and persistent fixed flags (fixed_ids_), and the
  // active edges in insertion order (`which`: their indices into edges_).
  void gather(std::vector<int>& ids, std::vector<double>& poses, std::vector<uint8_t>& fixed, std::vector<int32_t>& ij,
              std::vector<double>& meas, std::vector<double>& info, std::vector<size_t>* which = nullptr) const {
    std::map<int, int> index;
    for (auto& kv : estimates_) {
      index[kv.first] = (int)ids.size();
      ids.push_back(kv.first);
      poses.insert(poses.end(), kv.second.v, kv.second.v + 7);
    }
    fixed.assign(ids.size(), 0);
    for (size_t k = 0; k < ids.size(); k++)
      if (fixed_ids_.count(ids[k])) fixed[k] = 1;
    for (size_t e = 0; e < edges_.size(); e++) {
      if (!active_[e]) continue;
      ij.push_back(index[edges_[e].first]);
      ij.push_back(index[edges_[e].second]);
      meas.insert(meas.end(), meas_[e].v, meas_[e].v + 7);
      info.insert(info.end(), info_[e].m, info_[e].m + 36);
      if (which) which->push_back(e);
    }
  }

  // ---- graph_manager.cpp:1106-1246
  unsigned pruneEdgesWithErrorAbove(float thresh) {
    std::vector<int> ids;
    std::vector<double> poses, meas, info;
    std::vector<uint8_t> fixed;
    std::vector<int32_t> ij;
    std::vector<size_t> which;
    gather(ids, poses, fixed, ij, meas, info, &which);
    if (ij.empty()) return 0;
    std::vector<double> per_edge(which.size());
    double chi2 = 0;
    check(rgbdslam_b200_posegraph_chi2((int)ids.size(), poses.data(), (int)which.size(), ij.data(), meas.data(), info.data(),
                                       params.huber_delta, &chi2, per_edge.data()),
          "posegraph_chi2");
    std::map<int, int> degree;  // v->edges().size(): every edge ever added counts
    for (auto& e : edges_) { degree[e.first]++; degree[e.second]++; }
    unsigned counter = 0;
    for (size_t k = 0; k < which.size(); k++) {
      if (!(per_edge[k] > thresh)) continue;
      counter++;
      const size_t e = which[k];
      meas_[e] = Pose7::Identity();
      const int a = edges_[e].first, b = edges_[e].second;
      Matrix6d I;
      std::memset(&I, 0, sizeof(I));
      if (std::abs(a - b) != 1) {
        if (degree[a] > 1 && degree[b] > 1) { active_[e] = false; continue; }
        for (int i = 0; i < 6; i++) I.m[7 * i] = 1e-100;
      } else {
        for (int i = 0; i < 6; i++) I.m[7 * i] = 1.0;
      }
      info_[e] = I;
    }
    return counter;
  }

  // parameters maximum_depth (parameter_server.cpp, default +inf: no point is dropped for its range; < 0 also disables the
  // filter) and preserve_raster_on_save (default false) of saveAllClouds
  static double& maximum_depth() {
    static double v = INFINITY;
    return v;
  }
  static bool& preserve_raster_on_save() {
    static bool v = false;
    return v;
  }

  // parameter voxelfilter_size (parameter_server.cpp:159, default -1: no filter) of reducePointClouds
  static double& voxelfilter_size() {
    static double v = -1.0;
    return v;
  }
  // Node::reducePointCloud(voxelfilter_size) of every node of graph_ in one device call.  The reference's slot
  // (GraphManager::reducePointCloud, graph_manager.cpp:1310-1319) reduces the one node whose cloud pointer the GUI hands it after
  // drawing it, so that in the end every drawn node is reduced; without a GUI the whole graph is reduced at once.  Nodes without a
  // stored cloud are passed over; voxelfilter_size <= 0 warns and changes nothing.  Returns the number of nodes reduced.
  size_t reducePointClouds() {
    if (voxelfilter_size() <= 0.0) {
      std::fprintf(stderr, "Point Clouds can't be reduced because of invalid voxelfilter_size\n");
      return 0;
    }
    std::vector<uint64_t> handles;
    for (auto& kv : graph_) {
      int w = 0, h = 0;
      if (rgbdslam_b200_node_download_cloud(kv.second->handle(), 32, nullptr, &w, &h) == 0) handles.push_back(kv.second->handle());
    }
    std::vector<int32_t> counts(handles.size());
    check(rgbdslam_b200_reduce_clouds((int)handles.size(), handles.data(), voxelfilter_size(), counts.data()), "reduce_clouds");
    size_t reduced = 0;
    for (int32_t c : counts) reduced += c >= 0;
    return reduced;
  }

  // world2cam = cam2rgb * eigenTransf2TF(estimate of node id) in double (graph_mgr_io.cpp:526-541), row-major 3 x 4: cam2rgb has
  // rotation createQuaternionFromRPY(-1.57, 0, -1.57) (-1.57, not -pi/2) and origin (0, -0.04, 0); eigenTransf2TF takes the
  // rotation through a quaternion (Eigen's matrix -> quaternion, here normalised) and tf's quaternion -> matrix.
  void mapTransform(int id, double T[12]) const {
    double P[12], C[12];
    eigenTransf2TF(id, P);
    const double hr = -1.57 * 0.5, hp = 0.0, hy = -1.57 * 0.5;  // tf::Quaternion::setRPY(roll, pitch, yaw)
    const double cr = std::cos(hr), sr = std::sin(hr), cp = std::cos(hp), sp = std::sin(hp), cy = std::cos(hy), sy = std::sin(hy);
    const double qc[4] = {sr * cp * cy - cr * sp * sy, cr * sp * cy + sr * cp * sy, cr * cp * sy - sr * sp * cy,
                          cr * cp * cy + sr * sp * sy};
    tfSetRotation(qc, C);
    C[3] = 0.0, C[7] = -0.04, C[11] = 0.0;
    tfMul(C, P, T);
  }
  // eigenTransf2TF(estimate of node id) (misc.cpp), row-major 3 x 4: the VertexSE3 estimate as an Isometry3d, its rotation
  // through Eigen's matrix -> quaternion (here normalised) and tf's quaternion -> matrix, its translation as it is
  void eigenTransf2TF(int id, double P[12]) const {
    const Pose7& p = estimates_.at(id);
    double R[9], q[4];
    quatToRot(p.v + 3, R);
    rotToQuat(R, q);
    tfSetRotation(q, P);
    P[3] = p.v[0], P[7] = p.v[1], P[11] = p.v[2];
  }

  // GraphManager::saveAllCloudsToFile (graph_mgr_io.cpp:502-583): the stored clouds (Node::store_pointclouds()) of the nodes
  // with valid_tf_estimate_, in id order, each put through mapTransform and transformAndAppendPointCloud on the device, written
  // as a binary PCD v0.7 (x y z rgb, 16 bytes per point; width 1 x height n, or n x 1 with preserve_raster_on_save, as PCL
  // leaves the aggregate).  ".pcd" is appended when the name lacks it; a ".ply" name throws std::invalid_argument (PLY
  // output is not built).  Returns the number of points written.
  size_t saveAllClouds(std::string filename) const {
    if (endsWith(filename, ".ply")) throw std::invalid_argument("saveAllClouds: PLY output is not built (save as .pcd)");
    if (!endsWith(filename, ".pcd")) filename += ".pcd";
    std::vector<uint64_t> handles;
    std::vector<double> T;
    for (auto& kv : graph_) {
      const Node* n = kv.second;
      if (!n->valid_tf_estimate_ || !estimates_.count(n->vertex_id_)) continue;
      handles.push_back(n->handle());
      T.resize(T.size() + 12);
      mapTransform(n->vertex_id_, &T[T.size() - 12]);
    }
    const int preserve = preserve_raster_on_save() ? 1 : 0;
    int64_t count = 0;
    check(rgbdslam_b200_render_cloud((int)handles.size(), handles.data(), T.data(), maximum_depth(), preserve, 32, nullptr, 0, &count,
                                     nullptr),
          "render_cloud");
    std::vector<PointXYZRGB> pts((size_t)count);
    check(rgbdslam_b200_render_cloud((int)handles.size(), handles.data(), T.data(), maximum_depth(), preserve, 32, pts.data(), count,
                                     &count, nullptr),
          "render_cloud");
    const unsigned long long n = (unsigned long long)count;
    const float viewpoint[7] = {0, 0, 0, 1, 0, 0, 0};
    writePCD(filename, pts, preserve ? n : 1ull, preserve ? 1ull : n, viewpoint);
    return pts.size();
  }

  // parameter transform_individual_clouds (parameter_server.cpp:67, default false) of saveIndividualClouds
  static bool& transform_individual_clouds() {
    static bool v = false;
    return v;
  }
  // world2points of saveIndividualCloudsToFile (graph_mgr_io.cpp:384-396) without tf and ground truth:
  // computeFixedToBaseTransform (:56-90) init_base_pose_ * base2points * eigenTransf2TF(estimate) * base2points.inverse(), times
  // base2points, with init_base_pose_ and base2points identities.  The products are formed literally: an identity factor can
  // turn the sign of a zero, which the pose text shows.
  void worldToPoints(int id, double W[12]) const {
    const double I[12] = {1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1, 0};
    double M[12], inv[12], a[12], b[12], c[12];
    eigenTransf2TF(id, M);
    tfInverse(I, inv);
    tfMul(I, I, a);
    tfMul(a, M, b);
    tfMul(b, inv, c);
    tfMul(c, I, W);
  }
  // GraphManager::saveIndividualCloudsToFile (graph_mgr_io.cpp:330-433): in ascending id, every node with valid_tf_estimate_,
  // an estimate and a non-empty stored cloud (the test of updateCloudOrigin) writes basename_%04d.pcd (its stored cloud, binary,
  // x y z rgb, its own width x height, NaN points included) and basename_%04d.txt (the sensor pose as a 4 x 4, rows "R R R o ",
  // then "0 0 0 1").  With transform_individual_clouds the clouds are first transformed in place on the device by their
  // estimates (rgbdslam_b200_transform_clouds) and stay so; the pose is then the reference's Quaternionf(0, 0, 0, 1) --
  // (w, x, y, z): w = 0, z = 1, a half turn about z -- at origin 0.  Without it the pose is worldToPoints'.  Either way it
  // becomes the node's cloud sensor pose.  Floats are written as std::ostream writes them (ostreamFloat).  The _gt.pcd files
  // of ground_truth_frame_name are not built.  Returns the number of nodes written.
  size_t saveIndividualClouds(const std::string& basename) {
    std::vector<Node*> nodes;
    for (auto& kv : graph_)
      if (hasCloud(kv.second)) nodes.push_back(kv.second);
    const bool in_place = transform_individual_clouds();
    if (in_place) {
      std::vector<uint64_t> handles;
      std::vector<double> T;
      for (Node* n : nodes) {  // v->estimate().matrix()
        const Pose7& p = estimates_.at(n->vertex_id_);
        double R[9];
        quatToRot(p.v + 3, R);
        handles.push_back(n->handle());
        const double t[12] = {R[0], R[1], R[2], p.v[0], R[3], R[4], R[5], p.v[1], R[6], R[7], R[8], p.v[2]};
        T.insert(T.end(), t, t + 12);
      }
      check(rgbdslam_b200_transform_clouds((int)handles.size(), handles.data(), T.data()), "transform_clouds");
    }
    for (Node* n : nodes) {
      float q[4] = {0, 0, 1, 0}, o[3] = {0, 0, 0};  // sensor_orientation_ (x, y, z, w), sensor_origin_
      if (!in_place) {
        double W[12], g[4];
        worldToPoints(n->vertex_id_, W);
        tfGetRotation(W, g);
        for (int k = 0; k < 4; k++) q[k] = (float)g[k];
        o[0] = (float)W[3], o[1] = (float)W[7], o[2] = (float)W[11];
      }
      float R[12];
      quatfToRotationMatrix(q, R);
      std::memcpy(n->cloud_sensor_pose_, q, sizeof(q));
      std::memcpy(n->cloud_sensor_pose_ + 4, o, sizeof(o));
      int w = 0, h = 0;
      check(rgbdslam_b200_node_download_cloud(n->handle(), 32, nullptr, &w, &h), "node_download_cloud");
      std::vector<PointXYZRGB> pts((size_t)w * h);
      check(rgbdslam_b200_node_download_cloud(n->handle(), 32, pts.data(), &w, &h), "node_download_cloud");
      char suffix[32];
      std::snprintf(suffix, sizeof(suffix), "_%04d", n->id_);
      const float viewpoint[7] = {o[0], o[1], o[2], q[3], q[0], q[1], q[2]};
      writePCD(basename + suffix + ".pcd", pts, (unsigned long long)w, (unsigned long long)h, viewpoint);
      std::string text;
      for (int i = 0; i < 3; i++)
        text += ostreamFloat(R[4 * i]) + " " + ostreamFloat(R[4 * i + 1]) + " " + ostreamFloat(R[4 * i + 2]) + " " + ostreamFloat(o[i]) + " ";
      text += "0 0 0 1\n";
      writeFile(basename + suffix + ".txt", text);
    }
    return nodes.size();
  }

  // GraphManager::saveAllFeaturesToFile (graph_mgr_io.cpp:445-497) as OpenCV 4.13's cv::FileStorage writes it (YamlFileStorage):
  // Feature_Locations, a sequence of flow maps {x, y, z}, one per feature of every node with valid_tf_estimate_ in id order --
  // mapTransform cast to float applied to (x, y, z, 1) in float, each row ((c0 x + c1 y) + c2 z) + c3, non-finite values
  // included --, then Feature_Descriptors, the descriptors of graph_[0], graph_[1], ... graph_[size - 1] looked up by key, as one
  // CV_8U matrix of 32 columns; like the reference this includes the nodes whose locations were skipped.  The float chain
  // assumes a build without FMA contraction (x86-64's default; add -ffp-contract=off to -mfma builds).  A name not ending in
  // .yml / .yaml throws std::invalid_argument (XML, JSON and .gz storage are not built); an empty graph throws
  // std::runtime_error (the reference asserts) and an id missing from [0, size) std::out_of_range (the reference crashes),
  // before the file is opened.  Returns the number of feature locations written.
  size_t saveAllFeatures(const std::string& filename) const {
    if (!endsWith(filename, ".yml") && !endsWith(filename, ".yaml"))
      throw std::invalid_argument("saveAllFeatures: only YAML storage (.yml / .yaml) is built");
    if (graph_.empty()) throw std::runtime_error("saveAllFeatures: the graph is empty");
    std::vector<uint8_t> desc;
    for (int i = 0; i < (int)graph_.size(); i++) {
      const std::vector<uint8_t>& d = graph_.at(i)->feature_descriptors_;
      desc.insert(desc.end(), d.begin(), d.end());
    }
    YamlFileStorage fs;
    fs.startSeq("Feature_Locations");
    size_t count = 0;
    for (auto& kv : graph_) {
      const Node* n = kv.second;
      if (!n->valid_tf_estimate_) continue;
      double T[12];
      mapTransform(n->vertex_id_, T);
      float M[12];
      for (int k = 0; k < 12; k++) M[k] = (float)T[k];
      for (const Vector4f& loc : n->feature_locations_3d_) {
        fs.startFlowMap();
        fs.writeReal("x", ((M[0] * loc.x + M[1] * loc.y) + M[2] * loc.z) + M[3]);
        fs.writeReal("y", ((M[4] * loc.x + M[5] * loc.y) + M[6] * loc.z) + M[7]);
        fs.writeReal("z", ((M[8] * loc.x + M[9] * loc.y) + M[10] * loc.z) + M[11]);
        fs.endStruct();
        count++;
      }
    }
    fs.endStruct();
    fs.writeMatU8("Feature_Descriptors", desc.data(), (int)(desc.size() / 32), 32);
    writeFile(filename, fs.release());
    return count;
  }

  // parameters octomap_* (parameter_server.cpp:56-65) that ColorOctomapServer::reset and saveOctomapImpl read;
  // octomap_occupancy_threshold does not change the file
  static double& octomap_resolution() { static double v = 0.05; return v; }
  static double& octomap_prob_hit() { static double v = 0.9; return v; }
  static double& octomap_prob_miss() { static double v = 0.4; return v; }
  static double& octomap_clamping_min() { static double v = 0.001; return v; }
  static double& octomap_clamping_max() { static double v = 0.999; return v; }
  static double& octomap_occupancy_threshold() { static double v = 0.5; return v; }
  static int& octomap_autosave_step() { static int v = 50; return v; }
  static bool& octomap_clear_after_save() { static bool v = false; return v; }
  static bool& octomap_clear_raycasted_clouds() { static bool v = false; return v; }
  // octomap_online_creation (parameter_server.cpp:65): optimizeGraph ends by rendering the newest node into the map, firstNode
  // runs optimizeGraph, and saveOctomap only writes the map
  static bool& octomap_online_creation() { static bool v = false; return v; }
  // occupancy_filter_threshold (parameter_server.cpp:69) of occupancyFilterClouds
  static double& occupancy_filter_threshold() { static double v = 0.9; return v; }

  // GraphManager::updateCloudOrigin (graph_mgr_io.cpp:216-235): the node has a valid estimate, a vertex and a non-empty stored
  // cloud; the cloud then records the estimate as its sensor pose (Node::cloud_sensor_pose_, cloudSensorPose).  (The
  // reference's function lacks its final `return true`; true is its evident intent.)
  bool updateCloudOrigin(const Node* node) const {
    if (!hasCloud(node)) return false;
    const Pose7& p = estimates_.at(node->vertex_id_);
    double R[9];
    quatToRot(p.v + 3, R);
    cloudSensorPose(R, p.v, node->cloud_sensor_pose_, node->cloud_sensor_pose_ + 4);
    return true;
  }
  // GraphManager::occupancyFilterClouds (graph_manager.cpp:1372-1381): ColorOctomapServer::occupancyFilter of every node of
  // graph_ that has a stored cloud, each under the sensor pose its cloud holds, against the map, in one device call.  Without
  // a map yet an empty one is made first (as writeOctomap does): every cloud is then emptied, as in the reference.
  void occupancyFilterClouds() {
    if (!octomap_) resetOctomap();
    std::vector<uint64_t> handles;
    std::vector<float> sensor;
    for (auto& kv : graph_) {
      int w = 0, h = 0;
      if (rgbdslam_b200_node_download_cloud(kv.second->handle(), 32, nullptr, &w, &h) != 0) continue;
      handles.push_back(kv.second->handle());
      sensor.insert(sensor.end(), kv.second->cloud_sensor_pose_, kv.second->cloud_sensor_pose_ + 7);
    }
    check(rgbdslam_b200_octomap_filter_clouds(octomap_, (int)handles.size(), handles.data(), sensor.data(), occupancy_filter_threshold(),
                                              nullptr),
          "octomap_filter_clouds");
  }
  // octomapPose of the node's estimate
  void octomapTransform(int vertex_id, float T[12]) const {
    const Pose7& p = estimates_.at(vertex_id);
    double R[9];
    quatToRot(p.v + 3, R);  // the VertexSE3 estimate's rotation as an Isometry3d holds it
    octomapPose(R, p.v, T);
  }
  // ColorOctomapServer::reset: an empty map with the current octomap_* parameters
  void resetOctomap() {
    if (octomap_) check(rgbdslam_b200_octomap_destroy(octomap_), "octomap_destroy");
    octomap_ = 0;
    rgbdslam_b200_octomap_params p{octomap_resolution(), octomap_prob_hit(), octomap_prob_miss(), octomap_clamping_min(),
                                   octomap_clamping_max()};
    check(rgbdslam_b200_octomap_create(&p, &octomap_), "octomap_create");
  }
  // GraphManager::renderToOctomap (graph_mgr_io.cpp:318-329): insertCloudCallback of the node when updateCloudOrigin passes,
  // then, with octomap_clear_raycasted_clouds, Node::clearPointCloud whether it was rendered or not
  void renderToOctomap(Node* node) { renderToOctomap(std::vector<Node*>(1, node)); }
  // GraphManager::writeOctomap / ColorOctomapServer::save: the .ot file.  Virtual so that a caller can observe every write,
  // saveOctomap's autosaves included.
  virtual void writeOctomap(const std::string& filename) const {
    if (!octomap_) const_cast<GraphManager*>(this)->resetOctomap();
    int64_t n = 0;
    check(rgbdslam_b200_octomap_write(octomap_, nullptr, 0, &n), "octomap_write");
    std::vector<char> buf((size_t)n);
    check(rgbdslam_b200_octomap_write(octomap_, buf.data(), n, &n), "octomap_write");
    FILE* f = std::fopen(filename.c_str(), "wb");
    if (!f) throw std::runtime_error("cannot open " + filename);
    const bool ok = std::fwrite(buf.data(), 1, buf.size(), f) == buf.size();
    if (std::fclose(f) != 0 || !ok) throw std::runtime_error("cannot write " + filename);
  }
  // GraphManager::saveOctomapImpl (graph_mgr_io.cpp:253-310): the nodes passing updateCloudOrigin in ascending id order, a reset
  // map, each node rendered (octomap_clear_raycasted_clouds applied after it), the file written after every
  // octomap_autosave_step-th node (<= 0: never; the reference divides by it) and once more at the end, then with
  // octomap_clear_after_save a reset.  The nodes between two autosaves go to the device in one insert call: how many one
  // call takes does not change the map.  With octomap_online_creation the map is only written (no reset, autosave or clear).
  void saveOctomap(const std::string& filename) {
    if (octomap_online_creation()) {  // graph_mgr_io.cpp:238-240: the map is already built
      writeOctomap(filename);
      return;
    }
    std::vector<Node*> nodes;
    for (auto& kv : graph_)
      if (updateCloudOrigin(kv.second)) nodes.push_back(kv.second);
    resetOctomap();
    const int step = octomap_autosave_step();
    for (size_t k0 = 0; k0 < nodes.size();) {
      const size_t k1 = step > 0 ? std::min(nodes.size(), (k0 / step + 1) * (size_t)step) : nodes.size();
      renderToOctomap(std::vector<Node*>(nodes.begin() + k0, nodes.begin() + k1));
      if (step > 0 && k1 % step == 0) writeOctomap(filename);
      k0 = k1;
    }
    writeOctomap(filename);
    if (octomap_clear_after_save()) resetOctomap();
  }

  // TUM trajectory "timestamp tx ty tz qx qy qz qw" (logTransform, misc.cpp:90-93)
  void saveTrajectory(const std::string& filename) const {
    FILE* f = std::fopen(filename.c_str(), "w");
    if (!f) throw std::runtime_error("cannot open " + filename);
    std::fprintf(f, "# TF Coordinate Frame ID: (data: )\n");
    for (auto& kv : estimates_) {
      const double* p = kv.second.v;
      std::fprintf(f, "%f %f %f %f %f %f %f %f\n", graph_.at(kv.first)->stamp_, p[0], p[1], p[2], p[3], p[4], p[5], p[6]);
    }
    std::fclose(f);
  }

 private:
  std::map<int, std::set<int>> adj_;
  uint64_t octomap_ = 0;  // ColorOctomapServer co_server_ (graph_manager.h), created at the first reset or write

  void renderToOctomap(const std::vector<Node*>& nodes) {
    if (!octomap_) resetOctomap();
    std::vector<uint64_t> handles;
    std::vector<float> T;
    for (Node* n : nodes) {
      if (!updateCloudOrigin(n)) continue;
      handles.push_back(n->handle());
      T.resize(T.size() + 12);
      octomapTransform(n->vertex_id_, &T[T.size() - 12]);
    }
    check(rgbdslam_b200_octomap_insert(octomap_, (int)handles.size(), handles.data(), T.data(), maximum_depth()), "octomap_insert");
    if (octomap_clear_raycasted_clouds())
      for (Node* n : nodes) n->clearPointCloud();
  }

  // the test updateCloudOrigin and saveIndividualClouds share: valid_tf_estimate_, an estimate and a non-empty stored cloud
  bool hasCloud(const Node* node) const {
    if (!node->valid_tf_estimate_ || !estimates_.count(node->vertex_id_)) return false;
    int w = 0, h = 0;
    return rgbdslam_b200_node_download_cloud(node->handle(), 32, nullptr, &w, &h) == 0 && (long long)w * h != 0;
  }

  static bool endsWith(const std::string& name, const char* ext) {  // ext in lower case; the name's case does not matter
    const size_t n = std::strlen(ext);
    if (name.size() < n) return false;
    for (size_t i = 0; i < n; i++)
      if (std::tolower((unsigned char)name[name.size() - n + i]) != ext[i]) return false;
    return true;
  }
  static void writeFile(const std::string& filename, const std::string& text) {
    FILE* f = std::fopen(filename.c_str(), "wb");
    if (!f) throw std::runtime_error("cannot open " + filename);
    const bool ok = std::fwrite(text.data(), 1, text.size(), f) == text.size();
    if (std::fclose(f) != 0 || !ok) throw std::runtime_error("cannot write " + filename);
  }
  // pcl::io::savePCDFile(filename, cloud, true) of PointXYZRGB records: a binary PCD v0.7 of fields x y z rgb (16 bytes per
  // point), width x height, viewpoint ox oy oz qw qx qy qz as std::ostream writes floats
  static void writePCD(const std::string& filename, const std::vector<PointXYZRGB>& pts, unsigned long long width,
                       unsigned long long height, const float viewpoint[7]) {
    std::string head =
        "# .PCD v0.7 - Point Cloud Data file format\nVERSION 0.7\nFIELDS x y z rgb\nSIZE 4 4 4 4\nTYPE F F F F\nCOUNT 1 1 1 1\n"
        "WIDTH " + std::to_string(width) + "\nHEIGHT " + std::to_string(height) + "\nVIEWPOINT";
    for (int k = 0; k < 7; k++) head += " " + ostreamFloat(viewpoint[k]);
    head += "\nPOINTS " + std::to_string((unsigned long long)pts.size()) + "\nDATA binary\n";
    std::string body(16 * pts.size(), '\0');
    for (size_t i = 0; i < pts.size(); i++) {
      std::memcpy(&body[16 * i], &pts[i].x, 12);
      std::memcpy(&body[16 * i + 12], &pts[i].b, 4);
    }
    writeFile(filename, head + body);
  }

  struct Rand {  // rand() stand-in: the library's splitmix64 counter generator, stream 0xC0
    uint64_t key;
    uint32_t ctr = 0;
    static uint64_t mix(uint64_t z) {
      z += 0x9E3779B97F4A7C15ull;
      z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
      z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
      return z ^ (z >> 31);
    }
    Rand(uint64_t seed, uint64_t node) : key(mix(seed ^ mix(node))) {}
    uint32_t operator()() { return (uint32_t)(mix(key ^ ((0xC0ull << 32) | ctr++)) >> 33); }
  };

  // g2o::HyperDijkstra::shortestPaths(v, UniformCostFunction, maxDistance) + visited(): the source and every vertex whose
  // hop count is < maxDistance
  std::set<int> geodesicBall(int source, double max_distance) const {
    std::map<int, int> dist;
    dist[source] = 0;
    std::vector<int> frontier(1, source);
    while (!frontier.empty()) {
      std::vector<int> next;
      for (int u : frontier) {
        auto it = adj_.find(u);
        if (it == adj_.end()) continue;
        for (int z : it->second) {
          const int d = dist[u] + 1;
          if (!dist.count(z) && d < max_distance) {
            dist[z] = d;
            next.push_back(z);
          }
        }
      }
      frontier.swap(next);
    }
    std::set<int> out;
    for (auto& kv : dist) out.insert(kv.first);
    return out;
  }

  void firstNode(Node* n) {  // :361-409
    n->id_ = (int)graph_.size();
    n->vertex_id_ = n->id_;
    graph_[n->id_] = n;
    estimates_[n->id_] = Pose7::Identity();
    fixed_ids_.insert(n->id_);  // reference_pose->setFixed(true) (:381)
    adj_[n->id_];
    keyframe_ids_.push_back(n->id_);
    if (octomap_online_creation()) optimizeGraph();  // :395-399
  }

  // the end of optimizeGraph (graph_manager.cpp:1044-1049) with octomap_online_creation: the newest node, graph_[size - 1],
  // rendered when updateCloudOrigin passes
  void renderNewestOnline() {
    if (!octomap_online_creation()) return;
    auto it = graph_.find((int)graph_.size() - 1);
    if (it != graph_.end() && updateCloudOrigin(it->second)) renderToOctomap(it->second);
  }

  // ---- graph_manager.cpp:421-658
  bool nodeComparisons(Node* new_node, bool& edge_to_keyframe) {
    const int num_keypoints = (int)std::max(new_node->feature_locations_2d_.size(), new_node->feature_locations_3d_.size());
    if (num_keypoints < params.min_matches && !params.keep_all_nodes) return false;
    new_node->id_ = (int)graph_.size();
    earliest_loop_closure_node_ = new_node->id_;  // :444
    const size_t num_edges_before = edges_.size();
    edge_to_keyframe = false;
    const int sequentially_previous_id = graph_.rbegin()->second->id_;
    curr_best_result_ = MatchingResult();
    bool predecessor_matched = false;
    if (params.min_translation_meter > 0.0 || params.min_rotation_degree > 0.0) {  // initial comparison :458-513
      Node* prev = graph_[(int)graph_.size() - 1];
      // the reference draws this comparison's RANSAC samples from the same global rand() as the others; here it takes the key
      // 64 id + 63, which none of the (at most 12) batched comparisons below, keyed 64 id + k, shares
      MatchingResult mr = new_node->matchNodePair(prev, seed, 64 * (int64_t)new_node->id_ + 63);
      if (mr.edge.id1 >= 0 && mr.edge.id2 >= 0) {
        const double dt = new_node->stamp_ - prev->stamp_;
        if (!isBigTrafo(mr.edge.transform) || !isSmallTrafo(mr.edge.transform, dt)) {
          curr_best_result_ = mr;
          return false;
        }
        if (!addEdgeToG2O(mr.edge, prev, new_node, true, true)) return false;
        graph_[new_node->id_] = new_node;
        if (std::find(keyframe_ids_.begin(), keyframe_ids_.end(), mr.edge.id1) != keyframe_ids_.end()) edge_to_keyframe = true;
        prev->valid_tf_estimate_ = true;
        curr_best_result_ = mr;
        predecessor_matched = true;
      }
    }
    const int seq_cand = params.predecessor_candidates - 1, geod_cand = params.neighbor_candidates,
              samp_cand = params.min_sampled_candidates;
    std::vector<int> targets = predecessor_matched
        ? getPotentialEdgeTargetsWithDijkstra(new_node, seq_cand, geod_cand, samp_cand, curr_best_result_.edge.id1)
        : getPotentialEdgeTargetsWithDijkstra(new_node, seq_cand, geod_cand, samp_cand, sequentially_previous_id, true);
    if (on_edge_targets_) on_edge_targets_(targets);
    std::vector<const Node*> olds;
    for (int t : targets) olds.push_back(graph_[t]);
    // QtConcurrent::blockingMapped(nodes_to_comp, &Node::matchNodePair) (:548) as one batched call
    std::vector<MatchingResult> results = Node::matchNodePairs(new_node, olds, seed, 64 * (int64_t)new_node->id_);
    for (size_t i = 0; i < results.size(); i++) {
      MatchingResult& mr = results[i];
      if (mr.edge.id1 < 0) continue;
      Node* old = graph_[mr.edge.id1];
      const double dt = new_node->stamp_ - old->stamp_;
      const bool more = mr.inlier_matches.size() > curr_best_result_.inlier_matches.size();
      if (isSmallTrafo(mr.edge.transform, dt) && addEdgeToG2O(mr.edge, old, new_node, isBigTrafo(mr.edge.transform), more)) {
        graph_[new_node->id_] = new_node;
        if (mr.edge.id1 == mr.edge.id2 - 1) predecessor_matched = true;
        old->valid_tf_estimate_ = true;
        if (more) curr_best_result_ = mr;
        if (std::find(keyframe_ids_.begin(), keyframe_ids_.end(), mr.edge.id1) != keyframe_ids_.end()) edge_to_keyframe = true;
      }
    }
    const bool found_trafo = edges_.size() != num_edges_before;
    const bool keep_anyway = params.keep_all_nodes || ((int)new_node->feature_locations_3d_.size() > params.min_matches && params.keep_good_nodes);
    const double time_delta_sec = std::fabs(new_node->stamp_ - graph_[sequentially_previous_id]->stamp_);
    if ((!found_trafo && params.valid_odometry) || (!found_trafo && keep_anyway) || (!predecessor_matched && time_delta_sec < 0.1)) {
      LoadedEdge3D odom_edge;  // constant position assumption :636-655
      odom_edge.id1 = sequentially_previous_id;
      odom_edge.id2 = new_node->id_;
      std::memset(&odom_edge.transform, 0, sizeof(odom_edge.transform));
      std::memset(&odom_edge.informationMatrix, 0, sizeof(odom_edge.informationMatrix));
      for (int i = 0; i < 4; i++) odom_edge.transform.m[5 * i] = 1.0;
      // information = I / time_delta_sec (:647); nodes without stamps (dt == 0) would get an infinite information matrix
      // (NaN in the linearisation): the time delta is clamped to 1 ms
      for (int i = 0; i < 6; i++) odom_edge.informationMatrix.m[7 * i] = 1.0 / std::max(time_delta_sec, 1e-3);
      addEdgeToG2O(odom_edge, graph_[sequentially_previous_id], new_node, true, true);
      graph_[new_node->id_] = new_node;
      new_node->valid_tf_estimate_ = false;
      MatchingResult mr;
      mr.edge = odom_edge;
      curr_best_result_ = mr;
    }
    return edges_.size() > num_edges_before;
  }
};

}  // namespace rgbdslam_b200
