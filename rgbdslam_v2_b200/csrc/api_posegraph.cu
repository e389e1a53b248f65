// api_posegraph.cu -- C ABI of the pose-graph solve (declared in include/rgbdslam_b200.h).
#include <cmath>
#include <mutex>

#include "posegraph.h"
#include "state.h"

using namespace rb200;

extern "C" {

int rgbdslam_b200_posegraph_optimize(int nv, double* poses, const uint8_t* fixed, int ne, const int32_t* ij,
                                     const double* meas, const double* info, double stop, double huber_delta,
                                     double* chi2, int* iters, int* cg_iters) {
  RB200_ENTER_INITED();
  if (nv <= 0 || ne < 0 || !poses || !fixed || (ne > 0 && (!ij || !meas || !info)) || !(stop > 0) || !(huber_delta > 0)) {
    set_error("posegraph_optimize: bad arguments (nv > 0, stop > 0, huber_delta > 0)");
    return RGBDSLAM_B200_ERR_ARG;
  }
  for (size_t k = 0; k < (size_t)ne * 36; k++)
    if (!std::isfinite(info[k])) {  // 0 * inf = NaN in the linearisation: the solve would make no progress
      set_error("posegraph_optimize: non-finite entry in an information matrix");
      return RGBDSLAM_B200_ERR_ARG;
    }
  return posegraph_optimize(nv, poses, fixed, ne, ij, meas, info, stop, huber_delta, chi2, iters, cg_iters);
}

int rgbdslam_b200_posegraph_reserve(int nv, int ne) {
  RB200_ENTER_INITED();
  if (nv < 0 || ne < 0) {
    set_error("posegraph_reserve: negative size");
    return RGBDSLAM_B200_ERR_ARG;
  }
  return posegraph_reserve(nv, ne);
}

int rgbdslam_b200_posegraph_chi2(int nv, const double* poses, int ne, const int32_t* ij, const double* meas,
                                 const double* info, double huber_delta, double* chi2, double* per_edge_chi2) {
  RB200_ENTER_INITED();
  if (nv <= 0 || ne < 0 || !poses || (ne > 0 && (!ij || !meas || !info)) || !(huber_delta > 0)) {
    set_error("posegraph_chi2: bad arguments");
    return RGBDSLAM_B200_ERR_ARG;
  }
  return posegraph_chi2(nv, poses, ne, ij, meas, info, huber_delta, chi2, per_edge_chi2);
}

int rgbdslam_b200_landmark_ba(int n_cams, double* poses7, const uint8_t* fixed, int n_points, double* points3, int n_obs,
                              const int32_t* obs_cam, const int32_t* obs_point, const double* obs_uvd, const double* obs_info3,
                              const double* K4, int n_edges, const int32_t* ij, const double* meas7, const double* info36,
                              int iterations, double huber_delta, double* chi2_before, double* chi2_after, int* lm_iterations,
                              int* pcg_iterations) {
  RB200_ENTER_INITED();
  if (n_cams <= 0 || n_points < 0 || n_obs < 0 || n_edges < 0 || iterations < 0 || !poses7 || !fixed || !K4 ||
      (n_points > 0 && !points3) || (n_obs > 0 && (!obs_cam || !obs_point || !obs_uvd || !obs_info3)) ||
      (n_edges > 0 && (!ij || !meas7 || !info36)) || !(huber_delta > 0)) {
    set_error("landmark_ba: bad arguments");
    return RGBDSLAM_B200_ERR_ARG;
  }
  for (size_t k = 0; k < (size_t)n_obs * 3; k++)
    if (!std::isfinite(obs_info3[k]) || !std::isfinite(obs_uvd[k])) {
      set_error("landmark_ba: non-finite observation or information entry");
      return RGBDSLAM_B200_ERR_ARG;
    }
  for (size_t k = 0; k < (size_t)n_edges * 36; k++)
    if (!std::isfinite(info36[k])) {
      set_error("landmark_ba: non-finite entry in an information matrix");
      return RGBDSLAM_B200_ERR_ARG;
    }
  return landmark_ba(n_cams, poses7, fixed, n_points, points3, n_obs, obs_cam, obs_point, obs_uvd, obs_info3, K4, n_edges, ij, meas7,
                     info36, iterations, huber_delta, chi2_before, chi2_after, lm_iterations, pcg_iterations);
}

// ---- host glue: MatchingResults of an offline candidate list -> vertices and edges --------------------------------
namespace {
inline void qmul(const double* a, const double* b, double* o) {  // (x y z w)
  const double ax = a[0], ay = a[1], az = a[2], aw = a[3], bx = b[0], by = b[1], bz = b[2], bw = b[3];
  o[0] = aw * bx + ax * bw + ay * bz - az * by;
  o[1] = aw * by - ax * bz + ay * bw + az * bx;
  o[2] = aw * bz + ax * by - ay * bx + az * bw;
  o[3] = aw * bw - ax * bx - ay * by - az * bz;
}
inline void pose_compose(const double* a, const double* b, double* o) {  // a * b, 7-vectors (t, q): VertexSE3 estimate = v1 * T
  const double qv[4] = {b[0], b[1], b[2], 0.0}, qc[4] = {-a[3], -a[4], -a[5], a[6]};
  double t1[4], t2[4], q[4];
  qmul(a + 3, qv, t1);
  qmul(t1, qc, t2);
  qmul(a + 3, b + 3, q);
  o[0] = a[0] + t2[0]; o[1] = a[1] + t2[1]; o[2] = a[2] + t2[2];
  o[3] = q[0]; o[4] = q[1]; o[5] = q[2]; o[6] = q[3];
}
inline void mat_to_pose7(const float* Tcm, double* z) {  // column-major Matrix4f -> (t, Eigen::Quaterniond(R) normalised)
  double R[3][3];
  for (int r = 0; r < 3; r++)
    for (int c = 0; c < 3; c++) R[r][c] = (double)Tcm[4 * c + r];
  z[0] = (double)Tcm[12]; z[1] = (double)Tcm[13]; z[2] = (double)Tcm[14];
  double q[4];
  const double tr = R[0][0] + R[1][1] + R[2][2];
  if (tr > 0) {
    const double s = std::sqrt(tr + 1.0) * 2;
    q[0] = (R[2][1] - R[1][2]) / s; q[1] = (R[0][2] - R[2][0]) / s; q[2] = (R[1][0] - R[0][1]) / s; q[3] = 0.25 * s;
  } else {
    int i = 0;
    if (R[1][1] > R[0][0]) i = 1;
    if (R[2][2] > R[i][i]) i = 2;
    const int j = (i + 1) % 3, k = (i + 2) % 3;
    const double s = std::sqrt(R[i][i] - R[j][j] - R[k][k] + 1.0) * 2;
    q[i] = 0.25 * s;
    q[j] = (R[j][i] + R[i][j]) / s;
    q[k] = (R[k][i] + R[i][k]) / s;
    q[3] = (R[k][j] - R[j][k]) / s;
  }
  const double n = std::sqrt(q[0] * q[0] + q[1] * q[1] + q[2] * q[2] + q[3] * q[3]);
  for (int a = 0; a < 4; a++) z[3 + a] = q[a] / n;
}
}  // namespace

int rgbdslam_b200_graph_from_pairs(int n_frames, int n_pairs, const int32_t* pairs, const rgbdslam_b200_pair_result* results,
                                   double const_edge_dt, double* poses7, uint8_t* fixed, int32_t* ij, double* meas7, double* info36,
                                   int* n_edges, int* n_const_edges) {
  if (n_frames < 1 || n_pairs < 0 || (n_pairs > 0 && (!pairs || !results)) || !poses7 || !fixed || !ij || !meas7 || !info36 ||
      !n_edges || !(const_edge_dt > 0.0)) {
    set_error("graph_from_pairs: bad arguments");
    return RGBDSLAM_B200_ERR_ARG;
  }
  for (int k = 0; k < n_frames; k++) {
    for (int a = 0; a < 6; a++) poses7[7 * k + a] = 0.0;
    poses7[7 * k + 6] = 1.0;
    fixed[k] = k == 0 ? 1 : 0;  // pose_relative_to = first (graph_manager.cpp:933-936)
  }
  const double ident[7] = {0, 0, 0, 0, 0, 0, 1};
  int ne = 0, nconst = 0, p = 0;
  auto add_edge = [&](int from, int to, const double* z, double scale) {
    ij[2 * ne] = from;
    ij[2 * ne + 1] = to;
    for (int a = 0; a < 7; a++) meas7[7 * (size_t)ne + a] = z[a];
    for (int a = 0; a < 36; a++) info36[36 * (size_t)ne + a] = (a % 7 == 0) ? scale : 0.0;
    ne++;
  };
  for (int k = 1; k < n_frames; k++) {
    while (p < n_pairs && pairs[2 * p] < k) {
      if (pairs[2 * p] < 1) { p++; continue; }
      set_error("graph_from_pairs: pairs must be grouped by ascending newer frame");
      return RGBDSLAM_B200_ERR_ARG;
    }
    int best_inl = 0;
    bool have_vertex = false, pred = false;
    for (; p < n_pairs && pairs[2 * p] == k; p++) {
      const int older = pairs[2 * p + 1];
      const rgbdslam_b200_pair_result& r = results[p];
      if (older < 0 || older >= k) {
        set_error("graph_from_pairs: the older frame of a pair must precede the newer one");
        return RGBDSLAM_B200_ERR_ARG;
      }
      if (r.id1 < 0) continue;  // no transformation (node.cpp:1420)
      double z[7];
      mat_to_pose7(r.ransac_trafo, z);  // edge.transform = final_trafo.cast<double>() (node.cpp:1339)
      if (!have_vertex || r.n_inliers > best_inl) {  // addEdgeToG2O: new vertex = v1 * T, setEstimate when more inliers (:858, :566)
        pose_compose(poses7 + 7 * (size_t)older, z, poses7 + 7 * (size_t)k);
        have_vertex = true;
      }
      if (r.n_inliers > best_inl) best_inl = r.n_inliers;
      add_edge(older, k, z, r.info_scale);  // informationMatrix = I6 * n_inliers / rmse^2 (node.cpp:1335)
      if (older == k - 1) pred = true;
    }
    if (!pred) {  // constant position assumption (graph_manager.cpp:636-655): identity, information I / dt, set_estimate = true
      pose_compose(poses7 + 7 * (size_t)(k - 1), ident, poses7 + 7 * (size_t)k);
      add_edge(k - 1, k, ident, 1.0 / const_edge_dt);
      nconst++;
    }
  }
  *n_edges = ne;
  if (n_const_edges) *n_const_edges = nconst;
  return 0;
}

}  // extern "C"
