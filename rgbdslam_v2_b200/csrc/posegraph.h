// posegraph.h -- host side of the two back-end solvers: the pose-graph optimiser (posegraph.cu) and the landmark bundle
// adjustment (landmark_ba.cu), and the parts they share: the pose-edge module and the Levenberg-Marquardt driver.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include <cfloat>
#include <cmath>
#include <vector>

#include "state.h"

namespace rb200 {
// poses nv x 7 (t, q) in/out; returns 0 or an RGBDSLAM_B200_ERR_* code.
int posegraph_optimize(int nv, double* poses, const uint8_t* fixed, int ne, const int32_t* ij, const double* meas,
                       const double* info, double stop, double huber_delta, double* chi2_out, int* iters_out, int* cg_iters_out);
// chi2 (plain) of the poses and optionally the per-edge chi2 (ne doubles)
int posegraph_chi2(int nv, const double* poses, int ne, const int32_t* ij, const double* meas, const double* info,
                   double huber_delta, double* chi2_out, double* per_edge_chi2);
void posegraph_release();
int posegraph_reserve(int nv, int ne);  // pre-size the cached device buffers
int landmark_ba(int n_cams, double* poses7, const uint8_t* fixed, int n_points, double* points3, int n_obs, const int32_t* obs_cam,
                const int32_t* obs_point, const double* obs_uvd, const double* obs_info3, const double K4[4], int n_edges,
                const int32_t* ij, const double* meas7, const double* info36, int iterations, double huber_delta, double* chi2_before,
                double* chi2_after, int* lm_iterations, int* pcg_iterations);
int landmark_ba_release();  // frees the cached solver buffers (rgbdslam_b200_shutdown)

// Device copy of one set of EdgeSE3 constraints with the Huber kernel (grow-only buffers).  blk: per-edge normal-equation
// blocks (layout in se3_graph.cuh).  off / inc / oth: CSR of the incident edges of every vertex in edge order, inc = edge << 1 |
// role, oth = the vertex at the other end; h_off is its host copy.  The functions return 0 or an RGBDSLAM_B200_ERR_* code and
// count their kernel launches in `launches`.
struct PoseEdges {
  int ne = 0;
  double delta = 1.0;
  DevBuf ij, meas, info, off, inc, oth, blk;
  std::vector<int> h_off, h_inc, h_oth;
  ~PoseEdges() {
    for (DevBuf* b : {&ij, &meas, &info, &off, &inc, &oth, &blk}) b->release();
  }
  int ensure(int nv, int n_edges);
  // ERR_ARG (with last_error) before any device work unless 0 <= ij < nv; then queues the copies of the edges and, with
  // `incidence`, of the CSR
  int upload(int nv, int n_edges, const int32_t* h_ij, const double* h_meas, const double* h_info, double huber_delta, bool incidence,
             cudaStream_t st);
  int linearize(const double* x, cudaStream_t st, int64_t& launches);  // blk at the poses x
  // (robust, plain) chi2 partial sums of chi2_blocks() blocks of 256 edges into part; per_edge (ne doubles) may be null
  int chi2(const double* x, double* part, double* per_edge, cudaStream_t st, int64_t& launches) const;
  int chi2_blocks() const { return (ne + 255) / 256; }
};

// xout = xin * fromVectorMQT(dlt) for every vertex that is not fixed (VertexSE3::oplusImpl)
cudaError_t pg_launch_update(int nv, const double* xin, const double* dlt, const uint8_t* fixed, double* xout, cudaStream_t st);

// SparseOptimizer::optimize(iterations) with OptimizationAlgorithmLevenberg::solve.  The solver supplies
//   linearize(chi2, maxdiag): linearise at the current estimate; may re-evaluate its chi2 (computeActiveErrors); maxdiag is
//       non-null on the first iteration and receives max diag(H)
//   trial(lambda, chi2, scale, ok): solve with damping lambda, the trial estimate's chi2, computeScale, PCG did not break down
//   accept(): the trial estimate becomes the current one
// Each returns 0 or an error code, as does lm_optimize; *done = LM iterations run.
template <class Linearize, class Trial, class Accept>
int lm_optimize(int iterations, double& chi2, int* done, Linearize&& linearize, Trial&& trial, Accept&& accept) {
  double lambda = 0, ni = 2;
  *done = 0;
  for (int i = 0; i < iterations; i++) {
    double maxdiag = 0;
    if (int rc = linearize(chi2, i == 0 ? &maxdiag : nullptr)) return rc;
    if (i == 0) lambda = 1e-5 * maxdiag;  // computeLambdaInit: tau * max diag(H)
    double rho = 0;
    int qmax = 0;
    do {
      double temp, scale;
      bool ok;
      if (int rc = trial(lambda, temp, scale, ok)) return rc;
      if (!ok) temp = DBL_MAX;
      rho = (chi2 - temp) / (scale + 1e-3);
      if (rho > 0 && std::isfinite(temp)) {
        double alpha = 1. - std::pow(2 * rho - 1, 3);
        alpha = std::fmin(alpha, 2. / 3.);
        lambda *= std::fmax(1. / 3., alpha);
        ni = 2;
        chi2 = temp;
        accept();  // discardTop
      } else {
        lambda *= ni;  // pop
        ni *= 2;
        if (!std::isfinite(lambda)) break;
      }
      qmax++;
    } while (rho < 0 && qmax < 10);
    ++*done;
    if (qmax == 10 || rho == 0) break;  // Terminate
  }
  return 0;
}
}  // namespace rb200
