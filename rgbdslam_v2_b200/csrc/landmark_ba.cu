// landmark_ba.cu -- bundle adjustment over camera poses and 3-D landmarks with the landmarks marginalised (SURVEY.md 8f rank 4).
//
// What the reference builds with DO_FEATURE_OPTIMIZATION (src/landmark.cpp:97-187; optimised by optimizeGraphImpl's
// `optimize_landmarks` branch, src/graph_manager.cpp:963-967):
//   VertexSE3 cameras  +  VertexPointXYZ landmarks (initialised from their first observation, landmark.cpp:97-128)
//   one EdgeSE3PointXYZDepth per observation: error (fx x/z + cx - u, fy y/z + cy - v, z - depth) of the landmark in the camera
//   frame, information point_information_matrix(depth) = diag(1, 1, 1 / depth_covariance(depth)) (misc2.h:37-47), no robust
//   kernel (landmark.cpp:176 is commented out);  plus the camera-camera EdgeSE3 constraints with the shared Huber kernel.
// The reference leaves the point vertices in the linear system (it never calls setMarginalized, SURVEY 8a-a20) and hands the
// full (6 Ncam + 3 Npoint) system to CSparse.  Here every Levenberg-Marquardt step eliminates the 3x3 point blocks:
//   S = Hcc - Hcp Hpp^-1 Hpc,   g = bc - Hcp Hpp^-1 bp,   S dc = g,   dp = Hpp^-1 (bp - Hpc dc)
// -- the same normal equations, hence the same step and the same optimum.  S is never formed: the block-Jacobi PCG applies it
// matrix-free (per point: u = Hpp^-1 sum Hpc d; per camera: q = Hcc d + sum pose-edge blocks - sum Hcp u), two gather kernels
// and one single-CTA update kernel per iteration, all reductions in a fixed order (deterministic).
// The pose edges are the pose-graph solver's module (PoseEdges), the LM bookkeeping its driver (lm_optimize, posegraph.h).
// float64 throughout.  Oracles: oracle/landmark_oracle.py (dense solve of the FULL system), tests/ba_exact.py (float64
// restatement of every step at multi-CTA shapes).
#include <cuda_runtime.h>

#include <vector>

#include "posegraph.h"
#include "se3_graph.cuh"
#include "se3_point.cuh"
#include "state.h"

namespace rb200 {

// per observation: [Hcc 36 | Hcp 18 | Hpp 9 | bc 6 | bp 3] with b = -J' W e  (H delta = b)
constexpr int kObsBlk = 72;
constexpr int kOHcc = 0, kOHcp = 36, kOHpp = 54, kObc = 63, kObp = 69;

__device__ __forceinline__ void cam_from_pose(const double* p, Cam& c) {
  quat_to_R(p + 3, c.R);
  c.t[0] = p[0]; c.t[1] = p[1]; c.t[2] = p[2];
}

__global__ void __launch_bounds__(128) ba_linearize_kernel(int n_obs, const double* __restrict__ poses, const double* __restrict__ points,
                                                           const int* __restrict__ obs_cam, const int* __restrict__ obs_pt,
                                                           const double* __restrict__ uvd, const double* __restrict__ w3, double fx,
                                                           double fy, double cx, double cy, double* __restrict__ blk) {
  const int o = blockIdx.x * blockDim.x + threadIdx.x;
  if (o >= n_obs) return;
  Cam c;
  cam_from_pose(poses + 7 * (size_t)obs_cam[o], c);
  const double* pw = points + 3 * (size_t)obs_pt[o];
  const double m[3] = {uvd[3 * (size_t)o], uvd[3 * (size_t)o + 1], uvd[3 * (size_t)o + 2]};
  const double w[3] = {w3[3 * (size_t)o], w3[3 * (size_t)o + 1], w3[3 * (size_t)o + 2]};
  double e[3], Jc[18], Jp[9];
  edge_depth(c, pw, m, e, Jc, Jp, fx, fy, cx, cy);
  double* out = blk + (size_t)o * kObsBlk;
  for (int i = 0; i < 6; i++) {
    double b = 0;
    for (int r = 0; r < 3; r++) b -= Jc[6 * r + i] * w[r] * e[r];
    out[kObc + i] = b;
    for (int j = 0; j < 6; j++) {
      double h = 0;
      for (int r = 0; r < 3; r++) h += Jc[6 * r + i] * w[r] * Jc[6 * r + j];
      out[kOHcc + 6 * i + j] = h;
    }
    for (int j = 0; j < 3; j++) {
      double h = 0;
      for (int r = 0; r < 3; r++) h += Jc[6 * r + i] * w[r] * Jp[3 * r + j];
      out[kOHcp + 3 * i + j] = h;
    }
  }
  for (int i = 0; i < 3; i++) {
    double b = 0;
    for (int r = 0; r < 3; r++) b -= Jp[3 * r + i] * w[r] * e[r];
    out[kObp + i] = b;
    for (int j = 0; j < 3; j++) {
      double h = 0;
      for (int r = 0; r < 3; r++) h += Jp[3 * r + i] * w[r] * Jp[3 * r + j];
      out[kOHpp + 3 * i + j] = h;
    }
  }
}

// chi2 of the observations (no robust kernel): per-block partial sums
__global__ void __launch_bounds__(256) ba_chi2_obs_kernel(int n_obs, const double* __restrict__ poses, const double* __restrict__ points,
                                                          const int* __restrict__ obs_cam, const int* __restrict__ obs_pt,
                                                          const double* __restrict__ uvd, const double* __restrict__ w3, double fx,
                                                          double fy, double cx, double cy, double* __restrict__ part) {
  const int o = blockIdx.x * blockDim.x + threadIdx.x;
  double v = 0;
  if (o < n_obs) {
    Cam c;
    cam_from_pose(poses + 7 * (size_t)obs_cam[o], c);
    const double* pw = points + 3 * (size_t)obs_pt[o];
    const double d0 = pw[0] - c.t[0], d1 = pw[1] - c.t[1], d2 = pw[2] - c.t[2];
    const double x = c.R[0] * d0 + c.R[3] * d1 + c.R[6] * d2, y = c.R[1] * d0 + c.R[4] * d1 + c.R[7] * d2,
                 z = c.R[2] * d0 + c.R[5] * d1 + c.R[8] * d2;
    // same expression as edge_depth: (fx x + cx z) / z - u
    const double e0 = (fx * x + cx * z) / z - uvd[3 * (size_t)o], e1 = (fy * y + cy * z) / z - uvd[3 * (size_t)o + 1],
                 e2 = z - uvd[3 * (size_t)o + 2];
    v = e0 * e0 * w3[3 * (size_t)o] + e1 * e1 * w3[3 * (size_t)o + 1] + e2 * e2 * w3[3 * (size_t)o + 2];
  }
  __shared__ double sm[256];
  sm[threadIdx.x] = v;
  __syncthreads();
  for (int s = 128; s > 0; s >>= 1) {
    if (threadIdx.x < s) sm[threadIdx.x] += sm[threadIdx.x + s];
    __syncthreads();
  }
  if (threadIdx.x == 0) part[blockIdx.x] = sm[0];
}

// per point: Hpp = sum + lambda I -> inverse; bp = sum; max diagonal (undamped) per block
__global__ void __launch_bounds__(128) ba_points_kernel(int n_points, const int* __restrict__ pt_off, const int* __restrict__ pt_obs,
                                                        const double* __restrict__ blk, double lambda, double* __restrict__ Hppinv,
                                                        double* __restrict__ bp, double* __restrict__ maxdiag_part) {
  const int p = blockIdx.x * blockDim.x + threadIdx.x;
  double md = 0;
  if (p < n_points) {
    double H[9] = {0, 0, 0, 0, 0, 0, 0, 0, 0}, b[3] = {0, 0, 0};
    for (int q = pt_off[p]; q < pt_off[p + 1]; q++) {
      const double* o = blk + (size_t)pt_obs[q] * kObsBlk;
      for (int i = 0; i < 9; i++) H[i] += o[kOHpp + i];
      for (int i = 0; i < 3; i++) b[i] += o[kObp + i];
    }
    md = fmax(H[0], fmax(H[4], H[8]));
    H[0] += lambda; H[4] += lambda; H[8] += lambda;
    double inv[9];
    const bool ok = pt_off[p + 1] > pt_off[p] && inv3_sym(H, inv);
    for (int i = 0; i < 9; i++) Hppinv[9 * (size_t)p + i] = ok ? inv[i] : 0.0;
    for (int i = 0; i < 3; i++) bp[3 * (size_t)p + i] = ok ? b[i] : 0.0;
  }
  __shared__ double sm[128];
  sm[threadIdx.x] = md;
  __syncthreads();
  for (int s = 64; s > 0; s >>= 1) {
    if (threadIdx.x < s) sm[threadIdx.x] = fmax(sm[threadIdx.x], sm[threadIdx.x + s]);
    __syncthreads();
  }
  if (threadIdx.x == 0) maxdiag_part[blockIdx.x] = sm[0];
}

// per camera (one warp): Hcc (+ pose-edge diagonal blocks + lambda I), bc, the reduced right-hand side g and the block-Jacobi
// preconditioner (Hcc - sum Hcp Hpp^-1 Hpc)^-1
__global__ void __launch_bounds__(256) ba_cams_kernel(int n_cams, const int* __restrict__ cam_off, const int* __restrict__ cam_obs,
                                                      const int* __restrict__ obs_pt, const double* __restrict__ blk,
                                                      const int* __restrict__ e_off, const int* __restrict__ e_inc,
                                                      const double* __restrict__ eblk, const uint8_t* __restrict__ fixed, double lambda,
                                                      const double* __restrict__ Hppinv, const double* __restrict__ bp,
                                                      double* __restrict__ Hcc, double* __restrict__ bc, double* __restrict__ g,
                                                      double* __restrict__ Minv, double* __restrict__ maxdiag) {
  const int c = blockIdx.x * 8 + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (c >= n_cams) return;
  double H[36], b[6], S[36], gg[6];
#pragma unroll
  for (int i = 0; i < 36; i++) { H[i] = 0; S[i] = 0; }
#pragma unroll
  for (int i = 0; i < 6; i++) { b[i] = 0; gg[i] = 0; }
  for (int q = cam_off[c] + lane; q < cam_off[c + 1]; q += 32) {
    const int o = cam_obs[q];
    const double* ob = blk + (size_t)o * kObsBlk;
    const double* inv = Hppinv + 9 * (size_t)obs_pt[o];
    const double* bpp = bp + 3 * (size_t)obs_pt[o];
    double Y[18];  // Hcp Hpp^-1
#pragma unroll
    for (int r = 0; r < 6; r++)
#pragma unroll
      for (int k = 0; k < 3; k++) Y[3 * r + k] = ob[kOHcp + 3 * r] * inv[k] + ob[kOHcp + 3 * r + 1] * inv[3 + k] + ob[kOHcp + 3 * r + 2] * inv[6 + k];
#pragma unroll
    for (int r = 0; r < 6; r++) {
      b[r] += ob[kObc + r];
      gg[r] -= Y[3 * r] * bpp[0] + Y[3 * r + 1] * bpp[1] + Y[3 * r + 2] * bpp[2];
#pragma unroll
      for (int k = 0; k < 6; k++) {
        H[6 * r + k] += ob[kOHcc + 6 * r + k];
        S[6 * r + k] -= Y[3 * r] * ob[kOHcp + 3 * k] + Y[3 * r + 1] * ob[kOHcp + 3 * k + 1] + Y[3 * r + 2] * ob[kOHcp + 3 * k + 2];
      }
    }
  }
  if (e_off) {
    for (int q = e_off[c] + lane; q < e_off[c + 1]; q += 32) {
      const int code = e_inc[q];
      const double* eb = edge_blocks(eblk, code >> 1);
#pragma unroll
      for (int i = 0; i < 36; i++) H[i] += eb[edge_diag(code & 1) + i];
#pragma unroll
      for (int i = 0; i < 6; i++) b[i] -= eb[edge_grad(code & 1) + i];
    }
  }
#pragma unroll
  for (int i = 0; i < 36; i++) { H[i] = warp_sum_d(H[i]); S[i] = warp_sum_d(S[i]); }
#pragma unroll
  for (int i = 0; i < 6; i++) { b[i] = warp_sum_d(b[i]); gg[i] = warp_sum_d(gg[i]); }
  if (lane == 0) {
    const bool fx = fixed[c] != 0;
    double md = 0;
    for (int k = 0; k < 6; k++) md = fmax(md, H[7 * k]);
    maxdiag[c] = fx ? 0.0 : md;
    for (int k = 0; k < 6; k++) H[7 * k] += lambda;
    double A[36], Ai[36];
    for (int i = 0; i < 36; i++) {
      Hcc[36 * (size_t)c + i] = H[i];
      A[i] = H[i] + S[i];
    }
    const bool ok = !fx && inv6(A, Ai);
    for (int i = 0; i < 36; i++) Minv[36 * (size_t)c + i] = ok ? Ai[i] : 0.0;
    for (int i = 0; i < 6; i++) {
      bc[6 * (size_t)c + i] = fx ? 0.0 : b[i];
      g[6 * (size_t)c + i] = fx ? 0.0 : b[i] + gg[i];
    }
  }
}

// u_p = Hpp^-1 sum_o Hcp_o' d_cam(o)
__global__ void __launch_bounds__(128) ba_pt_gather_kernel(int n_points, const int* __restrict__ pt_off, const int* __restrict__ pt_obs,
                                                           const int* __restrict__ obs_cam, const double* __restrict__ blk,
                                                           const double* __restrict__ Hppinv, const double* __restrict__ d,
                                                           double* __restrict__ u) {
  const int p = blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= n_points) return;
  double t[3] = {0, 0, 0};
  for (int q = pt_off[p]; q < pt_off[p + 1]; q++) {
    const int o = pt_obs[q];
    const double* hcp = blk + (size_t)o * kObsBlk + kOHcp;
    const double* dc = d + 6 * (size_t)obs_cam[o];
#pragma unroll
    for (int r = 0; r < 6; r++) {
      t[0] += hcp[3 * r] * dc[r];
      t[1] += hcp[3 * r + 1] * dc[r];
      t[2] += hcp[3 * r + 2] * dc[r];
    }
  }
  const double* inv = Hppinv + 9 * (size_t)p;
  for (int k = 0; k < 3; k++) u[3 * (size_t)p + k] = inv[3 * k] * t[0] + inv[3 * k + 1] * t[1] + inv[3 * k + 2] * t[2];
}

// q_c = Hcc d_c + sum pose-edge off-diagonal blocks - sum_o Hcp_o u_point(o)   (one warp per camera); block partials of d.q
__global__ void __launch_bounds__(256) ba_cam_apply_kernel(int n_cams, const int* __restrict__ cam_off, const int* __restrict__ cam_obs,
                                                           const int* __restrict__ obs_pt, const double* __restrict__ blk,
                                                           const int* __restrict__ e_off, const int* __restrict__ e_inc,
                                                           const int* __restrict__ e_oth, const double* __restrict__ eblk,
                                                           const uint8_t* __restrict__ fixed, const double* __restrict__ Hcc,
                                                           const double* __restrict__ d, const double* __restrict__ u,
                                                           double* __restrict__ qv, double* __restrict__ part) {
  const int c = blockIdx.x * 8 + (threadIdx.x >> 5), lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  double acc[6] = {0, 0, 0, 0, 0, 0};
  double dq = 0;
  const bool act = c < n_cams && !fixed[c < n_cams ? c : 0];
  if (act) {
    for (int q = cam_off[c] + lane; q < cam_off[c + 1]; q += 32) {
      const int o = cam_obs[q];
      const double* hcp = blk + (size_t)o * kObsBlk + kOHcp;
      const double* up = u + 3 * (size_t)obs_pt[o];
#pragma unroll
      for (int r = 0; r < 6; r++) acc[r] -= hcp[3 * r] * up[0] + hcp[3 * r + 1] * up[1] + hcp[3 * r + 2] * up[2];
    }
    if (e_off) {
      for (int q = e_off[c] + lane; q < e_off[c + 1]; q += 32) {
        const int code = e_inc[q], other = e_oth[q];
        if (other == c) continue;
        const double* C = edge_blocks(eblk, code >> 1) + kEdgeC;
        const double* ov = d + 6 * (size_t)other;
        if ((code & 1) == 0) {
#pragma unroll
          for (int r = 0; r < 6; r++)
#pragma unroll
            for (int k = 0; k < 6; k++) acc[r] += C[6 * r + k] * ov[k];
        } else {
#pragma unroll
          for (int r = 0; r < 6; r++)
#pragma unroll
            for (int k = 0; k < 6; k++) acc[k] += C[6 * r + k] * ov[r];
        }
      }
    }
  }
#pragma unroll
  for (int r = 0; r < 6; r++) acc[r] = warp_sum_d(acc[r]);
  if (c < n_cams && lane < 6) {
    double s = 0;
    if (act) {
      const double* H = Hcc + 36 * (size_t)c + 6 * lane;
      const double* dc = d + 6 * (size_t)c;
#pragma unroll
      for (int k = 0; k < 6; k++) s += H[k] * dc[k];
      double t = 0;
#pragma unroll
      for (int r = 0; r < 6; r++) t = (r == lane) ? acc[r] : t;
      s += t;
      dq = s * dc[lane];
    }
    qv[6 * (size_t)c + lane] = s;
  }
  dq = warp_sum_d(dq);
  __shared__ double sm[8];
  if (lane == 0) sm[w] = dq;
  __syncthreads();
  if (threadIdx.x == 0) {
    double t = 0;
    for (int i = 0; i < 8; i++) t += sm[i];
    part[blockIdx.x] = t;
  }
}

// PCG state on the device: [0] dn = r'M^-1 r, [1] iterations, [2] status (0 running, 1 converged, 2 breakdown), [3] tolerance
// One CTA: mode 0 = initialise (x = 0, r = g, d = s = M^-1 r), mode 1 = one update after q = S d.
__global__ void __launch_bounds__(1024) ba_cg_step_kernel(int mode, int n_cams, int nparts, const double* __restrict__ part,
                                                          const double* __restrict__ g, const double* __restrict__ Minv,
                                                          const double* __restrict__ qv, double* __restrict__ x, double* __restrict__ r,
                                                          double* __restrict__ d, double* __restrict__ state, double rel_tol) {
  __shared__ double sm[32];
  __shared__ double s_val;
  const int n = 6 * n_cams;
  auto block_sum = [&](double v) -> double {
    v = warp_sum_d(v);
    __syncthreads();
    if ((threadIdx.x & 31) == 0) sm[threadIdx.x >> 5] = v;
    __syncthreads();
    if (threadIdx.x == 0) {
      double t = 0;
      for (int i = 0; i < 32; i++) t += sm[i];
      s_val = t;
    }
    __syncthreads();
    return s_val;
  };
  if (mode == 1 && state[2] != 0.0) return;  // finished: further launches of the fixed-length host loop are no-ops
  // dn of the previous step, read once before any barrier: thread 0 overwrites state[0] at the end of this launch, and a warp
  // still computing beta after that write would otherwise see the new value
  const double dn_old = mode == 1 ? state[0] : 0.0;
  double alpha = 0;
  if (mode == 1) {
    double t = 0;
    for (int i = threadIdx.x; i < nparts; i += blockDim.x) t += part[i];
    const double dq = block_sum(t);
    if (!(dq > 0)) {
      if (threadIdx.x == 0) state[2] = 2.0;
      return;
    }
    alpha = dn_old / dq;
  }
  double loc = 0;
  for (int i = threadIdx.x; i < n; i += blockDim.x) {
    double ri;
    if (mode == 0) {
      x[i] = 0.0;
      ri = g[i];
    } else {
      x[i] += alpha * d[i];
      ri = r[i] - alpha * qv[i];
    }
    r[i] = ri;
  }
  __syncthreads();
  // s = M^-1 r (block rows), dn_new = r.s ; kept in qv's place? no: computed on the fly twice (cheap) to avoid another vector
  for (int i = threadIdx.x; i < n; i += blockDim.x) {
    const int c = i / 6, rr = i % 6;
    double s = 0;
#pragma unroll
    for (int k = 0; k < 6; k++) s += Minv[36 * (size_t)c + 6 * rr + k] * r[6 * (size_t)c + k];
    loc += r[i] * s;
  }
  const double dn_new = block_sum(loc);
  const double beta = mode == 0 ? 0.0 : dn_new / dn_old;
  for (int i = threadIdx.x; i < n; i += blockDim.x) {
    const int c = i / 6, rr = i % 6;
    double s = 0;
#pragma unroll
    for (int k = 0; k < 6; k++) s += Minv[36 * (size_t)c + 6 * rr + k] * r[6 * (size_t)c + k];
    d[i] = s + beta * (mode == 0 ? 0.0 : d[i]);
  }
  if (threadIdx.x == 0) {
    if (mode == 0) {
      state[1] = 0.0;
      state[3] = dn_new * rel_tol;
      state[2] = dn_new <= 0.0 ? 1.0 : 0.0;
    } else {
      state[1] += 1.0;
      if (dn_new <= state[3]) state[2] = 1.0;
    }
    state[0] = dn_new;
  }
}

// dp = Hpp^-1 (bp - sum Hpc dc); trial points; partial sums of the LM scale  dp.(lambda dp + bp)
__global__ void __launch_bounds__(128) ba_pt_update_kernel(int n_points, const int* __restrict__ pt_off, const int* __restrict__ pt_obs,
                                                           const int* __restrict__ obs_cam, const double* __restrict__ blk,
                                                           const double* __restrict__ Hppinv, const double* __restrict__ bp,
                                                           const double* __restrict__ dxc, double lambda, const double* __restrict__ pts,
                                                           double* __restrict__ pts_trial, double* __restrict__ part) {
  const int p = blockIdx.x * blockDim.x + threadIdx.x;
  double sc = 0;
  if (p < n_points) {
    double t[3] = {bp[3 * (size_t)p], bp[3 * (size_t)p + 1], bp[3 * (size_t)p + 2]};
    for (int q = pt_off[p]; q < pt_off[p + 1]; q++) {
      const int o = pt_obs[q];
      const double* hcp = blk + (size_t)o * kObsBlk + kOHcp;
      const double* dc = dxc + 6 * (size_t)obs_cam[o];
#pragma unroll
      for (int r = 0; r < 6; r++) {
        t[0] -= hcp[3 * r] * dc[r];
        t[1] -= hcp[3 * r + 1] * dc[r];
        t[2] -= hcp[3 * r + 2] * dc[r];
      }
    }
    const double* inv = Hppinv + 9 * (size_t)p;
    for (int k = 0; k < 3; k++) {
      const double dp = inv[3 * k] * t[0] + inv[3 * k + 1] * t[1] + inv[3 * k + 2] * t[2];
      pts_trial[3 * (size_t)p + k] = pts[3 * (size_t)p + k] + dp;
      sc += dp * (lambda * dp + bp[3 * (size_t)p + k]);
    }
  }
  __shared__ double sm[128];
  sm[threadIdx.x] = sc;
  __syncthreads();
  for (int s = 64; s > 0; s >>= 1) {
    if (threadIdx.x < s) sm[threadIdx.x] += sm[threadIdx.x + s];
    __syncthreads();
  }
  if (threadIdx.x == 0) part[blockIdx.x] = sm[0];
}

// ================================================================================================
struct BaDevice {
  PoseEdges edges;  // the camera-camera constraints
  DevBuf poses, poses_trial, pts, pts_trial, fixed, obs_cam, obs_pt, uvd, w3, pt_off, pt_obs, cam_off, cam_obs, blk, Hppinv, bp, Hcc, bc, g,
      Minv, maxd_c, maxd_p, x, r, d, q, u, part, state, chipart, scpart;
  ~BaDevice() {
    DevBuf* all[] = {&poses, &poses_trial, &pts, &pts_trial, &fixed, &obs_cam, &obs_pt, &uvd, &w3, &pt_off, &pt_obs, &cam_off, &cam_obs, &blk,
                     &Hppinv, &bp, &Hcc, &bc, &g, &Minv, &maxd_c, &maxd_p, &x, &r, &d, &q, &u, &part, &state, &chipart, &scpart};
    for (DevBuf* b : all) b->release();
  }
};
static BaDevice* g_ba = nullptr;
int landmark_ba_release() {
  delete g_ba;
  g_ba = nullptr;
  return 0;
}

struct BaProblem {
  int nc, np, no;
  double K[4];
  cudaStream_t st;
  BaDevice* d;
  int64_t launches = 0;
  int pcg_iters = 0;
};

static int ba_chi2(BaProblem& P, const double* poses, const double* pts, double* chi2) {
  BaDevice& d = *P.d;
  const int nb = (P.no + 255) / 256, neb = d.edges.chi2_blocks();
  if (nb > 0) {
    ba_chi2_obs_kernel<<<nb, 256, 0, P.st>>>(P.no, poses, pts, (const int*)d.obs_cam.ptr, (const int*)d.obs_pt.ptr,
                                             (const double*)d.uvd.ptr, (const double*)d.w3.ptr, P.K[0], P.K[1], P.K[2], P.K[3],
                                             (double*)d.chipart.ptr);
    RB200_CUDA(cudaGetLastError());
    P.launches++;
  }
  if (int rc = d.edges.chi2(poses, (double*)d.chipart.ptr + nb, nullptr, P.st, P.launches)) return rc;
  std::vector<double> part(nb + 2 * (size_t)neb);
  RB200_CUDA(cudaMemcpyAsync(part.data(), d.chipart.ptr, sizeof(double) * part.size(), cudaMemcpyDeviceToHost, P.st));
  RB200_CUDA(cudaStreamSynchronize(P.st));
  double s = 0;
  for (int i = 0; i < nb; i++) s += part[i];
  for (int i = 0; i < neb; i++) s += part[nb + 2 * i];  // robust chi2 of the pose edges (activeRobustChi2)
  *chi2 = s;
  return 0;
}

// SparseOptimizer::optimize(iterations); the chi2 of an iteration's start is the one of the trial last accepted
static int ba_optimize(BaProblem& P, int iterations, double& chi2, int* done) {
  BaDevice& d = *P.d;
  const int npb = (P.np + 127) / 128, ncb = (P.nc + 7) / 8;
  const int* e_off = d.edges.ne > 0 ? (const int*)d.edges.off.ptr : nullptr;  // no pose-edge terms in ba_cams / ba_cam_apply
  auto assemble = [&](double lam) -> int {
    if (npb > 0)
      ba_points_kernel<<<npb, 128, 0, P.st>>>(P.np, (const int*)d.pt_off.ptr, (const int*)d.pt_obs.ptr, (const double*)d.blk.ptr, lam,
                                            (double*)d.Hppinv.ptr, (double*)d.bp.ptr, (double*)d.maxd_p.ptr);
    ba_cams_kernel<<<ncb, 256, 0, P.st>>>(P.nc, (const int*)d.cam_off.ptr, (const int*)d.cam_obs.ptr, (const int*)d.obs_pt.ptr,
                                          (const double*)d.blk.ptr, e_off, (const int*)d.edges.inc.ptr, (const double*)d.edges.blk.ptr,
                                          (const uint8_t*)d.fixed.ptr, lam, (const double*)d.Hppinv.ptr, (const double*)d.bp.ptr,
                                          (double*)d.Hcc.ptr, (double*)d.bc.ptr, (double*)d.g.ptr, (double*)d.Minv.ptr,
                                          (double*)d.maxd_c.ptr);
    P.launches += 2;
    RB200_CUDA(cudaGetLastError());
    return 0;
  };
  auto linearize = [&](double&, double* maxdiag) -> int {
    if (P.no > 0)
      ba_linearize_kernel<<<(P.no + 127) / 128, 128, 0, P.st>>>(P.no, (const double*)d.poses.ptr, (const double*)d.pts.ptr,
                                                              (const int*)d.obs_cam.ptr, (const int*)d.obs_pt.ptr, (const double*)d.uvd.ptr,
                                                              (const double*)d.w3.ptr, P.K[0], P.K[1], P.K[2], P.K[3], (double*)d.blk.ptr);
    RB200_CUDA(cudaGetLastError());
    P.launches++;
    if (int rc = d.edges.linearize((const double*)d.poses.ptr, P.st, P.launches)) return rc;
    if (!maxdiag) return 0;
    if (int rc = assemble(0.0)) return rc;
    std::vector<double> mc(P.nc), mp(npb);
    RB200_CUDA(cudaMemcpyAsync(mc.data(), d.maxd_c.ptr, 8 * (size_t)P.nc, cudaMemcpyDeviceToHost, P.st));
    RB200_CUDA(cudaMemcpyAsync(mp.data(), d.maxd_p.ptr, 8 * (size_t)npb, cudaMemcpyDeviceToHost, P.st));
    RB200_CUDA(cudaStreamSynchronize(P.st));
    double m = 0;
    for (double v : mc) m = v > m ? v : m;
    for (double v : mp) m = v > m ? v : m;
    *maxdiag = m;
    return 0;
  };
  auto trial = [&](double lambda, double& temp, double& scale, bool& ok) -> int {
    if (int rc = assemble(lambda)) return rc;
    // ---- PCG on the reduced camera system
    ba_cg_step_kernel<<<1, 1024, 0, P.st>>>(0, P.nc, 0, nullptr, (const double*)d.g.ptr, (const double*)d.Minv.ptr, nullptr, (double*)d.x.ptr,
                                            (double*)d.r.ptr, (double*)d.d.ptr, (double*)d.state.ptr, 1e-18);
    P.launches++;
    const int maxit = 6 * P.nc + 20;
    double st4[4] = {0, 0, 0, 0};
    for (int it = 0; it < maxit;) {
      const int burst = 16;
      for (int k = 0; k < burst; k++) {
        if (npb > 0)
          ba_pt_gather_kernel<<<npb, 128, 0, P.st>>>(P.np, (const int*)d.pt_off.ptr, (const int*)d.pt_obs.ptr, (const int*)d.obs_cam.ptr,
                                                   (const double*)d.blk.ptr, (const double*)d.Hppinv.ptr, (const double*)d.d.ptr,
                                                   (double*)d.u.ptr);
        ba_cam_apply_kernel<<<ncb, 256, 0, P.st>>>(P.nc, (const int*)d.cam_off.ptr, (const int*)d.cam_obs.ptr, (const int*)d.obs_pt.ptr,
                                                   (const double*)d.blk.ptr, e_off, (const int*)d.edges.inc.ptr,
                                                   (const int*)d.edges.oth.ptr, (const double*)d.edges.blk.ptr,
                                                   (const uint8_t*)d.fixed.ptr, (const double*)d.Hcc.ptr, (const double*)d.d.ptr,
                                                   (const double*)d.u.ptr, (double*)d.q.ptr, (double*)d.part.ptr);
        ba_cg_step_kernel<<<1, 1024, 0, P.st>>>(1, P.nc, ncb, (const double*)d.part.ptr, (const double*)d.g.ptr, (const double*)d.Minv.ptr,
                                                (const double*)d.q.ptr, (double*)d.x.ptr, (double*)d.r.ptr, (double*)d.d.ptr,
                                                (double*)d.state.ptr, 1e-18);
        P.launches += 3;
      }
      it += burst;
      RB200_CUDA(cudaMemcpyAsync(st4, d.state.ptr, sizeof(st4), cudaMemcpyDeviceToHost, P.st));
      RB200_CUDA(cudaStreamSynchronize(P.st));
      if (st4[2] != 0.0) break;
    }
    P.pcg_iters += (int)st4[1];
    ok = st4[2] != 2.0;
    // ---- back-substitution, trial update, gain ratio
    if (npb > 0)
      ba_pt_update_kernel<<<npb, 128, 0, P.st>>>(P.np, (const int*)d.pt_off.ptr, (const int*)d.pt_obs.ptr, (const int*)d.obs_cam.ptr,
                                               (const double*)d.blk.ptr, (const double*)d.Hppinv.ptr, (const double*)d.bp.ptr,
                                               (const double*)d.x.ptr, lambda, (const double*)d.pts.ptr, (double*)d.pts_trial.ptr,
                                               (double*)d.scpart.ptr);
    RB200_CUDA(pg_launch_update(P.nc, (const double*)d.poses.ptr, (const double*)d.x.ptr, (const uint8_t*)d.fixed.ptr,
                                (double*)d.poses_trial.ptr, P.st));
    P.launches += 2;
    std::vector<double> sp(npb), xc(6 * (size_t)P.nc), bcv(6 * (size_t)P.nc);
    RB200_CUDA(cudaMemcpyAsync(sp.data(), d.scpart.ptr, 8 * (size_t)npb, cudaMemcpyDeviceToHost, P.st));
    RB200_CUDA(cudaMemcpyAsync(xc.data(), d.x.ptr, 48 * (size_t)P.nc, cudaMemcpyDeviceToHost, P.st));
    RB200_CUDA(cudaMemcpyAsync(bcv.data(), d.bc.ptr, 48 * (size_t)P.nc, cudaMemcpyDeviceToHost, P.st));
    RB200_CUDA(cudaStreamSynchronize(P.st));
    scale = 0;
    for (double v : sp) scale += v;
    for (size_t i = 0; i < xc.size(); i++) scale += xc[i] * (lambda * xc[i] + bcv[i]);
    return ba_chi2(P, (const double*)d.poses_trial.ptr, (const double*)d.pts_trial.ptr, &temp);
  };
  auto accept = [&] {
    std::swap(d.poses, d.poses_trial);
    std::swap(d.pts, d.pts_trial);
  };
  return lm_optimize(iterations, chi2, done, linearize, trial, accept);
}

int landmark_ba(int n_cams, double* poses7, const uint8_t* fixed, int n_points, double* points3, int n_obs, const int32_t* obs_cam,
                const int32_t* obs_point, const double* obs_uvd, const double* obs_info3, const double K4[4], int n_edges,
                const int32_t* ij, const double* meas7, const double* info36, int iterations, double huber_delta, double* chi2_before,
                double* chi2_after, int* lm_iterations, int* pcg_iterations) {
  State& s = g_state;
  if (!g_ba) g_ba = new BaDevice();
  BaDevice& d = *g_ba;
  BaProblem P;
  P.nc = n_cams; P.np = n_points; P.no = n_obs;
  for (int k = 0; k < 4; k++) P.K[k] = K4[k];
  P.st = s.stream;
  P.d = g_ba;
  // CSR: observations by point and by camera (input order kept inside a row: deterministic sums)
  std::vector<int> pt_off(n_points + 1, 0), cam_off(n_cams + 1, 0), pt_obs(n_obs), cam_obs(n_obs);
  for (int o = 0; o < n_obs; o++) {
    if (obs_cam[o] < 0 || obs_cam[o] >= n_cams || obs_point[o] < 0 || obs_point[o] >= n_points) {
      set_error("landmark_ba: observation index out of range");
      return RGBDSLAM_B200_ERR_ARG;
    }
    pt_off[obs_point[o] + 1]++;
    cam_off[obs_cam[o] + 1]++;
  }
  for (int p = 0; p < n_points; p++) pt_off[p + 1] += pt_off[p];
  for (int c = 0; c < n_cams; c++) cam_off[c + 1] += cam_off[c];
  {
    std::vector<int> cp(pt_off.begin(), pt_off.end() - 1), cc(cam_off.begin(), cam_off.end() - 1);
    for (int o = 0; o < n_obs; o++) {
      pt_obs[cp[obs_point[o]]++] = o;
      cam_obs[cc[obs_cam[o]]++] = o;
    }
  }
  cudaStream_t st = P.st;
  int rc;
  if ((rc = d.edges.upload(n_cams, n_edges, ij, meas7, info36, huber_delta, true, st))) return rc;
  const size_t nc = (size_t)n_cams, np = (size_t)n_points, no = (size_t)(n_obs > 0 ? n_obs : 1);
  const int npb = (n_points + 127) / 128, ncb = (n_cams + 7) / 8, nchi = (n_obs + 255) / 256 + 2 * ((n_edges + 255) / 256) + 2;
  if ((rc = d.poses.ensure(56 * nc)) || (rc = d.poses_trial.ensure(56 * nc)) || (rc = d.pts.ensure(24 * np)) ||
      (rc = d.pts_trial.ensure(24 * np)) || (rc = d.fixed.ensure(nc)) || (rc = d.obs_cam.ensure(4 * no)) || (rc = d.obs_pt.ensure(4 * no)) ||
      (rc = d.uvd.ensure(24 * no)) || (rc = d.w3.ensure(24 * no)) || (rc = d.pt_off.ensure(4 * (np + 1))) || (rc = d.pt_obs.ensure(4 * no)) ||
      (rc = d.cam_off.ensure(4 * (nc + 1))) || (rc = d.cam_obs.ensure(4 * no)) || (rc = d.blk.ensure(8 * kObsBlk * no)) ||
      (rc = d.Hppinv.ensure(72 * np)) || (rc = d.bp.ensure(24 * np)) || (rc = d.Hcc.ensure(288 * nc)) || (rc = d.bc.ensure(48 * nc)) ||
      (rc = d.g.ensure(48 * nc)) || (rc = d.Minv.ensure(288 * nc)) || (rc = d.maxd_c.ensure(8 * nc)) ||
      (rc = d.maxd_p.ensure(8 * (size_t)(npb + 1))) || (rc = d.x.ensure(48 * nc)) || (rc = d.r.ensure(48 * nc)) || (rc = d.d.ensure(48 * nc)) ||
      (rc = d.q.ensure(48 * nc)) || (rc = d.u.ensure(24 * np)) || (rc = d.part.ensure(8 * (size_t)(ncb + 1))) || (rc = d.state.ensure(64)) ||
      (rc = d.chipart.ensure(8 * (size_t)nchi)) || (rc = d.scpart.ensure(8 * (size_t)(npb + 1))))
    return rc;
  RB200_CUDA(cudaMemcpyAsync(d.poses.ptr, poses7, 56 * nc, cudaMemcpyHostToDevice, st));
  RB200_CUDA(cudaMemcpyAsync(d.pts.ptr, points3, 24 * np, cudaMemcpyHostToDevice, st));
  RB200_CUDA(cudaMemcpyAsync(d.fixed.ptr, fixed, nc, cudaMemcpyHostToDevice, st));
  RB200_CUDA(cudaMemcpyAsync(d.pt_off.ptr, pt_off.data(), 4 * (np + 1), cudaMemcpyHostToDevice, st));
  RB200_CUDA(cudaMemcpyAsync(d.cam_off.ptr, cam_off.data(), 4 * (nc + 1), cudaMemcpyHostToDevice, st));
  if (n_obs > 0) {
    RB200_CUDA(cudaMemcpyAsync(d.obs_cam.ptr, obs_cam, 4 * (size_t)n_obs, cudaMemcpyHostToDevice, st));
    RB200_CUDA(cudaMemcpyAsync(d.obs_pt.ptr, obs_point, 4 * (size_t)n_obs, cudaMemcpyHostToDevice, st));
    RB200_CUDA(cudaMemcpyAsync(d.uvd.ptr, obs_uvd, 24 * (size_t)n_obs, cudaMemcpyHostToDevice, st));
    RB200_CUDA(cudaMemcpyAsync(d.w3.ptr, obs_info3, 24 * (size_t)n_obs, cudaMemcpyHostToDevice, st));
    RB200_CUDA(cudaMemcpyAsync(d.pt_obs.ptr, pt_obs.data(), 4 * (size_t)n_obs, cudaMemcpyHostToDevice, st));
    RB200_CUDA(cudaMemcpyAsync(d.cam_obs.ptr, cam_obs.data(), 4 * (size_t)n_obs, cudaMemcpyHostToDevice, st));
  }
  RB200_CUDA(cudaStreamSynchronize(st));
  double chi2 = 0;
  if ((rc = ba_chi2(P, (const double*)d.poses.ptr, (const double*)d.pts.ptr, &chi2))) return rc;
  if (chi2_before) *chi2_before = chi2;
  int done = 0;
  if ((rc = ba_optimize(P, iterations, chi2, &done))) return rc;
  RB200_CUDA(cudaMemcpyAsync(poses7, d.poses.ptr, 56 * nc, cudaMemcpyDeviceToHost, st));
  RB200_CUDA(cudaMemcpyAsync(points3, d.pts.ptr, 24 * np, cudaMemcpyDeviceToHost, st));
  RB200_CUDA(cudaStreamSynchronize(st));
  if (chi2_after) *chi2_after = chi2;
  if (lm_iterations) *lm_iterations = done;
  if (pcg_iterations) *pcg_iterations = P.pcg_iters;
  s.launches += P.launches;
  return 0;
}

}  // namespace rb200
