// se3_point.cuh -- camera / 3-D point geometry shared by the pairwise g2o refinement (frontend_kernels.cu) and the landmark
// bundle adjustment (landmark_ba.cu): g2o's EdgeSE3PointXYZDepth error with its Jacobians, VertexSE3::oplus, a 3x3 SPD inverse.
#pragma once
#include <cuda_runtime.h>

namespace rb200 {

struct Cam {
  double R[9], t[3];  // world-from-camera
};

// EdgeSE3PointXYZDepth: error and Jacobians (upstream g2o types/slam3d/edge_se3_pointxyz_depth.cpp)
__device__ __forceinline__ void edge_depth(const Cam& c, const double pw[3], const double meas[3], double e[3], double Jc[18],
                                           double Jp[9], double kfx = 521.0, double kfy = 521.0, double kcx = 319.5,
                                           double kcy = 239.5) {
  const double d0 = pw[0] - c.t[0], d1 = pw[1] - c.t[1], d2 = pw[2] - c.t[2];
  double zc[3];
#pragma unroll
  for (int k = 0; k < 3; k++) zc[k] = c.R[k] * d0 + c.R[3 + k] * d1 + c.R[6 + k] * d2;  // R^T (p - t)
  double J[3][9];
#pragma unroll
  for (int r = 0; r < 3; r++)
#pragma unroll
    for (int k = 0; k < 9; k++) J[r][k] = 0.0;
  J[0][0] = J[1][1] = J[2][2] = -1.0;
  J[0][4] = -2 * zc[2]; J[0][5] = 2 * zc[1];
  J[1][3] = 2 * zc[2];  J[1][5] = -2 * zc[0];
  J[2][3] = -2 * zc[1]; J[2][4] = 2 * zc[0];
#pragma unroll
  for (int r = 0; r < 3; r++)
#pragma unroll
    for (int k = 0; k < 3; k++) J[r][6 + k] = c.R[3 * k + r];
  const double zp0 = kfx * zc[0] + kcx * zc[2], zp1 = kfy * zc[1] + kcy * zc[2], zp2 = zc[2];
  const double iz2 = 1.0 / (zp2 * zp2);
#pragma unroll
  for (int k = 0; k < 9; k++) {
    const double j0 = kfx * J[0][k] + kcx * J[2][k], j1 = kfy * J[1][k] + kcy * J[2][k], j2 = J[2][k];
    const double h0 = iz2 * (j0 * zp2 - zp0 * j2), h1 = iz2 * (j1 * zp2 - zp1 * j2);
    if (k < 6) {
      Jc[k] = h0; Jc[6 + k] = h1; Jc[12 + k] = j2;
    } else {
      Jp[k - 6] = h0; Jp[3 + k - 6] = h1; Jp[6 + k - 6] = j2;
    }
  }
  e[0] = zp0 / zp2 - meas[0];
  e[1] = zp1 / zp2 - meas[1];
  e[2] = zp2 - meas[2];
}

__device__ __forceinline__ void cam_oplus(Cam& c, const double d[6]) {  // X <- X * fromVectorMQT(d)
  const double vx = d[3], vy = d[4], vz = d[5];
  double w = 1.0 - (vx * vx + vy * vy + vz * vz);
  double dR[9] = {1, 0, 0, 0, 1, 0, 0, 0, 1};
  if (w >= 0) {
    w = sqrt(w);
    dR[0] = 1 - 2 * (vy * vy + vz * vz); dR[1] = 2 * (vx * vy - vz * w);     dR[2] = 2 * (vx * vz + vy * w);
    dR[3] = 2 * (vx * vy + vz * w);     dR[4] = 1 - 2 * (vx * vx + vz * vz); dR[5] = 2 * (vy * vz - vx * w);
    dR[6] = 2 * (vx * vz - vy * w);     dR[7] = 2 * (vy * vz + vx * w);     dR[8] = 1 - 2 * (vx * vx + vy * vy);
  }
  double nR[9], nt[3];
#pragma unroll
  for (int r = 0; r < 3; r++) nt[r] = c.t[r] + c.R[3 * r] * d[0] + c.R[3 * r + 1] * d[1] + c.R[3 * r + 2] * d[2];
#pragma unroll
  for (int r = 0; r < 3; r++)
#pragma unroll
    for (int k = 0; k < 3; k++) nR[3 * r + k] = c.R[3 * r] * dR[k] + c.R[3 * r + 1] * dR[3 + k] + c.R[3 * r + 2] * dR[6 + k];
#pragma unroll
  for (int i = 0; i < 9; i++) c.R[i] = nR[i];
#pragma unroll
  for (int i = 0; i < 3; i++) c.t[i] = nt[i];
}

__device__ __forceinline__ bool inv3_sym(const double A[9], double inv[9]) {
  const double a = A[0], b = A[1], c = A[2], d = A[4], e = A[5], f = A[8];
  const double c00 = d * f - e * e, c01 = c * e - b * f, c02 = b * e - c * d;
  const double det = a * c00 + b * c01 + c * c02;
  if (!(det > 0.0)) return false;
  const double id = 1.0 / det;
  inv[0] = c00 * id; inv[1] = c01 * id; inv[2] = c02 * id;
  inv[3] = inv[1];   inv[4] = (a * f - c * c) * id; inv[5] = (b * c - a * e) * id;
  inv[6] = inv[2];   inv[7] = inv[5]; inv[8] = (a * d - b * b) * id;
  return true;
}

}  // namespace rb200
