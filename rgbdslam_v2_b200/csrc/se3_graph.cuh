// se3_graph.cuh -- small device helpers shared by the pose-graph solver (posegraph.cu) and the landmark bundle adjustment
// (landmark_ba.cu): quaternion / rotation conversions of the (t, q) pose vectors, a 6x6 inverse, a warp sum, the layout of
// the per-edge normal-equation blocks of the pose edges.
#pragma once
#include <cuda_runtime.h>

namespace rb200 {

// Per pose edge (written by pg_linearize_kernel), kEdgeBlk doubles: [A 36 | B 36 | C 36 | gi 6 | gj 6] with A = Ji'WJi,
// B = Jj'WJj, C = Ji'WJj, g = J'We, all scaled by the Huber weight.  An incidence code is edge << 1 | role, role 0 for the
// edge's vertex i, 1 for its vertex j.
constexpr int kEdgeBlk = 120, kEdgeA = 0, kEdgeB = 36, kEdgeC = 72, kEdgeGi = 108, kEdgeGj = 114;
__device__ __forceinline__ const double* edge_blocks(const double* blk, int edge) { return blk + (size_t)edge * kEdgeBlk; }
__device__ __forceinline__ int edge_diag(int role) { return kEdgeA + role * 36; }  // offset of A (role 0) or B (role 1)
__device__ __forceinline__ int edge_grad(int role) { return kEdgeGi + role * 6; }  // offset of gi (role 0) or gj (role 1)

// SE(3) helpers, poses are (tx,ty,tz,qx,qy,qz,qw)
__device__ __forceinline__ void quat_to_R(const double* q, double* R) {
  double x = q[0], y = q[1], z = q[2], w = q[3];
  const double n = 1.0 / sqrt(x * x + y * y + z * z + w * w);
  x *= n; y *= n; z *= n; w *= n;
  R[0] = 1 - 2 * (y * y + z * z); R[1] = 2 * (x * y - z * w);     R[2] = 2 * (x * z + y * w);
  R[3] = 2 * (x * y + z * w);     R[4] = 1 - 2 * (x * x + z * z); R[5] = 2 * (y * z - x * w);
  R[6] = 2 * (x * z - y * w);     R[7] = 2 * (y * z + x * w);     R[8] = 1 - 2 * (x * x + y * y);
}
__device__ __forceinline__ void quat_mul(const double* a, const double* b, double* o) {
  const double ax = a[0], ay = a[1], az = a[2], aw = a[3], bx = b[0], by = b[1], bz = b[2], bw = b[3];
  o[0] = aw * bx + ax * bw + ay * bz - az * by;
  o[1] = aw * by - ax * bz + ay * bw + az * bx;
  o[2] = aw * bz + ax * by - ay * bx + az * bw;
  o[3] = aw * bw - ax * bx - ay * by - az * bz;
}
__device__ __forceinline__ void quat_norm(double* q) {
  const double n = 1.0 / sqrt(q[0] * q[0] + q[1] * q[1] + q[2] * q[2] + q[3] * q[3]);
  q[0] *= n; q[1] *= n; q[2] *= n; q[3] *= n;
}

// 6x6 inverse by Gauss-Jordan with partial pivoting (block-Jacobi preconditioner)
__device__ inline bool inv6(const double* A, double* Ai) {
  double M[6][12];
  for (int r = 0; r < 6; r++)
    for (int c = 0; c < 6; c++) {
      M[r][c] = A[6 * r + c];
      M[r][6 + c] = (r == c) ? 1.0 : 0.0;
    }
  for (int c = 0; c < 6; c++) {
    int p = c;
    for (int r = c + 1; r < 6; r++)
      if (fabs(M[r][c]) > fabs(M[p][c])) p = r;
    if (fabs(M[p][c]) < 1e-300) return false;
    if (p != c)
      for (int k = 0; k < 12; k++) {
        const double t = M[c][k];
        M[c][k] = M[p][k];
        M[p][k] = t;
      }
    const double d = 1.0 / M[c][c];
    for (int k = 0; k < 12; k++) M[c][k] *= d;
    for (int r = 0; r < 6; r++)
      if (r != c) {
        const double f = M[r][c];
        for (int k = 0; k < 12; k++) M[r][k] -= f * M[c][k];
      }
  }
  for (int r = 0; r < 6; r++)
    for (int c = 0; c < 6; c++) Ai[6 * r + c] = M[r][6 + c];
  return true;
}

__device__ __forceinline__ double warp_sum_d(double v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

}  // namespace rb200
