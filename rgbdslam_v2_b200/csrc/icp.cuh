// icp.cuh -- device helpers shared by the two ICP methods (icp.cu: IterativeClosestPoint, icp_nl.cu:
// IterativeClosestPointNonLinear): the target's cells and keys, the nearest-target search, the finite test, the float
// transform and the fixed-order block sum.  Every float operation is an explicit _rn intrinsic.
#pragma once
#include "kernels.h"
#include "map.cuh"

namespace rb200 {

constexpr int kIcpThreads = 256;  // k_icp_cells and the align kernels; the order of the align sums is defined by it
constexpr double kIcpMaxD2 = 0.05 * 0.05;  // setMaxCorrespondenceDistance(0.05), squared in double as PCL does
constexpr int kIcpMaxIterations = 50;
constexpr double kIcpTransformEps = 1e-8;
constexpr double kIcpFitnessEps = 1.0;  // setEuclideanFitnessEpsilon(1): PCL 1.7's relative MSE threshold
constexpr float kIcpCellClamp = 32766.f;  // cells are clamped to [-32766, 32766]: the 27 neighbours stay in 16-bit fields

__device__ __forceinline__ bool icp_finite(float x, float y, float z) { return isfinite(x) && isfinite(y) && isfinite(z); }

// floor(16 v), clamped.  Clamping is monotone and moves no two values further apart, so two points within 0.05 m
// (16 * 0.0500001 < 1) still lie in the same or adjacent cells.
__device__ __forceinline__ int icp_cell(float v) { return (int)fminf(fmaxf(floorf(__fmul_rn(v, 16.f)), -kIcpCellClamp), kIcpCellClamp); }

__device__ __forceinline__ unsigned long long icp_key(int cx, int cy, int cz) {
  return ((unsigned long long)(unsigned)(cz + 32768) << 32) | ((unsigned long long)(unsigned)(cy + 32768) << 16) |
         (unsigned long long)(unsigned)(cx + 32768);
}

__device__ __forceinline__ float icp_dot3(float a0, float b0, float a1, float b1, float a2, float b2) {
  return __fadd_rn(__fadd_rn(__fmul_rn(a0, b0), __fmul_rn(a1, b1)), __fmul_rn(a2, b2));
}

// The nearest finite target point of q: the smallest ((dx dx + dy dy) + dz dz), the lowest index among equal ones.  Only the
// 27 cells around q's are searched, which holds every point within 0.05 m; -1 when none is there.
struct IcpTarget {
  const unsigned long long* key;
  const int* idx;
  int m;
  const float *x, *y, *z;
};

__device__ __forceinline__ int icp_nearest(const IcpTarget& t, float qx, float qy, float qz, float& best) {
  const int cx = icp_cell(qx), cy = icp_cell(qy), cz = icp_cell(qz);
  int bj = -1;
  best = INFINITY;
#pragma unroll 1
  for (int r = 0; r < 9; r++) {
    const unsigned long long lo = icp_key(cx - 1, cy + r % 3 - 1, cz + r / 3 - 1), hi = lo + 2;  // three cells in a row
    int a = 0, b = t.m;
    while (a < b) {
      const int mid = (a + b) >> 1;
      if (t.key[mid] < lo) a = mid + 1;
      else b = mid;
    }
    for (; a < t.m && t.key[a] <= hi; a++) {
      const int j = t.idx[a];
      const float dx = __fsub_rn(qx, t.x[j]), dy = __fsub_rn(qy, t.y[j]), dz = __fsub_rn(qz, t.z[j]);
      const float d = __fadd_rn(__fadd_rn(__fmul_rn(dx, dx), __fmul_rn(dy, dy)), __fmul_rn(dz, dz));
      if (d < best || (d == best && j < bj)) {
        best = d;
        bj = j;
      }
    }
  }
  return bj;
}

// The device's float sum of one value per thread: p[t] += p[t + s] for s = 128, 64, ..., 1.  Ends with a barrier.
template <int N>
__device__ __forceinline__ void icp_tree(float (*red)[kIcpThreads], const float (&v)[N]) {
#pragma unroll
  for (int c = 0; c < N; c++) red[c][threadIdx.x] = v[c];
  __syncthreads();
#pragma unroll 1
  for (int s = kIcpThreads / 2; s > 0; s >>= 1) {
    if (threadIdx.x < s)
#pragma unroll
      for (int c = 0; c < N; c++) red[c][threadIdx.x] = __fadd_rn(red[c][threadIdx.x], red[c][threadIdx.x + s]);
    __syncthreads();
  }
}

}  // namespace rb200
