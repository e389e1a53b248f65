// icp.cuh -- what the two ICP methods share (icp.cu: IterativeClosestPoint, icp_nl.cu: IterativeClosestPointNonLinear):
// the target's cells and keys, the nearest-target search, the finite test, the float transform, the fixed-order block sum
// and the align kernel, which takes the transformation estimator as a template parameter.  Every float operation is an
// explicit _rn intrinsic.
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

// ---- alignment ------------------------------------------------------------------------------------------------------------

// One iteration's correspondences: source point i, as the iterations have moved it, pairs with target point cr[i] >= 0.
// Thread t searched the points t, t + 256, ...
struct IcpPass {
  const float *x, *y, *z;
  const int* cr;
  int ns;
  IcpTarget tg;
};

// IterativeClosestPoint::computeTransformation of PCL 1.7, one persistent CTA per pair.  Each iteration finds the
// correspondences in source order, has the estimator E turn them into T_inc, then on thread 0 accumulates final = T_inc final,
// computes calculateMSE and DefaultConvergenceCriteria, and moves the source.  The estimator (icp.cu: IcpSvd, icp_nl.cu: IcpLm)
// provides:
//   kMinCorrespondences     fewer correspondences end the alignment, not converged
//   kMinBlocks              the CTAs per SM its register budget is set for
//   kPlanes                 its pair's work planes (wplane floats apart, at w0 in each); planes 0-2 hold the moving source
//   Shared                  its shared memory, passed to every hook below
//   E(sh, w, wplane)        its state in every thread, from the pair's work planes w, before the first barrier
//   add(x, y, z, tx, ty, tz)  called in the search by the thread of source point i for each correspondence i -> j, i
//                           ascending, with the target point j
//   count(sh, pass, c)      every thread, after the search (c: the calling thread's correspondences): their number in every
//                           thread; ends with a barrier when there are any
//   estimate(sh, pass, n)   every thread, when n >= kMinCorrespondences
//   increment(sh, T)        thread 0, after estimate: T_inc as 12 row-major floats
template <class E>
__global__ void __launch_bounds__(kIcpThreads, E::kMinBlocks)
    k_icp_align(const IcpPair* __restrict__ pairs, const IcpNode* __restrict__ nodes, const float* __restrict__ pts, long long plane,
                const int* __restrict__ nf, const unsigned long long* __restrict__ key, const int* __restrict__ idx,
                const int* __restrict__ nfin, float* __restrict__ work, long long wplane, int* __restrict__ corr,
                float* __restrict__ dist, rgbdslam_b200_icp_result* __restrict__ results) {
  __shared__ typename E::Shared sh;
  __shared__ float s_T[12];
  __shared__ int s_stop;
  const IcpPair pr = pairs[blockIdx.x];
  const long long fs = nodes[pr.s].f0, ft = nodes[pr.t].f0;
  const int ns = nf[pr.s];
  IcpTarget tg;
  tg.key = key + ft;
  tg.idx = idx + ft;
  tg.m = nfin[pr.t];
  tg.x = pts + ft;
  tg.y = tg.x + plane;
  tg.z = tg.y + plane;
  float* wx = work + pr.w0;  // the source as the iterations move it
  float* wy = wx + wplane;
  float* wz = wy + wplane;
  int* cr = corr + pr.w0;
  float* ds = dist + pr.w0;
  const IcpPass pass{wx, wy, wz, cr, ns, tg};
  E est(sh, wx, wplane);
  for (int i = threadIdx.x; i < ns; i += kIcpThreads) {
    wx[i] = pts[fs + i];
    wy[i] = pts[plane + fs + i];
    wz[i] = pts[2 * plane + fs + i];
  }
  // thread 0's bookkeeping
  float final_T[16];
#pragma unroll
  for (int k = 0; k < 16; k++) final_T[k] = k % 5 == 0 ? 1.f : 0.f;
  double prev = 1.7976931348623157e308, mse = 0.0;
  int iterations = 0, criterion = 0, cnt = 0;
  __syncthreads();
#pragma unroll 1
  for (;;) {
    // 1. the correspondences in source order
    int c = 0;
    for (int i = threadIdx.x; i < ns; i += kIcpThreads) {
      const float x = wx[i], y = wy[i], z = wz[i];
      float d = INFINITY;
      int j = icp_finite(x, y, z) ? icp_nearest(tg, x, y, z, d) : -1;
      if (j >= 0 && !((double)d <= kIcpMaxD2)) j = -1;
      cr[i] = j;
      ds[i] = d;
      if (j >= 0) {
        c++;
        est.add(x, y, z, tg.x[j], tg.y[j], tg.z[j]);
      }
    }
    cnt = est.count(sh, pass, c);
    if (cnt < E::kMinCorrespondences) {  // too few correspondences: not converged
      criterion = 0;
      break;
    }
    // 2. T_inc
    est.estimate(sh, pass, cnt);
    // 3. thread 0: final = T_inc final, calculateMSE and DefaultConvergenceCriteria
    float T[12];
    if (threadIdx.x == 0) {
      est.increment(sh, T);
      float nf_T[16];
#pragma unroll
      for (int r = 0; r < 4; r++)
#pragma unroll
        for (int q = 0; q < 4; q++) {
          const float a0 = r < 3 ? T[4 * r] : 0.f, a1 = r < 3 ? T[4 * r + 1] : 0.f, a2 = r < 3 ? T[4 * r + 2] : 0.f,
                      a3 = r < 3 ? T[4 * r + 3] : 1.f;
          nf_T[4 * r + q] = __fadd_rn(__fadd_rn(__fadd_rn(__fmul_rn(a0, final_T[q]), __fmul_rn(a1, final_T[4 + q])),
                                                __fmul_rn(a2, final_T[8 + q])),
                                      __fmul_rn(a3, final_T[12 + q]));
        }
#pragma unroll
      for (int k = 0; k < 16; k++) final_T[k] = nf_T[k];
      iterations++;
      double acc = 0.0;
#pragma unroll 4
      for (int i = 0; i < ns; i++)
        if (cr[i] >= 0) acc = __dadd_rn(acc, (double)ds[i]);
      mse = __ddiv_rn(acc, (double)cnt);
      int stop = 0;
      const double cos_angle = __dmul_rn(0.5, (double)__fsub_rn(__fadd_rn(__fadd_rn(T[0], T[5]), T[10]), 1.f));
      const double trans2 = (double)__fadd_rn(__fadd_rn(__fmul_rn(T[3], T[3]), __fmul_rn(T[7], T[7])), __fmul_rn(T[11], T[11]));
      const double dmse = fabs(__dsub_rn(mse, prev));
      if (iterations >= kIcpMaxIterations) stop = 1;
      else if (cos_angle >= 1.0 - kIcpTransformEps && trans2 <= kIcpTransformEps) stop = 2;
      else if (dmse < 1e-12) stop = 3;
      else if (__ddiv_rn(dmse, prev) < kIcpFitnessEps) stop = 4;
      else prev = mse;
      criterion = stop;
#pragma unroll
      for (int k = 0; k < 12; k++) s_T[k] = T[k];
      s_stop = stop;
    }
    __syncthreads();
    if (s_stop) break;
    // 4. move the source: ((r0 x + r1 y) + r2 z) + t of every finite point
#pragma unroll
    for (int k = 0; k < 12; k++) T[k] = s_T[k];
    for (int i = threadIdx.x; i < ns; i += kIcpThreads) {
      const float x = wx[i], y = wy[i], z = wz[i];
      if (!icp_finite(x, y, z)) continue;
      wx[i] = __fadd_rn(icp_dot3(T[0], x, T[1], y, T[2], z), T[3]);
      wy[i] = __fadd_rn(icp_dot3(T[4], x, T[5], y, T[6], z), T[7]);
      wz[i] = __fadd_rn(icp_dot3(T[8], x, T[9], y, T[10], z), T[11]);
    }
    __syncthreads();
  }
  if (threadIdx.x == 0) {
    rgbdslam_b200_icp_result r;
    const bool converged = criterion != 0;
#pragma unroll
    for (int q = 0; q < 4; q++)
#pragma unroll
      for (int p = 0; p < 4; p++) r.T[4 * q + p] = converged ? final_T[4 * p + q] : (p == q ? 1.f : 0.f);
    r.converged = converged ? 1 : 0;
    r.iterations = iterations;
    r.criterion = criterion;
    r.n_source = ns;
    r.n_target = nf[pr.t];
    r.n_correspondences = cnt;
    r.mse = mse;
    results[blockIdx.x] = r;
  }
}

// The work planes and the launch of k_icp_align<E>.  launch_icp_align and icp_work_planes (icp.cu) choose E by method.
template <class E>
struct IcpAlign {
  static int planes();
  static cudaError_t launch(const IcpPair* pairs, int npairs, const IcpNode* d_nodes, const float* pts, long long plane,
                            const int* nf, const unsigned long long* key, const int* idx, const int* nfin, float* work,
                            long long wplane, int* corr, float* dist, rgbdslam_b200_icp_result* results, cudaStream_t st);
};

template <class E>
int IcpAlign<E>::planes() {
  return E::kPlanes;
}

template <class E>
cudaError_t IcpAlign<E>::launch(const IcpPair* pairs, int npairs, const IcpNode* d_nodes, const float* pts, long long plane,
                                const int* nf, const unsigned long long* key, const int* idx, const int* nfin, float* work,
                                long long wplane, int* corr, float* dist, rgbdslam_b200_icp_result* results, cudaStream_t st) {
  if (npairs <= 0) return cudaSuccess;
  k_icp_align<E><<<npairs, kIcpThreads, 0, st>>>(pairs, d_nodes, pts, plane, nf, key, idx, nfin, work, wplane, corr, dist, results);
  return cudaGetLastError();
}

struct IcpLm;
extern template struct IcpAlign<IcpLm>;  // instantiated in icp_nl.cu, with the estimator

}  // namespace rb200
