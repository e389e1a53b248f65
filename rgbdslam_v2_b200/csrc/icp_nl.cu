// icp_nl.cu -- icp_method "icp_nl" of the ICP fallback (icp.cpp:50-58): PCL 1.7's
// pcl::IterativeClosestPointNonLinear<PointXYZRGB, PointXYZRGB>, whose increments come from TransformationEstimationLM:
// Eigen's LevenbergMarquardt (MINPACK lmder) over NumericalDiff's forward differences of |warp(src_i) - tgt_i|, with
// WarpPointRigid6D's parameters (tx, ty, tz, qx, qy, qz).  The clouds come from icp.cu's k_icp_filter and k_icp_cells.
//   IcpLm  the estimator of k_icp_align<IcpLm> (icp.cuh): the correspondences, compacted in source order into the pair's
//          work rows, then the LM.
// The length-m work of the LM is spread over the CTA: residuals, Jacobian columns, blueNorm and squared column norms, the
// Householder tails and their updates, Q^T f and stableNorm.  Thread 0 does the 6 x 6 work: pivots, Householder scalars,
// lmpar2 / qrsolv and the LM bookkeeping.  Every length-m float sum is the fixed-order block sum of icp_tree over the row
// indices (thread t owns rows t, t + 256, ...); the rules are restated in include/rgbdslam_b200/icp.h.  Every float
// operation is an explicit _rn intrinsic, so tests/icp_nl_exact.py replays the kernel bit for bit.
#include <cfloat>

#include "icp.cuh"

namespace rb200 {

constexpr int kNlN = 6;                 // WarpPointRigid6D's dimension
constexpr int kNlMaxfev = 400;
constexpr int kNlStableBlock = 4096;    // stableNorm's block
constexpr float kNlEps = 0x1p-23f;  // NumTraits<float>::epsilon()
constexpr float kNlFactor = 100.f;
constexpr float kNlB1 = 0x1p-63f, kNlB2 = 0x1p52f, kNlS1m = 0x1p63f, kNlS2m = 0x1p-76f;  // blueNorm's constants for float

// The work planes of a pair after k_icp_align's moving source (planes 0-2)
enum { kSx = 3, kTx = 6, kF0 = 9, kQf = 11, kJ0 = 12 };

struct NlLm {  // thread 0's 6 x 6 state and what it broadcasts
  float R[kNlN][kNlN], S[kNlN][kNlN];
  float x[kNlN], xt[kNlN], wa1[kNlN], wa2[kNlN], diag[kNlN], qtf[kNlN], cn[kNlN], hc[kNlN], sq[kNlN], sdiag[kNlN], tmp[kNlN];
  int perm[kNlN];
  float tau, denom, inv;
  int big, zero_tail, cur, flag;
};

__device__ __forceinline__ float nl_max(float a, float b) { return a < b ? b : a; }  // std::max
__device__ __forceinline__ float nl_min(float a, float b) { return b < a ? b : a; }  // std::min
__device__ __forceinline__ float nl_nanmax(float a, float b) { return (b > a || b != b) ? b : a; }

// block_sum of six non-negative values at threads 0..5: ((p0 + p4) + p2) + ((p1 + p5) + p3)
__device__ __forceinline__ float nl_sum6(const float (&w)[kNlN]) {
  float p[kNlN];
#pragma unroll
  for (int i = 0; i < kNlN; i++) p[i] = __fadd_rn(0.f, w[i]);
  return __fadd_rn(__fadd_rn(__fadd_rn(p[0], p[4]), p[2]), __fadd_rn(__fadd_rn(p[1], p[5]), p[3]));
}

// stableNorm's per-block scale update (Eigen 3.3's stable_norm_kernel)
__device__ __forceinline__ void nl_stable_scale(float mx, float& scale, float& inv, float& ssq) {
  if (mx > scale) {
    const float r = __fdiv_rn(scale, mx);
    ssq = __fmul_rn(ssq, __fmul_rn(r, r));
    const float tmp = __fdiv_rn(1.f, mx);
    if (tmp > FLT_MAX) {
      inv = FLT_MAX;
      scale = __fdiv_rn(1.f, inv);
    } else if (mx > FLT_MAX) {
      inv = 1.f;
      scale = mx;
    } else {
      scale = mx;
      inv = tmp;
    }
  } else if (mx != mx) {
    scale = mx;
  }
}

__device__ float nl_stable6(const float* v) {
  float mx = 0.f, scale = 0.f, inv = 1.f, ssq = 0.f;
#pragma unroll
  for (int i = 0; i < kNlN; i++) mx = nl_nanmax(mx, fabsf(v[i]));
  nl_stable_scale(mx, scale, inv, ssq);
  if (scale > 0.f) {
    float w[kNlN];
#pragma unroll
    for (int i = 0; i < kNlN; i++) {
      const float t = __fmul_rn(v[i], inv);
      w[i] = __fmul_rn(t, t);
    }
    ssq = __fadd_rn(ssq, nl_sum6(w));
  }
  return __fmul_rn(scale, __fsqrt_rn(ssq));
}

// blueNorm after its three sums
__device__ float nl_blue_finish(float abig, float asml, float amed) {
  if (amed != amed) return amed;
  if (abig > 0.f) {
    abig = __fsqrt_rn(abig);
    if (abig > FLT_MAX) return abig;
    if (amed > 0.f) {
      abig = __fdiv_rn(abig, kNlS2m);
      amed = __fsqrt_rn(amed);
    } else {
      return __fdiv_rn(abig, kNlS2m);
    }
  } else if (asml > 0.f) {
    if (amed > 0.f) {
      abig = __fsqrt_rn(amed);
      amed = __fdiv_rn(__fsqrt_rn(asml), kNlS1m);
    } else {
      return __fdiv_rn(__fsqrt_rn(asml), kNlS1m);
    }
  } else {
    return __fsqrt_rn(amed);
  }
  asml = nl_min(abig, amed);
  abig = nl_max(abig, amed);
  if (asml <= __fmul_rn(abig, __fsqrt_rn(kNlEps))) return abig;
  const float r = __fdiv_rn(asml, abig);
  return __fmul_rn(abig, __fsqrt_rn(__fadd_rn(1.f, __fmul_rn(r, r))));
}

// blueNorm's classification of one |value|, added into the three sums
__device__ __forceinline__ void nl_blue_add(float a, float ab2, float& big, float& sml, float& med) {
  if (a > ab2) {
    const float z = __fmul_rn(a, kNlS2m);
    big = __fadd_rn(big, __fmul_rn(z, z));
  } else if (a < kNlB1) {
    const float z = __fmul_rn(a, kNlS1m);
    sml = __fadd_rn(sml, __fmul_rn(z, z));
  } else {
    med = __fadd_rn(med, __fmul_rn(a, a));
  }
}

__device__ float nl_blue6(const float* v) {
  const float ab2 = __fdiv_rn(kNlB2, (float)kNlN);
  float wb[kNlN], ws[kNlN], wm[kNlN];
#pragma unroll
  for (int i = 0; i < kNlN; i++) {
    wb[i] = ws[i] = wm[i] = 0.f;
    nl_blue_add(fabsf(v[i]), ab2, wb[i], ws[i], wm[i]);
  }
  return nl_blue_finish(nl_sum6(wb), nl_sum6(ws), nl_sum6(wm));
}

// WarpPointRigid6D::setParam(x).getTransform() as 12 row-major floats: q.q = (qx qx + qz qz) + qy qy, w = sqrt(1 - q.q)
// without renormalisation, the rotation of Quaternion::toRotationMatrix
__device__ __forceinline__ void nl_warp(const float (&x)[kNlN], float (&T)[12]) {
  const float qx = x[3], qy = x[4], qz = x[5];
  const float qq = __fadd_rn(__fadd_rn(__fmul_rn(qx, qx), __fmul_rn(qz, qz)), __fmul_rn(qy, qy));
  const float w = __fsqrt_rn(__fsub_rn(1.f, qq));
  const float tx = __fmul_rn(2.f, qx), ty = __fmul_rn(2.f, qy), tz = __fmul_rn(2.f, qz);
  const float twx = __fmul_rn(tx, w), twy = __fmul_rn(ty, w), twz = __fmul_rn(tz, w);
  const float txx = __fmul_rn(tx, qx), txy = __fmul_rn(ty, qx), txz = __fmul_rn(tz, qx);
  const float tyy = __fmul_rn(ty, qy), tyz = __fmul_rn(tz, qy), tzz = __fmul_rn(tz, qz);
  T[0] = __fsub_rn(1.f, __fadd_rn(tyy, tzz));
  T[1] = __fsub_rn(txy, twz);
  T[2] = __fadd_rn(txz, twy);
  T[3] = x[0];
  T[4] = __fadd_rn(txy, twz);
  T[5] = __fsub_rn(1.f, __fadd_rn(txx, tzz));
  T[6] = __fsub_rn(tyz, twx);
  T[7] = x[1];
  T[8] = __fsub_rn(txz, twy);
  T[9] = __fadd_rn(tyz, twx);
  T[10] = __fsub_rn(1.f, __fadd_rn(txx, tyy));
  T[11] = x[2];
}

// |warp(s) - t|: sqrt((dx dx + dz dz) + dy dy), the Vector4 norm with w = 0
__device__ __forceinline__ float nl_residual(const float (&T)[12], float sx, float sy, float sz, float tx, float ty, float tz) {
  const float dx = __fsub_rn(__fadd_rn(icp_dot3(T[0], sx, T[1], sy, T[2], sz), T[3]), tx);
  const float dy = __fsub_rn(__fadd_rn(icp_dot3(T[4], sx, T[5], sy, T[6], sz), T[7]), ty);
  const float dz = __fsub_rn(__fadd_rn(icp_dot3(T[8], sx, T[9], sy, T[10], sz), T[11]), tz);
  return __fsqrt_rn(__fadd_rn(__fadd_rn(__fmul_rn(dx, dx), __fmul_rn(dz, dz)), __fmul_rn(dy, dy)));
}

// The compact correspondences of a pair and its work rows
struct NlRows {
  float *sx, *sy, *sz, *tx, *ty, *tz;
  float* f[2];
  float* q;
  float* J[kNlN];
  int m;
};

// out_i = residual of row i at the parameters x (every thread computes the same warp)
__device__ __forceinline__ void nl_eval(const NlRows& r, const float* xs, float* out) {
  float x[kNlN], T[12];
#pragma unroll
  for (int k = 0; k < kNlN; k++) x[k] = xs[k];
  nl_warp(x, T);
  for (int i = threadIdx.x; i < r.m; i += kIcpThreads) out[i] = nl_residual(T, r.sx[i], r.sy[i], r.sz[i], r.tx[i], r.ty[i], r.tz[i]);
}

// stableNorm of v[0, m) for the whole CTA; the value is thread 0's.  Ends with a barrier.
__device__ float nl_stable_m(const float* v, int m, float (*red)[kIcpThreads], NlLm& L) {
  float scale = 0.f, inv = 1.f, ssq = 0.f;
  __syncthreads();
#pragma unroll 1
  for (int b = 0; b < m; b += kNlStableBlock) {
    const int e = min(b + kNlStableBlock, m);
    float mx = 0.f;
    for (int i = b + threadIdx.x; i < e; i += kIcpThreads) mx = nl_nanmax(mx, fabsf(v[i]));
    red[0][threadIdx.x] = mx;
    __syncthreads();
#pragma unroll 1
    for (int s = kIcpThreads / 2; s > 0; s >>= 1) {
      if (threadIdx.x < s) red[0][threadIdx.x] = nl_nanmax(red[0][threadIdx.x], red[0][threadIdx.x + s]);
      __syncthreads();
    }
    if (threadIdx.x == 0) {
      nl_stable_scale(red[0][0], scale, inv, ssq);
      L.inv = inv;
      L.flag = scale > 0.f;
    }
    __syncthreads();
    const float iv = L.inv;
    const int add = L.flag;
    float acc[1] = {0.f};
    for (int i = b + threadIdx.x; i < e; i += kIcpThreads) {
      const float w = __fmul_rn(v[i], iv);
      acc[0] = __fadd_rn(acc[0], __fmul_rn(w, w));
    }
    icp_tree<1>(red, acc);
    if (threadIdx.x == 0 && add) ssq = __fadd_rn(ssq, red[0][0]);
    __syncthreads();
  }
  return __fmul_rn(scale, __fsqrt_rn(ssq));
}

// ---- thread 0: qrsolv and lmpar2 ------------------------------------------------------------------------------------------

__device__ void nl_givens(float p, float q, float& c, float& s) {  // JacobiRotation::makeGivens, real
  if (q == 0.f) {
    c = p < 0.f ? -1.f : 1.f;
    s = 0.f;
  } else if (p == 0.f) {
    c = 0.f;
    s = q < 0.f ? 1.f : -1.f;
  } else if (fabsf(p) > fabsf(q)) {
    const float t = __fdiv_rn(q, p);
    float u = __fsqrt_rn(__fadd_rn(1.f, __fmul_rn(t, t)));
    if (p < 0.f) u = -u;
    c = __fdiv_rn(1.f, u);
    s = __fmul_rn(-t, c);
  } else {
    const float t = __fdiv_rn(p, q);
    float u = __fsqrt_rn(__fadd_rn(1.f, __fmul_rn(t, t)));
    if (q < 0.f) u = -u;
    s = __fdiv_rn(-1.f, u);
    c = __fmul_rn(-t, s);
  }
}

// qrsolv on L.S with the diagonal d: the solution into x (L.wa2 is free here), L.sdiag
__device__ void nl_qrsolv(NlLm& L, const float* d, float* x) {
  float xs[kNlN], wa[kNlN];
  for (int i = 0; i < kNlN; i++) {
    xs[i] = L.S[i][i];
    wa[i] = L.qtf[i];
    for (int j = 0; j < i; j++) L.S[i][j] = L.S[j][i];
    L.sdiag[i] = 0.f;
  }
  for (int j = 0; j < kNlN; j++) {
    const int l = L.perm[j];
    if (d[l] == 0.f) break;
    for (int i = j; i < kNlN; i++) L.sdiag[i] = 0.f;
    L.sdiag[j] = d[l];
    float qtbpj = 0.f;
    for (int k = j; k < kNlN; k++) {
      float c, s;
      nl_givens(-L.S[k][k], L.sdiag[k], c, s);
      L.S[k][k] = __fadd_rn(__fmul_rn(c, L.S[k][k]), __fmul_rn(s, L.sdiag[k]));
      const float temp = __fadd_rn(__fmul_rn(c, wa[k]), __fmul_rn(s, qtbpj));
      qtbpj = __fadd_rn(__fmul_rn(-s, wa[k]), __fmul_rn(c, qtbpj));
      wa[k] = temp;
      for (int i = k + 1; i < kNlN; i++) {
        const float t2 = __fadd_rn(__fmul_rn(c, L.S[i][k]), __fmul_rn(s, L.sdiag[i]));
        L.sdiag[i] = __fadd_rn(__fmul_rn(-s, L.S[i][k]), __fmul_rn(c, L.sdiag[i]));
        L.S[i][k] = t2;
      }
    }
  }
  int nsing = 0;
  for (int i = 0; i < kNlN; i++) L.sdiag[i] = L.S[i][i];
  while (nsing < kNlN && L.sdiag[nsing] != 0.f) nsing++;
  for (int i = nsing; i < kNlN; i++) wa[i] = 0.f;
  for (int i = nsing - 1; i >= 0; i--) {
    if (i < nsing - 1) {
      float dot = __fmul_rn(L.S[i + 1][i], wa[i + 1]);
      for (int l = i + 2; l < nsing; l++) dot = __fadd_rn(dot, __fmul_rn(L.S[l][i], wa[l]));
      wa[i] = __fsub_rn(wa[i], dot);
    }
    wa[i] = __fdiv_rn(wa[i], L.S[i][i]);
  }
  for (int i = 0; i < kNlN; i++) L.S[i][i] = xs[i];
  for (int j = 0; j < kNlN; j++) x[L.perm[j]] = wa[j];
}

// lmpar2: par and the step into L.wa1 (before LevenbergMarquardt negates it)
__device__ float nl_lmpar(NlLm& L, int rank, float delta, float par) {
  float w1[kNlN], w2[kNlN], x[kNlN];
  for (int i = 0; i < kNlN; i++) w1[i] = i < rank ? L.qtf[i] : 0.f;
  for (int i = rank - 1; i >= 0; i--)
    if (w1[i] != 0.f) {
      w1[i] = __fdiv_rn(w1[i], L.R[i][i]);
      for (int r = 0; r < i; r++) w1[r] = __fsub_rn(w1[r], __fmul_rn(w1[i], L.R[r][i]));
    }
  for (int i = 0; i < kNlN; i++) x[L.perm[i]] = w1[i];
  for (int i = 0; i < kNlN; i++) w2[i] = __fmul_rn(L.diag[i], x[i]);
  float dxnorm = nl_blue6(w2);
  float fp = __fsub_rn(dxnorm, delta);
  if (fp <= __fmul_rn(0.1f, delta)) {
    for (int i = 0; i < kNlN; i++) L.wa1[i] = x[i];
    return 0.f;
  }
  float parl = 0.f;
  if (rank == kNlN) {
    for (int i = 0; i < kNlN; i++) w1[i] = __fdiv_rn(__fmul_rn(L.diag[L.perm[i]], w2[L.perm[i]]), dxnorm);
    for (int i = 0; i < kNlN; i++) {
      if (i > 0) {
        float dot = __fmul_rn(L.R[0][i], w1[0]);
        for (int s = 1; s < i; s++) dot = __fadd_rn(dot, __fmul_rn(L.R[s][i], w1[s]));
        w1[i] = __fsub_rn(w1[i], dot);
      }
      w1[i] = __fdiv_rn(w1[i], L.R[i][i]);
    }
    const float temp = nl_blue6(w1);
    parl = __fdiv_rn(__fdiv_rn(__fdiv_rn(fp, delta), temp), temp);
  }
  for (int j = 0; j < kNlN; j++) {
    float dot = __fmul_rn(L.R[0][j], L.qtf[0]);
    for (int i = 1; i <= j; i++) dot = __fadd_rn(dot, __fmul_rn(L.R[i][j], L.qtf[i]));
    w1[j] = __fdiv_rn(dot, L.diag[L.perm[j]]);
  }
  const float gnorm = nl_stable6(w1);
  float paru = __fdiv_rn(gnorm, delta);
  if (paru == 0.f) paru = __fdiv_rn(FLT_MIN, nl_min(delta, 0.1f));
  par = nl_max(par, parl);
  par = nl_min(par, paru);
  if (par == 0.f) par = __fdiv_rn(gnorm, dxnorm);
  for (int i = 0; i < kNlN; i++)
    for (int j = 0; j < kNlN; j++) L.S[i][j] = L.R[i][j];
  for (int it = 1;; it++) {
    if (par == 0.f) par = nl_max(FLT_MIN, __fmul_rn(0.001f, paru));
    const float sp = __fsqrt_rn(par);
    float d[kNlN];
    for (int i = 0; i < kNlN; i++) d[i] = __fmul_rn(sp, L.diag[i]);
    nl_qrsolv(L, d, x);
    for (int i = 0; i < kNlN; i++) w2[i] = __fmul_rn(L.diag[i], x[i]);
    dxnorm = nl_blue6(w2);
    float temp = fp;
    fp = __fsub_rn(dxnorm, delta);
    if (fabsf(fp) <= __fmul_rn(0.1f, delta) || (parl == 0.f && fp <= temp && temp < 0.f) || it == 10) break;
    for (int i = 0; i < kNlN; i++) w1[i] = __fmul_rn(L.diag[L.perm[i]], __fdiv_rn(w2[L.perm[i]], dxnorm));
    for (int j = 0; j < kNlN; j++) {
      w1[j] = __fdiv_rn(w1[j], L.sdiag[j]);
      temp = w1[j];
      for (int i = j + 1; i < kNlN; i++) w1[i] = __fsub_rn(w1[i], __fmul_rn(L.S[i][j], temp));
    }
    temp = nl_blue6(w1);
    const float parc = __fdiv_rn(__fdiv_rn(__fdiv_rn(fp, delta), temp), temp);
    if (fp > 0.f) parl = nl_max(parl, par);
    if (fp < 0.f) paru = nl_min(paru, par);
    par = nl_max(parl, __fadd_rn(par, parc));
  }
  for (int i = 0; i < kNlN; i++) L.wa1[i] = x[i];
  return par;
}

// ---- the CTA's Levenberg-Marquardt -------------------------------------------------------------------------------------------

// LevenbergMarquardt<NumericalDiff<...>, float>::minimize from x = 0 over r.m >= 6 rows; leaves x in L.x
__device__ void nl_minimize(const NlRows& r, float (*red)[kIcpThreads], NlLm& L) {
  const int m = r.m, tid = threadIdx.x;
  const float sqrt_eps = __fsqrt_rn(kNlEps);
  if (tid == 0) {
    for (int k = 0; k < kNlN; k++) L.x[k] = 0.f;
    L.cur = 0;
  }
  __syncthreads();
  nl_eval(r, L.x, r.f[0]);
  float fnorm = nl_stable_m(r.f[0], m, red, L);
  // thread 0's bookkeeping
  float par = 0.f, delta = 0.f, xnorm = 0.f, temp = 0.f;
  int iter = 1, nfev = 1;
#pragma unroll 1
  for (;;) {
    // 1. the forward-difference Jacobian (f(x) is the current residual vector)
    const float* fv = r.f[L.cur];
#pragma unroll 1
    for (int j = 0; j < kNlN; j++) {
      float x[kNlN], T[12];
#pragma unroll
      for (int k = 0; k < kNlN; k++) x[k] = L.x[k];
      float h = __fmul_rn(sqrt_eps, fabsf(x[j]));
      if (h == 0.f) h = sqrt_eps;
      x[j] = __fadd_rn(x[j], h);
      nl_warp(x, T);
      float* Jj = r.J[j];
      for (int i = tid; i < m; i += kIcpThreads)
        Jj[i] = __fdiv_rn(__fsub_rn(nl_residual(T, r.sx[i], r.sy[i], r.sz[i], r.tx[i], r.ty[i], r.tz[i]), fv[i]), h);
    }
    nfev += kNlN + 1;
    // 2. blueNorm and the squared norm of every column
    {
      const float ab2 = __fdiv_rn(kNlB2, (float)m);
      float v[4 * kNlN];
#pragma unroll
      for (int k = 0; k < 4 * kNlN; k++) v[k] = 0.f;
      for (int i = tid; i < m; i += kIcpThreads)
#pragma unroll
        for (int c = 0; c < kNlN; c++) {
          const float a = r.J[c][i];
          nl_blue_add(fabsf(a), ab2, v[c], v[kNlN + c], v[2 * kNlN + c]);
          v[3 * kNlN + c] = __fadd_rn(v[3 * kNlN + c], __fmul_rn(a, a));
        }
      icp_tree<4 * kNlN>(red, v);
      if (tid == 0)
        for (int c = 0; c < kNlN; c++) {
          L.cn[c] = nl_blue_finish(red[c][0], red[kNlN + c][0], red[2 * kNlN + c][0]);
          L.sq[c] = red[3 * kNlN + c][0];
          L.perm[c] = c;
        }
      __syncthreads();
    }
    // 3. ColPivHouseholderQR: logical column k lives in plane J[perm[k]]
    float thr = 0.f, maxpivot = 0.f;
    int nonzero = kNlN;
    if (tid == 0) {
      float mx = L.sq[0];
      for (int c = 1; c < kNlN; c++)
        if (L.sq[c] > mx) mx = L.sq[c];
      thr = __fdiv_rn(__fmul_rn(mx, __fmul_rn(kNlEps, kNlEps)), (float)m);
    }
#pragma unroll 1
    for (int k = 0; k < kNlN; k++) {
      if (tid == 0) {
        int big = k;
        for (int c = k + 1; c < kNlN; c++)
          if (L.sq[c] > L.sq[big]) big = c;
        L.big = big;
      }
      __syncthreads();
      {
        const float* col = r.J[L.perm[L.big]];
        float v[2] = {0.f, 0.f};
        for (int i = tid; i < m; i += kIcpThreads) {
          const float a = col[i];
          if (i >= k) v[0] = __fadd_rn(v[0], __fmul_rn(a, a));
          if (i > k) v[1] = __fadd_rn(v[1], __fmul_rn(a, a));
        }
        icp_tree<2>(red, v);
      }
      if (tid == 0) {
        const int big = L.big;
        const float bsq = red[0][0], tsq = red[1][0];
        L.sq[big] = bsq;
        if (nonzero == kNlN && bsq < __fmul_rn(thr, (float)(m - k))) nonzero = k;
        if (big != k) {
          float t = L.sq[k];
          L.sq[k] = L.sq[big];
          L.sq[big] = t;
          const int p = L.perm[k];
          L.perm[k] = L.perm[big];
          L.perm[big] = p;
        }
        float* col = r.J[L.perm[k]];
        const float c0 = col[k];
        float tau, beta;
        if (tsq <= FLT_MIN) {
          tau = 0.f;
          beta = c0;
          L.zero_tail = 1;
        } else {
          beta = __fsqrt_rn(__fadd_rn(__fmul_rn(c0, c0), tsq));
          if (c0 >= 0.f) beta = -beta;
          L.denom = __fsub_rn(c0, beta);
          tau = __fdiv_rn(__fsub_rn(beta, c0), beta);
          L.zero_tail = 0;
        }
        col[k] = beta;
        L.hc[k] = tau;
        L.tau = tau;
        if (fabsf(beta) > maxpivot) maxpivot = fabsf(beta);
      }
      __syncthreads();
      float* colk = r.J[L.perm[k]];
      const float tau = L.tau;
      {
        const int zt = L.zero_tail;
        const float den = L.denom;
        for (int i = k + 1 + tid; i < m; i += kIcpThreads) colk[i] = zt ? 0.f : __fdiv_rn(colk[i], den);
      }
      __syncthreads();
      if (tau != 0.f) {  // applyHouseholderOnTheLeft to the logical columns k + 1 ... 5
        float v[kNlN - 1];
        const float* cols[kNlN - 1];
#pragma unroll
        for (int c = 0; c < kNlN - 1; c++) {
          v[c] = 0.f;
          cols[c] = k + 1 + c < kNlN ? r.J[L.perm[k + 1 + c]] : colk;
        }
        for (int i = tid; i < m; i += kIcpThreads) {
          if (i <= k) continue;
          const float e = colk[i];
#pragma unroll
          for (int c = 0; c < kNlN - 1; c++)
            if (k + 1 + c < kNlN) v[c] = __fadd_rn(v[c], __fmul_rn(e, cols[c][i]));
        }
        icp_tree<kNlN - 1>(red, v);
        if (tid == 0)
          for (int c = k + 1; c < kNlN; c++) {
            float* col = r.J[L.perm[c]];
            const float t = __fadd_rn(red[c - k - 1][0], col[k]);
            col[k] = __fsub_rn(col[k], __fmul_rn(tau, t));
            L.tmp[c] = t;
          }
        __syncthreads();
        for (int i = k + 1 + tid; i < m; i += kIcpThreads) {
          const float te = __fmul_rn(tau, colk[i]);
          for (int c = k + 1; c < kNlN; c++) {
            float* col = r.J[L.perm[c]];
            col[i] = __fsub_rn(col[i], __fmul_rn(te, L.tmp[c]));
          }
        }
        __syncthreads();
      }
      if (tid == 0)
        for (int c = k + 1; c < kNlN; c++) {
          const float a = r.J[L.perm[c]][k];
          L.sq[c] = __fsub_rn(L.sq[c], __fmul_rn(a, a));
        }
    }
    // 4. thread 0: R, the rank, the first iteration's scaling; all: Q^T f
    int rank = 0;
    if (tid == 0) {
      for (int i = 0; i < kNlN; i++)
        for (int j = 0; j < kNlN; j++) L.R[i][j] = r.J[L.perm[j]][i];
      const float pthr = __fmul_rn(maxpivot, __fmul_rn(kNlEps, (float)min(m, kNlN)));
      for (int i = 0; i < nonzero; i++) rank += fabsf(L.R[i][i]) > pthr;
      if (iter == 1) {
        float w[kNlN];
        for (int j = 0; j < kNlN; j++) L.diag[j] = L.cn[j] == 0.f ? 1.f : L.cn[j];
        for (int j = 0; j < kNlN; j++) w[j] = __fmul_rn(L.diag[j], L.x[j]);
        xnorm = nl_stable6(w);
        delta = __fmul_rn(kNlFactor, xnorm);
        if (delta == 0.f) delta = kNlFactor;
      }
    }
    for (int i = tid; i < m; i += kIcpThreads) r.q[i] = fv[i];
    __syncthreads();
#pragma unroll 1
    for (int k = 0; k < kNlN; k++) {
      const float tau = L.hc[k];
      if (tau == 0.f) continue;
      const float* ess = r.J[L.perm[k]];
      float v[1] = {0.f};
      for (int i = tid; i < m; i += kIcpThreads)
        if (i > k) v[0] = __fadd_rn(v[0], __fmul_rn(ess[i], r.q[i]));
      icp_tree<1>(red, v);
      if (tid == 0) {
        const float t = __fadd_rn(red[0][0], r.q[k]);
        r.q[k] = __fsub_rn(r.q[k], __fmul_rn(tau, t));
        L.tmp[0] = t;
      }
      __syncthreads();
      const float t = L.tmp[0];
      for (int i = k + 1 + tid; i < m; i += kIcpThreads) r.q[i] = __fsub_rn(r.q[i], __fmul_rn(__fmul_rn(tau, ess[i]), t));
      __syncthreads();
    }
    // 5. thread 0: the gradient test and the rescaling
    if (tid == 0) {
      for (int i = 0; i < kNlN; i++) L.qtf[i] = r.q[i];
      float gnorm = 0.f;
      if (fnorm != 0.f)
        for (int j = 0; j < kNlN; j++) {
          const float w = L.cn[L.perm[j]];
          if (w != 0.f) {
            float dot = __fmul_rn(L.R[0][j], __fdiv_rn(L.qtf[0], fnorm));
            for (int i = 1; i <= j; i++) dot = __fadd_rn(dot, __fmul_rn(L.R[i][j], __fdiv_rn(L.qtf[i], fnorm)));
            gnorm = nl_max(gnorm, fabsf(__fdiv_rn(dot, w)));
          }
        }
      L.flag = gnorm <= 0.f ? 2 : 0;  // CosinusTooSmall (gtol = 0)
      L.tau = gnorm;                  // kept for the GtolTooSmall test
      for (int j = 0; j < kNlN; j++) L.diag[j] = nl_max(L.diag[j], L.cn[j]);
    }
    __syncthreads();
    if (L.flag == 2) break;
    const float gnorm = L.tau;
    __syncthreads();
    // 6. the inner loop: trial steps until one succeeds or a test ends the minimisation
#pragma unroll 1
    for (;;) {
      float pnorm = 0.f;
      if (tid == 0) {
        par = nl_lmpar(L, rank, delta, par);
        float w[kNlN];
        for (int i = 0; i < kNlN; i++) {
          L.wa1[i] = -L.wa1[i];
          L.xt[i] = __fadd_rn(L.x[i], L.wa1[i]);
          w[i] = __fmul_rn(L.diag[i], L.wa1[i]);
        }
        pnorm = nl_stable6(w);
        if (iter == 1) delta = nl_min(delta, pnorm);
      }
      __syncthreads();
      float* ft = r.f[1 - L.cur];
      nl_eval(r, L.xt, ft);
      const float fnorm1 = nl_stable_m(ft, m, red, L);
      if (tid == 0) {
        nfev++;
        float actred = -1.f;
        if (__fmul_rn(0.1f, fnorm1) < fnorm) {
          const float q = __fdiv_rn(fnorm1, fnorm);
          actred = __double2float_rn(__dsub_rn(1.0, (double)__fmul_rn(q, q)));  // 1. - abs2(..) in double
        }
        float w3[kNlN];
        for (int rr = 0; rr < kNlN; rr++) {
          float s = 0.f;
          for (int i = rr; i < kNlN; i++) s = __fadd_rn(s, __fmul_rn(L.wa1[L.perm[i]], L.R[rr][i]));
          w3[rr] = s;
        }
        float q = __fdiv_rn(nl_stable6(w3), fnorm);
        const float temp1 = __fmul_rn(q, q);
        q = __fdiv_rn(__fmul_rn(__fsqrt_rn(par), pnorm), fnorm);
        const float temp2 = __fmul_rn(q, q);
        const float prered = __fadd_rn(temp1, __fdiv_rn(temp2, 0.5f));
        const float dirder = -__fadd_rn(temp1, temp2);
        float ratio = 0.f;
        if (prered != 0.f) ratio = __fdiv_rn(actred, prered);
        if (ratio <= 0.25f) {
          if (actred >= 0.f) temp = 0.5f;
          if (actred < 0.f) temp = __fdiv_rn(__fmul_rn(0.5f, dirder), __fadd_rn(dirder, __fmul_rn(0.5f, actred)));
          if (__fmul_rn(0.1f, fnorm1) >= fnorm || temp < 0.1f) temp = 0.1f;
          delta = __fmul_rn(temp, nl_min(delta, __fdiv_rn(pnorm, 0.1f)));
          par = __fdiv_rn(par, temp);
        } else if (!(par != 0.f && ratio < 0.75f)) {
          delta = __fdiv_rn(pnorm, 0.5f);
          par = __fmul_rn(0.5f, par);
        }
        if (ratio >= 1e-4f) {
          float w[kNlN];
          for (int i = 0; i < kNlN; i++) {
            L.x[i] = L.xt[i];
            w[i] = __fmul_rn(L.diag[i], L.x[i]);
          }
          xnorm = nl_stable6(w);
          L.cur = 1 - L.cur;
          fnorm = fnorm1;
          iter++;
        }
        const bool small = fabsf(actred) <= sqrt_eps && prered <= sqrt_eps && __fmul_rn(0.5f, ratio) <= 1.f;
        const bool done = (small && delta <= __fmul_rn(sqrt_eps, xnorm)) || small || delta <= __fmul_rn(sqrt_eps, xnorm) ||
                          nfev >= kNlMaxfev ||
                          (fabsf(actred) <= kNlEps && prered <= kNlEps && __fmul_rn(0.5f, ratio) <= 1.f) ||
                          delta <= __fmul_rn(kNlEps, xnorm) || gnorm <= kNlEps;
        L.flag = done ? 2 : (ratio < 1e-4f ? 0 : 1);
      }
      __syncthreads();
      const int flag = L.flag;
      __syncthreads();
      if (flag == 2) return;
      if (flag == 1) break;
    }
  }
}

// ---- the estimator -----------------------------------------------------------------------------------------------------------

// TransformationEstimationLM for k_icp_align: the correspondences compacted in source order into the pair's work rows, the
// LM from x = 0, and T_inc = WarpPointRigid6D(x).  With fewer rows than parameters Eigen refuses and x stays 0.
struct IcpLm {
  static constexpr int kMinCorrespondences = 4;
  static constexpr int kMinBlocks = 2;  // at most 128 registers: the LM fits them without spills
  static constexpr int kPlanes = kJ0 + kNlN;
  struct Shared {
    float red[4 * kNlN][kIcpThreads];
    NlLm L;
    int warp[kIcpThreads / 32];
  };
  NlRows rows;

  __device__ IcpLm(Shared&, float* w, long long wplane) {
    const auto plane = [&](int k) { return w + k * wplane; };
    rows.sx = plane(kSx), rows.sy = plane(kSx + 1), rows.sz = plane(kSx + 2);
    rows.tx = plane(kTx), rows.ty = plane(kTx + 1), rows.tz = plane(kTx + 2);
    rows.f[0] = plane(kF0);
    rows.f[1] = plane(kF0 + 1);
    rows.q = plane(kQf);
#pragma unroll
    for (int c = 0; c < kNlN; c++) rows.J[c] = plane(kJ0 + c);
  }
  __device__ void add(float, float, float, float, float, float) {}
  __device__ int count(Shared& sh, const IcpPass& p, int) {  // the compaction; this thread reads only the cr it wrote in the search
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    int m = 0;
#pragma unroll 1
    for (int base = 0; base < p.ns; base += kIcpThreads) {
      const int i = base + threadIdx.x;
      const int j = i < p.ns ? p.cr[i] : -1;
      const unsigned bal = __ballot_sync(0xffffffffu, j >= 0);
      if (lane == 0) sh.warp[wid] = __popc(bal);
      __syncthreads();
      int before = 0, sum = 0;
#pragma unroll
      for (int q = 0; q < kIcpThreads / 32; q++) {
        const int c = sh.warp[q];
        before += q < wid ? c : 0;
        sum += c;
      }
      if (j >= 0) {
        const int at = m + before + __popc(bal & ((1u << lane) - 1u));
        rows.sx[at] = p.x[i];
        rows.sy[at] = p.y[i];
        rows.sz[at] = p.z[i];
        rows.tx[at] = p.tg.x[j];
        rows.ty[at] = p.tg.y[j];
        rows.tz[at] = p.tg.z[j];
      }
      m += sum;
      __syncthreads();
    }
    return m;
  }
  __device__ void estimate(Shared& sh, const IcpPass&, int n) {
    if (n >= kNlN) {
      rows.m = n;
      nl_minimize(rows, sh.red, sh.L);
    } else if (threadIdx.x == 0) {
      for (int k = 0; k < kNlN; k++) sh.L.x[k] = 0.f;
    }
  }
  __device__ void increment(Shared& sh, float (&T)[12]) {
    float x[kNlN];
    for (int k = 0; k < kNlN; k++) x[k] = sh.L.x[k];
    nl_warp(x, T);
  }
};

template struct IcpAlign<IcpLm>;

}  // namespace rb200
