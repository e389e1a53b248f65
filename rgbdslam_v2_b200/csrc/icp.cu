// icp.cu -- the ICP fallback of Node::matchNodePair (node.cpp:1356-1377): icpAlignment(filterCloud(older->pc_col),
// filterCloud(this->pc_col), Identity) (icp.cpp:20-89), PCL 1.7's pcl::IterativeClosestPoint<PointXYZRGB, PointXYZRGB>.
//   k_icp_filter  one CTA per distinct node: stable compaction of the points whose z is not NaN, filterCloud's float step walk
//                 (one thread: it is a chain of float additions), then the kept points' coordinates
//   k_icp_cells   one CTA per distinct target: the finite kept points' cells of side 1/16 m, stably sorted by cell key
//                 (8-bit LSD radix passes in global memory), so that a cell's points stay in index order
//   IcpSvd        the estimator of k_icp_align<IcpSvd> (icp.cuh): the Umeyama sums, then on thread 0 the 3 x 3 Jacobi SVD
// Points are read through map_point (map.cuh), as stored.  Every float operation is an explicit _rn intrinsic (no
// contraction, no approximate division or square root), so tests/icp_exact.py replays the kernels bit for bit.
#include "icp.cuh"

namespace rb200 {

constexpr int kIcpFilterThreads = 1024;
constexpr int kIcpSvdSweeps = 32;       // never reached by a float 3 x 3 in practice; it bounds the loop

__device__ __forceinline__ MapArgs icp_args() { return MapArgs{0.f, 0, 1, 0, 32}; }  // as stored: no filter, no transform

// ---- filterCloud ----------------------------------------------------------------------------------------------------------

__global__ void __launch_bounds__(kIcpFilterThreads) k_icp_filter(const IcpNode* __restrict__ nodes, int desired,
                                                                  int* __restrict__ scratch, float* __restrict__ pts, long long plane,
                                                                  int* __restrict__ nf) {
  __shared__ int warp_cnt[kIcpFilterThreads / 32];
  __shared__ int s_n;
  const IcpNode& u = nodes[blockIdx.x];
  const MapArgs a = icp_args();
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  int* list = scratch + u.scratch0;
  int total = 0;
  for (int base = 0; base < u.P; base += kIcpFilterThreads) {  // the indices of the non-NaN z, in storage order
    const int i = base + threadIdx.x;
    bool keep = false;
    if (i < u.P) {
      MapOut o;
      map_point(u.src, i, a, o);
      keep = !isnan(o.z);
    }
    const unsigned bal = __ballot_sync(0xffffffffu, keep);
    if (lane == 0) warp_cnt[wid] = __popc(bal);
    __syncthreads();
    int before = 0, sum = 0;
#pragma unroll 8
    for (int w = 0; w < kIcpFilterThreads / 32; w++) {
      const int c = warp_cnt[w];
      before += w < wid ? c : 0;
      sum += c;
    }
    if (keep) list[total + before + __popc(bal & ((1u << lane) - 1u))] = i;
    total += sum;
    __syncthreads();
  }
  float* px = pts + u.f0;
  float* py = px + plane;
  float* pz = py + plane;
  int* rank = reinterpret_cast<int*>(pz);  // the walk's ranks, replaced by z point by point below
  // float step = n / (float)desired, at least 1; for (float i = 0; i < n; i += step) keep rank (unsigned)i
  const float step0 = __fdiv_rn((float)total, (float)desired);
  const float step = step0 < 1.0f ? 1.0f : step0;
  const bool walk = step != 1.0f;  // with step 1 the walk visits 0, 1, ..., n - 1 exactly (n < 2^24)
  int nout = total;
  if (walk) {
    if (threadIdx.x == 0) {
      int k = 0;
      for (float f = 0.f; f < (float)total; f = __fadd_rn(f, step), k++)
        if (k < u.cap) rank[k] = (int)f;
      s_n = k;
    }
    __syncthreads();
    nout = min(s_n, u.cap);
  }
  for (int k = threadIdx.x; k < nout; k += kIcpFilterThreads) {
    MapOut o;
    map_point(u.src, list[walk ? rank[k] : k], a, o);
    px[k] = o.x;
    py[k] = o.y;
    pz[k] = o.z;
  }
  if (threadIdx.x == 0) nf[blockIdx.x] = walk ? s_n : total;  // > cap only if the host's bound were wrong: reported as an error
}

// ---- the target's cells ---------------------------------------------------------------------------------------------------

__global__ void __launch_bounds__(kIcpThreads) k_icp_cells(const IcpNode* __restrict__ nodes, const int* __restrict__ targets,
                                                           const float* __restrict__ pts, long long plane, const int* __restrict__ nf,
                                                           unsigned long long* __restrict__ key0, int* __restrict__ idx0,
                                                           unsigned long long* __restrict__ key1, int* __restrict__ idx1,
                                                           int* __restrict__ nfin) {
  __shared__ int warp_cnt[kIcpThreads / 32];
  __shared__ int warp_pos[kIcpThreads / 32][256];
  __shared__ int next[256];
  __shared__ int s_single;
  const int u = targets[blockIdx.x];
  const long long f0 = nodes[u].f0;
  const int n = nf[u];
  const float* px = pts + f0;
  const float* py = px + plane;
  const float* pz = py + plane;
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  unsigned long long *kin = key0 + f0, *kout = key1 + f0;
  int *iin = idx0 + f0, *iout = idx1 + f0;
  int m = 0;
  for (int base = 0; base < n; base += kIcpThreads) {  // the finite points with their keys, in index order
    const int i = base + threadIdx.x;
    const bool fin = i < n && icp_finite(px[i], py[i], pz[i]);
    const unsigned bal = __ballot_sync(0xffffffffu, fin);
    if (lane == 0) warp_cnt[wid] = __popc(bal);
    __syncthreads();
    int before = 0, sum = 0;
#pragma unroll
    for (int w = 0; w < kIcpThreads / 32; w++) {
      const int c = warp_cnt[w];
      before += w < wid ? c : 0;
      sum += c;
    }
    if (fin) {
      const int at = m + before + __popc(bal & ((1u << lane) - 1u));
      kin[at] = icp_key(icp_cell(px[i]), icp_cell(py[i]), icp_cell(pz[i]));
      iin[at] = i;
    }
    m += sum;
    __syncthreads();
  }
#pragma unroll 1
  for (int shift = 0; shift < 48; shift += 8) {  // stable LSD radix sort; a pass whose digit is the same everywhere is skipped
    int* hist = next;
    hist[threadIdx.x] = 0;
    __syncthreads();
    for (int i = threadIdx.x; i < m; i += kIcpThreads) atomicAdd(&hist[(int)((kin[i] >> shift) & 255u)], 1);
    __syncthreads();
    if (threadIdx.x == 0) {
      int run = 0, single = 0;
      for (int d = 0; d < 256; d++) {
        const int c = hist[d];
        single |= c == m;
        hist[d] = run;
        run += c;
      }
      s_single = single;
    }
    __syncthreads();
    if (s_single) continue;
#pragma unroll 1
    for (int base = 0; base < m; base += kIcpThreads) {
#pragma unroll
      for (int w = 0; w < kIcpThreads / 32; w++) warp_pos[w][threadIdx.x] = 0;
      __syncthreads();
      const int i = base + threadIdx.x;
      const bool valid = i < m;
      const unsigned long long k = valid ? kin[i] : 0ull;
      const int id = valid ? iin[i] : 0;
      const int d = (int)((k >> shift) & 255u);
      const unsigned peers = __match_any_sync(0xffffffffu, valid ? d : 256 + lane);
      if (valid && lane == __ffs(peers) - 1) warp_pos[wid][d] = __popc(peers);
      __syncthreads();
      {
        int acc = next[threadIdx.x];
#pragma unroll
        for (int w = 0; w < kIcpThreads / 32; w++) {
          const int t = warp_pos[w][threadIdx.x];
          warp_pos[w][threadIdx.x] = acc;
          acc += t;
        }
        next[threadIdx.x] = acc;
      }
      __syncthreads();
      if (valid) {
        const int dst = warp_pos[wid][d] + __popc(peers & ((1u << lane) - 1u));
        kout[dst] = k;
        iout[dst] = id;
      }
      __syncthreads();
    }
    unsigned long long* tk = kin;
    kin = kout;
    kout = tk;
    int* ti = iin;
    iin = iout;
    iout = ti;
  }
  if (kin != key0 + f0) {
    for (int i = threadIdx.x; i < m; i += kIcpThreads) {
      key0[f0 + i] = kin[i];
      idx0[f0 + i] = iin[i];
    }
  }
  if (threadIdx.x == 0) nfin[u] = m;
}

// ---- alignment ------------------------------------------------------------------------------------------------------------

// x' = c x + s y, y' = -s x + c y (Eigen's apply_rotation_in_the_plane)
__device__ __forceinline__ void icp_rot(float& x, float& y, float c, float s) {
  const float a = __fadd_rn(__fmul_rn(c, x), __fmul_rn(s, y));
  y = __fadd_rn(__fmul_rn(-s, x), __fmul_rn(c, y));
  x = a;
}

// One step of the two-sided Jacobi SVD on the (p, q) plane (Eigen's JacobiSVD, real_2x2_jacobi_svd and makeJacobi).
// Returns false when the off-diagonal pair is already below the threshold.
template <int p, int q>
__device__ __forceinline__ bool icp_jacobi(float (&W)[3][3], float (&U)[3][3], float (&V)[3][3]) {
  const float thr = fmaxf(1.40129846e-45f * 2.f, __fmul_rn(2.38418579e-7f, fmaxf(fabsf(W[p][p]), fabsf(W[q][q]))));
  if (!(fmaxf(fabsf(W[p][q]), fabsf(W[q][p])) > thr)) return false;
  const float m00 = W[p][p], m01 = W[p][q], m10 = W[q][p], m11 = W[q][q];
  const float t = __fadd_rn(m00, m11), d = __fsub_rn(m10, m01);
  float c1, s1;
  if (t == 0.f) {
    c1 = 0.f;
    s1 = d > 0.f ? 1.f : -1.f;
  } else {
    const float u = __fdiv_rn(d, t);
    c1 = __fdiv_rn(1.f, __fsqrt_rn(__fadd_rn(1.f, __fmul_rn(u, u))));
    s1 = __fmul_rn(c1, u);
  }
  float a00 = m00, a10 = m10, a01 = m01, a11 = m11;
  icp_rot(a00, a10, c1, s1);
  icp_rot(a01, a11, c1, s1);
  float c2 = 1.f, s2 = 0.f;
  if (a01 != 0.f) {
    const float tau = __fdiv_rn(__fsub_rn(a00, a11), __fmul_rn(2.f, fabsf(a01)));
    const float w = __fsqrt_rn(__fadd_rn(__fmul_rn(tau, tau), 1.f));
    const float tt = tau > 0.f ? __fdiv_rn(1.f, __fadd_rn(tau, w)) : __fdiv_rn(1.f, __fsub_rn(tau, w));
    const float nn = __fdiv_rn(1.f, __fsqrt_rn(__fadd_rn(__fmul_rn(tt, tt), 1.f)));
    const float mag = __fmul_rn(fabsf(tt), nn);
    s2 = (tt > 0.f) == (a01 > 0.f) ? -mag : mag;  // -sign(t) * sign(y) * |t| * n
    c2 = nn;
  }
  const float cl = __fadd_rn(__fmul_rn(c1, c2), __fmul_rn(s1, s2)), sl = __fsub_rn(__fmul_rn(s1, c2), __fmul_rn(c1, s2));
#pragma unroll
  for (int k = 0; k < 3; k++) icp_rot(W[p][k], W[q][k], cl, sl);
#pragma unroll
  for (int k = 0; k < 3; k++) icp_rot(U[k][p], U[k][q], cl, sl);
#pragma unroll
  for (int k = 0; k < 3; k++) icp_rot(W[k][p], W[k][q], c2, -s2);
#pragma unroll
  for (int k = 0; k < 3; k++) icp_rot(V[k][p], V[k][q], c2, -s2);
  return true;
}

template <int a, int b>
__device__ __forceinline__ void icp_swap(float (&s)[3], float (&U)[3][3], float (&V)[3][3]) {
  float t = s[a];
  s[a] = s[b];
  s[b] = t;
#pragma unroll
  for (int k = 0; k < 3; k++) {
    t = U[k][a], U[k][a] = U[k][b], U[k][b] = t;
    t = V[k][a], V[k][a] = V[k][b], V[k][b] = t;
  }
}

__device__ __forceinline__ float icp_det3(const float (&M)[3][3]) {
  const float a = __fsub_rn(__fmul_rn(M[1][1], M[2][2]), __fmul_rn(M[1][2], M[2][1]));
  const float b = __fsub_rn(__fmul_rn(M[1][0], M[2][2]), __fmul_rn(M[1][2], M[2][0]));
  const float c = __fsub_rn(__fmul_rn(M[1][0], M[2][1]), __fmul_rn(M[1][1], M[2][0]));
  return __fadd_rn(__fsub_rn(__fmul_rn(M[0][0], a), __fmul_rn(M[0][1], b)), __fmul_rn(M[0][2], c));
}

// TransformationEstimationSVD (Eigen's umeyama without scaling) from the sums: R = U S V^T, t = dst_mean - R src_mean.
__device__ __forceinline__ void icp_umeyama(const float (&sigma)[3][3], const float (&sm)[3], const float (&dm)[3], float (&T)[12]) {
  float W[3][3], U[3][3], V[3][3];
#pragma unroll
  for (int i = 0; i < 3; i++)
#pragma unroll
    for (int j = 0; j < 3; j++) {
      W[i][j] = sigma[i][j];
      U[i][j] = V[i][j] = i == j ? 1.f : 0.f;
    }
#pragma unroll 1
  for (int sweep = 0; sweep < kIcpSvdSweeps; sweep++) {
    bool rotated = icp_jacobi<1, 0>(W, U, V);
    rotated |= icp_jacobi<2, 0>(W, U, V);
    rotated |= icp_jacobi<2, 1>(W, U, V);
    if (!rotated) break;
  }
  float s[3];
#pragma unroll
  for (int i = 0; i < 3; i++) {
    s[i] = fabsf(W[i][i]);
    if (W[i][i] < 0.f)
#pragma unroll
      for (int k = 0; k < 3; k++) U[k][i] = -U[k][i];
  }
  // descending singular values; the first of equal maxima stays first; stop at a zero maximum
  if (!(s[0] == 0.f && s[1] == 0.f && s[2] == 0.f)) {
    const int p0 = s[1] > s[0] ? (s[2] > s[1] ? 2 : 1) : (s[2] > s[0] ? 2 : 0);
    if (p0 == 1) icp_swap<0, 1>(s, U, V);
    if (p0 == 2) icp_swap<0, 2>(s, U, V);
    if (s[2] > s[1] && s[1] != s[2]) icp_swap<1, 2>(s, U, V);
  }
  if (__fmul_rn(icp_det3(U), icp_det3(V)) < 0.f)
#pragma unroll
    for (int k = 0; k < 3; k++) U[k][2] = -U[k][2];
#pragma unroll
  for (int i = 0; i < 3; i++)
#pragma unroll
    for (int j = 0; j < 3; j++) T[4 * i + j] = icp_dot3(U[i][0], V[j][0], U[i][1], V[j][1], U[i][2], V[j][2]);
#pragma unroll
  for (int i = 0; i < 3; i++) T[4 * i + 3] = __fsub_rn(dm[i], icp_dot3(T[4 * i], sm[0], T[4 * i + 1], sm[1], T[4 * i + 2], sm[2]));
}

// TransformationEstimationSVD for k_icp_align: the means (summed in the search) and sigma, then Umeyama on thread 0.
struct IcpSvd {
  static constexpr int kMinCorrespondences = 3;
  static constexpr int kMinBlocks = 3;  // at most 80 registers, without spills
  static constexpr int kPlanes = 3;  // the moving source only
  struct Shared {
    float red[9][kIcpThreads];
    int cnt;
  };
  float v[6];  // this thread's sums of the source and target coordinates
  float inv_n, sm[3], dm[3];

  __device__ IcpSvd(Shared& sh, float*, long long) : v{0.f, 0.f, 0.f, 0.f, 0.f, 0.f} {
    if (threadIdx.x == 0) sh.cnt = 0;
  }
  __device__ void add(float x, float y, float z, float tx, float ty, float tz) {
    v[0] = __fadd_rn(v[0], x);
    v[1] = __fadd_rn(v[1], y);
    v[2] = __fadd_rn(v[2], z);
    v[3] = __fadd_rn(v[3], tx);
    v[4] = __fadd_rn(v[4], ty);
    v[5] = __fadd_rn(v[5], tz);
  }
  __device__ int count(Shared& sh, const IcpPass&, int c) {
    if (c) atomicAdd(&sh.cnt, c);
    icp_tree<6>(sh.red, v);
#pragma unroll
    for (int k = 0; k < 6; k++) v[k] = 0.f;
    return sh.cnt;
  }
  __device__ void estimate(Shared& sh, const IcpPass& p, int n) {
    inv_n = __fdiv_rn(1.f, (float)n);
#pragma unroll
    for (int k = 0; k < 3; k++) {
      sm[k] = __fmul_rn(sh.red[k][0], inv_n);
      dm[k] = __fmul_rn(sh.red[3 + k][0], inv_n);
    }
    __syncthreads();
    // sigma = (1/n) dst_demean src_demean^T
    float s[9] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
    for (int i = threadIdx.x; i < p.ns; i += kIcpThreads) {
      const int j = p.cr[i];
      if (j < 0) continue;
      const float sd[3] = {__fsub_rn(p.x[i], sm[0]), __fsub_rn(p.y[i], sm[1]), __fsub_rn(p.z[i], sm[2])};
      const float dd[3] = {__fsub_rn(p.tg.x[j], dm[0]), __fsub_rn(p.tg.y[j], dm[1]), __fsub_rn(p.tg.z[j], dm[2])};
#pragma unroll
      for (int r = 0; r < 3; r++)
#pragma unroll
        for (int q = 0; q < 3; q++) s[3 * r + q] = __fadd_rn(s[3 * r + q], __fmul_rn(dd[r], sd[q]));
    }
    icp_tree<9>(sh.red, s);
  }
  __device__ void increment(Shared& sh, float (&T)[12]) {
    float sigma[3][3];
#pragma unroll
    for (int r = 0; r < 3; r++)
#pragma unroll
      for (int q = 0; q < 3; q++) sigma[r][q] = __fmul_rn(inv_n, sh.red[3 * r + q][0]);
    icp_umeyama(sigma, sm, dm, T);
    sh.cnt = 0;  // every thread read it before estimate's barriers
  }
};

// ---- launchers -------------------------------------------------------------------------------------------------------------

cudaError_t launch_icp_filter(const IcpNode* d_nodes, int nnodes, int desired, int* scratch, float* pts, long long plane, int* nf,
                              cudaStream_t st) {
  if (nnodes <= 0) return cudaSuccess;
  k_icp_filter<<<nnodes, kIcpFilterThreads, 0, st>>>(d_nodes, desired, scratch, pts, plane, nf);
  return cudaGetLastError();
}

cudaError_t launch_icp_cells(const IcpNode* d_nodes, const int* targets, int ntargets, const float* pts, long long plane, const int* nf,
                             unsigned long long* key[2], int* idx[2], int* nfin, cudaStream_t st) {
  if (ntargets <= 0) return cudaSuccess;
  k_icp_cells<<<ntargets, kIcpThreads, 0, st>>>(d_nodes, targets, pts, plane, nf, key[0], idx[0], key[1], idx[1], nfin);
  return cudaGetLastError();
}

int icp_work_planes(int method) {
  return method == RGBDSLAM_B200_ICP_METHOD_ICP_NL ? IcpAlign<IcpLm>::planes() : IcpAlign<IcpSvd>::planes();
}

cudaError_t launch_icp_align(int method, const IcpPair* pairs, int npairs, const IcpNode* d_nodes, const float* pts, long long plane,
                             const int* nf, const unsigned long long* key, const int* idx, const int* nfin, float* work,
                             long long wplane, int* corr, float* dist, rgbdslam_b200_icp_result* results, cudaStream_t st) {
  return (method == RGBDSLAM_B200_ICP_METHOD_ICP_NL ? IcpAlign<IcpLm>::launch : IcpAlign<IcpSvd>::launch)(
      pairs, npairs, d_nodes, pts, plane, nf, key, idx, nfin, work, wplane, corr, dist, results, st);
}

}  // namespace rb200
