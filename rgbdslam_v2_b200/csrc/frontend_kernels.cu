// frontend_kernels.cu -- sm_90a kernels of the frame-pair hot path:
//   hamming_simt_kernel    : bruteForceSearchORB (features.cpp:168-182) for every query row of every pair
//   select_matches_kernel  : hd<128 filter, jitter distance, sort, keepStrongestMatches (node.cpp:572-573,674,1127)
//   ransac_hyp_kernel      : one warp per RANSAC hypothesis (node.cpp:1130-1169) -- sample 4, weighted Kabsch
//                            (transformation_estimation_euclidean.cpp:7-61), Mahalanobis scoring
//                            (node.cpp:968-1020, misc.cpp:697-770) with __ballot_sync inlier masks, <=19 refits
//   ransac_select_kernel   : sequential replay of the best-hypothesis bookkeeping incl. the n+=10 / break
//                            shortcuts (node.cpp:1170-1216), identity last resort, edge (node.cpp:1335-1339)
#include "kernels.h"
#include "se3_point.cuh"

namespace rb200 {

__constant__ DevParams c_params;

cudaError_t set_dev_params(const DevParams& p, cudaStream_t stream) {
  return cudaMemcpyToSymbolAsync(c_params, &p, sizeof(DevParams), 0, cudaMemcpyHostToDevice, stream);
}

// =====================================================================================================
// Hamming brute force, SIMT popcount version.
// One thread per query descriptor (8 x u32 in registers), train descriptors staged through shared
// memory in tiles and read as broadcast LDS.128.  Reference semantics kept bit-exactly:
//   - only train rows [0, nt-2] are examined (loop bound `i < size-1`, features.cpp:174)
//   - strict `<` while scanning upwards => lowest index wins ties (features.cpp:176)
//   - no candidate => (257, -1) (features.cpp:172-173)
constexpr int kHamQ = 128;  // queries per CTA
constexpr int kHamT = 128;  // train rows per smem tile

__global__ void __launch_bounds__(kHamQ) hamming_simt_kernel(const PairDesc* __restrict__ pairs,
                                                             int2* __restrict__ best, int stride) {
  const PairDesc pd = pairs[blockIdx.y];
  const int q0 = blockIdx.x * kHamQ;
  if (q0 >= pd.nq) return;
  __shared__ uint4 tile[kHamT * 2];
  const int qi = q0 + threadIdx.x;
  const bool qvalid = qi < pd.nq;
  uint4 qa = make_uint4(0, 0, 0, 0), qb = qa;
  if (qvalid) {
    const uint4* qp = reinterpret_cast<const uint4*>(pd.q_desc) + 2 * (size_t)qi;
    qa = __ldg(qp);
    qb = __ldg(qp + 1);
  }
  int best_hd = 257, best_idx = -1;
  const int nsearch = pd.nt - 1;
  const uint4* tp = reinterpret_cast<const uint4*>(pd.t_desc);
  for (int t0 = 0; t0 < nsearch; t0 += kHamT) {
    const int cnt = min(kHamT, nsearch - t0);
    __syncthreads();
    for (int k = threadIdx.x; k < 2 * cnt; k += kHamQ) tile[k] = __ldg(tp + 2 * (size_t)t0 + k);
    __syncthreads();
#pragma unroll 4
    for (int j = 0; j < cnt; j++) {
      const uint4 a = tile[2 * j], b = tile[2 * j + 1];
      const int d = (__popc(qa.x ^ a.x) + __popc(qa.y ^ a.y)) + (__popc(qa.z ^ a.z) + __popc(qa.w ^ a.w)) +
                    (__popc(qb.x ^ b.x) + __popc(qb.y ^ b.y)) + (__popc(qb.z ^ b.z) + __popc(qb.w ^ b.w));
      if (d < best_hd) {
        best_hd = d;
        best_idx = t0 + j;
      }
    }
  }
  if (qvalid) best[(size_t)blockIdx.y * stride + qi] = make_int2(best_hd, best_idx);
}

cudaError_t launch_hamming_simt(const PairDesc* pairs, int npairs, int max_nq, int2* best, int stride,
                                cudaStream_t stream) {
  if (npairs <= 0 || max_nq <= 0) return cudaSuccess;
  dim3 grid((max_nq + kHamQ - 1) / kHamQ, npairs);
  hamming_simt_kernel<<<grid, kHamQ, 0, stream>>>(pairs, best, stride);
  return cudaGetLastError();
}

// =====================================================================================================
// Match selection.  distance = hd/256.0 + (float)rand()/(1000.0*RAND_MAX) (node.cpp:573) with rand()
// replaced by rand31(pair key, stream 0, queryIdx); keepStrongestMatches + std::sort == ascending sort by
// (distance, queryIdx) and truncation to max_matches.  One CTA per pair, bitonic sort in shared memory.
// Switches for the two restructured selection kernels (the first versions stay in the file as the fallback).
#ifndef RB200_SELECT_PARTIAL
#define RB200_SELECT_PARTIAL 1  // select_matches_kernel: sort only the matches below the distance cut (0 = sort all keys)
#endif
#ifndef RB200_SELECT_STAGED
#define RB200_SELECT_STAGED 1  // ransac_select_kernel: loads issued up front, 32-wide scan (0 = the first, serial version)
#endif
constexpr int kSelThreads = 512;

__device__ __forceinline__ float match_distance(int hd, uint32_t r31) {
  const double d = __dadd_rn(__ddiv_rn((double)hd, 256.0), __ddiv_rn((double)(float)r31, 1000.0 * 2147483647.0));
  return __double2float_rn(d);
}

__global__ void __launch_bounds__(kSelThreads)
    select_matches_kernel(const PairDesc* __restrict__ pairs, const int2* __restrict__ best, int stride, uint64_t seed,
                          int64_t first_pair, rgbdslam_b200_dmatch* __restrict__ matches, float4* __restrict__ mfrom,
                          float4* __restrict__ mto, int32_t* __restrict__ n_all) {
  __shared__ unsigned long long keys[kMaxFeatures];
  __shared__ int s_count;
  const int p = blockIdx.x;
  const PairDesc pd = pairs[p];
  const int nq = min(pd.nq, kMaxFeatures);
  const uint64_t key = pair_key(seed, (uint64_t)(first_pair + p));
  const int2* bp = best + (size_t)p * stride;
  if (threadIdx.x == 0) s_count = 0;
#if RB200_SELECT_PARTIAL
  // Only the max_matches strongest matches survive (keepStrongestMatches, node.cpp:519-531,674), and the jitter (< 1e-3) never
  // reorders two different Hamming distances (1/256 apart): histogram the distances, find the cut that covers max_matches,
  // and sort only the matches at or below it (typically ~350 of 1000 keys: a 512-key instead of a 1024-key network).
  __shared__ int s_hist[128];
  __shared__ int s_cut, s_k;
  for (int i = threadIdx.x; i < 128; i += kSelThreads) s_hist[i] = 0;
  if (threadIdx.x == 0) s_k = 0;
  __syncthreads();
  for (int i = threadIdx.x; i < nq; i += kSelThreads) {
    const int2 b = bp[i];
    if (b.x < 128 && b.x >= 0 && b.y >= 0) atomicAdd(&s_hist[b.x], 1);  // node.cpp:572
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    int cum = 0, cut = 127;
    for (int h = 0; h < 128; h++) {
      cum += s_hist[h];
      if (cum >= c_params.max_matches) {
        cut = h;
        break;
      }
    }
    s_cut = cut;
  }
  __syncthreads();
  const int cut = s_cut;
  for (int i = threadIdx.x; i < nq; i += kSelThreads) {
    const int2 b = bp[i];
    if (b.x <= cut && b.x >= 0 && b.y >= 0) {
      const float dist = match_distance(b.x, rand31(key, 0u, (uint32_t)i));
      keys[atomicAdd(&s_k, 1)] = ((unsigned long long)__float_as_uint(dist) << 32) | (unsigned)i;
    }
  }
  __syncthreads();
  const int K = s_k;
  int N = 2;
  while (N < K) N <<= 1;
  for (int i = K + threadIdx.x; i < N; i += kSelThreads) keys[i] = ~0ULL;
  __syncthreads();
#else
  int N = 2;
  while (N < nq) N <<= 1;
  for (int i = threadIdx.x; i < N; i += kSelThreads) {
    unsigned long long k = ~0ULL;
    if (i < nq) {
      const int2 b = bp[i];
      if (b.x < 128 && b.y >= 0) {  // node.cpp:572
        const float dist = match_distance(b.x, rand31(key, 0u, (uint32_t)i));
        k = ((unsigned long long)__float_as_uint(dist) << 32) | (unsigned)i;
      }
    }
    keys[i] = k;
  }
  __syncthreads();
#endif
  for (int k = 2; k <= N; k <<= 1) {
    for (int j = k >> 1; j > 0; j >>= 1) {
      for (int t = threadIdx.x; t < (N >> 1); t += kSelThreads) {
        const int lo = ((t & ~(j - 1)) << 1) | (t & (j - 1));  // index with bit j cleared
        const int hi = lo | j;
        const bool up = (lo & k) == 0;
        const unsigned long long a = keys[lo], b = keys[hi];
        if ((a > b) == up) {
          keys[lo] = b;
          keys[hi] = a;
        }
      }
      __syncthreads();
    }
  }
  for (int i = threadIdx.x; i < N; i += kSelThreads)
    if (keys[i] != ~0ULL && (i == N - 1 || keys[i + 1] == ~0ULL)) s_count = i + 1;
  __syncthreads();
  const int maxM = c_params.max_matches;
  const int M = min(s_count, maxM);
  for (int k = threadIdx.x; k < M; k += kSelThreads) {
    const unsigned long long kk = keys[k];
    const int qi = (int)(kk & 0xffffffffULL);
    const int ti = bp[qi].y;
    rgbdslam_b200_dmatch m;
    m.queryIdx = qi;
    m.trainIdx = ti;
    m.imgIdx = -1;
    m.distance = __uint_as_float((unsigned)(kk >> 32));
    matches[(size_t)p * maxM + k] = m;
    mfrom[(size_t)p * maxM + k] = __ldg(pd.q_xyz + qi);
    mto[(size_t)p * maxM + k] = __ldg(pd.t_xyz + ti);
  }
  if (threadIdx.x == 0) n_all[p] = M;
}

cudaError_t launch_select_matches(const PairDesc* pairs, int npairs, const int2* best, int stride, uint64_t seed,
                                  int64_t first_pair, rgbdslam_b200_dmatch* matches, float4* mfrom, float4* mto,
                                  int32_t* n_all, int max_nq, cudaStream_t stream) {
  (void)max_nq;
  if (npairs <= 0) return cudaSuccess;
  select_matches_kernel<<<npairs, kSelThreads, 0, stream>>>(pairs, best, stride, seed, first_pair, matches, mfrom, mto,
                                                            n_all);
  return cudaGetLastError();
}

// =====================================================================================================
// RANSAC building blocks (warp-cooperative; every lane ends up with identical, warp-uniform results).

constexpr unsigned kFull = 0xffffffffu;
constexpr unsigned kFullMask = 0xffffffffu;
#ifndef RB200_SCORE_GROUP
#define RB200_SCORE_GROUP 5  // correspondences (mask words) scored per lane without an intervening branch
#endif

__device__ __forceinline__ float wsum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(kFull, v, o);
  return v;
}
// All-lanes sums of 16 values per lane.  Step with offset o: a lane keeps the half of its values selected by bit o of its id,
// hands the other half to lane ^ o and adds what it receives; after offsets 16, 8, 4, 2 one value per lane is left (index =
// lane bits 4..1), offset 1 completes it, 16 indexed shuffles hand every total to every lane.  Deterministic, warp-uniform.
__device__ __forceinline__ void wsum16(float (&v)[16], int lane) {
  float r8[8], r4[4], r2[2], r1;
  const bool b16 = lane & 16, b8 = lane & 8, b4 = lane & 4, b2 = lane & 2;
#pragma unroll
  for (int i = 0; i < 8; i++) r8[i] = (b16 ? v[i + 8] : v[i]) + __shfl_xor_sync(kFullMask, b16 ? v[i] : v[i + 8], 16);
#pragma unroll
  for (int i = 0; i < 4; i++) r4[i] = (b8 ? r8[i + 4] : r8[i]) + __shfl_xor_sync(kFullMask, b8 ? r8[i] : r8[i + 4], 8);
#pragma unroll
  for (int i = 0; i < 2; i++) r2[i] = (b4 ? r4[i + 2] : r4[i]) + __shfl_xor_sync(kFullMask, b4 ? r4[i] : r4[i + 2], 4);
  r1 = (b2 ? r2[1] : r2[0]) + __shfl_xor_sync(kFullMask, b2 ? r2[0] : r2[1], 2);
  r1 += __shfl_xor_sync(kFullMask, r1, 1);
  // value j lives in the lanes with (bit4, bit3, bit2, bit1) = (j>>3 &1, j>>2 &1, j>>1 &1, j &1)
#pragma unroll
  for (int j = 0; j < 16; j++) v[j] = __shfl_sync(kFullMask, r1, ((j & 8) ? 16 : 0) | ((j & 4) ? 8 : 0) | ((j & 2) ? 4 : 0) | ((j & 1) ? 2 : 0));
}
__device__ __forceinline__ double wsumd(double v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = __dadd_rn(v, __shfl_xor_sync(kFull, v, o));
  return v;
}

struct Rt {
  float R[9];  // row-major
  float t[3];
};

// Weighted rigid fit == getTransformFromMatches (transformation_estimation_euclidean.cpp:7-61):
// weight 1/(z_from*z_to) (:25), NaN-depth correspondences skipped (:22), then the closed form of
// pcl::TransformationFromCorrespondences: weighted means, C = sum w (to-m2)(from-m1)^T, C = U S V^T,
// R = U diag(1,1,det(U)det(V)) V^T, t = m2 - R m1.  The SVD is a Hestenes one-sided Jacobi; the
// reflection-corrected product is formed as u1 v1^T + u2 v2^T + (u1 x u2)(v1 x v2)^T, which equals
// U diag(1,1,det U det V) V^T for any sign choice of the third singular pair.
// Returns false if the result is not finite (the reference's `transformation != transformation` test,
// node.cpp:1144) or the correspondences are rank deficient (< 2 independent directions).
// cfrom / cto hold the correspondences CENTRED on the pair's centroids (ca, cb) with the ORIGINAL depth in .w:
// (x - cx, y - cy, z - cz, z).  Centring makes the single-pass raw-moment form of the weighted covariance
// (sum w b a^T / W - m2 m1^T) as accurate in float32 as the reference's running-mean update.
template <int NW>
__device__ bool fit_transform(const float4* __restrict__ cfrom, const float4* __restrict__ cto, const float* ca, const float* cb,
                              const uint32_t* sel, int nw, int lane, Rt& out) {
  float W = 0.f, f0 = 0.f, f1 = 0.f, f2 = 0.f, t0 = 0.f, t1 = 0.f, t2 = 0.f;
  float c[9] = {0, 0, 0, 0, 0, 0, 0, 0, 0};
  constexpr int kFitGroup = (NW % 5 == 0) ? 5 : 4;
#pragma unroll 1
  for (int g = 0; g < NW / kFitGroup; g++) {  // rolled for code size, see score_all
    uint32_t selg[kFitGroup];
#pragma unroll
    for (int gg = 0; gg < NW / kFitGroup; gg++)
      if (gg == g) {
#pragma unroll
        for (int j = 0; j < kFitGroup; j++) selg[j] = sel[gg * kFitGroup + j];
      }
#pragma unroll
    for (int j = 0; j < kFitGroup; j++) {
      const int w = g * kFitGroup + j;
      if (w < nw && ((selg[j] >> lane) & 1u)) {
        const float4 a = cfrom[w * 32 + lane], b = cto[w * 32 + lane];
        if (!isnan(a.w) && !isnan(b.w)) {  // transformation_estimation_euclidean.cpp:22
          const float wt = __fdiv_rn(1.0f, a.w * b.w);  // :25
          W += wt;
          f0 += wt * a.x; f1 += wt * a.y; f2 += wt * a.z;
          const float bx = wt * b.x, by = wt * b.y, bz = wt * b.z;
          t0 += bx; t1 += by; t2 += bz;
          c[0] += bx * a.x; c[1] += bx * a.y; c[2] += bx * a.z;
          c[3] += by * a.x; c[4] += by * a.y; c[5] += by * a.z;
          c[6] += bz * a.x; c[7] += bz * a.y; c[8] += bz * a.z;
        }
      }
    }
  }
  {  // 16 warp sums in 32 shuffles instead of 80: halve the value set at every butterfly step, then broadcast
    float v[16] = {W, f0, f1, f2, t0, t1, t2, c[0], c[1], c[2], c[3], c[4], c[5], c[6], c[7], c[8]};
    wsum16(v, lane);
    W = v[0]; f0 = v[1]; f1 = v[2]; f2 = v[3]; t0 = v[4]; t1 = v[5]; t2 = v[6];
#pragma unroll
    for (int i = 0; i < 9; i++) c[i] = v[7 + i];
  }
  if (!(W > 0.f)) return false;
  const float iW = __fdiv_rn(1.0f, W);
  const float m1x = f0 * iW, m1y = f1 * iW, m1z = f2 * iW;  // weighted means of the centred points
  const float m2x = t0 * iW, m2y = t1 * iW, m2z = t2 * iW;
  c[0] = c[0] * iW - m2x * m1x; c[1] = c[1] * iW - m2x * m1y; c[2] = c[2] * iW - m2x * m1z;
  c[3] = c[3] * iW - m2y * m1x; c[4] = c[4] * iW - m2y * m1y; c[5] = c[5] * iW - m2y * m1z;
  c[6] = c[6] * iW - m2z * m1x; c[7] = c[7] * iW - m2z * m1y; c[8] = c[8] * iW - m2z * m1z;

  // --- one-sided Jacobi SVD of c (row-major a[r][col]); v accumulates the right rotations ---
  float a00 = c[0], a01 = c[1], a02 = c[2], a10 = c[3], a11 = c[4], a12 = c[5], a20 = c[6], a21 = c[7], a22 = c[8];
  float v00 = 1, v01 = 0, v02 = 0, v10 = 0, v11 = 1, v12 = 0, v20 = 0, v21 = 0, v22 = 1;
#ifndef RB200_FAST_JACOBI
#define RB200_FAST_JACOBI 1
#endif
#if RB200_FAST_JACOBI
  // tan(theta) = sign(zeta) / (|zeta| + sqrt(1 + zeta^2)), zeta = (beta - alpha) / (2 gamma), written without the first
  // division; MUFU-based reciprocal / rsqrt (2 ulp): a Jacobi rotation only has to be orthogonal to rounding, the
  // iteration corrects any error in the angle on the next sweep.
#define RB200_JTEST(AL, BE, GA) ((GA) * (GA) > 1.6e-13f * ((AL) * (BE)))
#define RB200_JANGLE(AL, BE, GA, CS, SN)                                                             \
  {                                                                                                  \
    const float dd = (BE) - (AL), g2 = 2.f * (GA);                                                   \
    const float hh = sqrtf(fmaf(dd, dd, g2 * g2));                                                   \
    const float sg = ((dd < 0.f) != (g2 < 0.f)) ? -1.f : 1.f;                                        \
    const float tt = sg * __fdividef(fabsf(g2), fabsf(dd) + hh);                                     \
    CS = rsqrtf(fmaf(tt, tt, 1.f));                                                                  \
    SN = CS * tt;                                                                                    \
  }
#else
#define RB200_JTEST(AL, BE, GA) (fabsf(GA) > 4e-7f * sqrtf((AL) * (BE)) && (GA) != 0.f)
#define RB200_JANGLE(AL, BE, GA, CS, SN)                                                             \
  {                                                                                                  \
    const float zeta = ((BE) - (AL)) / (2.f * (GA));                                                 \
    const float tt = copysignf(1.f, zeta) / (fabsf(zeta) + sqrtf(1.f + zeta * zeta));               \
    CS = 1.f / sqrtf(1.f + tt * tt);                                                                 \
    SN = CS * tt;                                                                                    \
  }
#endif
#define RB200_JROT(AP0, AP1, AP2, AQ0, AQ1, AQ2, VP0, VP1, VP2, VQ0, VQ1, VQ2)                       \
  {                                                                                                  \
    const float alpha = AP0 * AP0 + AP1 * AP1 + AP2 * AP2;                                           \
    const float beta = AQ0 * AQ0 + AQ1 * AQ1 + AQ2 * AQ2;                                            \
    const float gamma = AP0 * AQ0 + AP1 * AQ1 + AP2 * AQ2;                                           \
    if (RB200_JTEST(alpha, beta, gamma)) {                                                           \
      if (gamma * gamma > 1e-7f * (alpha * beta)) rotated = true; /* else: converged after this one */ \
      float cs, sn;                                                                                  \
      RB200_JANGLE(alpha, beta, gamma, cs, sn)                                                       \
      float x, y;                                                                                    \
      x = AP0; y = AQ0; AP0 = cs * x - sn * y; AQ0 = sn * x + cs * y;                                \
      x = AP1; y = AQ1; AP1 = cs * x - sn * y; AQ1 = sn * x + cs * y;                                \
      x = AP2; y = AQ2; AP2 = cs * x - sn * y; AQ2 = sn * x + cs * y;                                \
      x = VP0; y = VQ0; VP0 = cs * x - sn * y; VQ0 = sn * x + cs * y;                                \
      x = VP1; y = VQ1; VP1 = cs * x - sn * y; VQ1 = sn * x + cs * y;                                \
      x = VP2; y = VQ2; VP2 = cs * x - sn * y; VQ2 = sn * x + cs * y;                                \
    }                                                                                                \
  }
  // `rotated` = some column pair was still more than 3e-4 from orthogonal before its rotation.  One-sided Jacobi converges
  // quadratically, so a sweep whose rotations were all below that leaves residuals ~1e-7 (float epsilon): no check sweep.
  for (int sweep = 0; sweep < 6; sweep++) {
    bool rotated = false;
    RB200_JROT(a00, a10, a20, a01, a11, a21, v00, v10, v20, v01, v11, v21)  // columns 0,1
    RB200_JROT(a00, a10, a20, a02, a12, a22, v00, v10, v20, v02, v12, v22)  // columns 0,2
    RB200_JROT(a01, a11, a21, a02, a12, a22, v01, v11, v21, v02, v12, v22)  // columns 1,2
    if (!rotated) break;
  }
#undef RB200_JROT
#undef RB200_JTEST
#undef RB200_JANGLE
  // column norms; pick the two largest columns (p >= q >= r)
  const float n0 = a00 * a00 + a10 * a10 + a20 * a20;
  const float n1 = a01 * a01 + a11 * a11 + a21 * a21;
  const float n2 = a02 * a02 + a12 * a12 + a22 * a22;
  float p0, p1, p2, q0, q1, q2, vp0, vp1, vp2, vq0, vq1, vq2, np, nq;
  // largest
  int ip = 0;
  if (n1 > n0) ip = 1;
  if (n2 > (ip == 0 ? n0 : n1)) ip = 2;
  int iq;  // second largest
  if (ip == 0) iq = (n2 > n1) ? 2 : 1;
  else if (ip == 1) iq = (n2 > n0) ? 2 : 0;
  else iq = (n1 > n0) ? 1 : 0;
#define RB200_COL(I, X0, X1, X2, Y0, Y1, Y2, NN)                                      \
  if (I == 0) { X0 = a00; X1 = a10; X2 = a20; Y0 = v00; Y1 = v10; Y2 = v20; NN = n0; } \
  else if (I == 1) { X0 = a01; X1 = a11; X2 = a21; Y0 = v01; Y1 = v11; Y2 = v21; NN = n1; } \
  else { X0 = a02; X1 = a12; X2 = a22; Y0 = v02; Y1 = v12; Y2 = v22; NN = n2; }
  RB200_COL(ip, p0, p1, p2, vp0, vp1, vp2, np)
  RB200_COL(iq, q0, q1, q2, vq0, vq1, vq2, nq)
#undef RB200_COL
  if (!(np > 0.f) || !(nq > 1e-24f * np)) return false;  // rank < 2: rotation undetermined
#if RB200_FAST_JACOBI
  const float ip_ = rsqrtf(np), iq_ = rsqrtf(nq);
#else
  const float ip_ = 1.f / sqrtf(np), iq_ = 1.f / sqrtf(nq);
#endif
  p0 *= ip_; p1 *= ip_; p2 *= ip_;
  q0 *= iq_; q1 *= iq_; q2 *= iq_;
  const float u30 = p1 * q2 - p2 * q1, u31 = p2 * q0 - p0 * q2, u32 = p0 * q1 - p1 * q0;
  const float v30 = vp1 * vq2 - vp2 * vq1, v31 = vp2 * vq0 - vp0 * vq2, v32 = vp0 * vq1 - vp1 * vq0;
  out.R[0] = p0 * vp0 + q0 * vq0 + u30 * v30;
  out.R[1] = p0 * vp1 + q0 * vq1 + u30 * v31;
  out.R[2] = p0 * vp2 + q0 * vq2 + u30 * v32;
  out.R[3] = p1 * vp0 + q1 * vq0 + u31 * v30;
  out.R[4] = p1 * vp1 + q1 * vq1 + u31 * v31;
  out.R[5] = p1 * vp2 + q1 * vq2 + u31 * v32;
  out.R[6] = p2 * vp0 + q2 * vq0 + u32 * v30;
  out.R[7] = p2 * vp1 + q2 * vq1 + u32 * v31;
  out.R[8] = p2 * vp2 + q2 * vq2 + u32 * v32;
  // t = mean2 - R mean1 with the centroids added back
  const float g1x = m1x + ca[0], g1y = m1y + ca[1], g1z = m1z + ca[2];
  out.t[0] = (m2x + cb[0]) - (out.R[0] * g1x + out.R[1] * g1y + out.R[2] * g1z);
  out.t[1] = (m2y + cb[1]) - (out.R[3] * g1x + out.R[4] * g1y + out.R[5] * g1z);
  out.t[2] = (m2z + cb[2]) - (out.R[6] * g1x + out.R[7] * g1y + out.R[8] * g1z);
  bool fin = true;
#pragma unroll
  for (int i = 0; i < 9; i++) fin = fin && (out.R[i] == out.R[i]);
#pragma unroll
  for (int i = 0; i < 3; i++) fin = fin && (out.t[i] == out.t[i]);
  return fin;
}

constexpr double kHuge = 1.7976931348623157e308;  // std::numeric_limits<double>::max()

__device__ __forceinline__ double depth_cov(double z) {  // misc2.h:20-35 (static cache emulated by cov_z_const)
  if (c_params.cov_z_const >= 0.0) return c_params.cov_z_const;
  const double sd = __dmul_rn(c_params.sigma_depth, __dmul_rn(z, z));
  return __dmul_rn(sd, sd);
}

// Per-hypothesis constants of the float64 scoring formula (warp-uniform).  Only built when some correspondence of the
// warp's current 32 cannot be classified in float32 (score_all).
struct ScoreCtx {
  double R[9], t[3];
  double P[6];   // rcx * r0_i r0_j + rcy * r1_i r1_j   (ij = 00,01,02,11,12,22), r_k = k-th row of R
  double O2[6];  // r2_i r2_j
};

__device__ __noinline__ void make_score_ctx(const Rt& T, ScoreCtx& c) {
#pragma unroll
  for (int i = 0; i < 9; i++) c.R[i] = (double)T.R[i];  // transformation4f.cast<double>() (node.cpp:984)
#pragma unroll
  for (int i = 0; i < 3; i++) c.t[i] = (double)T.t[i];
  const double rcx = c_params.raster_cov_x, rcy = c_params.raster_cov_y;
  const int I[6] = {0, 0, 0, 1, 1, 2}, J[6] = {0, 1, 2, 1, 2, 2};
#pragma unroll
  for (int k = 0; k < 6; k++) {
    c.P[k] = fma(__dmul_rn(rcx, c.R[I[k]]), c.R[J[k]], __dmul_rn(__dmul_rn(rcy, c.R[3 + I[k]]), c.R[3 + J[k]]));
    c.O2[k] = __dmul_rn(c.R[6 + I[k]], c.R[6 + J[k]]);
  }
}

// The same constants in float32 for the screening pass, plus the loop invariants of the covariance model.
struct ScreenCtx {
  float Pf[6], O2f[6];
  float rcx, rcy, sq_max, sigma_depth;
  float czc;  // constant depth covariance (misc2.h static cache), < 0: per-point (sigma_depth * z^2)^2 model
  float Cc[6], lim_c;  // czc >= 0: czc * O2f (+ czc on the zz entry) and the constant shortcut limit
};

__device__ __forceinline__ void make_screen_ctx(const Rt& T, ScreenCtx& c) {
  c.rcx = (float)c_params.raster_cov_x;
  c.rcy = (float)c_params.raster_cov_y;
  c.sq_max = (float)c_params.sq_max_dist;
  c.czc = (float)c_params.cov_z_const;
  c.sigma_depth = (float)c_params.sigma_depth;
  const int I[6] = {0, 0, 0, 1, 1, 2}, J[6] = {0, 1, 2, 1, 2, 2};
#pragma unroll
  for (int k = 0; k < 6; k++) {
    c.Pf[k] = fmaf(c.rcx * T.R[I[k]], T.R[J[k]], (c.rcy * T.R[3 + I[k]]) * T.R[3 + J[k]]);
    c.O2f[k] = T.R[6 + I[k]] * T.R[6 + J[k]];
    c.Cc[k] = c.czc * c.O2f[k] + (k == 5 ? c.czc : 0.f);
  }
  c.lim_c = 2.f * (fmaxf(c.rcx, c.czc) + fmaxf(c.rcx, c.czc));
}

// float32 screening of errorFunction2, branch-free so that the unrolled scoring loop interleaves several
// correspondences (the kernel is bound by dependent-instruction latency, not by issue slots).  Returns
//   m >= 0 : certainly an inlier, value = d^2 (float)          -1 : certainly rejected (shortcut of misc.cpp:726-735,
//   d^2 > thr, NaN depth)                                      NaN: too close to call in float32 -> the caller
//                                                                   evaluates the float64 reference formula
// Margins: 1e-3 relative on both tests, orders of magnitude above the float32 evaluation error (~1e-5 relative for
// the 3x3 SPD solve with condition number < 1e2).
template <bool kConstCov>
__device__ __forceinline__ float mahal_screen(const float4 x1, const float4 x2, const Rt& T, const ScreenCtx& c) {
  const float d0 = fmaf(T.R[0], x1.x, fmaf(T.R[1], x1.y, fmaf(T.R[2], x1.z, T.t[0] * x1.w))) - x2.x;
  const float d1 = fmaf(T.R[3], x1.x, fmaf(T.R[4], x1.y, fmaf(T.R[5], x1.z, T.t[1] * x1.w))) - x2.y;
  const float d2 = fmaf(T.R[6], x1.x, fmaf(T.R[7], x1.y, fmaf(T.R[8], x1.z, T.t[2] * x1.w))) - x2.z;
  const float rcx = c.rcx, rcy = c.rcy;
  const float dsq = fmaf(d0, d0, fmaf(d1, d1, d2 * d2));
  const float a2 = x1.z, b2 = x2.z;
  float lim, S00, S01, S02, S11, S12, S22;
  if (kConstCov) {  // the default configuration: depth covariance latched to a constant (misc2.h:30-35)
    lim = c.lim_c;
    S00 = fmaf(a2, c.Pf[0], fmaf(rcx, b2, c.Cc[0]));
    S01 = fmaf(a2, c.Pf[1], c.Cc[1]);
    S02 = fmaf(a2, c.Pf[2], c.Cc[2]);
    S11 = fmaf(a2, c.Pf[3], fmaf(rcy, b2, c.Cc[3]));
    S12 = fmaf(a2, c.Pf[4], c.Cc[4]);
    S22 = fmaf(a2, c.Pf[5], c.Cc[5]);
  } else {
    const float sd1 = c.sigma_depth * (x1.z * x1.z), sd2 = c.sigma_depth * (x2.z * x2.z);
    const float cz1 = sd1 * sd1, cz2 = sd2 * sd2;
    lim = 2.f * (fmaxf(rcx, cz1) + fmaxf(rcx, cz2));
    S00 = fmaf(a2, c.Pf[0], fmaf(cz1, c.O2f[0], rcx * b2));
    S01 = fmaf(a2, c.Pf[1], cz1 * c.O2f[1]);
    S02 = fmaf(a2, c.Pf[2], cz1 * c.O2f[2]);
    S11 = fmaf(a2, c.Pf[3], fmaf(cz1, c.O2f[3], rcy * b2));
    S12 = fmaf(a2, c.Pf[4], cz1 * c.O2f[4]);
    S22 = fmaf(a2, c.Pf[5], fmaf(cz1, c.O2f[5], cz2));
  }
  // scale to O(1) to stay far from float under/overflow in the cubic determinant (entries are 1e-5 .. 1e-2)
  const float k = 1024.f;
  const float s00 = S00 * k, s01 = S01 * k, s02 = S02 * k, s11 = S11 * k, s12 = S12 * k, s22 = S22 * k;
  const float A00 = fmaf(s11, s22, -s12 * s12), A01 = fmaf(s02, s12, -s01 * s22), A02 = fmaf(s01, s12, -s02 * s11);
  const float A11 = fmaf(s00, s22, -s02 * s02), A12 = fmaf(s01, s02, -s00 * s12), A22 = fmaf(s00, s11, -s01 * s01);
  const float det = fmaf(s00, A00, fmaf(s01, A01, s02 * A02));
  const float e0 = fmaf(A00, d0, fmaf(A01, d1, A02 * d2));
  const float e1 = fmaf(A01, d0, fmaf(A11, d1, A12 * d2));
  const float e2 = fmaf(A02, d0, fmaf(A12, d1, A22 * d2));
  const float m = __fdividef(fmaf(d0, e0, fmaf(d1, e1, d2 * e2)) * k, det);
  const float undecided = __int_as_float(0x7fc00000);
  const bool reject1 = isnan(x1.z) || isnan(x2.z) || dsq > lim * 1.001f;
  const bool unsure = !(dsq < lim * 0.999f) || !(m >= 0.f) || !(det > 0.f);
  const float r = (m > c.sq_max * 1.001f) ? -1.f : ((m < c.sq_max * 0.999f) ? m : undecided);
  return reject1 ? -1.f : (unsure ? undecided : r);
}

// errorFunction2 (misc.cpp:697-770) in float64.  Written with explicit rounding intrinsics only, so the
// hypothesis kernel and the selection kernel (which re-scores the winning transform) produce bit-identical
// values regardless of how the compiler inlines/contracts.
//   S = R^T diag(rcx z1, rcy z1, cz1) R + diag(rcx z2, rcy z2, cz2)  =  z1 * P + cz1 * O2 + diag(...)
// (P, O2 precomputed per hypothesis).  The 3x3 SPD solve uses the adjugate form
// d^T S^-1 d = d^T adj(S) d / det(S) instead of the reference's LLT (same value to rounding).
__device__ __forceinline__ double mahal_sq(const float4 x1, const float4 x2, const ScoreCtx& c) {
  if (isnan(x1.z) || isnan(x2.z)) return kHuge;
  const double a0 = x1.x, a1 = x1.y, a2 = x1.z, a3 = x1.w;
  const double b0 = x2.x, b1 = x2.y, b2 = x2.z;
  const double mu0 = fma(c.R[0], a0, fma(c.R[1], a1, fma(c.R[2], a2, __dmul_rn(c.t[0], a3))));
  const double mu1 = fma(c.R[3], a0, fma(c.R[4], a1, fma(c.R[5], a2, __dmul_rn(c.t[1], a3))));
  const double mu2 = fma(c.R[6], a0, fma(c.R[7], a1, fma(c.R[8], a2, __dmul_rn(c.t[2], a3))));
  const double d0 = __dsub_rn(mu0, b0), d1 = __dsub_rn(mu1, b1), d2 = __dsub_rn(mu2, b2);
  const double rcx = c_params.raster_cov_x, rcy = c_params.raster_cov_y;
  const double cz1 = depth_cov(a2), cz2 = depth_cov(b2);
  {
    const double dsq = fma(d0, d0, fma(d1, d1, __dmul_rn(d2, d2)));
    const double s1 = fmax(rcx, cz1), s2 = fmax(rcx, cz2);
    if (dsq > __dmul_rn(2.0, __dadd_rn(s1, s2))) return kHuge;  // misc.cpp:726-735
  }
  if (isnan(d2)) return kHuge;
  const double S00 = fma(a2, c.P[0], fma(cz1, c.O2[0], __dmul_rn(rcx, b2)));
  const double S01 = fma(a2, c.P[1], __dmul_rn(cz1, c.O2[1]));
  const double S02 = fma(a2, c.P[2], __dmul_rn(cz1, c.O2[2]));
  const double S11 = fma(a2, c.P[3], fma(cz1, c.O2[3], __dmul_rn(rcy, b2)));
  const double S12 = fma(a2, c.P[4], __dmul_rn(cz1, c.O2[4]));
  const double S22 = fma(a2, c.P[5], fma(cz1, c.O2[5], cz2));
  const double A00 = fma(S11, S22, -__dmul_rn(S12, S12));
  const double A01 = fma(S02, S12, -__dmul_rn(S01, S22));
  const double A02 = fma(S01, S12, -__dmul_rn(S02, S11));
  const double A11 = fma(S00, S22, -__dmul_rn(S02, S02));
  const double A12 = fma(S01, S02, -__dmul_rn(S00, S12));
  const double A22 = fma(S00, S11, -__dmul_rn(S01, S01));
  const double det = fma(S00, A00, fma(S01, A01, __dmul_rn(S02, A02)));
  const double e0 = fma(A00, d0, fma(A01, d1, __dmul_rn(A02, d2)));
  const double e1 = fma(A01, d0, fma(A11, d1, __dmul_rn(A12, d2)));
  const double e2 = fma(A02, d0, fma(A12, d1, __dmul_rn(A22, d2)));
  const double num = fma(d0, e0, fma(d1, e1, __dmul_rn(d2, e2)));
  const double m = __ddiv_rn(num, det);
  if (!(m >= 0.0)) return kHuge;
  return m;
}

__device__ __noinline__ double mahal_sq_slow(const float4 x1, const float4 x2, const ScoreCtx& c) { return mahal_sq(x1, x2, c); }

// computeInliersAndError (node.cpp:968-1020): returns #inliers, fills the mask words (warp-uniform) and
// the Mahalanobis RMS (1e9 if < 3 inliers).
template <int NW>
__device__ int score_all(const float4* __restrict__ sfrom, const float4* __restrict__ sto, int M, int nw, int lane,
                         const Rt& T, uint32_t* words, double& err) {
  ScreenCtx sc;
  make_screen_ctx(T, sc);
  const double sq_max = c_params.sq_max_dist;
  // Per group of kGroup mask words: pass 1 classifies the correspondences in float32 with no branch in between (kGroup
  // independent dependency chains per lane), pass 2 resolves the undecided ones with the float64 reference formula and
  // builds the inlier masks.  The group loop is NOT unrolled: the fully unrolled body made the hot loop ~28 KiB of code and
  // a quarter of all stall samples were instruction-cache misses (`stall_no_inst`); mask words are moved between the
  // register array and the loop body with compile-time indices under a predicate.
  constexpr int kGroup = (NW % RB200_SCORE_GROUP == 0) ? RB200_SCORE_GROUP : 4;
  constexpr int kGroups = NW / kGroup;
  ScoreCtx ctx;
  bool have_ctx = false;
  double esum = 0.0;
  int cnt = 0;
#pragma unroll 1
  for (int g = 0; g < kGroups; g++) {
    float code[kGroup];
    uint32_t wout[kGroup];
    if (g * kGroup < nw) {
      if (sc.czc >= 0.f) {  // warp-uniform; decided once per group so the kGroup chains stay branch-free
#pragma unroll
        for (int j = 0; j < kGroup; j++) {
          const int i = (g * kGroup + j) * 32 + lane;  // < kMaxMatchesCap: rows >= M hold stale but addressable memory
          const float4 a = sfrom[i], b = sto[i];
          const float cm = mahal_screen<true>(a, b, T, sc);
          code[j] = (i < M && !(a.z == 0.0f || b.z == 0.0f)) ? cm : -1.f;  // node.cpp:994 (does not trigger on NaN)
        }
      } else {
#pragma unroll
        for (int j = 0; j < kGroup; j++) {
          const int i = (g * kGroup + j) * 32 + lane;
          const float4 a = sfrom[i], b = sto[i];
          const float cm = mahal_screen<false>(a, b, T, sc);
          code[j] = (i < M && !(a.z == 0.0f || b.z == 0.0f)) ? cm : -1.f;
        }
      }
    } else {
#pragma unroll
      for (int j = 0; j < kGroup; j++) code[j] = -1.f;
    }
#pragma unroll
    for (int j = 0; j < kGroup; j++) {
      const int w = g * kGroup + j;
      uint32_t word = 0;
      if (w < nw) {
        const float cm = code[j];
        const bool undecided = isnan(cm);
        bool inl = cm >= 0.f;
        double m = (double)cm;
        if (__any_sync(kFull, undecided)) {  // rare: kept out of line
          if (!have_ctx) {
            make_score_ctx(T, ctx);
            have_ctx = true;
          }
          if (undecided) {
            const int i = w * 32 + lane;
            m = mahal_sq_slow(sfrom[i], sto[i], ctx);
            inl = !(m > sq_max) && (m >= 0.0);  // node.cpp:998-1005
          }
        }
        word = __ballot_sync(kFull, inl);
        if (inl) esum = __dadd_rn(esum, m);
        cnt += __popc(word);
      }
      wout[j] = word;
    }
#pragma unroll
    for (int gg = 0; gg < kGroups; gg++)
      if (gg == g) {
#pragma unroll
        for (int j = 0; j < kGroup; j++) words[gg * kGroup + j] = wout[j];
      }
  }
  esum = wsumd(esum);
  err = (cnt < 3) ? 1e9 : sqrt(__ddiv_rn(esum, (double)cnt));  // node.cpp:1011-1017
  return cnt;
}

__device__ __forceinline__ unsigned min_inlier_threshold(int M) {  // node.cpp:1094-1099
  unsigned thr = (unsigned)c_params.min_matches;
  if ((double)thr > 0.75 * (double)M) thr = (unsigned)(0.75 * (double)M);
  return thr;
}

// Tuning knobs (defaults are the shipped configuration; tools/build_variants.py overrides them for A/B timing).
#ifndef RB200_RANSAC_WARPS
#define RB200_RANSAC_WARPS 8
#endif
#ifndef RB200_RANSAC_MINBLOCKS
#define RB200_RANSAC_MINBLOCKS 3
#endif
#ifndef RB200_PH1
#define RB200_PH1 4
#endif
#ifndef RB200_PH2
#define RB200_PH2 4
#endif
constexpr int kRansacWarps = RB200_RANSAC_WARPS;
#ifdef RB200_PROFILE
// per phase: fit cycles, score cycles, refinement rounds, hypotheses, loop cycles, max loop cycles, max rounds
__device__ unsigned long long g_ransac_prof[3][8];
extern "C" int rb200_debug_ransac_profile(unsigned long long* out24, int reset) {
  cudaError_t e = cudaMemcpyFromSymbol(out24, g_ransac_prof, sizeof(unsigned long long) * 24);
  if (e == cudaSuccess && reset) {
    unsigned long long z[24] = {0};
    e = cudaMemcpyToSymbol(g_ransac_prof, z, sizeof(z));
  }
  return (int)e;
}
#endif

// The reference's bookkeeping over finished hypotheses (node.cpp:1170-1190), replayed in order over the
// records of hypotheses [0, n_limit): global best by (error <=, inliers >=), the "n += 10" shortcuts for
// > 50 % / > 75 % inliers and the break at > 80 %.  Returns the next hypothesis index the sequential loop
// would visit (>= n_limit) -- hypotheses below it that were jumped over are never looked at.
struct ScanState {
  float rmse;
  int best_cnt, best_n, valid, next_n;
  bool done;
};

// `cnt` / `err` are shared-memory copies of the records' count / err fields (staged in parallel by the
// caller: a dependent chain of 200 global loads would cost ~60 us).
__device__ ScanState ransac_scan(const int* cnt_s, const double* err_s, int M, unsigned min_thr, int n_limit) {
  ScanState st;
  st.rmse = 1e6f;  // node.cpp:1110
  st.best_cnt = 0;
  st.best_n = -1;
  st.valid = 0;
  st.done = false;
  int n = 0;
  for (; n < n_limit; n++) {  // node.cpp:1130
    const int cnt = cnt_s[n];
    if (cnt > 0) {  // node.cpp:1170
      st.valid++;
      const double err = err_s[n];
      if (err <= (double)st.rmse && cnt >= st.best_cnt && (unsigned)cnt >= min_thr) {  // node.cpp:1177-1179
        st.rmse = (float)err;
        st.best_cnt = cnt;
        st.best_n = n;
        if ((double)cnt > (double)M * 0.5) n += 10;   // node.cpp:1186
        if ((double)cnt > (double)M * 0.75) n += 10;  // node.cpp:1187
        if ((double)cnt > (double)M * 0.8) {          // node.cpp:1188
          st.done = true;
          break;
        }
      }
    }
  }
  st.next_n = n;
  return st;
}

// The same bookkeeping evaluated 32 records at a time (exactly equivalent to ransac_scan: between two improvements of the best
// model the loop state does not change, so the first improving record of a chunk in index order is the one the sequential
// loop would take; the chunk restarts behind every jump, records the sequential loop skips are never looked at).  Verified
// against the sequential form on 20 000 random record sets on the CPU.  next_n is NOT maintained (final scan only).
__device__ ScanState ransac_scan_warp(const int* cnt_s, const double* err_s, int M, unsigned min_thr, int n_limit, int lane) {
  ScanState st;
  st.rmse = 1e6f;
  st.best_cnt = 0;
  st.best_n = -1;
  st.valid = 0;
  st.done = false;
  int n = 0;
  while (n < n_limit) {
    const int i = n + lane;
    const int c = i < n_limit ? cnt_s[i] : 0;
    const double e = i < n_limit ? err_s[i] : 0.0;
    const bool val = c > 0;
    const bool imp = val && e <= (double)st.rmse && c >= st.best_cnt && (unsigned)c >= min_thr;
    const unsigned vmask = __ballot_sync(kFull, val), imask = __ballot_sync(kFull, imp);
    if (imask == 0) {
      st.valid += __popc(vmask);
      n += 32;
      continue;
    }
    const int f = __ffs(imask) - 1;
    st.valid += __popc(vmask & (0xffffffffu >> (31 - f)));
    const int cb = __shfl_sync(kFull, c, f);
    const double eb = __shfl_sync(kFull, e, f);
    st.rmse = (float)eb;
    st.best_cnt = cb;
    st.best_n = n + f;
    int nn = n + f;
    if ((double)cb > (double)M * 0.5) nn += 10;
    if ((double)cb > (double)M * 0.75) nn += 10;
    if ((double)cb > (double)M * 0.8) {
      st.done = true;
      n = nn;
      break;
    }
    n = nn + 1;
  }
  st.next_n = n;
  return st;
}

constexpr int kMaxScanPrefix = 64;  // largest n_begin of a non-final phase (phases: [0,8) [8,40) [40,H))

// Hypotheses [n_begin, n_end) of every pair.  The host launches this in growing phases ([0,8), [8,40),
// [40,H)); a CTA first replays the scan over the already finished prefix [0, n_begin) and skips work the
// sequential reference loop would never reach (pair finished by the > 80 % break, or index jumped over).
// NW = mask words compiled in (10 covers the default max_matches = 300, 16 the cap of 512): the unrolled
// per-word code is the bulk of the kernel, the smaller instantiation relieves the instruction cache.
template <int NW>
__global__ void __launch_bounds__(kRansacWarps * 32, RB200_RANSAC_MINBLOCKS)
    ransac_hyp_kernel(int H, int maxM, int n_begin, int n_end, uint64_t seed, int64_t first_pair,
                      const float4* __restrict__ mfrom, const float4* __restrict__ mto,
                      const int32_t* __restrict__ n_all, HypResult* __restrict__ hyp, float* __restrict__ cen,
                      int32_t* __restrict__ next_n) {
  // NW * 32 rows each (20 KiB in total for the default max_matches = 300): small enough for one CTA of this kernel to share
  // an SM with a CTA of the tensor-core match kernel of another batch in flight
  __shared__ float4 sfrom[NW * 32];
  __shared__ float4 sto[NW * 32];
  __shared__ float4 cfrom[NW * 32];  // centred copies for the fit (see fit_transform)
  __shared__ float4 cto[NW * 32];
  __shared__ float s_cen[8];
  __shared__ float s_part[kRansacWarps][6];
  __shared__ int s_next_n;
  __shared__ int s_cnt[kMaxScanPrefix];
  __shared__ double s_err[kMaxScanPrefix];
  const int p = blockIdx.y;
  const int M = n_all[p];
  if (M <= c_params.min_matches || M < 4) return;  // node.cpp:1087,1130 (selection kernel checks the same)
  const unsigned min_thr = min_inlier_threshold(M);
  // The first phase (one CTA per pair when n_end <= kRansacWarps) publishes the pair's centroids and, after its
  // hypotheses, the index the sequential loop would visit next; later phases read both instead of recomputing them
  // (20 CTAs per pair used to replay the scan just to find out that 75 % of the pairs were finished).
  const bool publish = n_begin == 0 && gridDim.x == 1 && next_n != nullptr;
  int skip_below = 0;
  if (n_begin > 0) {
    if (next_n != nullptr) {
      skip_below = next_n[p];
    } else {
      // records of hypotheses the sequential loop never visits are stale/unwritten: harmless, the scan skips them
      for (int i = threadIdx.x; i < n_begin; i += blockDim.x) {
        const HypResult* r = hyp + (size_t)p * H + i;
        s_cnt[i] = r->count;
        s_err[i] = r->err;
      }
      __syncthreads();
      if (threadIdx.x == 0) {
        const ScanState st = ransac_scan(s_cnt, s_err, M, min_thr, n_begin);
        s_next_n = st.done ? H : st.next_n;
      }
      __syncthreads();
      skip_below = s_next_n;
    }
    if (skip_below >= n_begin + (int)(blockIdx.x + 1) * kRansacWarps || skip_below >= n_end) return;
  }
  if (n_begin == 0 || next_n == nullptr) {
    float cs[6] = {0, 0, 0, 0, 0, 0};
    for (int i = threadIdx.x; i < M; i += blockDim.x) {
      const float4 a = mfrom[(size_t)p * maxM + i], b = mto[(size_t)p * maxM + i];
      sfrom[i] = a;
      sto[i] = b;
      if (!isnan(a.x + a.y + a.z + b.x + b.y + b.z)) {
        cs[0] += a.x; cs[1] += a.y; cs[2] += a.z; cs[3] += b.x; cs[4] += b.y; cs[5] += b.z;
      }
    }
#pragma unroll
    for (int k = 0; k < 6; k++) cs[k] = wsum(cs[k]);
    if ((threadIdx.x & 31) == 0)
      for (int k = 0; k < 6; k++) s_part[threadIdx.x >> 5][k] = cs[k];
    __syncthreads();
    if (threadIdx.x < 6) {
      float t = 0.f;
      for (int w = 0; w < kRansacWarps; w++) t += s_part[w][threadIdx.x];
      s_cen[threadIdx.x] = t / (float)M;  // any common offset is valid; the (NaN-free) mean keeps the centred data small
      if (publish) cen[(size_t)p * 8 + threadIdx.x] = s_cen[threadIdx.x];
    }
    __syncthreads();
    for (int i = threadIdx.x; i < M; i += blockDim.x) {
      const float4 a = sfrom[i], b = sto[i];
      cfrom[i] = make_float4(a.x - s_cen[0], a.y - s_cen[1], a.z - s_cen[2], a.z);
      cto[i] = make_float4(b.x - s_cen[3], b.y - s_cen[4], b.z - s_cen[5], b.z);
    }
  } else {
    if (threadIdx.x < 6) s_cen[threadIdx.x] = cen[(size_t)p * 8 + threadIdx.x];
    __syncthreads();
    for (int i = threadIdx.x; i < M; i += blockDim.x) {
      const float4 a = mfrom[(size_t)p * maxM + i], b = mto[(size_t)p * maxM + i];
      sfrom[i] = a;
      sto[i] = b;
      cfrom[i] = make_float4(a.x - s_cen[0], a.y - s_cen[1], a.z - s_cen[2], a.z);
      cto[i] = make_float4(b.x - s_cen[3], b.y - s_cen[4], b.z - s_cen[5], b.z);
    }
  }
  __syncthreads();
  const int lane = threadIdx.x & 31;
  const int n = n_begin + blockIdx.x * kRansacWarps + (threadIdx.x >> 5);
  const bool active = !(n >= n_end || (n_begin > 0 && n < skip_below));
  if (!active && !publish) return;
  if (active) {
  const int nw = (M + 31) >> 5;
  const uint64_t key = pair_key(seed, (uint64_t)(first_pair + p));

  // sample_matches_prefer_by_distance(4, ...) (node.cpp:1024-1047)
  int ids[4] = {-1, -1, -1, -1};
  {
    int cnt = 0, safety = 0;
    uint32_t ctr = 0;
    while (cnt < 4) {
      int id1 = (int)(rand31(key, 1u + (uint32_t)n, ctr) % (uint32_t)M);
      const int id2 = (int)(rand31(key, 1u + (uint32_t)n, ctr + 1) % (uint32_t)M);
      ctr += 2;
      if (id1 > id2) id1 = id2;
      if (id1 != ids[0] && id1 != ids[1] && id1 != ids[2] && id1 != ids[3]) {
        if (cnt == 0) ids[0] = id1;
        else if (cnt == 1) ids[1] = id1;
        else if (cnt == 2) ids[2] = id1;
        else ids[3] = id1;
        cnt++;
      }
      if (++safety > 10000) break;
    }
  }
  uint32_t sel[NW];
#pragma unroll
  for (int w = 0; w < NW; w++) {
    uint32_t word = 0;
#pragma unroll
    for (int k = 0; k < 4; k++)
      if (ids[k] >= 0 && (ids[k] >> 5) == w) word |= 1u << (ids[k] & 31);
    sel[w] = word;
  }

  double refined_err = 1e6;
  int refined_cnt = 0;
  Rt refined;
#pragma unroll
  for (int i = 0; i < 9; i++) refined.R[i] = (i % 4 == 0) ? 1.f : 0.f;
  refined.t[0] = refined.t[1] = refined.t[2] = 0.f;

#ifdef RB200_PROFILE
  long long pf_fit = 0, pf_score = 0, pf_rounds = 0;
  const long long pf_t0 = clock64();
#endif
  for (int refinements = 1; refinements < 20; refinements++) {  // node.cpp:1140
    Rt T;
#ifdef RB200_PROFILE
    const long long c0 = clock64();
#endif
    const bool fit_ok = fit_transform<NW>(cfrom, cto, s_cen, s_cen + 3, sel, nw, lane, T);
#ifdef RB200_PROFILE
    const long long c1 = clock64();
    pf_fit += c1 - c0;
    pf_rounds++;
#endif
    if (!fit_ok) break;  // node.cpp:1142-1145
    double err;
    const int cnt = score_all<NW>(sfrom, sto, M, nw, lane, T, sel, err);  // node.cpp:1148
#ifdef RB200_PROFILE
    pf_score += clock64() - c1;
#endif
    if ((unsigned)cnt < min_thr || err > (double)c_params.max_dist_m) break;  // node.cpp:1154
    if (cnt >= refined_cnt && err <= refined_err) {                             // node.cpp:1160
      const int prev = refined_cnt;
      refined = T;
      refined_cnt = cnt;
      refined_err = err;
      if (cnt == prev) break;  // node.cpp:1166
    } else
      break;
  }
#ifdef RB200_PROFILE
  if (lane == 0) {
    const int ph = n_begin == 0 ? 0 : (n_end < H ? 1 : 2);
    atomicAdd(&g_ransac_prof[ph][0], (unsigned long long)pf_fit);
    atomicAdd(&g_ransac_prof[ph][1], (unsigned long long)pf_score);
    atomicAdd(&g_ransac_prof[ph][2], (unsigned long long)pf_rounds);
    atomicAdd(&g_ransac_prof[ph][3], 1ull);
    atomicAdd(&g_ransac_prof[ph][4], (unsigned long long)(clock64() - pf_t0));
    atomicMax(&g_ransac_prof[ph][5], (unsigned long long)(clock64() - pf_t0));
    atomicMax(&g_ransac_prof[ph][6], (unsigned long long)pf_rounds);
  }
#endif
  if (lane == 0) {
    HypResult r;
    r.err = refined_err;
    r.count = refined_cnt;
    r.pad_ = 0;
#pragma unroll
    for (int i = 0; i < 9; i++) r.T[i] = refined.R[i];
#pragma unroll
    for (int i = 0; i < 3; i++) r.T[9 + i] = refined.t[i];
    hyp[(size_t)p * H + n] = r;
    if (publish) {
      s_cnt[n] = refined_cnt;
      s_err[n] = refined_err;
    }
  }
  }  // active
  if (publish) {
    __syncthreads();
    if (threadIdx.x == 0) {
      const ScanState st = ransac_scan(s_cnt, s_err, M, min_thr, n_end < H ? n_end : H);
      next_n[p] = st.done ? H : st.next_n;
    }
  }
}

cudaError_t launch_ransac_hypotheses(int npairs, int ransac_iterations, int max_matches, uint64_t seed,
                                     int64_t first_pair, const float4* mfrom, const float4* mto,
                                     const int32_t* n_all, HypResult* hyp, float* cen, int32_t* next_n, cudaStream_t stream,
                                     int* n_launches) {
  if (n_launches) *n_launches = 0;
  if (npairs <= 0 || ransac_iterations <= 0) return cudaSuccess;
  const int H = ransac_iterations;
  const int bounds[4] = {0, RB200_PH1, RB200_PH2, H};  // non-final phase ends must stay <= kMaxScanPrefix
  // the first phase can hand its scan result to the later ones when it runs as ONE CTA per pair
  const int first_end = bounds[1] < H ? bounds[1] : H;
  int32_t* nn = (first_end <= kRansacWarps && bounds[2] == bounds[1]) ? next_n : nullptr;
  for (int ph = 0; ph < 3; ph++) {
    const int n_begin = bounds[ph], n_end = bounds[ph + 1] < H ? bounds[ph + 1] : H;
    if (n_begin >= n_end) continue;
    dim3 grid((n_end - n_begin + kRansacWarps - 1) / kRansacWarps, npairs);
    if (max_matches <= 320)
      ransac_hyp_kernel<10><<<grid, kRansacWarps * 32, 0, stream>>>(H, max_matches, n_begin, n_end, seed, first_pair, mfrom, mto,
                                                                    n_all, hyp, cen, nn);
    else
      ransac_hyp_kernel<kMaxMaskWords><<<grid, kRansacWarps * 32, 0, stream>>>(H, max_matches, n_begin, n_end, seed, first_pair,
                                                                               mfrom, mto, n_all, hyp, cen, nn);
    if (n_launches) (*n_launches)++;
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) return e;
  }
  return cudaSuccess;
}

// One warp per pair.
template <int NW>
__global__ void __launch_bounds__(32)
    ransac_select_kernel(const PairDesc* __restrict__ pairs, int H, int maxM, const float4* __restrict__ mfrom,
                         const float4* __restrict__ mto, const int32_t* __restrict__ n_all,
                         const rgbdslam_b200_dmatch* __restrict__ matches, const HypResult* __restrict__ hyp,
                         rgbdslam_b200_pair_result* __restrict__ results,
                         rgbdslam_b200_dmatch* __restrict__ inlier_matches) {
  const int p = blockIdx.x;
  const int lane = threadIdx.x;
  const PairDesc pd = pairs[p];
  const int M = n_all[p];
#if RB200_SELECT_STAGED
  // One warp per pair is a chain of dependent global-memory round trips (records -> scan -> winner -> points -> matches);
  // issue every independent load up front: the hypothesis records, the match points and the match list go to shared memory /
  // registers together, the scan and the scoring then run from on-chip data.
  extern __shared__ double sel_smem[];  // H err | H count | NW*32 from | NW*32 to
  float4* sfrom = reinterpret_cast<float4*>(sel_smem + ((H + (H + 1) / 2 + 1) & ~1));  // 16-byte aligned
  float4* sto = sfrom + NW * 32;
  rgbdslam_b200_dmatch mreg[NW];
  {
    const float4* gfrom = mfrom + (size_t)p * maxM;
    const float4* gto = mto + (size_t)p * maxM;
#pragma unroll
    for (int w = 0; w < NW; w++) {
      const int i = w * 32 + lane;
      if (i < M) {
        sfrom[i] = gfrom[i];
        sto[i] = gto[i];
        mreg[w] = matches[(size_t)p * maxM + i];
      }
    }
  }
#else
  const float4* sfrom = mfrom + (size_t)p * maxM;
  const float4* sto = mto + (size_t)p * maxM;
#endif

  rgbdslam_b200_pair_result res;
  res.id1 = res.id2 = -1;
  res.n_all_matches = M;
  res.n_inliers = 0;
  res.rmse = 0.f;  // MatchingResult(): rmse(0.0)
  res.valid_iterations = 0;
#pragma unroll
  for (int i = 0; i < 16; i++) res.ransac_trafo[i] = (i % 5 == 0) ? 1.f : 0.f;
  res.info_scale = 0.0;
  res.used_identity = 0;
  res.inlier_points = res.outlier_points = res.occluded_points = res.all_points = 0;
  res.reserved_ = 0;

  // matchNodePair: all_matches.size() < min_matches -> no RANSAC (node.cpp:1319);
  // getRelativeTransformationTo: size <= min_matches -> false (node.cpp:1087)
  const bool run = (M >= c_params.min_matches) && (M > c_params.min_matches);
  if (run) {
    const int nw = (M + 31) >> 5;
    const unsigned min_thr = min_inlier_threshold(M);
    const HypResult* hp = hyp + (size_t)p * H;
#if !RB200_SELECT_STAGED
    extern __shared__ double sel_smem[];  // H doubles (err) followed by H ints (count)
#endif
    double* err_s = sel_smem;
    int* cnt_s = reinterpret_cast<int*>(sel_smem + H);
    if (M >= 4) {
      for (int i = lane; i < H; i += 32) {
        cnt_s[i] = hp[i].count;
        err_s[i] = hp[i].err;
      }
    }
    __syncwarp();
#if RB200_SELECT_STAGED
    const ScanState st = ransac_scan_warp(cnt_s, err_s, M, min_thr, M >= 4 ? H : 0, lane);
#else
    const ScanState st = ransac_scan(cnt_s, err_s, M, min_thr, M >= 4 ? H : 0);
#endif
    float rmse = st.rmse;
    int best_n = st.best_n, valid = st.valid;
    Rt T;
#pragma unroll
    for (int i = 0; i < 9; i++) T.R[i] = (i % 4 == 0) ? 1.f : 0.f;
    T.t[0] = T.t[1] = T.t[2] = 0.f;
    uint32_t words[NW];
#pragma unroll
    for (int w = 0; w < NW; w++) words[w] = 0;
    int n_inl = 0;
    if (best_n >= 0) {
#pragma unroll
      for (int i = 0; i < 9; i++) T.R[i] = hp[best_n].T[i];
#pragma unroll
      for (int i = 0; i < 3; i++) T.t[i] = hp[best_n].T[9 + i];
      double err;
      n_inl = score_all<NW>(sfrom, sto, M, nw, lane, T, words, err);  // bit-identical to the hypothesis kernel's pass
    } else if (valid == 0) {  // identity as last resort (node.cpp:1192-1215)
      double err;
      const int cnt = score_all<NW>(sfrom, sto, M, nw, lane, T, words, err);
      if ((unsigned)cnt > min_thr && err < (double)c_params.max_dist_m) {
        n_inl = cnt;
        rmse = (float)err;
        valid = 1;
        res.used_identity = 1;
      } else {
#pragma unroll
        for (int w = 0; w < NW; w++) words[w] = 0;
      }
    }
    res.valid_iterations = valid;
    res.rmse = rmse;
    res.n_inliers = n_inl;
    // column-major Matrix4f
    res.ransac_trafo[0] = T.R[0]; res.ransac_trafo[1] = T.R[3]; res.ransac_trafo[2] = T.R[6];
    res.ransac_trafo[4] = T.R[1]; res.ransac_trafo[5] = T.R[4]; res.ransac_trafo[6] = T.R[7];
    res.ransac_trafo[8] = T.R[2]; res.ransac_trafo[9] = T.R[5]; res.ransac_trafo[10] = T.R[8];
    res.ransac_trafo[12] = T.t[0]; res.ransac_trafo[13] = T.t[1]; res.ransac_trafo[14] = T.t[2];
    // compact the inlier matches in all_matches order
    if (inlier_matches) {
      int base = 0;
#pragma unroll
      for (int w = 0; w < NW; w++) {
        if (w < nw) {
          const uint32_t word = words[w];
          if ((word >> lane) & 1u) {
            const int pos = base + __popc(word & ((1u << lane) - 1u));
#if RB200_SELECT_STAGED
            inlier_matches[(size_t)p * maxM + pos] = mreg[w];
#else
            inlier_matches[(size_t)p * maxM + pos] = matches[(size_t)p * maxM + w * 32 + lane];
#endif
          }
          base += __popc(word);
        }
      }
    }
    if ((unsigned)n_inl >= min_thr) {  // node.cpp:1275, then node.cpp:1335-1339
      res.info_scale = (double)((float)n_inl / (rmse * rmse));
      res.id1 = pd.id_t;
      res.id2 = pd.id_q;
    }
  }
  if (lane == 0) results[p] = res;
}

cudaError_t launch_ransac_select(const PairDesc* pairs, int npairs, int ransac_iterations, int max_matches,
                                 const float4* mfrom, const float4* mto, const int32_t* n_all,
                                 const rgbdslam_b200_dmatch* matches, const HypResult* hyp,
                                 rgbdslam_b200_pair_result* results, rgbdslam_b200_dmatch* inlier_matches,
                                 cudaStream_t stream) {
  if (npairs <= 0) return cudaSuccess;
#if RB200_SELECT_STAGED
  const int nwords = max_matches <= 320 ? 10 : kMaxMaskWords;
  const size_t smem = (size_t)((ransac_iterations + (ransac_iterations + 1) / 2 + 1) & ~1) * 8 + (size_t)nwords * 32 * 32 + 16;
#else
  const size_t smem = (size_t)ransac_iterations * 12 + 16;
#endif
  if (smem > 48 * 1024) {
    cudaError_t e = cudaFuncSetAttribute(ransac_select_kernel<10>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e == cudaSuccess)
      e = cudaFuncSetAttribute(ransac_select_kernel<kMaxMaskWords>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) return e;
  }
  if (max_matches <= 320)
    ransac_select_kernel<10><<<npairs, 32, smem, stream>>>(pairs, ransac_iterations, max_matches, mfrom, mto, n_all, matches, hyp,
                                                           results, inlier_matches);
  else
    ransac_select_kernel<kMaxMaskWords><<<npairs, 32, smem, stream>>>(pairs, ransac_iterations, max_matches, mfrom, mto, n_all,
                                                                      matches, hyp, results, inlier_matches);
  return cudaGetLastError();
}

// =====================================================================================================
// Pairwise g2o refinement (SURVEY.md 8a row a16; parameter g2o_transformation_refinement, default 0 = off).
// getTransformFromMatchesG2O (transformation_estimation.cpp:126-170): a 2-camera bundle adjustment over the current
// inliers -- camera 2 (newer node) fixed at identity, camera 1 (earlier node) seeded with the estimate, one
// VertexPointXYZ per match seeded with the newer node's 3-D position, two EdgeSE3PointXYZDepth per match with
// measurement (u, v, depth), information diag(1, 1, 1 / depth_covariance) (misc2.h:37-47), Kcam (521, 521, 319.5, 239.5)
// (:56), `iterations` undamped Gauss-Newton steps.  The reference solves the full (6 + 3n) system with cholmod (no
// marginalisation); here the 3x3 point blocks are eliminated analytically (Schur complement onto the 6x6 camera block),
// which is the same linear solution.  One warp per pair, lanes own matches l, l+32, ...; float64 throughout.
__device__ __forceinline__ void cam_from_rt(const Rt& T, Cam& c) {  // Quaterniond(Matrix3d) -> normalise -> rotation matrix
  double m[3][3];
#pragma unroll
  for (int r = 0; r < 3; r++)
#pragma unroll
    for (int k = 0; k < 3; k++) m[r][k] = (double)T.R[3 * r + k];
  double q[4];
  const double tr = m[0][0] + m[1][1] + m[2][2];
  if (tr > 0) {
    double s = sqrt(tr + 1.0);
    q[3] = 0.5 * s;
    s = 0.5 / s;
    q[0] = (m[2][1] - m[1][2]) * s; q[1] = (m[0][2] - m[2][0]) * s; q[2] = (m[1][0] - m[0][1]) * s;
  } else {
    int i = 0;
    if (m[1][1] > m[0][0]) i = 1;
    if (m[2][2] > m[i][i]) i = 2;
    const int j = (i + 1) % 3, k = (j + 1) % 3;
    double s = sqrt(m[i][i] - m[j][j] - m[k][k] + 1.0);
    q[i] = 0.5 * s;
    s = 0.5 / s;
    q[3] = (m[k][j] - m[j][k]) * s;
    q[j] = (m[j][i] + m[i][j]) * s;
    q[k] = (m[k][i] + m[i][k]) * s;
  }
  const double n = sqrt(q[0] * q[0] + q[1] * q[1] + q[2] * q[2] + q[3] * q[3]);
  const double x = q[0] / n, y = q[1] / n, z = q[2] / n, w = q[3] / n;
  c.R[0] = 1 - 2 * (y * y + z * z); c.R[1] = 2 * (x * y - z * w);     c.R[2] = 2 * (x * z + y * w);
  c.R[3] = 2 * (x * y + z * w);     c.R[4] = 1 - 2 * (x * x + z * z); c.R[5] = 2 * (y * z - x * w);
  c.R[6] = 2 * (x * z - y * w);     c.R[7] = 2 * (y * z + x * w);     c.R[8] = 1 - 2 * (x * x + y * y);
#pragma unroll
  for (int r = 0; r < 3; r++) c.t[r] = (double)T.t[r];
}

// The normal-equation blocks of one match (both edges).  Hpp / Hcc symmetric (full storage), Hcp 6x3.
struct PointBlocks {
  double Hpp[9], bp[3], Hcp[18], Hcc[36], bc[6];
};

__device__ __forceinline__ void point_blocks(const Cam& c1, const double pw[3], const double m1[3], double w1, const double m2[3],
                                             double w2, PointBlocks& B) {
  double e[3], Jc[18], Jp[9];
  edge_depth(c1, pw, m1, e, Jc, Jp);
  const double om1[3] = {1.0, 1.0, w1};
#pragma unroll
  for (int i = 0; i < 3; i++) {
    B.bp[i] = 0;
#pragma unroll
    for (int j = 0; j < 3; j++) B.Hpp[3 * i + j] = 0;
  }
#pragma unroll
  for (int i = 0; i < 6; i++) {
    B.bc[i] = 0;
#pragma unroll
    for (int j = 0; j < 6; j++) B.Hcc[6 * i + j] = 0;
#pragma unroll
    for (int j = 0; j < 3; j++) B.Hcp[3 * i + j] = 0;
  }
#pragma unroll
  for (int r = 0; r < 3; r++) {
#pragma unroll
    for (int i = 0; i < 3; i++) {
      B.bp[i] -= Jp[3 * r + i] * om1[r] * e[r];
#pragma unroll
      for (int j = 0; j < 3; j++) B.Hpp[3 * i + j] += Jp[3 * r + i] * om1[r] * Jp[3 * r + j];
    }
#pragma unroll
    for (int i = 0; i < 6; i++) {
      B.bc[i] -= Jc[6 * r + i] * om1[r] * e[r];
#pragma unroll
      for (int j = 0; j < 6; j++) B.Hcc[6 * i + j] += Jc[6 * r + i] * om1[r] * Jc[6 * r + j];
#pragma unroll
      for (int j = 0; j < 3; j++) B.Hcp[3 * i + j] += Jc[6 * r + i] * om1[r] * Jp[3 * r + j];
    }
  }
  Cam c2;
#pragma unroll
  for (int i = 0; i < 9; i++) c2.R[i] = (i % 4 == 0) ? 1.0 : 0.0;
  c2.t[0] = c2.t[1] = c2.t[2] = 0.0;
  edge_depth(c2, pw, m2, e, Jc, Jp);  // camera 2 is fixed: only the point block
  const double om2[3] = {1.0, 1.0, w2};
#pragma unroll
  for (int r = 0; r < 3; r++)
#pragma unroll
    for (int i = 0; i < 3; i++) {
      B.bp[i] -= Jp[3 * r + i] * om2[r] * e[r];
#pragma unroll
      for (int j = 0; j < 3; j++) B.Hpp[3 * i + j] += Jp[3 * r + i] * om2[r] * Jp[3 * r + j];
    }
}

// Runs the bundle adjustment over the matches selected by `mask` (warp-uniform words); T in: estimate, out: result.
template <int NW>
__device__ void ba_refine(const float4* __restrict__ xyz_n, const float4* __restrict__ xyz_e, const float2* __restrict__ kp_n,
                          const float2* __restrict__ kp_e, const uint32_t* mask, int nw, int lane, int iterations, Rt& T,
                          double* __restrict__ pts /* 3 doubles per match, indexed like the match list */) {
  Cam c1;
  cam_from_rt(T, c1);
  const double cz_const = c_params.cov_z_const;
#pragma unroll 1
  for (int w = 0; w < nw; w++)
    if ((mask[w] >> lane) & 1u) {
      const int i = w * 32 + lane;
      const float4 pn = xyz_n[i];
      double* q = pts + 3 * i;
      if (!isnan(pn.z)) { q[0] = pn.x; q[1] = pn.y; q[2] = pn.z; }
      else { q[0] = (double)pn.x * 10; q[1] = (double)pn.y * 10; q[2] = 10.0; }
    }
  __syncwarp();
  for (int it = 0; it < iterations; it++) {
    double S[27];  // 21 unique entries of the reduced 6x6 (upper triangle, row-major) + 6 right-hand sides
#pragma unroll
    for (int k = 0; k < 27; k++) S[k] = 0.0;
    bool ok = true;
#pragma unroll 1
    for (int w = 0; w < nw; w++)
      if ((mask[w] >> lane) & 1u) {
        const int i = w * 32 + lane;
        const float4 pe = xyz_e[i], pn = xyz_n[i];
        const float2 ke = kp_e[i], kn = kp_n[i];
        const double d1 = isnan(pe.z) ? 10.0 : (double)pe.z, d2 = isnan(pn.z) ? 10.0 : (double)pn.z;
        const double m1[3] = {ke.x, ke.y, d1}, m2[3] = {kn.x, kn.y, d2};
        const double w1 = 1.0 / (cz_const >= 0.0 ? cz_const : depth_cov(d1)), w2 = 1.0 / (cz_const >= 0.0 ? cz_const : depth_cov(d2));
        PointBlocks B;
        point_blocks(c1, pts + 3 * i, m1, w1, m2, w2, B);
        double inv[9];
        if (!inv3_sym(B.Hpp, inv)) { ok = false; continue; }
        double Y[18];  // Hcp * Hpp^-1
#pragma unroll
        for (int r = 0; r < 6; r++)
#pragma unroll
          for (int k = 0; k < 3; k++) Y[3 * r + k] = B.Hcp[3 * r] * inv[k] + B.Hcp[3 * r + 1] * inv[3 + k] + B.Hcp[3 * r + 2] * inv[6 + k];
        int idx = 0;
#pragma unroll
        for (int r = 0; r < 6; r++) {
#pragma unroll
          for (int k = r; k < 6; k++)
            S[idx++] += B.Hcc[6 * r + k] - (Y[3 * r] * B.Hcp[3 * k] + Y[3 * r + 1] * B.Hcp[3 * k + 1] + Y[3 * r + 2] * B.Hcp[3 * k + 2]);
        }
#pragma unroll
        for (int r = 0; r < 6; r++) S[21 + r] += B.bc[r] - (Y[3 * r] * B.bp[0] + Y[3 * r + 1] * B.bp[1] + Y[3 * r + 2] * B.bp[2]);
      }
#pragma unroll
    for (int k = 0; k < 27; k++) S[k] = wsumd(S[k]);
    ok = __all_sync(kFull, ok);
    // 6x6 Cholesky solve (warp-uniform)
    double L[36], dc[6];
    {
      int idx = 0;
#pragma unroll
      for (int r = 0; r < 6; r++)
#pragma unroll
        for (int k = r; k < 6; k++) { L[6 * k + r] = S[idx]; L[6 * r + k] = S[idx]; idx++; }
    }
#pragma unroll
    for (int j = 0; j < 6; j++) {
      double sj = L[6 * j + j];
#pragma unroll
      for (int k = 0; k < 6; k++) if (k < j) sj -= L[6 * j + k] * L[6 * j + k];
      if (!(sj > 0.0)) ok = false;
      const double l = sqrt(sj);
      L[6 * j + j] = l;
#pragma unroll
      for (int i = 0; i < 6; i++)
        if (i > j) {
          double v = L[6 * i + j];
#pragma unroll
          for (int k = 0; k < 6; k++) if (k < j) v -= L[6 * i + k] * L[6 * j + k];
          L[6 * i + j] = v / l;
        }
    }
    if (!ok) break;  // the linear solver failed: the optimisation stops (g2o returns from optimize())
#pragma unroll
    for (int i = 0; i < 6; i++) {
      double v = S[21 + i];
#pragma unroll
      for (int k = 0; k < 6; k++) if (k < i) v -= L[6 * i + k] * dc[k];
      dc[i] = v / L[6 * i + i];
    }
#pragma unroll
    for (int ii = 0; ii < 6; ii++) {
      const int i = 5 - ii;
      double v = dc[i];
#pragma unroll
      for (int k = 0; k < 6; k++) if (k > i) v -= L[6 * k + i] * dc[k];
      dc[i] = v / L[6 * i + i];
    }
    // back-substitution of the points (same blocks, recomputed) BEFORE the camera moves
#pragma unroll 1
    for (int w = 0; w < nw; w++)
      if ((mask[w] >> lane) & 1u) {
        const int i = w * 32 + lane;
        const float4 pe = xyz_e[i], pn = xyz_n[i];
        const float2 ke = kp_e[i], kn = kp_n[i];
        const double d1 = isnan(pe.z) ? 10.0 : (double)pe.z, d2 = isnan(pn.z) ? 10.0 : (double)pn.z;
        const double m1[3] = {ke.x, ke.y, d1}, m2[3] = {kn.x, kn.y, d2};
        const double w1 = 1.0 / (cz_const >= 0.0 ? cz_const : depth_cov(d1)), w2 = 1.0 / (cz_const >= 0.0 ? cz_const : depth_cov(d2));
        PointBlocks B;
        point_blocks(c1, pts + 3 * i, m1, w1, m2, w2, B);
        double inv[9];
        inv3_sym(B.Hpp, inv);
        double r3[3];
#pragma unroll
        for (int k = 0; k < 3; k++) {
          double v = B.bp[k];
#pragma unroll
          for (int r = 0; r < 6; r++) v -= B.Hcp[3 * r + k] * dc[r];
          r3[k] = v;
        }
#pragma unroll
        for (int k = 0; k < 3; k++) pts[3 * i + k] += inv[3 * k] * r3[0] + inv[3 * k + 1] * r3[1] + inv[3 * k + 2] * r3[2];
      }
    __syncwarp();
    cam_oplus(c1, dc);
  }
  // cams.first->estimate().cast<float>().inverse().matrix()
  float Rf[9], tf[3];
#pragma unroll
  for (int i = 0; i < 9; i++) Rf[i] = (float)c1.R[i];
#pragma unroll
  for (int i = 0; i < 3; i++) tf[i] = (float)c1.t[i];
#pragma unroll
  for (int r = 0; r < 3; r++) {
#pragma unroll
    for (int k = 0; k < 3; k++) T.R[3 * r + k] = Rf[3 * k + r];
    T.t[r] = -(__fmul_rn(Rf[r], tf[0]) + __fmul_rn(Rf[3 + r], tf[1]) + __fmul_rn(Rf[6 + r], tf[2]));
  }
}

// node.cpp:1225-1268 on the result of ransac_select_kernel.  One warp per pair.
template <int NW>
__global__ void __launch_bounds__(32)
    refine_g2o_kernel(const PairDesc* __restrict__ pairs, int maxM, int iterations, const float4* __restrict__ mfrom,
                      const float4* __restrict__ mto, const int32_t* __restrict__ n_all,
                      const rgbdslam_b200_dmatch* __restrict__ matches, rgbdslam_b200_pair_result* __restrict__ results,
                      rgbdslam_b200_dmatch* __restrict__ inlier_matches) {
  extern __shared__ double refine_smem[];  // pts: 3 * maxM doubles, then keypoints 2 x maxM float2
  const int p = blockIdx.x, lane = threadIdx.x;
  const PairDesc pd = pairs[p];
  const int M = n_all[p];
  rgbdslam_b200_pair_result res = results[p];
  const unsigned min_thr = min_inlier_threshold(M);
  if (!(M > c_params.min_matches && M >= 4 && (unsigned)res.n_inliers > min_thr)) return;  // :1226
  double* pts = refine_smem;
  float2* kp_n = reinterpret_cast<float2*>(refine_smem + 3 * maxM);
  float2* kp_e = kp_n + maxM;
  const float4* sfrom = mfrom + (size_t)p * maxM;
  const float4* sto = mto + (size_t)p * maxM;
  for (int i = lane; i < M; i += 32) {
    const rgbdslam_b200_dmatch m = matches[(size_t)p * maxM + i];
    kp_n[i] = make_float2(pd.q_kp[m.queryIdx].x, pd.q_kp[m.queryIdx].y);
    kp_e[i] = make_float2(pd.t_kp[m.trainIdx].x, pd.t_kp[m.trainIdx].y);
  }
  __syncwarp();
  const int nw = (M + 31) >> 5;
  Rt T;
  T.R[0] = res.ransac_trafo[0]; T.R[1] = res.ransac_trafo[4]; T.R[2] = res.ransac_trafo[8];
  T.R[3] = res.ransac_trafo[1]; T.R[4] = res.ransac_trafo[5]; T.R[5] = res.ransac_trafo[9];
  T.R[6] = res.ransac_trafo[2]; T.R[7] = res.ransac_trafo[6]; T.R[8] = res.ransac_trafo[10];
  T.t[0] = res.ransac_trafo[12]; T.t[1] = res.ransac_trafo[13]; T.t[2] = res.ransac_trafo[14];
  uint32_t words0[NW], words1[NW];
  double err0;
  const int cnt0 = score_all<NW>(sfrom, sto, M, nw, lane, T, words0, err0);  // == the inlier set ransac_select stored
  Rt T1 = T;
  ba_refine<NW>(sfrom, sto, kp_n, kp_e, words0, nw, lane, iterations, T1, pts);
  double err1;
  int cnt1 = score_all<NW>(sfrom, sto, M, nw, lane, T1, words1, err1);
  bool accept = false;
  if (cnt1 >= cnt0 || ((unsigned)cnt1 >= min_thr && err1 < (double)res.rmse)) {  // :1241
    if (cnt1 > cnt0) {                                                           // :1243-1251
      ba_refine<NW>(sfrom, sto, kp_n, kp_e, words1, nw, lane, iterations, T1, pts);
      cnt1 = score_all<NW>(sfrom, sto, M, nw, lane, T1, words1, err1);
    }
    accept = cnt1 >= cnt0;  // :1254
  }
  if (!accept) return;
  res.n_inliers = cnt1;
  res.rmse = (float)err1;
  res.valid_iterations += 1;
  res.ransac_trafo[0] = T1.R[0]; res.ransac_trafo[1] = T1.R[3]; res.ransac_trafo[2] = T1.R[6];
  res.ransac_trafo[4] = T1.R[1]; res.ransac_trafo[5] = T1.R[4]; res.ransac_trafo[6] = T1.R[7];
  res.ransac_trafo[8] = T1.R[2]; res.ransac_trafo[9] = T1.R[5]; res.ransac_trafo[10] = T1.R[8];
  res.ransac_trafo[12] = T1.t[0]; res.ransac_trafo[13] = T1.t[1]; res.ransac_trafo[14] = T1.t[2];
  if (inlier_matches) {
    int base = 0;
#pragma unroll
    for (int w = 0; w < NW; w++) {
      if (w < nw) {
        const uint32_t word = words1[w];
        if ((word >> lane) & 1u) {
          const int pos = base + __popc(word & ((1u << lane) - 1u));
          inlier_matches[(size_t)p * maxM + pos] = matches[(size_t)p * maxM + w * 32 + lane];
        }
        base += __popc(word);
      }
    }
  }
  if ((unsigned)cnt1 >= min_thr) {
    res.info_scale = (double)((float)cnt1 / (res.rmse * res.rmse));
    res.id1 = pd.id_t;
    res.id2 = pd.id_q;
  }
  if (lane == 0) results[p] = res;
}

cudaError_t launch_refine_g2o(const PairDesc* pairs, int npairs, int max_matches, int iterations, const float4* mfrom,
                              const float4* mto, const int32_t* n_all, const rgbdslam_b200_dmatch* matches,
                              rgbdslam_b200_pair_result* results, rgbdslam_b200_dmatch* inlier_matches, cudaStream_t stream) {
  if (npairs <= 0 || iterations <= 0) return cudaSuccess;
  const size_t smem = (size_t)max_matches * (24 + 16);
  if (max_matches <= 320)
    refine_g2o_kernel<10><<<npairs, 32, smem, stream>>>(pairs, max_matches, iterations, mfrom, mto, n_all, matches, results,
                                                        inlier_matches);
  else
    refine_g2o_kernel<kMaxMaskWords><<<npairs, 32, smem, stream>>>(pairs, max_matches, iterations, mfrom, mto, n_all, matches,
                                                                   results, inlier_matches);
  return cudaGetLastError();
}

}  // namespace rb200
