// sift_l2.cu -- the SIFT-128 float-descriptor path (BASELINE config C3):
//   k_sift_prepare      squareroot_descriptor_space (RootSIFT, node.cpp:1557-1571) + bf16 operand tiles + |b|^2
//   tc_match_kernel<1>  (hamming_tc.cu) N x M score matrix 2 a.b - |b|^2 as a bf16 wgmma GEMM, 4 best per query
//   k_l2_refine         exact fp32 squared L2 of the 4 candidates -> exact 2-NN among them
//   k_select_sift       ratio test (nn_distance_ratio) + first-come uniqueness of trainIdx + keepStrongestMatches
//                       (node.cpp:638-667, 674) -- replaces the approximate FLANN kd-tree 2-NN of node.cpp:493-514,610-636
#include <cuda_bf16.h>

#include "kernels.h"

namespace rb200 {

// one warp per descriptor row (128 floats: 4 per lane)
__global__ void __launch_bounds__(256) k_sift_prepare(const SiftJob* __restrict__ jobs, int root_sift, int siftgpu) {
  const SiftJob job = jobs[blockIdx.y];
  const int row = blockIdx.x * 8 + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (row >= job.n_pad) return;
  float4 v = make_float4(0, 0, 0, 0);
  if (row < job.n) {
    v = reinterpret_cast<const float4*>(job.in + (size_t)row * 128)[lane];
    if (root_sift) {
      v.x = fabsf(v.x); v.y = fabsf(v.y); v.z = fabsf(v.z); v.w = fabsf(v.w);  // descriptors = cv::abs(descriptors)
      float s = (v.x + v.y) + (v.z + v.w);
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
      if (s != 0.f) {  // node.cpp:1565 (zero rows are left alone)
        v.x = sqrtf(__fdiv_rn(v.x, s)); v.y = sqrtf(__fdiv_rn(v.y, s));
        v.z = sqrtf(__fdiv_rn(v.z, s)); v.w = sqrtf(__fdiv_rn(v.w, s));
      }
    }
    reinterpret_cast<float4*>(job.root + (size_t)row * 128)[lane] = v;
  }
  const int tile = row >> 7, rg = (row >> 3) & 15, rr = row & 7;
  if (siftgpu) {
    // SiftMatchCU::SetDescriptors (SiftMatchCU.cpp:87-101): unsigned char(int(512 * d + 0.5)); 128 B of data per row in
    // k-chunks 0..7 of the 256 B tile row, chunks 8..15 zero (the MMA only walks the first 4 k-steps).
    const float q[4] = {v.x, v.y, v.z, v.w};
    uint32_t pk = 0;
#pragma unroll
    for (int k = 0; k < 4; k++) {
      const int iv = (int)((double)__fmul_rn(512.0f, q[k]) + 0.5);
      pk |= ((uint32_t)iv & 0xFFu) << (8 * k);
    }
    uint8_t* base = reinterpret_cast<uint8_t*>(job.tiles) + (size_t)tile * 32768 + rg * 2048 + rr * 16;
    *reinterpret_cast<uint32_t*>(base + (lane >> 2) * 128 + (lane & 3) * 4) = pk;
    *reinterpret_cast<uint32_t*>(base + (8 + (lane >> 2)) * 128 + (lane & 3) * 4) = 0u;
    if (lane == 0) job.norms[row] = 0.f;
    return;
  }
  const __nv_bfloat16 b0 = __float2bfloat16_rn(v.x), b1 = __float2bfloat16_rn(v.y), b2 = __float2bfloat16_rn(v.z),
                      b3 = __float2bfloat16_rn(v.w);
  const float f0 = __bfloat162float(b0), f1 = __bfloat162float(b1), f2 = __bfloat162float(b2), f3 = __bfloat162float(b3);
  float nrm = (f0 * f0 + f1 * f1) + (f2 * f2 + f3 * f3);
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) nrm += __shfl_xor_sync(0xffffffffu, nrm, o);
  if (lane == 0) job.norms[row] = nrm;
  // tile layout [row_group 16][k_chunk 16][row_in_group 8][16 B]; lane's 4 elements = 8 B of chunk lane/2
  const int kc = lane >> 1, half = lane & 1;
  uint2 pk;
  pk.x = (uint32_t)__bfloat16_as_ushort(b0) | ((uint32_t)__bfloat16_as_ushort(b1) << 16);
  pk.y = (uint32_t)__bfloat16_as_ushort(b2) | ((uint32_t)__bfloat16_as_ushort(b3) << 16);
  uint8_t* dst = reinterpret_cast<uint8_t*>(job.tiles) + (size_t)tile * 32768 + rg * 2048 + kc * 128 + rr * 16 + half * 8;
  *reinterpret_cast<uint2*>(dst) = pk;
}

cudaError_t launch_sift_prepare(const SiftJob* d_jobs, int njobs, int max_n_pad, int root_sift, int siftgpu, cudaStream_t stream) {
  if (njobs <= 0 || max_n_pad <= 0) return cudaSuccess;
  k_sift_prepare<<<dim3((max_n_pad + 7) / 8, njobs), 256, 0, stream>>>(d_jobs, siftgpu ? 0 : root_sift, siftgpu);
  return cudaGetLastError();
}

// exact fp32 re-ranking of the 4 tensor-core candidates: one warp per query.  knn[i] = {idx1, idx2, d1, d2}
__global__ void __launch_bounds__(256) k_l2_refine(const PairDesc* __restrict__ pairs, const int4* __restrict__ top4, int stride,
                                                   float4* __restrict__ knn) {
  const PairDesc pd = pairs[blockIdx.y];
  const int i = blockIdx.x * 8 + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (i >= pd.nq) return;
  const float4 a = reinterpret_cast<const float4*>(pd.q_f32 + (size_t)i * 128)[lane];
  const int4 c = top4[(size_t)blockIdx.y * stride + i];
  const int cand[4] = {c.x, c.y, c.z, c.w};
  float d[4];
#pragma unroll
  for (int k = 0; k < 4; k++) {
    float s = 3.0e38f;
    if (cand[k] >= 0) {
      const float4 b = reinterpret_cast<const float4*>(pd.t_f32 + (size_t)cand[k] * 128)[lane];
      const float dx = a.x - b.x, dy = a.y - b.y, dz = a.z - b.z, dw = a.w - b.w;
      s = (dx * dx + dy * dy) + (dz * dz + dw * dw);
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    }
    d[k] = s;
  }
  if (lane == 0) {
    int b1 = -1, b2 = -1;
    float d1 = 3.0e38f, d2 = 3.0e38f;
#pragma unroll
    for (int k = 0; k < 4; k++) {
      if (cand[k] < 0) continue;
      if (d[k] < d1 || (d[k] == d1 && cand[k] < b1)) {
        d2 = d1; b2 = b1; d1 = d[k]; b1 = cand[k];
      } else if (d[k] < d2 || (d[k] == d2 && cand[k] < b2)) {
        d2 = d[k]; b2 = cand[k];
      }
    }
    knn[(size_t)blockIdx.y * stride + i] = make_float4(__int_as_float(b1), __int_as_float(b2), d1, d2);
  }
}

cudaError_t launch_l2_refine(const PairDesc* pairs, int npairs, int max_nq, const int4* top4, int stride, float4* knn,
                             cudaStream_t stream) {
  if (npairs <= 0 || max_nq <= 0) return cudaSuccess;
  k_l2_refine<<<dim3((max_nq + 7) / 8, npairs), 256, 0, stream>>>(pairs, top4, stride, knn);
  return cudaGetLastError();
}

// node.cpp:638-667 + 674 + 1127: ratio = d1/d2 (squared distances, as cv::flann returns them); accept if
// nn_distance_ratio > ratio and the train index was not taken by an earlier query; distance = ratio; keep the
// max_matches strongest, sorted.  One CTA per pair.
__global__ void __launch_bounds__(512) k_select_sift(const PairDesc* __restrict__ pairs, const float4* __restrict__ knn, int stride,
                                                     float nn_ratio, int maxM, rgbdslam_b200_dmatch* __restrict__ matches,
                                                     float4* __restrict__ mfrom, float4* __restrict__ mto, int32_t* __restrict__ n_all) {
  extern __shared__ unsigned long long sift_smem[];  // keys[kMaxFeatures] then owner[kMaxFeatures]
  unsigned long long* keys = sift_smem;
  int* owner = reinterpret_cast<int*>(sift_smem + kMaxFeatures);
  __shared__ int s_count;
  const int p = blockIdx.x;
  const PairDesc pd = pairs[p];
  const int nq = min(pd.nq, kMaxFeatures);
  int N = 2;
  while (N < nq) N <<= 1;
  const float4* kp = knn + (size_t)p * stride;
  if (threadIdx.x == 0) s_count = 0;
  for (int i = threadIdx.x; i < kMaxFeatures; i += blockDim.x) owner[i] = 0x7fffffff;
  __syncthreads();
  for (int i = threadIdx.x; i < nq; i += blockDim.x) {
    const float4 k = kp[i];
    const int t1 = __float_as_int(k.x), t2 = __float_as_int(k.y);
    if (t1 >= 0 && t2 >= 0) {
      const float ratio = __fdiv_rn(k.z, k.w);
      if (nn_ratio > ratio) atomicMin(&owner[t1], i);  // first query (lowest index) keeps the train feature
    }
  }
  __syncthreads();
  for (int i = threadIdx.x; i < N; i += blockDim.x) {
    unsigned long long key = ~0ULL;
    if (i < nq) {
      const float4 k = kp[i];
      const int t1 = __float_as_int(k.x), t2 = __float_as_int(k.y);
      if (t1 >= 0 && t2 >= 0) {
        const float ratio = __fdiv_rn(k.z, k.w);
        if (nn_ratio > ratio && owner[t1] == i) key = ((unsigned long long)__float_as_uint(ratio) << 32) | (unsigned)i;
      }
    }
    keys[i] = key;
  }
  __syncthreads();
  for (int k = 2; k <= N; k <<= 1) {
    for (int j = k >> 1; j > 0; j >>= 1) {
      for (int t = threadIdx.x; t < (N >> 1); t += blockDim.x) {
        const int lo = ((t & ~(j - 1)) << 1) | (t & (j - 1));
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
  for (int i = threadIdx.x; i < N; i += blockDim.x)
    if (keys[i] != ~0ULL && (i == N - 1 || keys[i + 1] == ~0ULL)) s_count = i + 1;
  __syncthreads();
  const int M = min(s_count, maxM);
  for (int k = threadIdx.x; k < M; k += blockDim.x) {
    const unsigned long long kk = keys[k];
    const int qi = (int)(kk & 0xffffffffULL);
    const int ti = __float_as_int(kp[qi].x);
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

cudaError_t launch_select_sift(const PairDesc* pairs, int npairs, const float4* knn, int stride, float nn_ratio, int maxM,
                               rgbdslam_b200_dmatch* matches, float4* mfrom, float4* mto, int32_t* n_all, cudaStream_t stream) {
  if (npairs <= 0) return cudaSuccess;
  const int smem = kMaxFeatures * 12;
  static bool attr = false;
  if (!attr) {
    cudaError_t e = cudaFuncSetAttribute(k_select_sift, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
    if (e != cudaSuccess) return e;
    attr = true;
  }
  k_select_sift<<<npairs, 512, smem, stream>>>(pairs, knn, stride, nn_ratio, maxM, matches, mfrom, mto, n_all);
  return cudaGetLastError();
}

// matcher_type == "SIFTGPU" (node.cpp:553-557): SiftMatchGPU::GetSiftMatch(num1, buf, 0.9, 0.9) with mutual best match
// (SiftMatchCU.cpp:139-176) followed by SiftGPUWrapper::match's float L2 distance (sift_gpu_wrapper.cpp:169-227) and
// keepStrongestMatches + sort (node.cpp:674, 1127).  rowres / colres = {best dot, arg, runner-up dot, -} per query / train
// row from tc_match256_kernel<2>.  One CTA per pair.
__device__ __forceinline__ bool siftgpu_accept(int best, int next, float distmax, float ratiomax) {
  // ProgramCU.cu:1739-1742: acos(min(dot * 2^-18f, 1.0)) -- float product, double min / acos, stored to float
  const float dist = (float)acos(fmin((double)__fmul_rn((float)best, 0.000003814697265625f), 1.0));
  const float distn = (float)acos(fmin((double)__fmul_rn((float)next, 0.000003814697265625f), 1.0));
  return (dist < distmax) && (dist < __fmul_rn(distn, ratiomax));
}

__global__ void __launch_bounds__(512) k_select_siftgpu(const PairDesc* __restrict__ pairs, const int4* __restrict__ rowres,
                                                        const int4* __restrict__ colres, int stride, int maxM,
                                                        rgbdslam_b200_dmatch* __restrict__ matches, float4* __restrict__ mfrom,
                                                        float4* __restrict__ mto, int32_t* __restrict__ n_all) {
  extern __shared__ unsigned long long sift_smem[];  // keys[kMaxFeatures] then train index per query [kMaxFeatures]
  unsigned long long* keys = sift_smem;
  int* tidx = reinterpret_cast<int*>(sift_smem + kMaxFeatures);
  __shared__ int s_count, s_number, s_zero;
  const int p = blockIdx.x;
  const PairDesc pd = pairs[p];
  const int nq = min(pd.nq, kMaxFeatures), nt = min(pd.nt, kMaxFeatures);
  int N = 2;
  while (N < nq) N <<= 1;
  const int4* rr = rowres + (size_t)p * stride;
  const int4* cr = colres + (size_t)p * stride;
  if (threadIdx.x == 0) s_count = s_number = s_zero = 0;
  __syncthreads();
  const float distmax = 0.9f, ratiomax = 0.9f;  // sift_gpu_wrapper.cpp:184
  for (int i = threadIdx.x; i < nq; i += blockDim.x) {
    int j = -1;
    if (nt > 0) {
      const int4 r = rr[i];
      if (r.y >= 0 && siftgpu_accept(r.x, r.z, distmax, ratiomax)) {
        const int4 c = cr[r.y];
        if (c.y == i && siftgpu_accept(c.x, c.z, distmax, ratiomax)) j = r.y;  // buffer2[j] == i (SiftMatchCU.cpp:167)
      }
    }
    tidx[i] = j;
    if (j >= 0) {
      atomicAdd(&s_number, 1);
      if (i == 0 || j == 0) atomicAdd(&s_zero, 1);
    }
  }
  __syncthreads();
  // "matches bad due to context error": more than half of the matches involve index 0 (sift_gpu_wrapper.cpp:204-213)
  const bool cleared = (float)s_zero > 0.5f * (float)s_number;
  for (int i = threadIdx.x; i < N; i += blockDim.x) {
    unsigned long long key = ~0ULL;
    if (i < nq && !cleared && tidx[i] >= 0) {
      const float* a = pd.q_f32 + (size_t)i * 128;
      const float* b = pd.t_f32 + (size_t)tidx[i] * 128;
      float sum = 0.f;
      for (int k = 0; k < 128; k++) {  // sequential float accumulation like the host loop (:215-219)
        const float d = __fsub_rn(a[k], b[k]);
        sum = __fadd_rn(sum, __fmul_rn(d, d));
      }
      key = ((unsigned long long)__float_as_uint(__fsqrt_rn(sum)) << 32) | (unsigned)i;
    }
    keys[i] = key;
  }
  __syncthreads();
  for (int k = 2; k <= N; k <<= 1) {
    for (int j = k >> 1; j > 0; j >>= 1) {
      for (int t = threadIdx.x; t < (N >> 1); t += blockDim.x) {
        const int lo = ((t & ~(j - 1)) << 1) | (t & (j - 1));
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
  for (int i = threadIdx.x; i < N; i += blockDim.x)
    if (keys[i] != ~0ULL && (i == N - 1 || keys[i + 1] == ~0ULL)) s_count = i + 1;
  __syncthreads();
  const int M = min(s_count, maxM);
  for (int k = threadIdx.x; k < M; k += blockDim.x) {
    const unsigned long long kk = keys[k];
    const int qi = (int)(kk & 0xffffffffULL);
    const int ti = tidx[qi];
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

cudaError_t launch_select_siftgpu(const PairDesc* pairs, int npairs, const int4* rowres, const int4* colres, int stride, int maxM,
                                  rgbdslam_b200_dmatch* matches, float4* mfrom, float4* mto, int32_t* n_all, cudaStream_t stream) {
  if (npairs <= 0) return cudaSuccess;
  const int smem = kMaxFeatures * 12;
  static bool attr = false;
  if (!attr) {
    cudaError_t e = cudaFuncSetAttribute(k_select_siftgpu, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
    if (e != cudaSuccess) return e;
    attr = true;
  }
  k_select_siftgpu<<<npairs, 512, smem, stream>>>(pairs, rowres, colres, stride, maxM, matches, mfrom, mto, n_all);
  return cudaGetLastError();
}

}  // namespace rb200
