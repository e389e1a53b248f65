// emm.cu -- Environment Measurement Model (SURVEY.md 8f rank 3; parameter observability_threshold > 0):
//   k_build_cloud        the z-plane of createXYZRGBPointCloud (misc.cpp:467-556): every cloud_creation_skip_step-th pixel,
//                        NaN where !(Z >= minimum_depth); x / y are recomputed from the pixel grid (backProject, misc2.h:49-65)
//   k_split_cloud        Node::pc_col of the point-cloud constructor (node.cpp:261): x / y / z planes of an organised cloud
//   k_emm_pairs          pairwiseObservationLikelihood (node.cpp:1520-1554) = observationLikelihood (misc.cpp:814-969) in both
//                        directions + observation_criterion_met (misc.cpp:1136-1148) applied to the pair result
// Both EMM kernels are instantiated per point source (EmmPoints): depth-image nodes (the sub-sampled z-plane) and nodes that
// keep the organised cloud of the point-cloud constructor (RGBDSLAM_B200_KEEP_CLOUD).
// Dense projective data association on the sub-sampled clouds: embarrassingly parallel per sampled pixel, HBM / latency bound
// (<= 9 random depth reads per sample, 2 x (W/s/k) x (H/s/k) samples per pair: 2400 at the defaults s = 2, k = 8; kept clouds
// are sampled at full resolution, s = 1: 9600).
#include "kernels.h"

namespace rb200 {


__global__ void __launch_bounds__(256) k_build_cloud(const float* __restrict__ depth, int w, int h, int step, float scaling,
                                                     float min_depth, float* __restrict__ cloud_z, int cw, int ch) {
  const int i = blockIdx.x * 256 + threadIdx.x;
  if (i >= cw * ch) return;
  const int rx = i % cw, ry = i / cw;
  const int u = rx * step, v = ry * step;
  float z = __int_as_float(0x7fc00000);
  if (u < w && v < h) {
    const float Z = depth[(size_t)v * w + u] * scaling;  // misc.cpp:520
    if (Z >= min_depth) z = Z;                            // :523 (also rejects NaN)
  }
  cloud_z[i] = z;
}

cudaError_t launch_build_cloud(const float* d_depth, int w, int h, int step, float scaling, float min_depth, float* cloud_z, int cw,
                               int ch, cudaStream_t stream) {
  if (cw <= 0 || ch <= 0) return cudaSuccess;
  k_build_cloud<<<(cw * ch + 255) / 256, 256, 0, stream>>>(d_depth, w, h, step, scaling, min_depth, cloud_z, cw, ch);
  return cudaGetLastError();
}

// De-interleave one organised cloud (n points of `stride` floats, x / y / z at 0 / 1 / 2) into three planes.
__global__ void __launch_bounds__(256) k_split_cloud(const float* __restrict__ cloud, int stride, int n, float* __restrict__ x,
                                                     float* __restrict__ y, float* __restrict__ z) {
  const int i = blockIdx.x * 256 + threadIdx.x;
  if (i >= n) return;
  const float* p = cloud + (size_t)i * stride;
  x[i] = p[0];
  y[i] = p[1];
  z[i] = p[2];
}

cudaError_t launch_split_cloud(const float* d_cloud, int stride, int n, float* x, float* y, float* z, cudaStream_t stream) {
  if (n <= 0) return cudaSuccess;
  k_split_cloud<<<(n + 255) / 256, 256, 0, stream>>>(d_cloud, stride, n, x, y, z);
  return cudaGetLastError();
}

struct EmmView {
  const float* z;   // cloud z-plane
  const float* x;   // kept clouds (EmmPoints::kCloud) only: x / y planes of the organised cloud
  const float* y;
  int cw, ch;
  float fx, fy, cx, cy;  // depth nodes: full-resolution intrinsics of the camera that took it; kept clouds: the camera the
                         // model projects into (the reference's depth_camera_fx / fy / cx / cy)
};

__device__ __forceinline__ int round_like_ref(float d) { return (int)floor((double)d + 0.5); }  // misc.cpp:804-807
// The same as x86-64 evaluates it: cvttsd2si gives INT_MIN for NaN, +-inf and values outside int32, and INT_MIN fails the
// `< 0` bound.  A device (int) cast gives 0 for NaN instead, which is inside the raster.  Only kept clouds reach the
// conversion with NaN (an untransformed point with NaN x and finite z, or +-inf x with +inf z).
__device__ __forceinline__ int round_x86(float d) {
  const double r = floor((double)d + 0.5);
  return (r >= -2147483648.0 && r < 2147483648.0) ? (int)r : INT_MIN;
}

// One direction of the model: the `src` cloud transformed by T (row-major R, t: src frame -> dst frame) and projected into
// the `dst` depth raster.  Each thread takes samples; returns this thread's (good, bad, occluded, all).
// The float chain (back-projection, R p + t, projection) and the double sigma sums are written with explicit _rn intrinsics
// in the reference's operation order: nvcc would otherwise contract them into FMAs, which the reference (built without
// -mfma) does not do, and a projection near a floor(x + 0.5) boundary could then pick a different neighbourhood.
__device__ __forceinline__ float dot3_rn(float a0, float b0, float a1, float b1, float a2, float b2) {  // (a0 b0 + a1 b1) + a2 b2
  return __fadd_rn(__fadd_rn(__fmul_rn(a0, b0), __fmul_rn(a1, b1)), __fmul_rn(a2, b2));
}

// Where the source points of a direction come from.
enum class EmmPoints {
  kDepth,  // depth-image nodes: the z-plane every cloud_creation_skip_step-th pixel, x / y back-projected from the pixel grid
  kCloud,  // kept organised clouds (RGBDSLAM_B200_KEEP_CLOUD): x / y / z as stored, full resolution.  With clouds as input the
           // reference sets topic_points, so cloud_creation_skip_step is 1 there: no division of the intrinsics, no sigma scaling
           // (misc.cpp:856-863, 903-905)
};

template <EmmPoints P>
__device__ void emm_direction(const EmmView& src, const EmmView& dst, const float R[9], const float t[3], int cloud_step_param,
                              int skip_step, double cov_z_const, double sigma_depth, unsigned& good, unsigned& bad, unsigned& occl,
                              unsigned& all) {
  constexpr bool kCloud = P == EmmPoints::kCloud;
  // a direction whose two clouds differ in width contributes nothing, not even to `all` (misc.cpp:844-847).  The
  // `width <= 1 || height <= 1` branch before it (:836-843) is unreachable: nodes_create* rejects frames below 96 px for
  // both detectors (orb_prepare), and clouds only come from there.
  if (kCloud && src.cw != dst.cw) return;
  const int cloud_step = kCloud ? 1 : cloud_step_param;
  const float sfxinv = (float)(1.0 / (double)src.fx), sfyinv = (float)(1.0 / (double)src.fy);  // misc.cpp:64-69
  // "downsampled cloud?" branch (misc.cpp:854-861): intrinsics of the raster the old cloud lives on
  const float fx = kCloud ? dst.fx : dst.fx / cloud_step, fy = kCloud ? dst.fy : dst.fy / cloud_step;
  const float cx = kCloud ? dst.cx : dst.cx / cloud_step, cy = kCloud ? dst.cy : dst.cy / cloud_step;
  const int nsx = (src.cw + skip_step - 1) / skip_step, nsy = (src.ch + skip_step - 1) / skip_step;
  for (int sidx = threadIdx.x; sidx < nsx * nsy; sidx += blockDim.x) {
    all++;  // the loop header increments `all` for every sampled raster cell (:872)
    const int rx = (sidx % nsx) * skip_step, ry = (sidx / nsx) * skip_step;
    const size_t si = (size_t)ry * src.cw + rx;
    float qx, qy, qz;
    if (kCloud) {
      // the stored point; pcl::transformPointCloud on a cloud that is not dense copies the input and leaves a point with any
      // non-finite coordinate untransformed (a +inf z stays +inf and is not skipped below)
      const float px = src.x[si], py = src.y[si], pz = src.z[si];
      if (isfinite(px) && isfinite(py) && isfinite(pz)) {
        qx = __fadd_rn(dot3_rn(R[0], px, R[1], py, R[2], pz), t[0]);
        qy = __fadd_rn(dot3_rn(R[3], px, R[4], py, R[5], pz), t[1]);
        qz = __fadd_rn(dot3_rn(R[6], px, R[7], py, R[8], pz), t[2]);
      } else {
        qx = px;
        qy = py;
        qz = pz;
      }
    } else {
      const float Z = src.z[si];
      // the source point: NaN depth keeps x / y of the 1 m ray (misc.cpp:525-529) -> the transformed z is NaN as well
      const float u = (float)(rx * cloud_step), v = (float)(ry * cloud_step);
      const float zs = isnan(Z) ? 1.0f : Z;
      const float px = __fmul_rn(__fmul_rn(__fsub_rn(u, src.cx), zs), sfxinv);
      const float py = __fmul_rn(__fmul_rn(__fsub_rn(v, src.cy), zs), sfyinv);
      const float pz = Z;
      qx = __fadd_rn(dot3_rn(R[0], px, R[1], py, R[2], pz), t[0]);  // pcl::transformPointCloud
      qy = __fadd_rn(dot3_rn(R[3], px, R[4], py, R[5], pz), t[1]);
      qz = __fadd_rn(dot3_rn(R[6], px, R[7], py, R[8], pz), t[2]);
    }
    if (qz != qz) continue;   // NaN
    if (qz < 0) continue;     // behind the camera
    const float xc = __fadd_rn(__fmul_rn(__fdiv_rn(qx, qz), fx), cx), yc = __fadd_rn(__fmul_rn(__fdiv_rn(qy, qz), fy), cy);
    const int ocx = kCloud ? round_x86(xc) : round_like_ref(xc);
    const int ocy = kCloud ? round_x86(yc) : round_like_ref(yc);
    if (ocx >= dst.cw || ocx < 0 || ocy >= dst.ch || ocy < 0) continue;
    const int nbhd = 2;
    bool good_point = false, occluded_point = false, bad_point = false;
    const int startx = max(0, ocx - nbhd), starty = max(0, ocy - nbhd);
    const int endx = min(dst.cw, ocx + nbhd + 1), endy = min(dst.ch, ocy + nbhd + 1);
    for (int oy = starty; oy < endy; oy += 2)
      for (int ox = startx; ox < endx; ox += 2) {
        const float oz = dst.z[(size_t)oy * dst.cw + ox];
        if (oz != oz) continue;
        const double sd_old = sigma_depth * (double)oz * (double)oz, sd_new = sigma_depth * (double)qz * (double)qz;
        const double old_sigma = __dmul_rn((double)cloud_step, cov_z_const >= 0.0 ? cov_z_const : sd_old * sd_old);
        const double new_sigma = __dmul_rn((double)cloud_step, cov_z_const >= 0.0 ? cov_z_const : sd_new * sd_new);
        const double joint_sigma = __dadd_rn(old_sigma, new_sigma);
        // cdf(old_p.z, p.z, sqrt(joint_sigma)) with the reference's truncated SQRT_2 (misc.cpp:801, 809-812)
        const double p_new_in_front = 0.5 * (1 + erf(((double)oz - (double)qz) / (sqrt(joint_sigma) * 1.41421)));
        if (p_new_in_front < 0.001) occluded_point = true;
        else if (p_new_in_front < 0.999) good_point = true;
        else bad_point = true;
      }
    if (good_point) good++;
    else if (occluded_point) occl++;
    else if (bad_point) bad++;
  }
}

__device__ __forceinline__ unsigned block_sum(unsigned v, unsigned* scratch) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  __syncthreads();
  if ((threadIdx.x & 31) == 0) scratch[threadIdx.x >> 5] = v;
  __syncthreads();
  unsigned s = 0;
  for (int w = 0; w < (int)(blockDim.x >> 5); w++) s += scratch[w];
  return s;
}

struct EmmArgs {
  int cloud_step, skip_step;
  double cov_z_const, sigma_depth, observability_threshold;
};

// counts[4] = inlier, outlier, occluded, all points (MatchingResult, matching_result.h:40-42)
template <EmmPoints P>
__device__ void emm_pair(const EmmView& newer, const EmmView& older, const float* T16 /* column-major, newer -> older */,
                         const EmmArgs& a, unsigned counts[4], unsigned* scratch) {
  float R[9], t[3], Ri[9], ti[3];
#pragma unroll
  for (int r = 0; r < 3; r++) {
#pragma unroll
    for (int c = 0; c < 3; c++) R[3 * r + c] = T16[4 * c + r];
    t[r] = T16[12 + r];
  }
  // mr.final_trafo.inverse(): cofactor inverse of the affine matrix in float, uncontracted like the reference
  const float c00 = __fsub_rn(__fmul_rn(R[4], R[8]), __fmul_rn(R[5], R[7]));
  const float c01 = __fsub_rn(__fmul_rn(R[5], R[6]), __fmul_rn(R[3], R[8]));
  const float c02 = __fsub_rn(__fmul_rn(R[3], R[7]), __fmul_rn(R[4], R[6]));
  const float det = dot3_rn(R[0], c00, R[1], c01, R[2], c02);
  const float id = __fdiv_rn(1.0f, det);
  Ri[0] = __fmul_rn(c00, id);
  Ri[1] = __fmul_rn(__fsub_rn(__fmul_rn(R[2], R[7]), __fmul_rn(R[1], R[8])), id);
  Ri[2] = __fmul_rn(__fsub_rn(__fmul_rn(R[1], R[5]), __fmul_rn(R[2], R[4])), id);
  Ri[3] = __fmul_rn(c01, id);
  Ri[4] = __fmul_rn(__fsub_rn(__fmul_rn(R[0], R[8]), __fmul_rn(R[2], R[6])), id);
  Ri[5] = __fmul_rn(__fsub_rn(__fmul_rn(R[2], R[3]), __fmul_rn(R[0], R[5])), id);
  Ri[6] = __fmul_rn(c02, id);
  Ri[7] = __fmul_rn(__fsub_rn(__fmul_rn(R[1], R[6]), __fmul_rn(R[0], R[7])), id);
  Ri[8] = __fmul_rn(__fsub_rn(__fmul_rn(R[0], R[4]), __fmul_rn(R[1], R[3])), id);
#pragma unroll
  for (int r = 0; r < 3; r++) ti[r] = -dot3_rn(Ri[3 * r], t[0], Ri[3 * r + 1], t[1], Ri[3 * r + 2], t[2]);
  unsigned g = 0, b = 0, o = 0, al = 0;
  emm_direction<P>(newer, older, R, t, a.cloud_step, a.skip_step, a.cov_z_const, a.sigma_depth, g, b, o, al);   // node.cpp:1527-1535
  emm_direction<P>(older, newer, Ri, ti, a.cloud_step, a.skip_step, a.cov_z_const, a.sigma_depth, g, b, o, al);  // :1538-1548
  counts[0] = block_sum(g, scratch);
  counts[1] = block_sum(b, scratch);
  counts[2] = block_sum(o, scratch);
  counts[3] = block_sum(al, scratch);
}

// One CTA per pair; a pair whose nodes are of the other kind is left to the other instantiation.
template <EmmPoints P>
__global__ void __launch_bounds__(256) k_emm_pairs(const PairDesc* __restrict__ pairs, EmmArgs a,
                                                   rgbdslam_b200_pair_result* __restrict__ results) {
  __shared__ unsigned scratch[8];
  const int p = blockIdx.x;
  rgbdslam_b200_pair_result res = results[p];
  if (res.id1 < 0) return;  // the model only judges transformations RANSAC accepted (node.cpp:1336-1345)
  const PairDesc pd = pairs[p];
  if ((pd.emm_cloud != 0) != (P == EmmPoints::kCloud)) return;
  EmmView nv{pd.q_cloud, pd.q_cloud_x, pd.q_cloud_y, pd.q_cw, pd.q_ch, pd.q_K[0], pd.q_K[1], pd.q_K[2], pd.q_K[3]};
  EmmView ov{pd.t_cloud, pd.t_cloud_x, pd.t_cloud_y, pd.t_cw, pd.t_ch, pd.t_K[0], pd.t_K[1], pd.t_K[2], pd.t_K[3]};
  unsigned counts[4];
  emm_pair<P>(nv, ov, res.ransac_trafo, a, counts, scratch);
  if (threadIdx.x == 0) {
    res.inlier_points = counts[0];
    res.outlier_points = counts[1];
    res.occluded_points = counts[2];
    res.all_points = counts[3];
    // observation_criterion_met(inliers, outliers, occluded + inliers + outliers, quality) (misc.cpp:1136-1148)
    const double quality = counts[0] / (double)(counts[0] + counts[1]);
    const double certainty = counts[0] / (double)(counts[2] + counts[0] + counts[1]);
    if (!(quality > a.observability_threshold && certainty > 0.25)) res.id1 = res.id2 = -1;  // node.cpp:1420
    results[p] = res;
  }
}

cudaError_t launch_emm_pairs(const PairDesc* pairs, int npairs, bool depth_pairs, bool cloud_pairs, int cloud_step, int skip_step,
                             double cov_z_const, double sigma_depth, double observability_threshold,
                             rgbdslam_b200_pair_result* results, cudaStream_t stream, int* n_launches) {
  if (npairs <= 0) return cudaSuccess;
  EmmArgs a{cloud_step, skip_step, cov_z_const, sigma_depth, observability_threshold};
  if (depth_pairs) {
    k_emm_pairs<EmmPoints::kDepth><<<npairs, 256, 0, stream>>>(pairs, a, results);
    ++*n_launches;
  }
  if (cloud_pairs) {
    k_emm_pairs<EmmPoints::kCloud><<<npairs, 256, 0, stream>>>(pairs, a, results);
    ++*n_launches;
  }
  return cudaGetLastError();
}

// rgbdslam_b200_observation_likelihood: one pair, explicit transformation, counts only
template <EmmPoints P>
__global__ void __launch_bounds__(256) k_emm_single(EmmView newer, EmmView older, const float* __restrict__ T16, EmmArgs a,
                                                    unsigned* __restrict__ counts_out) {
  __shared__ unsigned scratch[8];
  __shared__ float sT[16];
  if (threadIdx.x < 16) sT[threadIdx.x] = T16[threadIdx.x];
  __syncthreads();
  unsigned counts[4];
  emm_pair<P>(newer, older, sT, a, counts, scratch);
  if (threadIdx.x == 0)
    for (int k = 0; k < 4; k++) counts_out[k] = counts[k];
}

cudaError_t launch_emm_single(const EmmNode& q, const EmmNode& t, bool cloud, const float* d_T16, int cloud_step, int skip_step,
                              double cov_z_const, double sigma_depth, unsigned* d_counts, cudaStream_t stream) {
  EmmArgs a{cloud_step, skip_step, cov_z_const, sigma_depth, 0.0};
  EmmView nv{q.z, q.x, q.y, q.cw, q.ch, q.K[0], q.K[1], q.K[2], q.K[3]};
  EmmView ov{t.z, t.x, t.y, t.cw, t.ch, t.K[0], t.K[1], t.K[2], t.K[3]};
  if (cloud) k_emm_single<EmmPoints::kCloud><<<1, 256, 0, stream>>>(nv, ov, d_T16, a, d_counts);
  else k_emm_single<EmmPoints::kDepth><<<1, 256, 0, stream>>>(nv, ov, d_T16, a, d_counts);
  return cudaGetLastError();
}

}  // namespace rb200
