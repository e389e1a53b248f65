// common.cuh -- shared device/host definitions for the sm_90a front-end kernels.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "../../include/rgbdslam_b200.h"

namespace rb200 {

constexpr int kMaxMatchesCap = RGBDSLAM_B200_MAX_MATCHES_CAP;  // 512
constexpr int kMaxMaskWords = kMaxMatchesCap / 32;             // 16
constexpr int kMaxFeatures = 4096;                             // per node (SiftGPU limit too: sift_gpu_wrapper.cpp:231)

// One frame pair as the kernels see it (device pointers).
struct PairDesc {
  const uint32_t* q_desc;  // newer node descriptors, nq x 8 u32 (16 B aligned)
  const uint32_t* t_desc;  // older node descriptors, nt x 8 u32
  const float4* q_xyz;     // newer node points (x,y,z,1)
  const float4* t_xyz;     // older node points
  int32_t nq, nt;
  int32_t id_q, id_t;  // node ids (newer, older)
  const int8_t* q_i8;  // float-descriptor nodes: operand tiles (bf16 RootSIFT rows / u8 SiftGPU rows), else nullptr
  const int8_t* t_i8;
  const float* q_f32;  // SIFT nodes only: fp32 (Root)SIFT rows and train-row norms
  const float* t_f32;
  const float* t_norm;
  const rgbdslam_b200_keypoint* q_kp;  // 2-D keypoints (nullptr unless the node has them): pairwise g2o refinement only
  const rgbdslam_b200_keypoint* t_kp;
  const float* q_cloud;  // depth-cloud z-planes (environment measurement model), nullptr if the node has none
  const float* t_cloud;
  const float* q_cloud_x;  // kept organised clouds (RGBDSLAM_B200_KEEP_CLOUD): x / y planes, nullptr for depth-image nodes
  const float* q_cloud_y;
  const float* t_cloud_x;
  const float* t_cloud_y;
  int32_t q_cw, q_ch, t_cw, t_ch;
  float q_K[4], t_K[4];  // fx, fy, cx, cy of the full-resolution cameras (kept clouds: the camera the model projects into)
  int32_t sift_kind;   // float-descriptor nodes: 0 = RootSIFT / exact 2-NN ratio matcher, 1 = SiftGPU matcher (u8 tiles, raw rows)
  int32_t emm_cloud;   // 1: the newer node keeps its organised cloud (match_pairs* only runs the model on pairs of one kind)
};

// One work item of the tensor-core match kernels = 256 queries of one pair against all train rows.
struct HamItem {
  const int8_t* a;     // query block: ORB -- 32-byte descriptor rows; float descriptors -- operand tiles (2 x 32 KiB)
  const int8_t* b;     // train rows of the older node: ORB -- descriptor rows; float descriptors -- n_btiles x 32 KiB tiles
  int2* out;           // best[] slot of the block's first query row
  int32_t nq_valid;    // valid rows in this block (1..256)
  int32_t nsearch;     // ORB: nt - 1, only train rows [0, nt-2] are examined (features.cpp:174); float descriptors: nt
  int32_t n_btiles;    // ceil(nsearch / 128)
  int32_t pad_;        // SiftGPU pass: tie rule of the arg-max (0 = RowMatch_Kernel's thread-major order, 1 = lowest index)
  const float* bnorm;  // SIFT L2 only: |b|^2 of the train rows (bf16-rounded values); out then points to int4 records
};

// One node of the SIFT preparation kernel (RootSIFT + bf16 tiles + norms).
struct SiftJob {
  const float* in;     // n x 128 raw descriptors
  float* root;         // n x 128 RootSIFT (or copy) fp32, used for the exact re-ranking
  uint16_t* tiles;     // n_pad x 128 bf16, tiled like the int8 Hamming operands (256 B per row)
  float* norms;        // n_pad
  int32_t n, n_pad;
};

// Constant-memory copy of the parameters the kernels read.
struct DevParams {
  int32_t min_matches;
  int32_t max_matches;
  int32_t ransac_iterations;
  int32_t pad_;
  float max_dist_m;      // (float) max_dist_for_inliers        node.cpp:1105
  double sq_max_dist;    // (double)(max_dist_m*max_dist_m)     node.cpp:1152
  double sigma_depth;    // misc2.h:23
  double cov_z_const;    // (sigma*z0^2)^2 if the static-cache quirk is emulated, else <0
  double raster_cov_x;   // misc.cpp:702-709
  double raster_cov_y;
};

// Per-hypothesis record written by the RANSAC kernel and replayed by the selection kernel.
struct HypResult {
  double err;     // refined_error (1e6 if the hypothesis never produced a model)
  int32_t count;  // refined_matches.size()
  int32_t pad_;
  float T[12];  // R row-major (9) + t (3)
};

// ---- counter-based RNG (DESIGN.md "Random numbers"; same stream as oracle_rand31) -------------
__host__ __device__ __forceinline__ uint64_t mix64(uint64_t z) {
  z += 0x9E3779B97F4A7C15ULL;
  z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ULL;
  z = (z ^ (z >> 27)) * 0x94D049BB133111EBULL;
  return z ^ (z >> 31);
}
__host__ __device__ __forceinline__ uint64_t pair_key(uint64_t seed, uint64_t pair) { return mix64(seed ^ mix64(pair)); }
__host__ __device__ __forceinline__ uint32_t rand31(uint64_t key, uint32_t stream, uint32_t ctr) {
  return (uint32_t)(mix64(key ^ (((uint64_t)stream << 32) | ctr)) >> 33);
}

}  // namespace rb200
