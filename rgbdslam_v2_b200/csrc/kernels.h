// kernels.h -- host-side launchers of the sm_90a kernels (implemented in *.cu).
#pragma once
#include "common.cuh"

namespace rb200 {

// Upload the constant-memory parameter block (synchronous w.r.t. `stream`).
cudaError_t set_dev_params(const DevParams& p, cudaStream_t stream);

// Hamming N x M brute force (features.cpp:168-182 batched): best[p*stride + i] = {hd, idx}.
cudaError_t launch_hamming_simt(const PairDesc* pairs, int npairs, int max_nq, int2* best, int stride,
                                cudaStream_t stream);

// Hamming brute force on the tensor cores, 32-byte descriptors expanded to int8 operands inside the kernel (HamItem::a / b =
// descriptor rows); same output as launch_hamming_simt.
cudaError_t launch_hamming_tc_expand(const HamItem* d_items, int n_items, int sm_count, cudaStream_t stream);
cudaError_t launch_l2_tc256(const HamItem* d_items, int n_items, int sm_count, cudaStream_t stream);

// SIFT-128 path (sift_l2.cu / hamming_tc.cu MODE 1)
cudaError_t launch_sift_prepare(const SiftJob* d_jobs, int njobs, int max_n_pad, int root_sift, int siftgpu, cudaStream_t stream);
cudaError_t launch_build_cloud(const float* d_depth, int w, int h, int step, float scaling, float min_depth, float* cloud_z, int cw,
                               int ch, cudaStream_t stream);
cudaError_t launch_emm_pairs(const PairDesc* pairs, int npairs, int cloud_step, int skip_step, double cov_z_const,
                             double sigma_depth, double observability_threshold, rgbdslam_b200_pair_result* results,
                             cudaStream_t stream);
cudaError_t launch_emm_single(const float* q_cloud, int q_cw, int q_ch, const float* qK, const float* t_cloud, int t_cw, int t_ch,
                              const float* tK, const float* d_T16, int cloud_step, int skip_step, double cov_z_const,
                              double sigma_depth, unsigned* d_counts, cudaStream_t stream);
cudaError_t launch_refine_g2o(const PairDesc* pairs, int npairs, int max_matches, int iterations, const float4* mfrom,
                              const float4* mto, const int32_t* n_all, const rgbdslam_b200_dmatch* matches,
                              rgbdslam_b200_pair_result* results, rgbdslam_b200_dmatch* inlier_matches, cudaStream_t stream);
cudaError_t launch_siftgpu_tc256(const HamItem* d_items, int n_items, int sm_count, cudaStream_t stream);
cudaError_t launch_select_siftgpu(const PairDesc* pairs, int npairs, const int4* rowres, const int4* colres, int stride, int maxM,
                                  rgbdslam_b200_dmatch* matches, float4* mfrom, float4* mto, int32_t* n_all, cudaStream_t stream);
cudaError_t launch_l2_refine(const PairDesc* pairs, int npairs, int max_nq, const int4* top4, int stride, float4* knn,
                             cudaStream_t stream);
cudaError_t launch_select_sift(const PairDesc* pairs, int npairs, const float4* knn, int stride, float nn_ratio, int maxM,
                               rgbdslam_b200_dmatch* matches, float4* mfrom, float4* mto, int32_t* n_all, cudaStream_t stream);

// hd<128 filter + jitter distance + sort + keep max_matches (node.cpp:572-573,674,1127).
cudaError_t launch_select_matches(const PairDesc* pairs, int npairs, const int2* best, int stride, uint64_t seed,
                                  int64_t first_pair, rgbdslam_b200_dmatch* matches, float4* mfrom, float4* mto,
                                  int32_t* n_all, int max_nq, cudaStream_t stream);

// RANSAC hypotheses (node.cpp:1130-1169) -- one warp per hypothesis, launched in phases [0,8) [8,40) [40,H).
cudaError_t launch_ransac_hypotheses(int npairs, int ransac_iterations, int max_matches, uint64_t seed, int64_t first_pair,
                                     const float4* mfrom, const float4* mto, const int32_t* n_all, HypResult* hyp, float* cen,
                                     int32_t* next_n, cudaStream_t stream, int* n_launches);

// Sequential replay of the hypothesis bookkeeping (node.cpp:1170-1216,1275) + edge (node.cpp:1335-1339).
cudaError_t launch_ransac_select(const PairDesc* pairs, int npairs, int ransac_iterations, int max_matches,
                                 const float4* mfrom, const float4* mto, const int32_t* n_all,
                                 const rgbdslam_b200_dmatch* matches, const HypResult* hyp,
                                 rgbdslam_b200_pair_result* results, rgbdslam_b200_dmatch* inlier_matches,
                                 cudaStream_t stream);

}  // namespace rb200
