// kernels.h -- host-side launchers of the sm_90a kernels (implemented in *.cu).
#pragma once
#include "common.cuh"

namespace rb200 {

// Upload the constant-memory parameter block (synchronous w.r.t. `stream`).
cudaError_t set_dev_params(const DevParams& p, cudaStream_t stream);

// Hamming N x M brute force (features.cpp:168-182 batched): best[p*stride + i] = {hd, idx}.
cudaError_t launch_hamming_simt(const PairDesc* pairs, int npairs, int max_nq, int2* best, int stride,
                                cudaStream_t stream);

// Work-item counter of a persistent kernel whose CTAs claim items dynamically: `ticket` (device) only grows, `base` is its
// value when the next launch on the owner's stream starts.  One per slot, since slots run concurrently on their own streams.
struct ClaimCounter {
  unsigned long long* ticket = nullptr;
  unsigned long long base = 0;
};

// Hamming brute force on the tensor cores, 32-byte descriptors expanded to int8 operands inside the kernel (HamItem::a / b =
// descriptor rows); same output as launch_hamming_simt.  Advances claim.base past the tickets the launch takes.
cudaError_t launch_hamming_tc_expand(const HamItem* d_items, int n_items, int sm_count, ClaimCounter& claim,
                                     cudaStream_t stream);
cudaError_t launch_l2_tc256(const HamItem* d_items, int n_items, int sm_count, cudaStream_t stream);

// SIFT-128 path (sift_l2.cu / hamming_tc.cu MODE 1)
cudaError_t launch_sift_prepare(const SiftJob* d_jobs, int njobs, int max_n_pad, int root_sift, int siftgpu, cudaStream_t stream);
// Environment measurement model.  launch_emm_pairs launches the depth-node instantiation when depth_pairs, the kept-cloud one
// when cloud_pairs (each skips the other kind's pairs) and adds the launches to *n_launches.
cudaError_t launch_emm_pairs(const PairDesc* pairs, int npairs, bool depth_pairs, bool cloud_pairs, int cloud_step, int skip_step,
                             double cov_z_const, double sigma_depth, double observability_threshold,
                             rgbdslam_b200_pair_result* results, cudaStream_t stream, int* n_launches);
// One pair, explicit transformation; the kind of q (q.x != nullptr: organised clouds) selects the instantiation.
cudaError_t launch_emm_single(const CloudView& q, const CloudView& t, const float* d_T16, int cloud_step, int skip_step,
                              double cov_z_const, double sigma_depth, unsigned* d_counts, cudaStream_t stream);
// The nodes' clouds, Node::pc_col (map.cu).  Per node `node_words` 4-byte words: depth-image frames a z-plane at the skip-step
// raster (ceil(w / step) x ceil(h / step)), clouds [x | y | z] planes of n points; each followed by a colour plane when
// d_visual / rgb is given.  vis_kind: 0 grey, 1 three-channel, 2 Bayer GRBG.
cudaError_t launch_store_depth_cloud(int nframes, const float* d_depth, const uint8_t* d_visual, int vis_kind, bool bgr, int w, int h,
                                     int step, double scaling, float min_depth, float* out, size_t node_words, cudaStream_t st);
cudaError_t launch_store_cloud_points(int nframes, const float* d_cloud, int stride, int n, bool rgb, float* out, size_t node_words,
                                      cudaStream_t st);
// One node of a rgbdslam_b200_render_cloud / node_download_cloud call.
struct MapNode {
  const float *x, *y, *z;  // depth-image nodes: z only
  const uint32_t* rgb;     // colour words
  int cw, ch;
  int step;                // > 0: depth-image node (x / y from pixel (rx * step, ry * step)); 0: x / y planes stored
  float fxinv, fyinv, cx, cy;
  float m[12];             // row-major 3 x 4 float transform
};
struct MapArgs {
  float maxd2;     // maximum_depth^2 in float
  int filter;      // maximum_depth >= 0
  int preserve;    // preserve_raster_on_save
  int transform;   // 0: the points as stored (node_download_cloud)
  int point_bytes; // 16 or 32
};
constexpr int kMapBlockPoints = 1024;  // points per block of the count / scatter kernels
cudaError_t launch_map_count(const MapNode* d_nodes, const int2* d_blocks, int nblocks, const MapArgs& a, int* d_counts,
                             cudaStream_t st);
cudaError_t launch_map_scan(const int* d_counts, int nblocks, long long* d_offs, cudaStream_t st);
cudaError_t launch_map_scatter(const MapNode* d_nodes, const int2* d_blocks, const long long* d_offs, int b0, int b1, long long lo,
                               long long hi, const MapArgs& a, void* d_out, cudaStream_t st);
cudaError_t launch_refine_g2o(const PairDesc* pairs, int npairs, int max_matches, int iterations, const float4* mfrom,
                              const float4* mto, const int32_t* n_all, const rgbdslam_b200_dmatch* matches,
                              rgbdslam_b200_pair_result* results, rgbdslam_b200_dmatch* inlier_matches, cudaStream_t stream);
cudaError_t launch_siftgpu_tc256(const HamItem* d_items, int n_items, int sm_count, cudaStream_t stream);
cudaError_t launch_select_siftgpu(const PairDesc* pairs, int npairs, const int4* rowres, const int4* colres, int stride, int maxM,
                                  rgbdslam_b200_dmatch* matches, float4* mfrom, float4* mto, int32_t* n_all, cudaStream_t stream);
cudaError_t launch_l2_refine(const PairDesc* pairs, int npairs, int max_nq, const int4* top4, int stride, float4* knn,
                             cudaStream_t stream);
cudaError_t launch_select_sift(const PairDesc* pairs, int npairs, const float4* knn, int stride, double nn_ratio, int maxM,
                               rgbdslam_b200_dmatch* matches, float4* mfrom, float4* mto, int32_t* n_all, cudaStream_t stream);

// hd<128 filter + jitter distance + sort + keep max_matches (node.cpp:572-573,674,1127).
cudaError_t launch_select_matches(const PairDesc* pairs, int npairs, const int2* best, int stride, uint64_t seed,
                                  int64_t first_pair, rgbdslam_b200_dmatch* matches, float4* mfrom, float4* mto,
                                  int32_t* n_all, cudaStream_t stream);

// RANSAC hypotheses (node.cpp:1130-1169) -- one warp per hypothesis, launched in two phases [0,4) [4,H).
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
