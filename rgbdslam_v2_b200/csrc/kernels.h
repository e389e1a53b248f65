// kernels.h -- host-side launchers of the sm_90a kernels (implemented in *.cu).
#pragma once
#include "../../include/rgbdslam_b200/icp.h"
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

// Hamming brute force on the tensor cores as a binary GEMM (popcount(a & b) of the raw 32-byte descriptor rows, HamItem::a /
// b = descriptor rows); same output as launch_hamming_simt.  Advances claim.base past the tickets the launch takes.
cudaError_t launch_hamming_tc_b1(const HamItem* d_items, int n_items, int sm_count, ClaimCounter& claim, cudaStream_t stream);
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
  int point0_one;          // x / y planes: point 0 came from a depth image, its data[3] is 1.0f
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
// pcl::transformPointCloud of the stored clouds of a chunk of nodes (rgbdslam_b200_transform_clouds), each by its MapNode::m:
// node k's new planes [x | y | z | colour] of P_k points each start at word 4 * d_first[k] of slab
cudaError_t launch_transform_clouds(const MapNode* d_nodes, const int2* d_blocks, int nblocks, const long long* d_first, float* slab,
                                    cudaStream_t st);
// The voxel filter of the stored clouds, Node::reducePointCloud (voxel.cu).  A call works on a chunk of whole nodes whose
// points lie back to back in the work buffers; the (node, first point) block table is the map's.
struct VoxSeg {        // one node of the chunk
  int pt0, npts;       // its points are [pt0, pt0 + npts) of the chunk
  int blk0, nblk;      // its blocks of the block table
};
struct VoxGrid {       // written by k_vox_grid
  int min_b[3];        // floor(min_p * inv) per axis
  int mul[3];          // 1, div_b.x, div_b.x * div_b.y
  int cells;           // div_b.x * div_b.y * div_b.z; 0: no voxel (no finite point, or too many cells)
  int too_small;       // 1: the leaf size is too small for this cloud (more than INT32_MAX cells): the cloud stays as it is
};
struct VoxBufs {
  const MapNode* nodes;
  const int2* blocks;
  const VoxSeg* segs;
  uint32_t *bmin, *bmax;  // nnodes x 3 ordered-integer images of the float bounds
  VoxGrid* grid;
  uint32_t* key[2];       // ping-pong: voxel index, 0xffffffff for a point that takes no part
  uint32_t* idx[2];       //            raster index inside the node
  int* hist;              // nblocks x 256 digit counts, then output positions
  int* counts;            // run heads per block
  long long* offs;        // their exclusive scan (nblocks + 1)
  int2* heads;            // per voxel of the chunk: (position of its first point in the sorted chunk, node)
};
// bounds -> grid -> keys into key[0] / idx[0]
cudaError_t launch_vox_keys(const VoxBufs& b, int nnodes, int nblocks, float inv_leaf, cudaStream_t st, int* n_launches);
// `passes` stable 8-bit radix passes inside every node's segment, then the run heads and their scan; the sorted arrays are
// key[passes & 1] / idx[passes & 1]
cudaError_t launch_vox_sort(const VoxBufs& b, int nnodes, int nblocks, int passes, cudaStream_t st, int* n_launches);
// One point per voxel into the chunk's slab: node k's planes [x | y | z | colour] of its n_k voxels start at word
// 4 * offs[blk0_k]
cudaError_t launch_vox_centroids(const VoxBufs& b, int passes, long long nvoxels, float* slab, cudaStream_t st);
// The ICP fallback of matchNodePair (icp.cu).  The kept points of every distinct node of a call lie in three planes of `plane`
// floats each (x | y | z), node u's at [f0, f0 + cap).
struct IcpNode {
  MapNode src;          // its stored cloud, as stored
  int P;                // src.cw * src.ch
  int cap;              // room for its kept points
  long long f0;         // their first slot in the point planes (and in the cell arrays)
  long long scratch0;   // its non-NaN index list in the scratch of the filter launch that treats it
};
struct IcpPair {
  int s, t;             // source and target node
  long long w0;         // the pair's working source, correspondences and distances: [w0, w0 + cap of s)
};
// filterCloud of nnodes nodes: kept points into pts, their counts into nf (one CTA per node)
cudaError_t launch_icp_filter(const IcpNode* d_nodes, int nnodes, int desired, int* scratch, float* pts, long long plane, int* nf,
                              cudaStream_t st);
// the cell keys of the finite kept points of the listed nodes, sorted, into key[0] / idx[0] at f0; counts into nfin
cudaError_t launch_icp_cells(const IcpNode* d_nodes, const int* targets, int ntargets, const float* pts, long long plane, const int* nf,
                             unsigned long long* key[2], int* idx[2], int* nfin, cudaStream_t st);
// the alignment of every pair by icp_method `method` (RGBDSLAM_B200_ICP_METHOD_*, one CTA per pair); work holds
// icp_work_planes(method) planes of wplane floats
int icp_work_planes(int method);
cudaError_t launch_icp_align(int method, const IcpPair* pairs, int npairs, const IcpNode* d_nodes, const float* pts, long long plane,
                             const int* nf, const unsigned long long* key, const int* idx, const int* nfin, float* work,
                             long long wplane, int* corr, float* dist, rgbdslam_b200_icp_result* results, cudaStream_t st);
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
