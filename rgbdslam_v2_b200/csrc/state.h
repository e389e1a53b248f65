// state.h -- host-side library state shared by the api_*.cu translation units.
#pragma once
#include <cuda_runtime.h>

#include <mutex>
#include <string>
#include <vector>

#include "common.cuh"

namespace rb200 {

struct DevBuf {  // grow-only device buffer
  void* ptr = nullptr;
  size_t cap = 0;
  int ensure(size_t bytes);
  void release();
};
struct PinBuf {  // grow-only pinned host buffer
  void* ptr = nullptr;
  size_t cap = 0;
  int ensure(size_t bytes);
  void release();
};

// One device allocation shared by all nodes of a rgbdslam_b200_nodes_create call (no per-node cudaMalloc); freed when
// its last node is destroyed.
struct NodeSlab {
  void* base = nullptr;
  int refs = 0;
};

// Device copy of what the reference's Node keeps per frame (node.h:167-174).
struct NodeDev {
  static constexpr uint32_t kMagic = 0x4e4f4445u;  // 'NODE'
  uint32_t magic = 0;
  int32_t id = -1;
  int32_t n = 0;
  uint8_t* desc = nullptr;    // n x 32 B ORB descriptors
  float4* xyz = nullptr;      // n x (x,y,z,1)
  rgbdslam_b200_keypoint* kp = nullptr;  // n x cv::KeyPoint (only for nodes built from images)
  float* desc_f32 = nullptr;  // SIFT nodes: n x 128 fp32 (Root)SIFT rows (desc == nullptr then)
  float* norms = nullptr;     // SIFT nodes: n_pad |b|^2 of the bf16-rounded rows
  int8_t* desc_i8 = nullptr;  // float-descriptor nodes only: n_pad x 256 B operand tiles (bf16 RootSIFT rows / u8 SiftGPU rows)
  int32_t n_pad = 0;
  float* cloud_z = nullptr;   // depth cloud z-plane (cw x ch) for the environment measurement model
  int32_t cw = 0, ch = 0;
  float K[4] = {0, 0, 0, 0};  // fx, fy, cx, cy of the full-resolution camera
  int32_t sift_kind = 0;      // SIFT nodes: 0 = RootSIFT rows + bf16 tiles, 1 = raw rows + u8 tiles (SiftGPU matcher)
  NodeSlab* slab = nullptr;   // desc / xyz / kp live inside this shared allocation (cloud_z is always separate)
};

constexpr int kSlots = 8;  // independent in-flight match_pairs pipelines (stream + workspace each)

struct Workspace {
  cudaStream_t stream = nullptr;  // slot 0: the library / user stream; slots 1..: own non-blocking streams
  cudaEvent_t ev[8] = {nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr};
  bool timing_valid = false;
  bool host_path = false;  // last call uploaded host features (ev[4], ev[5] valid)
  bool pending = false;
  cudaEvent_t ev_gather = nullptr;  // rgbdslam_b200_allgather_slot_edges: the slot's collective + download have finished
  bool gather_pending = false;
  DevBuf d_pairs, d_best, d_matches, d_inliers, d_mfrom, d_mto, d_nall, d_hyp, d_results;
  DevBuf d_feat_a, d_feat_b, d_xyz_a, d_xyz_b;
  DevBuf d_i8_a, d_i8_b, d_jobs, d_items, d_top4, d_knn, d_cen, d_nextn;
  PinBuf h_pairs, h_jobs, h_items;
  void release() {
    DevBuf* all[] = {&d_pairs, &d_best, &d_matches, &d_inliers, &d_mfrom, &d_mto, &d_nall, &d_hyp, &d_results, &d_feat_a,
                     &d_feat_b, &d_xyz_a, &d_xyz_b, &d_i8_a, &d_i8_b, &d_jobs, &d_items, &d_top4, &d_knn, &d_cen, &d_nextn};
    for (DevBuf* b : all) b->release();
    h_pairs.release();
    h_jobs.release();
    h_items.release();
  }
};

struct State {
  std::mutex mu;
  bool inited = false;
  int device = 0;
  int sm_count = 0;
  rgbdslam_b200_params params;
  DevParams dp;
  cudaEvent_t epoch = nullptr;  // reference point of rgbdslam_b200_slot_timeline
  double z0 = 0.0;  // latched first depth for depth_covariance (misc2.h:30-35)
  cudaStream_t own_stream = nullptr, stream = nullptr;  // stream of the synchronous entry points (= slot 0)
  int64_t launches = 0;
  int comm_count = 0;  // live NCCL communicators (rgbdslam_b200_comm_init)
  Workspace ws[kSlots];
  Workspace* cur = &ws[0];
  Workspace& W() { return *cur; }
  DevBuf d_f32_a, d_f32_b, d_root_a, d_root_b, d_norm_a, d_norm_b;  // SIFT staging of the synchronous calls
  int sift_matcher = 0;  // float-descriptor nodes created from now on: 0 = exact 2-NN ratio matcher (FLANN branch), 1 = SiftGPU matcher
  int hamming_path = 1;  // 1 = wgmma int8 GEMM, operands expanded inside the kernel (default); 0 = SIMT popcount (cross-check)
  void release_workspaces() {
    for (Workspace& w : ws) w.release();
    DevBuf* all[] = {&d_f32_a, &d_f32_b, &d_root_a, &d_root_b, &d_norm_a, &d_norm_b};
    for (DevBuf* b : all) b->release();
  }
};

extern State g_state;
void set_error(const std::string& s);
int cuda_fail(cudaError_t e, const char* what);
int check_inited();
int node_build_cloud(NodeDev* nd, const float* d_depth, int w, int h, const float K4[4], cudaStream_t st);
void free_node(NodeDev* nd);  // frees everything a (possibly half-built) node owns (api.cu)

}  // namespace rb200
