// state.h -- host-side library state shared by the api_*.cu translation units.
#pragma once
#include <cuda_runtime.h>

#include <mutex>
#include <string>
#include <vector>

#include "common.cuh"
#include "kernels.h"

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

// A node's point cloud, the reference's Node::pc_col (node.cpp:126-131, 261), read by the environment measurement model and
// the map.  Depth-image nodes keep the z-plane of createXYZRGBPointCloud at every step-th pixel (x / y follow from the pixel
// and K); point-cloud nodes keep the x / y / z planes of the organised cloud.
struct NodeCloud {
  float *x = nullptr, *y = nullptr, *z = nullptr;  // x / y only for organised (point-cloud) nodes; z == nullptr: no cloud
  uint32_t* rgb = nullptr;      // colour words (b, g, r, a bytes): RGBDSLAM_B200_STORE_CLOUD only
  int32_t w = 0, h = 0, step = 0;  // step > 0: depth-image raster, point (rx, ry) is pixel (rx * step, ry * step)
  float K[4] = {0, 0, 0, 0};    // fx, fy, cx, cy of the call that built it (0 when it passed none)
  NodeSlab* slab = nullptr;     // the allocation the planes live in
  CloudView view() const { return CloudView{z, x, y, w, h, {K[0], K[1], K[2], K[3]}}; }
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
  int32_t sift_kind = 0;      // SIFT nodes: 0 = RootSIFT rows + bf16 tiles, 1 = raw rows + u8 tiles (SiftGPU matcher)
  NodeSlab* slab = nullptr;   // desc / xyz / kp live inside this shared allocation
  NodeCloud pc;
};

constexpr int kSlots = 8;  // independent in-flight match_pairs pipelines (stream + workspace each)

// The timing events of a slot, in the order a match_pairs* call records them on the slot's stream.
enum SlotEvent {
  kEvSubmit,       // host-feature calls: before the feature uploads
  kEvUploaded,     // host-feature calls: feature uploads queued
  kEvTables,       // pair table and work items uploaded: the device part of the call starts
  kEvMatchBegin,   // match kernel (Hamming / L2 / SiftGPU) start
  kEvMatchEnd,     // match kernel end
  kEvStagesEnd,    // match selection, RANSAC and the optional refinement / EMM done
  kEvDownloaded,   // result downloads done
  kEvGatherDep,    // rgbdslam_b200_allgather_slot_edges: everything the slot had queued
  kSlotEvents
};

struct Workspace {
  cudaStream_t stream = nullptr;  // slot 0: State::stream (set by init / set_stream); slots 1..: own non-blocking streams
  cudaEvent_t ev[kSlotEvents] = {};
  bool timing_valid = false;
  bool host_path = false;  // last call uploaded host features (kEvSubmit, kEvUploaded valid)
  bool pending = false;
  cudaEvent_t ev_gather = nullptr;  // rgbdslam_b200_allgather_slot_edges: the slot's collective + download have finished
  bool gather_pending = false;
  DevBuf d_pairs, d_best, d_matches, d_inliers, d_mfrom, d_mto, d_nall, d_hyp, d_results;
  DevBuf d_feat_a, d_feat_b, d_xyz_a, d_xyz_b;
  DevBuf d_jobs, d_items, d_top4, d_knn, d_cen, d_nextn;
  PinBuf h_pairs, h_jobs, h_items;
  DevBuf d_claim;      // ticket of claim (zeroed when allocated)
  ClaimCounter claim;  // work-item counter of the ORB match kernel
  void release() {
    DevBuf* all[] = {&d_pairs, &d_best, &d_matches, &d_inliers, &d_mfrom, &d_mto, &d_nall, &d_hyp, &d_results, &d_feat_a,
                     &d_feat_b, &d_xyz_a, &d_xyz_b, &d_jobs, &d_items, &d_top4, &d_knn, &d_cen, &d_nextn, &d_claim};
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
  DevBuf d_f32_a, d_f32_b, d_root_a, d_root_b, d_norm_a, d_norm_b, d_i8_a, d_i8_b;  // SIFT staging of the synchronous calls
  int sift_matcher = 0;  // float-descriptor nodes created from now on: 0 = exact 2-NN ratio matcher (FLANN branch), 1 = SiftGPU matcher
  int hamming_path = 1;  // 1 = wgmma int8 GEMM, operands expanded inside the kernel (default); 0 = SIMT popcount (cross-check)
  void release_workspaces() {
    for (Workspace& w : ws) w.release();
    DevBuf* all[] = {&d_f32_a, &d_f32_b, &d_root_a, &d_root_b, &d_norm_a, &d_norm_b, &d_i8_a, &d_i8_b};
    for (DevBuf* b : all) b->release();
  }
};

extern State g_state;
void set_error(const std::string& s);
int cuda_fail(cudaError_t e, const char* what);
int check_inited();
NodeDev* get_node(uint64_t h);  // nullptr (and last_error set) unless h is a live node handle
Workspace* get_slot(int slot);  // nullptr (and last_error set) unless 0 <= slot < kSlots

// Return cuda_fail(...) from the enclosing function when a CUDA runtime call fails.
#define RB200_CUDA(call)                                  \
  do {                                                    \
    cudaError_t e__ = (call);                             \
    if (e__ != cudaSuccess) return cuda_fail(e__, #call); \
  } while (0)

// Preamble of every entry point that needs an initialised library: holds the library lock for the rest of the scope and
// returns ERR_STATE (or ERR_CUDA) unless rgbdslam_b200_init has succeeded.
#define RB200_ENTER_INITED()                                    \
  std::lock_guard<std::mutex> entry_lock__(rb200::g_state.mu); \
  if (int entry_rc__ = rb200::check_inited()) return entry_rc__
void free_node(NodeDev* nd);  // frees everything a (possibly half-built) node owns (api.cu)

}  // namespace rb200
