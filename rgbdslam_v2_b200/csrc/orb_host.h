// orb_host.h -- host-side launchers of the ORB kernels (orb.cu).
#pragma once
#include <cuda_runtime.h>

#include "../../include/rgbdslam_b200.h"
#include "orb.cuh"

namespace rb200 {

cudaError_t orb_upload_constants(const OrbGeom& g, const int* umax, cudaStream_t st);

// d_depth_for_mask != nullptr: detection mask = depthToCV8UC1(depth) != 0 (misc.cpp:414-418), d_mask ignored.
// detector: RGBDSLAM_B200_DETECTOR_ORB (8-level cell pyramids) or _FAST (level 0 only, cv::FAST's 3 px border).
// cand_cap: candidates per (frame, cell) in d_cand, as orb_prepare sizes it (at least kOrbCandCap).
cudaError_t orb_run_detect(const OrbGeom& g, const OrbTables& tab, int nframes, const uint8_t* d_gray, const uint8_t* d_mask,
                           const float* d_depth_for_mask, int detector, uint8_t* d_cell_img, uint8_t* d_cell_mask, OrbCand* d_cand,
                           int* d_cand_count, int* d_hist, int* d_mask_any, int cand_cap, cudaStream_t st, int* launches);

// How a call's detection thresholds come about (createDetector, features.cpp:101-112)
enum class OrbThresholds {
  kHistogram,   // the adjuster's recurrence on the score histograms (FAST, and ORB where no quota can change its count)
  kQuotaTable,  // the same recurrence on orb_run_quota_counts' tables: ORB where a cell's maximum reaches cv::ORB's smallest quota
  kFixed,       // adjuster_max_iterations <= 0: the bare DetectorAdjuster detects once at its persistent threshold
};

// the thresholds of the F frames of a chunk, on the device (no host round trip): d_hist holds the score histograms or, for
// kQuotaTable, the count tables
cudaError_t orb_run_adapt(const OrbGeom& g, int nframes, const int* d_hist, const int* d_cand_count, const int* d_mask_any,
                          double* d_state, int* d_thr, int min_features, int max_features, int max_iters, int* d_err,
                          int cand_cap, OrbThresholds mode, cudaStream_t st, int* launches);

// d_table[(f * ncells + c) * 256 + t] = the number of keypoints cv::ORB(10000, ..., t).detect returns on cell c of frame f,
// t = 0..255 (k_quota_counts), from the candidates of orb_run_detect.  Overwrites d_thr_scratch (nframes x ncells) and d_resp.
cudaError_t orb_run_quota_counts(const OrbGeom& g, int nframes, const uint8_t* d_cell_img, const OrbCand* d_cand,
                                 const int* d_cand_count, int* d_thr_scratch, float* d_resp, int cand_cap, int* d_table,
                                 cudaStream_t st, int* launches);

// cvtColor(CV_RGB2GRAY) of nframes packed w*h*3 colour images into grey (node.cpp:139-144, 275-277).
cudaError_t orb_run_rgb_to_gray(int nframes, size_t px, const uint8_t* d_rgb, uint8_t* d_gray, cudaStream_t st, int* launches);
// calculateDepthMask (openni_listener.cpp:520-534) of nframes organised clouds, cloud_stride floats per point.
cudaError_t orb_run_cloud_mask(int nframes, size_t px, const float* d_cloud, int cloud_stride, uint8_t* d_mask, cudaStream_t st,
                               int* launches);
// the listener's depth input of nframes w x h frames (openni_listener.cpp:633-659) from dw x dh images d_src, 16UC1 millimetres
// (u16) or float metres: the nearest-neighbour resize to w x h (:651-656; d_col[w] / d_row[h] source columns / rows, both NULL
// when dw == w and dh == h), then for u16 the conversion to metres and depthToCV8UC1's mask into d_mask unless it is NULL;
// the float plane goes to d_depth.  One launch.
cudaError_t orb_run_depth_gather(int nframes, int w, int h, const void* d_src, bool u16, int dw, int dh, const uint16_t* d_col,
                                 const uint16_t* d_row, float* d_depth, uint8_t* d_mask, cudaStream_t st, int* launches);
// cvtColor(COLOR_BayerGR2RGB) then cvtColor(CV_RGB2GRAY) of nframes w x h Bayer mosaics (openni_listener.cpp:638-641).
cudaError_t orb_run_bayer_gr_to_gray(int nframes, int w, int h, const uint8_t* d_raw, uint8_t* d_gray, cudaStream_t st, int* launches);

// Where the Node constructor takes a keypoint's 3-D point from (removeDepthless and projectTo3D).
enum class OrbPoints {
  kDepthPixel,  // the depth image at the rounded position (node.cpp:67-97, 900-965); the only source of mode 0
  kMinDepth,    // use_feature_min_depth: the minimum depth of the keypoint's neighbourhood (misc.cpp:774-791)
  kCloud,       // the point-cloud constructor (node.cpp:252-369): the organised cloud's point at the truncated position
};

// The candidates of every (frame, cell) and their responses (written by orb_run_select).
struct OrbCandidates {
  const OrbCand* cand;
  const int* count;
  const int* thr;
  float* resp;
  int cap;  // candidates per (frame, cell): the stride of cand and resp
};

// What k_min_depth, k_frame_finalize and k_frame_emit read and write, passed by value.
struct OrbFrameArgs {
  unsigned long long* cell_out;  // keepStrongest survivors: nframes x ncells x out_stride keys, written by k_cell_select
  int* cell_out_count;
  int out_stride;                // = the cell's keepStrongest cap
  const float* depth;            // depth images, or organised clouds of cloud_stride floats per point (x, y, z first)
  int cloud_stride;
  float* cand_z;                 // OrbPoints::kMinDepth: the neighbourhood depth of every cell_out key
  const uint8_t* cell_img;       // the detector's cell pyramids (orientation)
  float depth_scaling;
  float4 Kinv;                   // 1/fx, 1/fy, cx, cy
  void* scratch;                 // nframes x 2 x kOrbFrameCap records of kOrbFrameKpBytes
  rgbdslam_b200_keypoint* kp_out;
  float4* xyz_out;
  float2* trig_out;              // mode 1: (cos, sin) of every keypoint's orientation for orb_run_describe, may be NULL
  int* n_out;
  int kp_stride;
  int max_keypoints;
  int mode;                      // 0: detector output (OrbPoints::kDepthPixel), 1: Node constructor
};

// Whole-frame detectors: every frame's keypoints before k_frame_precap caps them at kOrbFrameCap (stride >= cand_cap)
struct OrbSurvivors {
  unsigned long long* keys;
  int* count;
  float* z;  // OrbPoints::kMinDepth
  int stride;
};

// detector ORB: Harris responses, cv::ORB's per-level quotas (k_cell_select), orientation, size 31 * scale; FAST:
// response = corner score, angle -1, size 7.  all != NULL (one whole-frame cell): no keepStrongest, the survivors go through
// `all` to k_frame_precap; d_err bit 1: a detector output (mode 0) of more than kOrbFrameCap keypoints.
cudaError_t orb_run_select(const OrbGeom& g, int nframes, int detector, OrbPoints points, const OrbCandidates& c,
                           const OrbFrameArgs& a, const OrbSurvivors* all, int* d_err, cudaStream_t st, int* launches);

// levels: extractor pyramid levels built and blurred (cv::ORB::compute builds 1 + the largest keypoint octave)
cudaError_t orb_run_describe(const OrbGeom& g, const OrbTables& tab, int nframes, int levels, const uint8_t* d_gray,
                             uint8_t* d_pyr_raw, uint8_t* d_pyr_blur, const rgbdslam_b200_keypoint* d_kp, const int* d_n,
                             int kp_stride, int max_kp, const float2* d_trig, uint8_t* d_desc, cudaStream_t st, int* launches);

constexpr int kOrbFrameCap = 4096;       // == kFrameCap in orb.cu
constexpr int kOrbFrameKpBytes = 24;     // sizeof(FrameKpZ), the larger of the two per-keypoint records of k_frame_finalize

}  // namespace rb200
