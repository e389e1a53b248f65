// orb_host.h -- host-side launchers of the ORB kernels (orb.cu).
#pragma once
#include <cuda_runtime.h>

#include "../../include/rgbdslam_b200.h"
#include "orb.cuh"

namespace rb200 {

cudaError_t orb_upload_constants(const OrbGeom& g, const int* umax, cudaStream_t st);

// d_depth_for_mask != nullptr: detection mask = depthToCV8UC1(depth) != 0 (misc.cpp:414-418), d_mask ignored.
// detector: RGBDSLAM_B200_DETECTOR_ORB (8-level cell pyramids) or _FAST (level 0 only, cv::FAST's 3 px border).
cudaError_t orb_run_detect(const OrbGeom& g, const OrbTables& tab, int nframes, const uint8_t* d_gray, const uint8_t* d_mask,
                           const float* d_depth_for_mask, int detector, uint8_t* d_cell_img, uint8_t* d_cell_mask, OrbCand* d_cand,
                           int* d_cand_count, int* d_hist, int* d_mask_any, cudaStream_t st, int* launches);

// the adaptive-threshold recurrence of the F frames of a chunk, on the device (no host round trip)
cudaError_t orb_run_adapt(const OrbGeom& g, int nframes, const int* d_hist, const int* d_cand_count, const int* d_mask_any,
                          double* d_state, int* d_thr, int min_features, int max_features, int max_iters, int* d_err,
                          cudaStream_t st, int* launches);

// cvtColor(CV_RGB2GRAY) of nframes packed w*h*3 colour images into grey (node.cpp:139-144, 275-277).
cudaError_t orb_run_rgb_to_gray(int nframes, size_t px, const uint8_t* d_rgb, uint8_t* d_gray, cudaStream_t st, int* launches);
// calculateDepthMask (openni_listener.cpp:520-534) of nframes organised clouds, cloud_stride floats per point.
cudaError_t orb_run_cloud_mask(int nframes, size_t px, const float* d_cloud, int cloud_stride, uint8_t* d_mask, cudaStream_t st,
                               int* launches);

// detector ORB: Harris responses, orientation, size 31 * scale; FAST: response = corner score, angle -1, size 7.
// min_depth (mode 1 only; params.use_feature_min_depth): removeDepthless and projectTo3D take the minimum depth of each
// keypoint's neighbourhood (misc.cpp:774-791), one float per keepStrongest survivor in d_cand_z (nframes x ncells x max_per_cell).
// cloud_stride > 0 (mode 1 only): the point-cloud constructor (node.cpp:252-369) -- d_depth is an organised cloud of
// cloud_stride floats per point (x, y, z first); min_depth, depth_scaling and Kinv are not read.
cudaError_t orb_run_select(const OrbGeom& g, int nframes, int mode, int detector, int max_per_cell, int max_keypoints,
                           const uint8_t* d_cell_img, const OrbCand* d_cand, const int* d_cand_count, const int* d_thr,
                           float* d_resp, unsigned long long* d_cell_out, int* d_cell_out_count, const float* d_depth,
                           float depth_scaling, float4 Kinv, void* d_scratch, rgbdslam_b200_keypoint* d_kp, float4* d_xyz,
                           float2* d_trig /* mode 1: (cos, sin) of every keypoint's orientation for orb_run_describe, may be NULL */,
                           int* d_n, int kp_stride, bool min_depth, float* d_cand_z, int cloud_stride, cudaStream_t st,
                           int* launches);

// levels: extractor pyramid levels built and blurred (cv::ORB::compute builds 1 + the largest keypoint octave)
cudaError_t orb_run_describe(const OrbGeom& g, const OrbTables& tab, int nframes, int levels, const uint8_t* d_gray,
                             uint8_t* d_pyr_raw, uint8_t* d_pyr_blur, const rgbdslam_b200_keypoint* d_kp, const int* d_n,
                             int kp_stride, int max_kp, const float2* d_trig, uint8_t* d_desc, cudaStream_t st, int* launches);

constexpr int kOrbFrameCap = 4096;       // == kFrameCap in orb.cu
constexpr int kOrbFrameKpBytes = 24;     // sizeof(FrameKpZ), the larger of the two per-keypoint records of k_frame_finalize

}  // namespace rb200
