/*
 * rgbdslam_b200/depth_resize.h -- C ABI of the Node constructor for a depth image of another size than the visual: the
 * listener's nearest-neighbour resize of the depth (OpenNIListener::noCloudCallback, openni_listener.cpp:651-656,
 * cv::resize(depth, depth, visual.size(), 0, 0, cv::INTER_NEAREST), before depthToCV8UC1 builds the mask at :659) on the
 * device.  The conventions of ../rgbdslam_b200.h hold; the calls need an initialised library (ERR_STATE before
 * rgbdslam_b200_init).
 */
#ifndef RGBDSLAM_B200_DEPTH_RESIZE_H
#define RGBDSLAM_B200_DEPTH_RESIZE_H

#include "../rgbdslam_b200.h"

#ifdef __cplusplus
extern "C" {
#endif

/* rgbdslam_b200_nodes_create_ex for depth images of depth_w x depth_h pixels and visuals of w x h: `depth` holds nframes
 * depth_w x depth_h images, float metres or, with RGBDSLAM_B200_DEPTH_U16, uint16_t millimetres.  The visual, the caller's
 * mask, K4 (the visual camera's intrinsics, as the listener's cam_info), the frame size limits and STORE_CLOUD's skip-step
 * rule all refer to w x h.  Each frame's depth is first resized to w x h as cv2 4.13's INTER_NEAREST (resizeNN) does:
 *   ifx = 1.0 / ((double)w / depth_w),  ify = 1.0 / ((double)h / depth_h)                         (double)
 *   depth'(x, y) = depth(min((int)floor(x * ifx), depth_w - 1), min((int)floor(y * ify), depth_h - 1))
 * (the exact quotient x * depth_w / w picks another pixel at some sizes).  The resize only gathers pixels, so it commutes
 * with every per-pixel rule after it -- the 16-bit conversion (float)d * 0.001f, both depthToCV8UC1 masks (MASK_FROM_DEPTH),
 * depth_scaling_factor -- and a call is bit-identical to rgbdslam_b200_nodes_create_ex on the same visuals and cv::resize(depth, (w, h),
 * INTER_NEAREST): features, 3-D points and counts, the detector thresholds after the call, the stored cloud (STORE_CLOUD) and
 * the depth the environment measurement model keeps.  With depth_w == w and depth_h == h the call is
 * rgbdslam_b200_nodes_create_ex.  The depth is uploaded at its own size (2 or 4 bytes per depth pixel) and resized on the device
 * into the w x h float plane the constructor reads; the index tables are built on the host once per (w, h, depth_w, depth_h).
 * ERR_ARG before any device work, nothing launched: depth_w or depth_h outside [1, 4095]; any of RGBDSLAM_B200_CLOUD_XYZRGB,
 * CLOUD_XYZ, MASK_FROM_CLOUD and KEEP_CLOUD (the listener drops clouds of another size, openni_listener.cpp:713-719); every
 * case rgbdslam_b200_nodes_create_ex rejects. */
int rgbdslam_b200_nodes_create_resized(uint64_t detector, int nframes, const uint8_t* gray, const void* depth, int depth_w, int depth_h,
                                       const uint8_t* mask, int w, int h, const float* K4, const int32_t* ids, int flags,
                                       uint64_t* node_handles, int32_t* n_features);
/* rgbdslam_b200_nodes_create_sharded for depth images of depth_w x depth_h pixels: each rank passes its own frames' depth at
 * that size, resized on the device as above.  Bit-identical to rgbdslam_b200_nodes_create_resized on one GPU.  Rejected with
 * ERR_ARG before any device work: the cases of rgbdslam_b200_nodes_create_resized and of rgbdslam_b200_nodes_create_sharded. */
int rgbdslam_b200_nodes_create_sharded_resized(uint64_t detector, uint64_t comm_handle, int total_frames, const uint8_t* gray,
                                               const void* depth, int depth_w, int depth_h, const uint8_t* mask, int w, int h,
                                               const float* K4, const int32_t* ids, int flags, uint64_t* node_handles,
                                               int32_t* n_features);

#ifdef __cplusplus
}
#endif
#endif /* RGBDSLAM_B200_DEPTH_RESIZE_H */
