// orb.cu -- ORB keypoint detection / description kernels for sm_90a (see orb.cuh for provenance).
//
// Node constructor path (src/node.cpp:101-240), batched over frames:
//   detector->detect(gray, kp, mask)      VideoGridAdaptedFeatureDetector (feature_adjuster.cpp:286-317) over
//                                         VideoDynamicAdaptedFeatureDetector (:185-224) over cv::ORB (:94)
//     k_cell_extract / k_resize_cells     per-cell 8-level pyramids, chained INTER_LINEAR_EXACT; mask pyramid
//     k_fast_nms                          threshold-free FAST-9/16 corner score S, strict 3x3 NMS, mask + 15 px border
//                                         -> candidate list + histogram of S per (frame, cell)
//     (host) adaptive thresholds          the x0.7 / x1.3 recurrence only needs #candidates(S >= t): a histogram lookup
//     k_harris                            Harris response of the candidates that pass the final threshold
//     k_cell_select                       cv::ORB's per-level quotas, then keepStrongest(maxTotal / cells) by |response|
//                                         (feature_adjuster.cpp:247-255)
//   removeDepthless / retainBest / compute() border filter + octave sort / projectTo3D      (node.cpp:186-210)
//     k_frame_finalize<P>                 one CTA per frame; P (OrbPoints) = where a keypoint's 3-D point comes from
//     k_frame_emit<D, P>                  one warp per keypoint: orientation, cv::KeyPoint, projectTo3D; D = detector
//   extractor->compute(gray, kp, desc)    cv::ORB::create() defaults (features.cpp:117-119)
//     k_resize / k_blur / k_describe      full-image pyramid, 7-tap float Gaussian, steered BRIEF (one warp / keypoint)
//
// The FAST detector (feature_detector_type FAST: DetectorAdjuster("FAST", 20) -> cv::FastFeatureDetector::create(thresh),
// feature_adjuster.cpp:88-91, under the same dynamic and grid wrappers) runs the same chain on level 0 only: k_cell_extract
// (no k_resize_cells), k_fast9_nms (the k_fast_nms body with cv::FAST's 3 px frame, whose scores read as 0 in the NMS),
// k_adapt_thresholds, k_fast_response (response = S) in place of k_harris, k_cell_sort (k_cell_select without
// quotas where orb_prepare sizes the candidate buffer by area), k_frame_finalize,
// k_frame_emit<FAST, P> (size 7, angle -1, no orientation) and level 0 of the extractor pyramid.
//
// Apart from k_cell_sort, the kernels are the same at every frame size and candidate capacity: the candidate buffer's stride
// per (frame, cell) is a kernel argument (api_orb.cu sizes it), and the selection keys hold 12-bit level coordinates (CellPos,
// up to kOrbMaxSide).
//
// use_feature_min_depth (parameter_server.cpp:90) adds k_min_depth after k_cell_select: the minimum depth in each keypoint's
// neighbourhood (misc.cpp:774-791), which the kMinDepth instantiations of finalize and emit use for removeDepthless and
// projectTo3D.
//
// Colour input (node.cpp:139-144, 275-277: cvtColor(visual, gray, CV_RGB2GRAY)) adds k_rgb_to_gray in front of the chain.
// The point-cloud constructor (node.cpp:252-369) adds k_cloud_mask when the caller derives the mask from the cloud
// (calculateDepthMask, openni_listener.cpp:520-534) and runs k_frame_finalize<kCloud> / k_frame_emit<D, kCloud> in place
// of the depth-image finalize and emit: projectTo3D (node.cpp:855-898) on the detector's output, then compute().
// The listener's raw inputs (openni_listener.cpp:633-659) add k_depth_gather<uint16_t> (16UC1 millimetres -> metres and,
// optionally, the detection mask) and k_bayer_gr_to_gray (Bayer GRBG -> grey) in front of the chain; a depth image of another
// size than the visual adds its nearest-neighbour resize (:651-656), k_depth_gather<uint16_t> or <float>.  Everything after
// them is the grey, float-depth, caller-mask path.
#include "orb.cuh"

#include <cuda_runtime.h>

#include <type_traits>

#include "orb_tables_generated.h"
#include "orb_host.h"

namespace rb200 {

__constant__ OrbGeom c_geom;
__constant__ float c_gauss[7];
__constant__ int8_t c_pattern[256][4];
__constant__ int c_umax[kOrbHalfPatch + 2];
constexpr int kFT_W = 56, kFT_H = 30;  // output pixels per CTA
constexpr int kFS_W = 64, kFS_H = 32;  // scores computed per CTA: x in [-4, 60), y in [-1, 31) relative to the tile origin
constexpr int kFI_W = 72, kFI_H = 38;  // image pixels staged: x in [-8, 64), y in [-4, 34)
constexpr int kFastEdge = 15;          // ORB::create(..., edgeThreshold = 15, ...)  feature_adjuster.cpp:94
constexpr int kFast9Edge = 3;          // cv::FAST scores rows / columns [3, n-4] only

struct FastTiling {  // tiles of the fused kernel: per level the tile grid of the LARGEST cell, prefix sums over levels
  int32_t tiles_x[kOrbLevels], tiles_y[kOrbLevels], first[kOrbLevels + 1];
};
__constant__ FastTiling c_fast_tiling;  // ORB detector (all levels)

// CTAs per (frame, cell) of the fused FAST + NMS kernel, per detector type; the FAST detector tiles level 0 only, with its
// own border, and takes its tile-grid width as a kernel argument
static int g_fast_tiles[2] = {0, 0};
static int g_fast9_tiles_x = 1;

cudaError_t orb_upload_constants(const OrbGeom& g, const int* umax, cudaStream_t st) {
  cudaError_t e = cudaMemcpyToSymbolAsync(c_geom, &g, sizeof(OrbGeom), 0, cudaMemcpyHostToDevice, st);
  if (e != cudaSuccess) return e;
  e = cudaMemcpyToSymbolAsync(c_gauss, kOrbGaussBits, sizeof(float) * 7, 0, cudaMemcpyHostToDevice, st);
  if (e != cudaSuccess) return e;
  e = cudaMemcpyToSymbolAsync(c_pattern, kOrbPattern, sizeof(kOrbPattern), 0, cudaMemcpyHostToDevice, st);
  if (e != cudaSuccess) return e;
  e = cudaMemcpyToSymbolAsync(c_umax, umax, sizeof(int) * (kOrbHalfPatch + 2), 0, cudaMemcpyHostToDevice, st);
  if (e != cudaSuccess) return e;
  FastTiling ft;
  ft.first[0] = 0;
  for (int l = 0; l < kOrbLevels; l++) {
    int lw = 0, lh = 0;
    for (int c = 0; c < g.ncells; c++) {
      lw = g.cell[c][l].w > lw ? g.cell[c][l].w : lw;
      lh = g.cell[c][l].h > lh ? g.cell[c][l].h : lh;
    }
    const int iw = lw - 2 * kFastEdge, ih = lh - 2 * kFastEdge;  // pixels that can become keypoints
    ft.tiles_x[l] = iw > 0 ? (iw + kFT_W - 1) / kFT_W : 0;
    ft.tiles_y[l] = ih > 0 ? (ih + kFT_H - 1) / kFT_H : 0;
    if (ft.tiles_x[l] == 0 || ft.tiles_y[l] == 0) ft.tiles_x[l] = ft.tiles_y[l] = 0;
    ft.first[l + 1] = ft.first[l] + ft.tiles_x[l] * ft.tiles_y[l];
    if (ft.tiles_x[l] == 0) ft.tiles_x[l] = 1;  // never divided by for an empty level (no CTA maps to it)
  }
  g_fast_tiles[RGBDSLAM_B200_DETECTOR_ORB] = ft.first[kOrbLevels];
  {
    int lw = 0, lh = 0;
    for (int c = 0; c < g.ncells; c++) {
      lw = g.cell[c][0].w > lw ? g.cell[c][0].w : lw;
      lh = g.cell[c][0].h > lh ? g.cell[c][0].h : lh;
    }
    const int iw = lw - 2 * kFast9Edge, ih = lh - 2 * kFast9Edge;
    const int tx = iw > 0 ? (iw + kFT_W - 1) / kFT_W : 0, ty = ih > 0 ? (ih + kFT_H - 1) / kFT_H : 0;
    g_fast_tiles[RGBDSLAM_B200_DETECTOR_FAST] = tx * ty;
    g_fast9_tiles_x = tx > 0 ? tx : 1;
  }
  return cudaMemcpyToSymbolAsync(c_fast_tiling, &ft, sizeof(ft), 0, cudaMemcpyHostToDevice, st);
}

// -------------------------------------------------------------------------------------------------
// level 0 of the per-cell pyramids: sub-image copy; mask binarised (cv2: any non-zero mask pixel is valid).
// depth != nullptr: the detection mask is derived on the device as the caller of the reference does on the host --
// depthToCV8UC1 (misc.cpp:414-418): depth.convertTo(mono8, CV_8UC1, 100, 0) = saturate_cast<uchar>(cvRound(d * 100.f)),
// NaN -> 0 -- of which only "non-zero" matters: valid iff d * 100.f rounds (half to even) to an int in [1, 2^31).
// mask_any[f * ncells + c] receives 1 when the cell's mask has any non-zero pixel (hasNonZero, feature_adjuster.cpp:176-183).
__global__ void __launch_bounds__(256) k_cell_extract(const uint8_t* __restrict__ gray, const uint8_t* __restrict__ mask,
                                                      const float* __restrict__ depth, uint8_t* __restrict__ cell_img,
                                                      uint8_t* __restrict__ cell_mask, int* __restrict__ mask_any) {
  const int f = blockIdx.z / c_geom.ncells, c = blockIdx.z % c_geom.ncells;
  const OrbPlane& p = c_geom.cell[c][0];
  const int x = blockIdx.x * 32 + (threadIdx.x & 31), y = blockIdx.y * 8 + (threadIdx.x >> 5);
  bool nz = false;
  if (x < p.w && y < p.h) {
    const size_t src = (size_t)f * c_geom.W * c_geom.H + (size_t)(c_geom.cell_y0[c] + y) * c_geom.W + c_geom.cell_x0[c] + x;
    const size_t dst = (size_t)f * c_geom.cell_bytes + p.off + (size_t)y * p.w + x;
    cell_img[dst] = gray[src];
    if (depth) {
      const float v = __fmul_rn(depth[src], 100.f);
      nz = v == v && v < 2147483648.f && __float2int_rn(v) >= 1;  // cvRound of +inf / >= 2^31 is INT_MIN -> saturates to 0
    } else {
      nz = mask ? mask[src] != 0 : true;
    }
    cell_mask[dst] = nz ? 255 : 0;
  }
  // one (conditional) flag write per CTA: thousands of warps storing to the same word serialise in L2
  if (__syncthreads_or(nz) && threadIdx.x == 0 && mask_any[blockIdx.z] == 0) mask_any[blockIdx.z] = 1;
}

// cvtColor(visual, gray, CV_RGB2GRAY) (node.cpp:139-144, 275-277) of n packed 3-byte pixels, channel 0 weighted as R whatever
// the image's real channel order: OpenCV 4's 15-bit fixed point, (R * 9798 + G * 19235 + B * 3735 + 2^14) >> 15 (equal to
// cv2 4.13 on all 2^24 triples; DESIGN.md 4.5.3).  Four pixels per thread: three 32-bit loads, one 32-bit store (the same four
// pixels byte by byte when a buffer is not 4-byte aligned, and for the last < 4 pixels).
__device__ __forceinline__ uint32_t rgb_to_gray_px(uint32_t r, uint32_t g, uint32_t b) {
  return (r * 9798u + g * 19235u + b * 3735u + (1u << 14)) >> 15;
}

__global__ void __launch_bounds__(256) k_rgb_to_gray(const uint8_t* __restrict__ rgb, uint8_t* __restrict__ gray, size_t n) {
  const size_t p = ((size_t)blockIdx.x * blockDim.x + threadIdx.x) * 4;
  const bool aligned = ((reinterpret_cast<uintptr_t>(rgb) | reinterpret_cast<uintptr_t>(gray)) & 3) == 0;
  if (p + 4 <= n && aligned) {
    const uint32_t* w = reinterpret_cast<const uint32_t*>(rgb + 3 * p);
    const uint32_t w0 = w[0], w1 = w[1], w2 = w[2];  // bytes r0 g0 b0 r1 | g1 b1 r2 g2 | b2 r3 g3 b3
    const uint32_t v0 = rgb_to_gray_px(w0 & 0xFF, (w0 >> 8) & 0xFF, (w0 >> 16) & 0xFF);
    const uint32_t v1 = rgb_to_gray_px(w0 >> 24, w1 & 0xFF, (w1 >> 8) & 0xFF);
    const uint32_t v2 = rgb_to_gray_px((w1 >> 16) & 0xFF, w1 >> 24, w2 & 0xFF);
    const uint32_t v3 = rgb_to_gray_px((w2 >> 8) & 0xFF, (w2 >> 16) & 0xFF, w2 >> 24);
    *reinterpret_cast<uint32_t*>(gray + p) = v0 | (v1 << 8) | (v2 << 16) | (v3 << 24);
  } else {
    for (size_t i = p, e = min(p + 4, n); i < e; i++) gray[i] = (uint8_t)rgb_to_gray_px(rgb[3 * i], rgb[3 * i + 1], rgb[3 * i + 2]);
  }
}

// calculateDepthMask (openni_listener.cpp:520-534) of n organised-cloud points (stride floats per point, z at float 2):
// static_cast<uchar>(z * 50.0) as x86-64 compilers emit it -- cvttsd2si to int32 (0x80000000 when the truncated value does
// not fit), then the low byte -- and 0 for NaN.  So the byte is 0 below 0.02 m, wraps every 5.12 m, and is 0 for |z| >= ~43e6 m
// and +-inf.  CUDA's saturating conversions differ, hence the explicit range test.
__global__ void __launch_bounds__(256) k_cloud_mask(const float* __restrict__ cloud, int stride, uint8_t* __restrict__ mask, size_t n) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const float z = cloud[i * stride + 2];
  const double v = __dmul_rn((double)z, 50.0);
  const int iv = (v > -2147483649.0 && v < 2147483648.0) ? __double2int_rz(v) : (int)0x80000000;  // NaN fails the test
  mask[i] = z != z ? 0 : (uint8_t)(iv & 0xFF);
}

// The listener's depth input (openni_listener.cpp:633-659) of one w x h frame per blockIdx.z, read from the caller's dw x dh
// images: pixel (x, y) takes source pixel (col[x], row[y]), cv::resize(depth, depth, visual.size(), 0, 0, INTER_NEAREST)
// (:651-656) with the tables of nn_resize_tables (api_orb.cu); col == row == NULL is the identity (dw == w, dh == h).  The
// resize only gathers, so it commutes with the per-pixel rules after it.
//   T = uint16_t, 16UC1 millimetres, then the listener's conversions:
//     depth = convertTo(CV_32FC1, 0.001)                            = (float)d * 0.001f, so a hole (0) reads as 0 m, not NaN
//     mask  = depthToCV8UC1: convertTo(CV_8UC1, 0.05, -25) (misc.cpp:414-425) = saturate_cast<uchar>(fmaf(d, 0.05f, -25.f)),
//             non-zero iff d >= 510 (an unfused d * 0.05f - 25 gives 0.5 -> 0 at d = 510); written only when mask != nullptr.
//     Both equal cv2 4.13 on all 65536 values.
//   T = float, metres: the gather alone (bits copied, NaN kept); the float mask rule is k_cell_extract's.
template <class T>
__global__ void __launch_bounds__(256) k_depth_gather(const T* __restrict__ src, int dw, int dh, const uint16_t* __restrict__ col,
                                                      const uint16_t* __restrict__ row, float* __restrict__ depth,
                                                      uint8_t* __restrict__ mask, int w, int h) {
  const int x = blockIdx.x * 32 + (threadIdx.x & 31), y = blockIdx.y * 8 + (threadIdx.x >> 5);
  if (x >= w || y >= h) return;
  const int sx = col ? col[x] : x, sy = row ? row[y] : y;
  const T v = src[(size_t)blockIdx.z * dw * dh + (size_t)sy * dw + sx];
  const size_t i = (size_t)blockIdx.z * w * h + (size_t)y * w + x;
  if constexpr (std::is_same<T, uint16_t>::value) {
    const float d = (float)v;
    depth[i] = __fmul_rn(d, 0.001f);
    if (mask) mask[i] = (uint8_t)min(max(__float2int_rn(__fmaf_rn(d, 0.05f, -25.f)), 0), 255);
  } else {
    depth[i] = v;
  }
}

// cvtColor(raw, rgb, COLOR_BayerGR2RGB) (openni_listener.cpp:638-641; bayer_gr_rgb, orb.cuh) then cvtColor(CV_RGB2GRAY)
// (node.cpp:139-144) of one w x h frame per blockIdx.z.  RGB is rounded to u8 before the grey rule, as the two calls do (cv2's
// fused BayerGR2GRAY rounds differently).
__global__ void __launch_bounds__(256) k_bayer_gr_to_gray(const uint8_t* __restrict__ raw, uint8_t* __restrict__ gray, int w, int h) {
  const int x = blockIdx.x * 32 + (threadIdx.x & 31), y = blockIdx.y * 8 + (threadIdx.x >> 5);
  if (x >= w || y >= h) return;
  const size_t frame = (size_t)blockIdx.z * w * h;
  uint32_t r, g, b;
  bayer_gr_rgb(raw, frame, w, h, x, y, r, g, b);
  gray[frame + (size_t)y * w + x] = (uint8_t)rgb_to_gray_px(r, g, b);
}

// level of the full-image pyramid = INTER_LINEAR_EXACT resize of the previous level (8.8 fixed-point taps, round to nearest at
// the end).  One frame per blockIdx.z.
__global__ void __launch_bounds__(256) k_resize(uint8_t* __restrict__ buf, int frame_stride, int level, OrbTables tab) {
  const int f = blockIdx.z;
  const OrbPlane& d = c_geom.full[level];
  const OrbPlane& s = c_geom.full[level - 1];
  const int x = blockIdx.x * 32 + (threadIdx.x & 31), y = blockIdx.y * 8 + (threadIdx.x >> 5);
  if (x >= d.w || y >= d.h) return;
  const uint8_t* sp = buf + (size_t)f * frame_stride + s.off;
  const int ox = tab.ofs[d.tx + x], ax1 = tab.w1[d.tx + x], ax0 = 256 - ax1;
  const int oy = tab.ofs[d.ty + y], ay1 = tab.w1[d.ty + y], ay0 = 256 - ay1;
  const int x1 = min(ox + 1, s.w - 1), y1 = min(oy + 1, s.h - 1);
  const int h0 = sp[oy * s.w + ox] * ax0 + sp[oy * s.w + x1] * ax1;
  const int h1 = sp[y1 * s.w + ox] * ax0 + sp[y1 * s.w + x1] * ax1;
  const int v = (h0 * ay0 + h1 * ay1 + (1 << 15)) >> 16;
  buf[(size_t)f * frame_stride + d.off + (size_t)y * d.w + x] = (uint8_t)v;
}

// -------------------------------------------------------------------------------------------------
// Fused FAST score + NMS for ALL pyramid levels of all (frame, cell) planes in one launch.  The threshold-free score:
//   S + 1 = max( v - min_k max_{j<9} p[k+j] ,  max_k min_{j<9} p[k+j] - v )       (k, j on the 16-pixel circle)
// which equals the largest threshold t for which 9 contiguous circle pixels are all darker than v - t or all brighter than
// v + t (== cv::FAST's cornerScore<16>), clamped at 0.  Two horizontally adjacent pixels share a register as s16x2 halves
// (VIMNMX3.S16x2: three-input packed min / max), the image tile is staged in shared memory as 16-bit values so that a pixel
// pair is one aligned 32-bit word (even offsets) or one PRMT of two words (odd offsets).  The 8-bit scores of a tile plus a
// one-pixel halo stay in shared memory for the 3x3 non-maximum suppression: the score plane never goes to global memory.
__device__ __forceinline__ uint32_t pair_at(const uint16_t (*simg)[kFI_W], int row, int col) {  // pixels (col, col+1) as s16x2
  const uint32_t* r = reinterpret_cast<const uint32_t*>(simg[row]);
  const uint32_t w0 = r[col >> 1];
  if ((col & 1) == 0) return w0;
  return __byte_perm(w0, r[(col >> 1) + 1], 0x5432);
}

__device__ __forceinline__ uint32_t fast_score_pair(const uint16_t (*simg)[kFI_W], int row, int col) {
  // circle offsets in cv::FAST order (any rotation of the ring gives the same arcs)
  constexpr int dx[16] = {0, 1, 2, 3, 3, 3, 2, 1, 0, -1, -2, -3, -3, -3, -2, -1};
  constexpr int dy[16] = {3, 3, 2, 1, 0, -1, -2, -3, -3, -3, -2, -1, 0, 1, 2, 3};
  uint32_t r[16];
#pragma unroll
  for (int k = 0; k < 16; k++) r[k] = pair_at(simg, row + dy[k], col + dx[k]);
  const uint32_t v = pair_at(simg, row, col);
  uint32_t hi3[16], lo3[16];
#pragma unroll
  for (int k = 0; k < 16; k++) {
    hi3[k] = __vimax3_s16x2(r[k], r[(k + 1) & 15], r[(k + 2) & 15]);
    lo3[k] = __vimin3_s16x2(r[k], r[(k + 1) & 15], r[(k + 2) & 15]);
  }
  uint32_t mn = 0x7fff7fffu, mx = 0u;  // min over arcs of the arc maximum / max over arcs of the arc minimum
#pragma unroll
  for (int k = 0; k < 16; k += 2) {
    const uint32_t a0 = __vimax3_s16x2(hi3[k], hi3[(k + 3) & 15], hi3[(k + 6) & 15]);
    const uint32_t a1 = __vimax3_s16x2(hi3[k + 1], hi3[(k + 4) & 15], hi3[(k + 7) & 15]);
    mn = __vimin3_s16x2(mn, a0, a1);
    const uint32_t b0 = __vimin3_s16x2(lo3[k], lo3[(k + 3) & 15], lo3[(k + 6) & 15]);
    const uint32_t b1 = __vimin3_s16x2(lo3[k + 1], lo3[(k + 4) & 15], lo3[(k + 7) & 15]);
    mx = __vimax3_s16x2(mx, b0, b1);
  }
  // per half: S = max(v - mn, mx - v) - 1, clamped at 0 (all quantities within [-255, 255]: no cross-half borrow after biasing)
  const uint32_t bias = 0x01000100u;
  const uint32_t apos = (v + bias) - mn;  // v - mn + 256 in [1, 511]
  const uint32_t aneg = (mx + bias) - v;  // mx - v + 256
  const uint32_t m = __vmaxs2(apos, aneg);
  return __vmaxs2(m, 0x01010101u) - 0x01010101u;  // (max(., 257) - 257) per half = max(A - 1, 0)
}

// kFast = false: the ORB detector -- every level, candidates at least 15 px inside the level, whose NMS sees the real scores
// of the pixels around them.  kFast = true: the FAST detector -- level 0 only (tiles_x9 tiles per row); cv::FAST scores only
// the pixels [3, n-4] of the cell and its NMS reads every other pixel as score 0, so the scores outside that band are zeroed
// before the NMS.
template <bool kFast>
__device__ __forceinline__ void fast_nms_tile(const uint8_t* __restrict__ cell_img, const uint8_t* __restrict__ cell_mask,
                                              OrbCand* __restrict__ cand, int* __restrict__ cand_count, int* __restrict__ hist,
                                              int tiles_x9, int cap) {
  constexpr int kEdge = kFast ? kFast9Edge : kFastEdge;
  __shared__ __align__(16) uint16_t simg[kFI_H][kFI_W];
  __shared__ __align__(16) uint8_t ssc[kFS_H][kFS_W];
  int level = 0, tx, ty;
  if constexpr (kFast) {
    tx = blockIdx.x % tiles_x9;
    ty = blockIdx.x / tiles_x9;
  } else {
#pragma unroll
    for (int l = 1; l < kOrbLevels; l++)
      if ((int)blockIdx.x >= c_fast_tiling.first[l]) level = l;
    const int t = blockIdx.x - c_fast_tiling.first[level];
    tx = t % c_fast_tiling.tiles_x[level];
    ty = t / c_fast_tiling.tiles_x[level];
  }
  const int fc = blockIdx.y;
  const int f = fc / c_geom.ncells, c = fc % c_geom.ncells;
  const int pw = c_geom.cell[c][level].w, ph = c_geom.cell[c][level].h;
  const int ox0 = kEdge + tx * kFT_W, oy0 = kEdge + ty * kFT_H;
  if (ox0 >= pw - kEdge || oy0 >= ph - kEdge) return;
  const size_t base = (size_t)f * c_geom.cell_bytes + c_geom.cell[c][level].off;
  const uint8_t* im = cell_img + base;
  for (int i = threadIdx.x; i < kFI_H * kFI_W; i += 256) {
    const int rr = i / kFI_W, cc = i - rr * kFI_W;
    const int gx = ox0 - 8 + cc, gy = oy0 - 4 + rr;
    simg[rr][cc] = (gx >= 0 && gx < pw && gy >= 0 && gy < ph) ? im[gy * pw + gx] : 0;
  }
  __syncthreads();
  {  // scores: thread = (quad of 4 columns, row), two row passes
    const int q = threadIdx.x & 15, r0 = threadIdx.x >> 4;
    // rows below the last output row of this tile (+ 1 for the NMS) are never read: skipping them (a warp owns two
    // adjacent rows per pass) removes most of the waste of partially covered tiles
    const int sy_last = min(kFT_H, ph - kEdge - oy0) + 1;
#pragma unroll
    for (int pass = 0; pass < 2; pass++) {
      const int sy = r0 + 16 * pass;  // score row (relative y = sy - 1) -> image row sy + 3
      if (sy > sy_last) continue;
      const uint32_t s01 = fast_score_pair(simg, sy + 3, 4 * q + 4);
      const uint32_t s23 = fast_score_pair(simg, sy + 3, 4 * q + 6);
      // halves hold 0..254: pack the four scores into bytes
      uint32_t s4 = __byte_perm(s01, s23, 0x6420);
      if constexpr (kFast) {  // outside cv::FAST's scored band [3, n-4]: score 0
        const int gy = oy0 + sy - 1, gx = ox0 + 4 * q - 4;
        uint32_t keep = 0;
        if (gy >= kEdge && gy < ph - kEdge) {
#pragma unroll
          for (int b = 0; b < 4; b++)
            if (gx + b >= kEdge && gx + b < pw - kEdge) keep |= 0xFFu << (8 * b);
        }
        s4 &= keep;
      }
      reinterpret_cast<uint32_t*>(ssc[sy])[q] = s4;
    }
  }
  __syncthreads();
  // strict 3x3 non-maximum suppression on S, runByPixelsMask, runByImageBorder(kEdge) -> candidates + histogram
  for (int i = threadIdx.x; i < kFT_W * kFT_H; i += 256) {
    const int oy = i / kFT_W, ox = i - oy * kFT_W;
    const int gx = ox0 + ox, gy = oy0 + oy;
    if (gx >= pw - kEdge || gy >= ph - kEdge) continue;
    const int sx = ox + 4, sy = oy + 1;
    const int v = ssc[sy][sx];
    if (v < 2) continue;  // the adaptive threshold never drops below 2 (DetectorAdjuster min_thresh)
    const bool mxm = v > ssc[sy - 1][sx - 1] && v > ssc[sy - 1][sx] && v > ssc[sy - 1][sx + 1] && v > ssc[sy][sx - 1] &&
                     v > ssc[sy][sx + 1] && v > ssc[sy + 1][sx - 1] && v > ssc[sy + 1][sx] && v > ssc[sy + 1][sx + 1];
    if (!mxm) continue;
    if (cell_mask && cell_mask[base + (size_t)gy * pw + gx] == 0) continue;
    atomicAdd(&hist[fc * 256 + v], 1);
    const int slot = atomicAdd(&cand_count[fc], 1);
    if (slot < cap) {
      OrbCand cd;
      cd.x = (uint16_t)gx;
      cd.y = (uint16_t)gy;
      cd.level = (uint8_t)level;
      cd.score = (uint8_t)v;
      cd.pad_ = 0;
      cand[(size_t)fc * cap + slot] = cd;
    }
  }
}

// cap: candidates per (frame, cell), the stride of cand
__global__ void __launch_bounds__(256) k_fast_nms(const uint8_t* __restrict__ cell_img, const uint8_t* __restrict__ cell_mask,
                                                  OrbCand* __restrict__ cand, int* __restrict__ cand_count, int* __restrict__ hist,
                                                  int cap) {
  fast_nms_tile<false>(cell_img, cell_mask, cand, cand_count, hist, 0, cap);
}

__global__ void __launch_bounds__(256) k_fast9_nms(const uint8_t* __restrict__ cell_img, const uint8_t* __restrict__ cell_mask,
                                                   OrbCand* __restrict__ cand, int* __restrict__ cand_count, int* __restrict__ hist,
                                                   int tiles_x, int cap) {
  fast_nms_tile<true>(cell_img, cell_mask, cand, cand_count, hist, tiles_x, cap);
}

// All cell planes of one level from the previous level, image and mask together (INTER_LINEAR_EXACT, 8.8 fixed-point taps;
// the mask level is THRESH_TOZERO(254) of its resize, i.e. 255 exactly when every tap with a non-zero weight is 255).
__global__ void __launch_bounds__(256) k_resize_cells(uint8_t* __restrict__ cell_img, uint8_t* __restrict__ cell_mask, int level,
                                                      OrbTables tab) {
  const int fc = blockIdx.z;
  const int f = fc / c_geom.ncells, c = fc - f * c_geom.ncells;
  const int dw = c_geom.cell[c][level].w, dh = c_geom.cell[c][level].h;
  const int x = blockIdx.x * 32 + (threadIdx.x & 31), y = blockIdx.y * 8 + (threadIdx.x >> 5);
  if (x >= dw || y >= dh) return;
  const int sw = c_geom.cell[c][level - 1].w, sh = c_geom.cell[c][level - 1].h;
  const unsigned fbase = (unsigned)f * (unsigned)c_geom.cell_bytes;
  const unsigned soff = fbase + c_geom.cell[c][level - 1].off, doff = fbase + c_geom.cell[c][level].off;
  const int tx = c_geom.cell[c][level].tx + x, ty = c_geom.cell[c][level].ty + y;
  const int ox = tab.ofs[tx], ax1 = tab.w1[tx], ax0 = 256 - ax1;
  const int oy = tab.ofs[ty], ay1 = tab.w1[ty], ay0 = 256 - ay1;
  const int x1 = min(ox + 1, sw - 1), y1 = min(oy + 1, sh - 1);
  const unsigned i00 = soff + oy * sw + ox, i01 = soff + oy * sw + x1, i10 = soff + y1 * sw + ox, i11 = soff + y1 * sw + x1;
  {
    const int h0 = cell_img[i00] * ax0 + cell_img[i01] * ax1;
    const int h1 = cell_img[i10] * ax0 + cell_img[i11] * ax1;
    cell_img[doff + y * dw + x] = (uint8_t)((h0 * ay0 + h1 * ay1 + (1 << 15)) >> 16);
  }
  if (cell_mask) {
    const int h0 = cell_mask[i00] * ax0 + cell_mask[i01] * ax1;
    const int h1 = cell_mask[i10] * ax0 + cell_mask[i11] * ax1;
    const int v = (h0 * ay0 + h1 * ay1 + (1 << 15)) >> 16;
    cell_mask[doff + y * dw + x] = v <= 254 ? 0 : (uint8_t)v;
  }
}

// VideoDynamicAdaptedFeatureDetector::detect (feature_adjuster.cpp:185-224) on the histogram of corner scores, for the
// F frames of a chunk IN ORDER (the threshold of a cell persists from frame to frame, feature_adjuster.cpp:131-150).
// The re-detect loop (x0.7 while too few, <= max_iters detections) only needs #candidates(S >= t): a histogram lookup.
// One warp per grid cell; lane l owns score bins [8l, 8l+8).  state[c] = the detector's persistent threshold (double, as in
// the reference); thr_out[f * ncells + c] = the integer FAST threshold of the LAST detection call of that frame.
// err_flag bit 0: a cell overflowed the candidate buffer (cap candidates per cell).
// kTable: hist holds, per (frame, cell), the count cv::ORB's detect returns at each threshold t = 0..255 (k_quota_counts) in
// place of the score histogram.
template <bool kTable>
__device__ __forceinline__ void adapt_thresholds(const int* __restrict__ hist, const int* __restrict__ cand_count,
                                                 const int* __restrict__ mask_any, double* __restrict__ state,
                                                 int* __restrict__ thr_out, int nframes, int ncells, int min_features,
                                                 int max_features, int max_iters, int* __restrict__ err_flag, int cap) {
  const int c = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (c >= ncells) return;
  double thresh = state[c];
  for (int f = 0; f < nframes; f++) {
    const int fc = f * ncells + c;
    int h[8];
    if constexpr (!kTable) {
      const int4 a = reinterpret_cast<const int4*>(hist + (size_t)fc * 256)[lane * 2];
      const int4 b = reinterpret_cast<const int4*>(hist + (size_t)fc * 256)[lane * 2 + 1];
      h[0] = a.x; h[1] = a.y; h[2] = a.z; h[3] = a.w; h[4] = b.x; h[5] = b.y; h[6] = b.z; h[7] = b.w;
    }
    const int cnt = cand_count[fc];
    if (cnt > cap && lane == 0) atomicOr(err_flag, 1);
    const bool mask_nonzero = cnt > 0 || mask_any[fc] != 0;
    int iter = max_iters, used = 0;
    bool checked = false;
    do {
      const int t = (int)thresh;  // static_cast<int>(thresh_) feature_adjuster.cpp:94
      used = t;
      int part = 0;
      if constexpr (kTable) {
        part = t < 256 ? hist[(size_t)fc * 256 + t] : 0;
      } else {
#pragma unroll
        for (int k = 0; k < 8; k++) part += (lane * 8 + k >= t) ? h[k] : 0;
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) part += __shfl_xor_sync(0xffffffffu, part, o);
      }
      const int found = part;  // t > 255 -> 0
      if (found < min_features) {
        thresh = __dmul_rn(thresh, 0.7);  // tooFew
        if (thresh < 2.0) thresh = 2.0;
        if (found == 0 && !checked) {
          checked = true;
          if (!mask_nonzero) break;
        }
      } else if (found > max_features) {
        thresh = __dmul_rn(thresh, 1.3);  // tooMany
        if (thresh > 10000.0) thresh = 10000.0;
        break;
      } else
        break;
      iter--;
    } while (iter > 0 && thresh > 2.0 && thresh < 10000.0);
    if (lane == 0) thr_out[fc] = used;
  }
  if (lane == 0) state[c] = thresh;
}

__global__ void __launch_bounds__(32 * kOrbMaxCells) k_adapt_thresholds(const int* __restrict__ hist, const int* __restrict__ cand_count,
                                                                         const int* __restrict__ mask_any, double* __restrict__ state,
                                                                         int* __restrict__ thr_out, int nframes, int ncells,
                                                                         int min_features, int max_features, int max_iters,
                                                                         int* __restrict__ err_flag, int cap) {
  adapt_thresholds<false>(hist, cand_count, mask_any, state, thr_out, nframes, ncells, min_features, max_features, max_iters,
                          err_flag, cap);
}

// The same recurrence on k_quota_counts' tables: ORB geometries whose per-cell maximum reaches cv::ORB's smallest quota.
__global__ void __launch_bounds__(32 * kOrbMaxCells) k_adapt_thresholds_quota(const int* __restrict__ table,
                                                                               const int* __restrict__ cand_count,
                                                                               const int* __restrict__ mask_any,
                                                                               double* __restrict__ state, int* __restrict__ thr_out,
                                                                               int nframes, int ncells, int min_features,
                                                                               int max_features, int max_iters,
                                                                               int* __restrict__ err_flag, int cap) {
  adapt_thresholds<true>(table, cand_count, mask_any, state, thr_out, nframes, ncells, min_features, max_features, max_iters,
                         err_flag, cap);
}

// The bare DetectorAdjuster (adjuster_max_iterations <= 0, features.cpp:101-112): every frame is detected once at the
// persistent threshold, which never changes.  One thread per (frame, cell); err_flag bit 0 as in adapt_thresholds.
__global__ void __launch_bounds__(256) k_fixed_thresholds(const int* __restrict__ cand_count, const double* __restrict__ state,
                                                          int* __restrict__ thr_out, int n, int ncells, int* __restrict__ err_flag,
                                                          int cap) {
  const int fc = blockIdx.x * blockDim.x + threadIdx.x;
  if (fc >= n) return;
  if (cand_count[fc] > cap) atomicOr(err_flag, 1);
  thr_out[fc] = (int)state[fc % ncells];
}

// HarrisResponses(img, pts, blockSize 7, k 0.04): Sobel-3 sums over 7x7, float formula evaluated in the same order
__device__ __forceinline__ float harris_response(const uint8_t* __restrict__ im, int w, int x0, int y0) {
  int a = 0, b = 0, c = 0;
  for (int dy = -3; dy <= 3; dy++) {
#pragma unroll
    for (int dx = -3; dx <= 3; dx++) {
      const uint8_t* p = im + (y0 + dy) * w + x0 + dx;
      const int Ix = (p[1] - p[-1]) * 2 + (p[-w + 1] - p[-w - 1]) + (p[w + 1] - p[w - 1]);
      const int Iy = (p[w] - p[-w]) * 2 + (p[w - 1] - p[-w - 1]) + (p[w + 1] - p[-w + 1]);
      a += Ix * Ix;
      b += Iy * Iy;
      c += Ix * Iy;
    }
  }
  const float scale = __fdiv_rn(1.f, 4.f * 7.f * 255.f);
  const float s4 = __fmul_rn(__fmul_rn(__fmul_rn(scale, scale), scale), scale);
  const float fa = (float)a, fb = (float)b, fc = (float)c;
  const float sum = __fadd_rn(fa, fb);
  const float r = __fsub_rn(__fsub_rn(__fmul_rn(fa, fb), __fmul_rn(fc, fc)), __fmul_rn(__fmul_rn(0.04f, sum), sum));
  return __fmul_rn(r, s4);
}

// cv::fastAtan2 (degrees)
__device__ __forceinline__ float fast_atan2_deg(float y, float x) {
  const float k = 57.29577951308232f;  // (float)(180/CV_PI)
  const float p1 = __fmul_rn(0.9997878412794807f, k), p3 = __fmul_rn(-0.3258083974640975f, k);
  const float p5 = __fmul_rn(0.1555786518463281f, k), p7 = __fmul_rn(-0.04432655554792128f, k);
  const float ax = fabsf(x), ay = fabsf(y);
  const float eps = 2.220446049250313e-16f;
  float a, c, c2;
  if (ax >= ay) {
    c = __fdiv_rn(ay, __fadd_rn(ax, eps));
    c2 = __fmul_rn(c, c);
    a = __fmul_rn(__fadd_rn(__fmul_rn(__fadd_rn(__fmul_rn(__fadd_rn(__fmul_rn(p7, c2), p5), c2), p3), c2), p1), c);
  } else {
    c = __fdiv_rn(ax, __fadd_rn(ay, eps));
    c2 = __fmul_rn(c, c);
    a = __fsub_rn(90.f, __fmul_rn(__fadd_rn(__fmul_rn(__fadd_rn(__fmul_rn(__fadd_rn(__fmul_rn(p7, c2), p5), c2), p3), c2), p1), c));
  }
  if (x < 0) a = __fsub_rn(180.f, a);
  if (y < 0) a = __fsub_rn(360.f, a);
  return a;
}

// IC_Angle: intensity-centroid orientation over the radius-15 disc; one warp per keypoint
__device__ float ic_angle_warp(const uint8_t* __restrict__ im, int w, int x0, int y0, int lane) {
  int m01 = 0, m10 = 0;
  const uint8_t* ctr = im + y0 * w + x0;
  if (lane < 31) m10 += (lane - 15) * ctr[lane - 15];  // v = 0 row
  for (int v = 1; v <= kOrbHalfPatch; v++) {
    const int d = c_umax[v];
    const int u = lane - d;  // lanes cover u = -d .. d (d <= 15 -> <= 31 lanes)
    if (u <= d) {
      const int vp = ctr[u + v * w], vm = ctr[u - v * w];
      m01 += v * (vp - vm);
      m10 += u * (vp + vm);
    }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    m01 += __shfl_xor_sync(0xffffffffu, m01, o);
    m10 += __shfl_xor_sync(0xffffffffu, m10, o);
  }
  return fast_atan2_deg((float)m01, (float)m10);
}

// Harris response for candidates with S >= the cell's final threshold; others get NaN (excluded).
__global__ void __launch_bounds__(256) k_harris(const uint8_t* __restrict__ cell_img, const OrbCand* __restrict__ cand,
                                                const int* __restrict__ cand_count, const int* __restrict__ thr,
                                                float* __restrict__ resp, int cap) {
  const int fc = blockIdx.y;
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  const int n = min(cand_count[fc], cap);
  if (i >= n) return;
  const OrbCand cd = cand[(size_t)fc * cap + i];
  float r = __int_as_float(0x7fc00000);
  if (cd.score >= thr[fc]) {
    const int f = fc / c_geom.ncells, c = fc % c_geom.ncells;
    const OrbPlane& p = c_geom.cell[c][cd.level];
    r = harris_response(cell_img + (size_t)f * c_geom.cell_bytes + p.off, p.w, cd.x, cd.y);
  }
  resp[(size_t)fc * cap + i] = r;
}

// FAST detector: a keypoint's response is its corner score S (cv::FAST); NaN below the cell's final threshold (excluded).
__global__ void __launch_bounds__(256) k_fast_response(const OrbCand* __restrict__ cand, const int* __restrict__ cand_count,
                                                       const int* __restrict__ thr, float* __restrict__ resp, int cap) {
  const int fc = blockIdx.y;
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  const int n = min(cand_count[fc], cap);
  if (i >= n) return;
  const int s = cand[(size_t)fc * cap + i].score;
  resp[(size_t)fc * cap + i] = s >= thr[fc] ? (float)s : __int_as_float(0x7fc00000);
}

__device__ __forceinline__ uint32_t f32_ordered(float f) {  // ascending unsigned order == ascending float order
  const uint32_t b = __float_as_uint(f);
  return (b & 0x80000000u) ? ~b : (b | 0x80000000u);
}

__device__ void bitonic_sort_u64(unsigned long long* keys, int N) {
  for (int k = 2; k <= N; k <<= 1) {
    for (int j = k >> 1; j > 0; j >>= 1) {
      for (int t = threadIdx.x; t < (N >> 1); t += blockDim.x) {
        const int lo = ((t & ~(j - 1)) << 1) | (t & (j - 1));
        const int hi = lo | j;
        const bool up = (lo & k) == 0;
        const unsigned long long a = keys[lo], b = keys[hi];
        if ((a > b) == up) {
          keys[lo] = b;
          keys[hi] = a;
        }
      }
      __syncthreads();
    }
  }
}

// A keypoint's position in k_cell_select's keys (bits 0-31): [level : 3][y : 12][x : 12] from bit 5 up, the sign of the
// response in bit 0.  Monotone in (level, y, x), so the keys of a cell sort by position after |response|.
struct CellPos {
  static constexpr int kBits = 12, kShift = 5;
  static constexpr uint32_t kCoord = (1u << kBits) - 1, kMask = (1u << (3 + 2 * kBits)) - 1;
  static_assert(kOrbMaxSide <= (int)kCoord && kShift + 3 + 2 * kBits <= 32, "a level coordinate must fit its field");
  __device__ static uint32_t pack(int level, int y, int x) {
    return (((uint32_t)level << (2 * kBits)) | ((uint32_t)y << kBits) | (uint32_t)x) << kShift;
  }
  __device__ static void unpack(unsigned long long key, int& level, int& y, int& x) {
    const uint32_t pos = (uint32_t)(key >> kShift) & kMask;
    level = pos >> (2 * kBits);
    y = (pos >> kBits) & kCoord;
    x = pos & kCoord;
  }
};

// Shared-memory histogram add with the lanes that hit the same bin merged (bin < 0: no add).  Called by whole warps.
__device__ __forceinline__ void hist_add_warp(int* h, int bin) {
  const unsigned peers = __match_any_sync(0xffffffffu, bin);
  if (bin >= 0 && (threadIdx.x & 31) == __ffs(peers) - 1) atomicAdd(&h[bin], __popc(peers));
}

// The count cv::ORB(10000, 1.2, 8, 15, 0, 2, HARRIS, 31, t).detect returns on a cell, for every t = 0..255, from the cell's
// threshold-free candidates and their Harris responses (resp, every candidate: k_harris with a threshold of 0).  With
// B_l(t) = {S >= max(t, s_l)}, s_l the 2 n_l-th largest score of level l (0 when it has fewer candidates: retainBest(2 n_l)
// does not cut), level l keeps q_l(t) = |B_l| when |B_l| <= n_l and otherwise the keypoints of B_l whose Harris response is
// at least the n_l-th largest of B_l (retainBest keeps ties); k_cell_select applies the same rule at one threshold.
// One CTA per (frame, cell, level): the level's score histogram gives s_l and every |B_l|; each warp then finds the n_l-th
// largest response of one B_l (radix select, 8 bits per pass, over the cell's candidates) for the thresholds in
// [s_l, u_hi], the ones where |B_l| > n_l.  table[fc * 256 + t] += q_l(t) (zeroed by the caller).
__global__ void __launch_bounds__(1024) k_quota_counts(const OrbCand* __restrict__ cand, const int* __restrict__ cand_count,
                                                       const float* __restrict__ resp, int cap, int* __restrict__ table) {
  __shared__ int s_n[256];  // the level's score histogram, then |{S >= u}|
  __shared__ int s_q[256];  // q_l(u) for u >= s_l
  __shared__ int s_wh[32][256];
  __shared__ int s_cut, s_hi;
  const int fc = blockIdx.x, l = blockIdx.y, t = threadIdx.x, warp = t >> 5, lane = t & 31;
  const int n = min(cand_count[fc], cap), nl = c_geom.n_per_level[l];
  const OrbCand* cc = cand + (size_t)fc * cap;
  const float* rr = resp + (size_t)fc * cap;
  if (t < 256) s_n[t] = 0;
  __syncthreads();
  for (int i = t; i < ((n + 31) & ~31); i += blockDim.x) {
    int bin = -1;
    if (i < n) {
      const OrbCand cd = cc[i];
      if (cd.level == l) bin = cd.score;
    }
    hist_add_warp(s_n, bin);
  }
  __syncthreads();
  if (t == 0) {
    int cum = 0, cut = -1;
    for (int u = 255; u >= 0; u--) {
      cum += s_n[u];
      s_n[u] = cum;
      if (cut < 0 && cum >= 2 * nl) cut = u;
    }
    if (cut < 0) cut = 0;
    int hi = cut - 1;
    while (hi < 255 && s_n[hi + 1] > nl) hi++;
    s_cut = cut;
    s_hi = hi;
  }
  __syncthreads();
  const int cut = s_cut, hi = s_hi;
  if (t < 256) s_q[t] = s_n[t];  // |B_l(u)| <= n_l above u_hi
  __syncthreads();
  int* wh = s_wh[warp];
  for (int v = cut + warp; v <= hi; v += 32) {
    uint32_t prefix = 0;
    int want = nl;
    for (int shift = 24; shift >= 0; shift -= 8) {
      for (int b = lane; b < 256; b += 32) wh[b] = 0;
      __syncwarp();
      const uint32_t mask = shift == 24 ? 0u : ~0u << (shift + 8);
      for (int i = lane; i < n; i += 32) {
        const OrbCand cd = cc[i];
        if (cd.level == l && cd.score >= v) {
          const uint32_t o = f32_ordered(rr[i] + 0.f);  // + 0.f: -0 ties +0, as k_cell_select
          if ((o & mask) == (prefix & mask)) atomicAdd(&wh[(o >> shift) & 255], 1);
        }
      }
      __syncwarp();
      if (lane == 0) {
        int cum = 0;
        for (int b = 255; b >= 0; b--) {
          if (cum + wh[b] >= want) {
            prefix |= (uint32_t)b << shift;
            want -= cum;
            break;
          }
          cum += wh[b];
        }
      }
      prefix = __shfl_sync(0xffffffffu, prefix, 0);
      want = __shfl_sync(0xffffffffu, want, 0);
      __syncwarp();
    }
    int q = 0;
    for (int i = lane; i < n; i += 32) {
      const OrbCand cd = cc[i];
      q += (cd.level == l && cd.score >= v && f32_ordered(rr[i] + 0.f) >= prefix) ? 1 : 0;
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) q += __shfl_xor_sync(0xffffffffu, q, o);
    if (lane == 0) s_q[v] = q;
  }
  __syncthreads();
  if (t < 256) {
    const int q = s_q[max(t, cut)];
    if (q) atomicAdd(&table[(size_t)fc * 256 + t], q);
  }
}

// keepStrongest(maxPerCell) by |response| (feature_adjuster.cpp:247-255; nth_element order is unspecified in the reference ->
// canonical tie rule: (level, y, x) ascending) of every grid cell at every frame size except those of k_cell_sort; a cell's
// valid candidates (cap per cell) can outnumber any shared-memory sort.  max_per_cell <= 1024 (orb_prepare: 1.5 K <= 4096 over
// >= 4 cells).
// quotas (ORB detector): first cv::ORB's per-level culls (orb.cpp computeKeyPoints, nfeatures 10000: c_geom.n_per_level),
//   retainBest(2 n_l) by FAST score, then retainBest(n_l) by Harris response; retainBest keeps every keypoint whose response
//   equals the n-th largest.  The adjuster's count is unaffected while max_per_cell < min n_l (DESIGN.md 4.5.5).
// Then keepStrongest: the max_per_cell smallest keys (|response| descending, then level, y, x) by an 8-bit radix select over
// the 64-bit keys (unique per cell), sorted in shared memory.  One CTA of 1024 threads per (frame, cell); every pass re-reads
// the cell's candidates (L2-resident).
// key = [~ordered(|resp|) : 32][CellPos : 27][0 : 4][sign : 1]
// kAll (k_cell_quota_all): no keepStrongest; every survivor of the quotas goes to cell_out, unsorted.
template <bool kAll>
__device__ __forceinline__ void cell_select(const OrbCand* __restrict__ cand, const int* __restrict__ cand_count,
                                            const float* __restrict__ resp, int cap, int quotas, int max_per_cell,
                                            unsigned long long* __restrict__ cell_out, int* __restrict__ cell_out_count,
                                            int out_stride) {
  __shared__ int hist[kOrbLevels * 256];
  __shared__ unsigned long long keys[1024];
  __shared__ int s_score_cut[kOrbLevels], s_want[kOrbLevels];
  __shared__ uint32_t s_resp_cut[kOrbLevels];
  __shared__ unsigned long long s_prefix;
  __shared__ int s_shift, s_done, s_n;
  const int fc = blockIdx.x;
  if (max_per_cell <= 0) {
    if (threadIdx.x == 0) cell_out_count[fc] = 0;
    return;
  }
  const int n = min(cand_count[fc], cap);
  const int n_warps = (n + 31) & ~31;  // loop bound for whole warps (hist_add_warp)
  const OrbCand* cc = cand + (size_t)fc * cap;
  const float* rr = resp + (size_t)fc * cap;
  const int t = threadIdx.x;
  // candidate i passes the per-level culls decided so far (all, until they are decided)
  auto survives = [&](int i, OrbCand& cd, float& r) -> bool {
    r = rr[i];
    if (!(r == r)) return false;
    cd = cc[i];
    if (!quotas) return true;
    return cd.score >= s_score_cut[cd.level] && f32_ordered(r + 0.f) >= s_resp_cut[cd.level];  // + 0.f: -0 ties +0
  };
  if (t < kOrbLevels) {
    s_score_cut[t] = 0;
    s_resp_cut[t] = 0;
  }
  if (quotas) {
    // retainBest(2 n_l) by FAST score: cut at the (2 n_l)-th largest score of the level
    for (int i = t; i < kOrbLevels * 256; i += blockDim.x) hist[i] = 0;
    __syncthreads();
    for (int i = t; i < n_warps; i += blockDim.x) {
      OrbCand cd;
      float r;
      const bool ok = i < n && survives(i, cd, r);
      hist_add_warp(hist, ok ? cd.level * 256 + cd.score : -1);
    }
    __syncthreads();
    if (t < kOrbLevels) {
      const int q = 2 * c_geom.n_per_level[t];
      int cum = 0, cut = 0, kept = 0;
      for (int s = 255; s >= 0; s--) {
        cum += hist[t * 256 + s];
        if (cum >= q) {
          cut = s;
          break;
        }
      }
      for (int s = cut; s < 256; s++) kept += hist[t * 256 + s];
      s_score_cut[t] = cut;
      // retainBest(n_l) by Harris response: radix select of the n_l-th largest ordered response (want < 0: nothing to cut)
      s_want[t] = kept > c_geom.n_per_level[t] ? c_geom.n_per_level[t] : -1;
    }
    __syncthreads();
    for (int shift = 24; shift >= 0; shift -= 8) {
      for (int i = t; i < kOrbLevels * 256; i += blockDim.x) hist[i] = 0;
      __syncthreads();
      const uint32_t hi = shift == 24 ? 0u : ~0u << (shift + 8);
      for (int i = t; i < n_warps; i += blockDim.x) {
        OrbCand cd;
        float r;
        int bin = -1;
        if (i < n && survives(i, cd, r) && s_want[cd.level] > 0) {
          const uint32_t o = f32_ordered(r + 0.f);
          if ((o & hi) == (s_resp_cut[cd.level] & hi)) bin = cd.level * 256 + ((o >> shift) & 255);
        }
        hist_add_warp(hist, bin);
      }
      __syncthreads();
      if (t < kOrbLevels && s_want[t] > 0) {
        int cum = 0;
        for (int b = 255; b >= 0; b--) {
          const int h = hist[t * 256 + b];
          if (cum + h >= s_want[t]) {
            s_resp_cut[t] |= (uint32_t)b << shift;  // survives() compares the full word only after the last pass
            s_want[t] -= cum;
            break;
          }
          cum += h;
        }
      }
      __syncthreads();
    }
    // s_resp_cut is now the n_l-th largest ordered response of each level that had one to cut, 0 (keep all) elsewhere
  }
  // keepStrongest(max_per_cell): radix select of the max_per_cell-th smallest key, 8 bits per pass from the top; a pass whose
  // boundary bin holds exactly the keys still wanted ends the select (every key is unique, so the last pass always does)
  auto key_of = [&](const OrbCand& cd, float r) -> unsigned long long {
    return ((unsigned long long)(~f32_ordered(fabsf(r))) << 32) | CellPos::pack(cd.level, cd.y, cd.x) | (r < 0.f ? 1ull : 0ull);
  };
  if constexpr (kAll) {
    if (t == 0) s_n = 0;
    __syncthreads();
    for (int i = t; i < n; i += blockDim.x) {
      OrbCand cd;
      float r;
      if (survives(i, cd, r)) cell_out[(size_t)fc * out_stride + atomicAdd(&s_n, 1)] = key_of(cd, r);
    }
    __syncthreads();
    if (t == 0) cell_out_count[fc] = s_n;
    return;
  }
  if (t == 0) {
    s_prefix = 0;
    s_shift = 64;
    s_done = 0;
    s_want[0] = max_per_cell;
    s_n = 0;
  }
  __syncthreads();
  for (int shift = 56; shift >= 0; shift -= 8) {
    for (int i = t; i < 256; i += blockDim.x) hist[i] = 0;
    __syncthreads();
    const unsigned long long hi = shift == 56 ? 0ull : ~0ull << (shift + 8), prefix = s_prefix;
    for (int i = t; i < n_warps; i += blockDim.x) {
      OrbCand cd;
      float r;
      int bin = -1;
      if (i < n && survives(i, cd, r)) {
        const unsigned long long k = key_of(cd, r);
        if ((k & hi) == (prefix & hi)) bin = (int)((k >> shift) & 255);
      }
      hist_add_warp(hist, bin);
    }
    __syncthreads();
    if (t == 0) {
      int cum = 0, b = 0;
      for (; b < 256; b++) {
        if (cum + hist[b] >= s_want[0]) break;
        cum += hist[b];
      }
      if (b == 256) {  // fewer survivors than max_per_cell (first pass only): keep them all
        s_prefix = ~0ull;
        s_shift = 0;
        s_done = 1;
      } else {
        s_prefix |= (unsigned long long)b << shift;
        s_want[0] -= cum;
        if (hist[b] == s_want[0]) {
          s_shift = shift;
          s_done = 1;
        }
      }
    }
    __syncthreads();
    if (s_done) break;
  }
  const int sel_shift = s_shift;  // < 64: the last pass always ends the select
  const unsigned long long sel = s_prefix >> sel_shift;
  for (int i = t; i < n; i += blockDim.x) {
    OrbCand cd;
    float r;
    if (survives(i, cd, r)) {
      const unsigned long long k = key_of(cd, r);
      if ((k >> sel_shift) <= sel) keys[atomicAdd(&s_n, 1)] = k;
    }
  }
  __syncthreads();
  const int cnt = s_n;
  int N = 2;
  while (N < cnt) N <<= 1;
  for (int i = cnt + t; i < N; i += blockDim.x) keys[i] = ~0ull;
  __syncthreads();
  bitonic_sort_u64(keys, N);
  for (int i = t; i < cnt; i += blockDim.x) cell_out[(size_t)fc * out_stride + i] = keys[i];
  if (t == 0) cell_out_count[fc] = cnt;
}

__global__ void __launch_bounds__(1024) k_cell_select(const OrbCand* __restrict__ cand, const int* __restrict__ cand_count,
                                                      const float* __restrict__ resp, int cap, int quotas, int max_per_cell,
                                                      unsigned long long* __restrict__ cell_out, int* __restrict__ cell_out_count,
                                                      int out_stride) {
  cell_select<false>(cand, cand_count, resp, cap, quotas, max_per_cell, cell_out, cell_out_count, out_stride);
}

// The same keepStrongest for cells without quotas (FAST) and with at most kOrbCandCap candidates: every valid key sorted in
// kCellSortBytes of dynamic shared memory.  At 640x480 this is faster than k_cell_select's radix passes (0.63 against
// 1.03 us per frame on an H100, DESIGN.md 4.5.1) and keeps the same keys, as the keys of a cell are unique.
constexpr int kCellSortBytes = 16384 * 8;  // the next power of two above kOrbCandCap keys
__global__ void __launch_bounds__(1024) k_cell_sort(const OrbCand* __restrict__ cand, const int* __restrict__ cand_count,
                                                    const float* __restrict__ resp, int cap, int max_per_cell,
                                                    unsigned long long* __restrict__ cell_out, int* __restrict__ cell_out_count,
                                                    int out_stride) {
  extern __shared__ unsigned long long keys[];
  __shared__ int s_n;
  const int fc = blockIdx.x;
  const int n = min(cand_count[fc], cap);
  if (threadIdx.x == 0) s_n = 0;
  __syncthreads();
  for (int i = threadIdx.x; i < n; i += blockDim.x) {
    const float r = resp[(size_t)fc * cap + i];
    if (r == r) {
      const OrbCand cd = cand[(size_t)fc * cap + i];
      keys[atomicAdd(&s_n, 1)] =
          ((unsigned long long)(~f32_ordered(fabsf(r))) << 32) | CellPos::pack(cd.level, cd.y, cd.x) | (r < 0.f ? 1ull : 0ull);
    }
  }
  __syncthreads();
  const int cnt = s_n;
  int N = 2;
  while (N < cnt) N <<= 1;
  for (int i = cnt + threadIdx.x; i < N; i += blockDim.x) keys[i] = ~0ull;
  __syncthreads();
  bitonic_sort_u64(keys, N);
  const int keep = min(cnt, max_per_cell);
  for (int i = threadIdx.x; i < keep; i += blockDim.x) cell_out[(size_t)fc * out_stride + i] = keys[i];
  if (threadIdx.x == 0) cell_out_count[fc] = keep;
}

// Whole-frame detectors (one cell, up to kOrbNarrowMax px): cv::ORB's quotas (quotas != 0) or none (FAST), no keepStrongest;
// out_stride >= cap.  k_frame_precap then caps each frame's survivors for k_frame_finalize.
__global__ void __launch_bounds__(1024) k_cell_quota_all(const OrbCand* __restrict__ cand, const int* __restrict__ cand_count,
                                                         const float* __restrict__ resp, int cap, int quotas,
                                                         unsigned long long* __restrict__ cell_out, int* __restrict__ cell_out_count,
                                                         int out_stride) {
  cell_select<true>(cand, cand_count, resp, cap, quotas, 1, cell_out, cell_out_count, out_stride);
}

// -------------------------------------------------------------------------------------------------
// Per frame: aggregate the cells (feature_adjuster.cpp:259-282), removeDepthless (node.cpp:67-97), retainBest(K)
// (node.cpp:187-191), the extractor's border filter + octave sort (cv::ORB::compute), orientation, projectTo3D
// (node.cpp:900-965).  mode 0: stop after aggregation (== detector->detect output, with angles);
// mode 1: full Node constructor.
struct FrameKp {
  float x, y, resp;
  uint16_t lx, ly;  // level coordinates inside the cell pyramid
  uint8_t level, cell;
  uint16_t flag;
};
struct FrameKpZ : FrameKp {  // use_feature_min_depth: the keypoint carries its neighbourhood depth (k_min_depth)
  float z;
};
template <OrbPoints P>
using FrameKpOf = std::conditional_t<P == OrbPoints::kMinDepth, FrameKpZ, FrameKp>;
// k_min_depth, k_frame_finalize and k_frame_emit take their buffers in one OrbFrameArgs.  Members of a struct cannot be
// __restrict__, so each kernel reads through __restrict__ locals, and k_frame_finalize, where that is not enough, through
// __ldg: the loads keep the read-only path they had when the buffers were __restrict__ kernel parameters.
constexpr int kFrameCap = 4096;  // >= ncells * max_per_cell
static_assert(kFrameCap == kOrbFrameCap && sizeof(FrameKpZ) == kOrbFrameKpBytes && sizeof(FrameKp) <= sizeof(FrameKpZ),
              "orb_host.h sizes the finalize scratch");

// -------------------------------------------------------------------------------------------------
// use_feature_min_depth (parameter_server.cpp:90): Z = getMinDepthInNeighborhood(depth, kp.pt, kp.size) (misc.cpp:774-791) for
// every keepStrongest survivor of every frame, in place of depth(round(y), round(x)) -- removeDepthless (node.cpp:82-83) and
// projectTo3D (:940-941) both read it.  The keypoint is the one k_frame_finalize / k_frame_emit will build: image coordinates
// from the cell pyramid, size 31 * scale (ORB) or 7 (FAST).  radius = int((size - 1) / 2); the window is the half-open
// [int(y - r), int(y + r)) x [int(x - r), int(x + r)) of the raw depth image (float arithmetic, truncation toward zero),
// clamped to the image -- 2r x 2r, not centred.  Z = the minimum over the window, NaN pixels ignored (fminf), NaN when the
// window holds no number or its minimum is 0 (the reference's FIXME branch; -0 == 0).  One warp per candidate, lanes stride
// the columns of each window row.  cand_z[fc * out_stride + i] pairs with cell_out[fc * out_stride + i].
__global__ void __launch_bounds__(256) k_min_depth(OrbFrameArgs a, int fast) {
  const unsigned long long* __restrict__ cell_out = a.cell_out;
  const int* __restrict__ cell_out_count = a.cell_out_count;
  const float* __restrict__ depth = a.depth;
  float* __restrict__ cand_z = a.cand_z;
  const int fc = blockIdx.y;
  const int i = blockIdx.x * 8 + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (i >= cell_out_count[fc]) return;
  const int W = c_geom.W, H = c_geom.H;
  const int f = fc / c_geom.ncells, c = fc % c_geom.ncells;
  int level, ly, lx;
  CellPos::unpack(cell_out[(size_t)fc * a.out_stride + i], level, ly, lx);
  const float sc = c_geom.cell[c][level].scale;
  const float x = __fadd_rn(__fmul_rn((float)lx, sc), (float)c_geom.cell_x0[c]);  // as k_frame_finalize
  const float y = __fadd_rn(__fmul_rn((float)ly, sc), (float)c_geom.cell_y0[c]);
  const float size = fast ? 7.f : __fmul_rn(31.f, sc);  // as k_frame_emit
  const float r = (float)__float2int_rz(__fdiv_rn(__fsub_rn(size, 1.f), 2.f));
  const int top = max(__float2int_rz(__fsub_rn(y, r)), 0), left = max(__float2int_rz(__fsub_rn(x, r)), 0);
  const int bot = min(__float2int_rz(__fadd_rn(y, r)), H), right = min(__float2int_rz(__fadd_rn(x, r)), W);
  const float* d = depth + (size_t)f * W * H;
  float m = __int_as_float(0x7fc00000);
  for (int yy = top; yy < bot; yy++)
    for (int xx = left + lane; xx < right; xx += 32) m = fminf(m, d[(size_t)yy * W + xx]);
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) m = fminf(m, __shfl_xor_sync(0xffffffffu, m, o));
  if (lane == 0) cand_z[(size_t)fc * a.out_stride + i] = m == 0.f ? __int_as_float(0x7fc00000) : m;
}

// mode 0: detector output, cell-major, inside a cell |response| descending (canonical stand-in for the unspecified
//         nth_element order), ties by (level, y, x).
// mode 1: Node constructor: removeDepthless -> retainBest(K) by signed response (ties canonical, cut at K) ->
//         extractor border filter (31 px on cvRound'ed coordinates) -> stable sort by octave -> orientation ->
//         projectTo3D.  Final order = (octave, response descending, cell, level, y, x).
// The point source P (mode 1 only; mode 0 is OrbPoints::kDepthPixel):
// kDepthPixel: removeDepthless tests the depth pixel at the rounded position.
// kMinDepth (use_feature_min_depth): removeDepthless tests k_min_depth's Z of the keypoint (cand_z, aligned with cell_out)
// instead of the depth pixel, and the record carries Z on to k_frame_emit's projectTo3D.
// kCloud: the point-cloud constructor (node.cpp:252-369).  No removeDepthless and no retainBest: projectTo3D
// (:855-898) walks the detector output in its order (mode 0's) and keeps a keypoint when the organised cloud's point at the
// truncated position ((int)x, (int)y) has no NaN coordinate, up to max_keypoints kept; then compute()'s border filter and
// octave sort.  Final order = (octave, cell, |response| descending, y, x).  maximum_depth is fixed at its default, +inf, so
// the reference's z > maximum_depth test never drops a point.  `depth` is the cloud, cloud_stride floats per point.
template <OrbPoints P>
__global__ void __launch_bounds__(1024) k_frame_finalize(OrbFrameArgs a) {
  using Kp = FrameKpOf<P>;
  const int mode = P == OrbPoints::kDepthPixel ? a.mode : 1;
  const int W = c_geom.W, H = c_geom.H, out_stride = a.out_stride;
  __shared__ unsigned long long keys[kFrameCap];
  __shared__ int s_n, s_m;
  const int f = blockIdx.x;
  Kp* ka = reinterpret_cast<Kp*>(a.scratch) + (size_t)f * 2 * kFrameCap;  // gather order
  Kp* kc = ka + kFrameCap;                                                // canonical order
  if (threadIdx.x == 0) { s_n = 0; s_m = 0; }
  __syncthreads();
  // A. gather, shift to image coordinates (pt *= scale; pt += cell origin: feature_adjuster.cpp:259-282), depth check
  for (int c = 0; c < c_geom.ncells; c++) {
    const int fc = f * c_geom.ncells + c;
    const int n = __ldg(&a.cell_out_count[fc]);
    for (int i = threadIdx.x; i < n; i += blockDim.x) {
      const unsigned long long k = __ldg(&a.cell_out[(size_t)fc * out_stride + i]);
      int level, ly, lx;
      CellPos::unpack(k, level, ly, lx);
      const uint32_t ord = ~(uint32_t)(k >> 32);
      float r = __uint_as_float(ord & 0x7FFFFFFFu);  // |resp| (ordered() of a non-negative float only sets bit 31)
      if (k & 1ull) r = -r;
      const float sc = c_geom.cell[c][level].scale;
      Kp q;
      q.x = __fadd_rn(__fmul_rn((float)lx, sc), (float)c_geom.cell_x0[c]);
      q.y = __fadd_rn(__fmul_rn((float)ly, sc), (float)c_geom.cell_y0[c]);
      q.resp = r;
      q.lx = (uint16_t)lx;
      q.ly = (uint16_t)ly;
      q.level = (uint8_t)level;
      q.cell = (uint8_t)c;
      q.flag = 0;
      bool ok = true;
      if (P != OrbPoints::kCloud && mode == 1) {  // removeDepthless (node.cpp:67-97)
        ok = !(q.x >= W || q.x < 0 || q.y >= H || q.y < 0);
        if constexpr (P == OrbPoints::kMinDepth) {
          q.z = __ldg(&a.cand_z[(size_t)fc * out_stride + i]);  // getMinDepthInNeighborhood (node.cpp:82-83)
          ok = ok && !(q.z != q.z);
        } else if (ok) {
          const int rx = (int)floorf(q.x + 0.5f), ry = (int)floorf(q.y + 0.5f);  // round(): half away from zero
          const size_t idx = (size_t)ry * W + rx;
          const float Z = idx < (size_t)W * H ? __ldg(&a.depth[(size_t)f * W * H + idx]) : __int_as_float(0x7fc00000);
          ok = !(Z != Z);
        }
      }
      if (ok) {
        const int slot = atomicAdd(&s_n, 1);
        if (slot < kFrameCap) ka[slot] = q;
      }
    }
  }
  __syncthreads();
  const int cnt = min(s_n, kFrameCap);
  int N = 2;
  while (N < cnt) N <<= 1;
  // B. canonical order (cell, level, y, x)
  for (int i = threadIdx.x; i < N; i += blockDim.x) {
    unsigned long long k = ~0ull;
    if (i < cnt) {
      const Kp q = ka[i];
      const unsigned long long canon = ((unsigned long long)q.cell << 27) | ((unsigned long long)q.level << 24) |
                                       ((unsigned long long)q.ly << 12) | q.lx;
      k = (canon << 16) | (unsigned)i;
    }
    keys[i] = k;
  }
  __syncthreads();
  bitonic_sort_u64(keys, N);
  for (int r = threadIdx.x; r < cnt; r += blockDim.x) kc[r] = ka[keys[r] & 0xFFFFu];
  __threadfence_block();
  __syncthreads();
  int n_final = cnt;
  if (mode == 1) {
    int keepK;
    if constexpr (P == OrbPoints::kCloud) {
      // C'. projectTo3D (node.cpp:870-896) in detector order (mode 0's key below); keypoints outside the image or whose cloud
      //     point has a NaN coordinate get bit 63 and sort behind every kept one; cut at K kept
      static_assert(kOrbMaxCells <= 128, "the cell (bits 56-62) must stay below the invalid flag (bit 63)");
      __shared__ int s_v;
      if (threadIdx.x == 0) s_v = 0;
      __syncthreads();
      for (int r = threadIdx.x; r < N; r += blockDim.x) {
        unsigned long long k = ~0ull;
        if (r < cnt) {
          const Kp q = kc[r];
          bool ok = !(q.x >= W || q.x < 0 || q.y >= H || q.y < 0 || q.x != q.x || q.y != q.y);
          if (ok) {
            const float* p = a.depth + ((size_t)f * W * H + (size_t)__float2int_rz(q.y) * W + __float2int_rz(q.x)) * a.cloud_stride;
            const float px = __ldg(p), py = __ldg(p + 1), pz = __ldg(p + 2);
            ok = !(px != px || py != py || pz != pz);
          }
          if (ok) atomicAdd(&s_v, 1);
          k = ((unsigned long long)!ok << 63) | ((unsigned long long)q.cell << 56) |
              ((unsigned long long)(~f32_ordered(fabsf(q.resp))) << 16) | (unsigned)r;
        }
        keys[r] = k;
      }
      __syncthreads();
      bitonic_sort_u64(keys, N);
      keepK = min(s_v, a.max_keypoints);
    } else {
      // C. retainBest(max_keypoints) (node.cpp:187-191): signed response descending, ties canonical, cut at K
      for (int r = threadIdx.x; r < N; r += blockDim.x)
        keys[r] = r < cnt ? (((unsigned long long)(~f32_ordered(kc[r].resp)) << 32) | (unsigned)r) : ~0ull;
      __syncthreads();
      bitonic_sort_u64(keys, N);
      keepK = min(cnt, a.max_keypoints);
    }
    // D. extractor->compute(): runByImageBorder(31) on cvRound'ed coordinates, then stable sort by octave
    unsigned long long mine[4];  // up to 4 keys per thread (kFrameCap / 1024)
    int nm = 0;
    for (int j = threadIdx.x; j < N; j += blockDim.x) {
      unsigned long long k2 = ~0ull;
      if (j < keepK) {
        const int r = (int)(keys[j] & 0xFFFFu);
        const Kp q = kc[r];
        const int rx = __float2int_rn(q.x), ry = __float2int_rn(q.y);
        if (rx >= 31 && rx < W - 31 && ry >= 31 && ry < H - 31) {
          k2 = ((unsigned long long)q.level << 40) | ((unsigned long long)j << 16) | (unsigned)r;
          atomicAdd(&s_m, 1);
        }
      }
      mine[nm++] = k2;
    }
    __syncthreads();
    nm = 0;
    for (int j = threadIdx.x; j < N; j += blockDim.x) keys[j] = mine[nm++];
    __syncthreads();
    bitonic_sort_u64(keys, N);
    n_final = s_m;
  } else {
    for (int r = threadIdx.x; r < N; r += blockDim.x) {
      unsigned long long k = ~0ull;
      if (r < cnt) {
        const Kp q = kc[r];
        k = ((unsigned long long)q.cell << 56) | ((unsigned long long)(~f32_ordered(fabsf(q.resp))) << 16) | (unsigned)r;
      }
      keys[r] = k;
    }
    __syncthreads();
    bitonic_sort_u64(keys, N);
  }
  // E. hand the final order to k_frame_emit (one warp per keypoint across the whole grid: orientation, cv::KeyPoint,
  //    projectTo3D); the gather-order half of the scratch is free by now and receives the 16-bit indices into kc
  uint16_t* ord = reinterpret_cast<uint16_t*>(ka);
  for (int t = threadIdx.x; t < n_final; t += blockDim.x) ord[t] = (uint16_t)(keys[t] & 0xFFFFu);
  if (threadIdx.x == 0) a.n_out[f] = n_final;
}

template __global__ void k_frame_finalize<OrbPoints::kDepthPixel>(OrbFrameArgs);
template __global__ void k_frame_finalize<OrbPoints::kMinDepth>(OrbFrameArgs);
template __global__ void k_frame_finalize<OrbPoints::kCloud>(OrbFrameArgs);

// Whole-frame detectors return up to about 10^4 keypoints (ORB) or more (FAST), k_frame_finalize holds kFrameCap.  Per frame
// (one cell), from k_cell_quota_all's survivors src[f * src_stride ...] (and, kMinDepth, their depths src_z), this keeps the
// kFrameCap first of the keypoints k_frame_finalize would keep, in the order of its cut at max_keypoints: mode 1 the
// removeDepthless / cloud test of its step A, then signed response descending (retainBest) or, kCloud, |response| descending
// (the detector order projectTo3D walks), ties by (level, y, x).  max_keypoints <= 2730 < kFrameCap, so finalize's result is
// unchanged.  Mode 0 (the detector output itself) cannot be cut: more than kFrameCap keypoints sets err_flag bit 1.  The
// kept keys (and depths) go to a.cell_out (a.cand_z) at stride a.out_stride; radix select of the kFrameCap-th smallest
// order key as in k_cell_select.
template <OrbPoints P>
__global__ void __launch_bounds__(1024) k_frame_precap(OrbFrameArgs a, const unsigned long long* __restrict__ src,
                                                       const int* __restrict__ src_count, const float* __restrict__ src_z,
                                                       int src_stride, int* __restrict__ err_flag) {
  __shared__ int hist[256];
  __shared__ unsigned long long s_prefix;
  __shared__ int s_shift, s_done, s_want, s_n;
  const int mode = P == OrbPoints::kDepthPixel ? a.mode : 1;
  const int f = blockIdx.x, t = threadIdx.x, W = c_geom.W, H = c_geom.H;
  const int n = src_count[f];
  const unsigned long long* sk = src + (size_t)f * src_stride;
  if (mode == 0 && n > kFrameCap) {
    if (t == 0) {
      atomicOr(err_flag, 2);
      a.cell_out_count[f] = 0;
    }
    return;
  }
  // order key of survivor i, ~0 when k_frame_finalize's step A would drop it
  auto order = [&](int i) -> unsigned long long {
    const unsigned long long k = sk[i];
    if (mode == 0) return k;
    int level, ly, lx;
    CellPos::unpack(k, level, ly, lx);
    const float sc = c_geom.cell[0][level].scale;
    const float x = __fadd_rn(__fmul_rn((float)lx, sc), (float)c_geom.cell_x0[0]);
    const float y = __fadd_rn(__fmul_rn((float)ly, sc), (float)c_geom.cell_y0[0]);
    bool ok = !(x >= W || x < 0 || y >= H || y < 0);
    if constexpr (P == OrbPoints::kMinDepth) {
      const float z = src_z[(size_t)f * src_stride + i];
      ok = ok && !(z != z);
    } else if constexpr (P == OrbPoints::kCloud) {
      if (ok) {
        const float* p = a.depth + ((size_t)f * W * H + (size_t)__float2int_rz(y) * W + __float2int_rz(x)) * a.cloud_stride;
        ok = !(p[0] != p[0] || p[1] != p[1] || p[2] != p[2]);
      }
    } else if (ok) {
      const int rx = (int)floorf(x + 0.5f), ry = (int)floorf(y + 0.5f);
      const size_t idx = (size_t)ry * W + rx;
      ok = idx < (size_t)W * H && !(a.depth[(size_t)f * W * H + idx] != a.depth[(size_t)f * W * H + idx]);
    }
    if (!ok) return ~0ull;
    const uint32_t ord = ~(uint32_t)(k >> 32);  // ordered |response|
    float r = __uint_as_float(ord & 0x7FFFFFFFu);
    if (P != OrbPoints::kCloud && (k & 1ull)) r = -r;
    return ((unsigned long long)(~f32_ordered(r)) << 32) | CellPos::pack(level, ly, lx);
  };
  if (t == 0) {
    s_prefix = 0;
    s_shift = 64;
    s_done = 0;
    s_want = kFrameCap;
    s_n = 0;
  }
  __syncthreads();
  for (int shift = 56; shift >= 0; shift -= 8) {
    for (int i = t; i < 256; i += blockDim.x) hist[i] = 0;
    __syncthreads();
    const unsigned long long hi = shift == 56 ? 0ull : ~0ull << (shift + 8), prefix = s_prefix;
    for (int i = t; i < ((n + 31) & ~31); i += blockDim.x) {
      int bin = -1;
      if (i < n) {
        const unsigned long long k = order(i);
        if (k != ~0ull && (k & hi) == (prefix & hi)) bin = (int)((k >> shift) & 255);
      }
      hist_add_warp(hist, bin);
    }
    __syncthreads();
    if (t == 0) {
      int cum = 0, b = 0;
      for (; b < 256; b++) {
        if (cum + hist[b] >= s_want) break;
        cum += hist[b];
      }
      if (b == 256) {  // at most kFrameCap kept (first pass only): all of them
        s_prefix = ~0ull;
        s_shift = 0;
        s_done = 1;
      } else {
        s_prefix |= (unsigned long long)b << shift;
        s_want -= cum;
        if (hist[b] == s_want) {
          s_shift = shift;
          s_done = 1;
        }
      }
    }
    __syncthreads();
    if (s_done) break;
  }
  const int sel_shift = s_shift;
  const unsigned long long sel = s_prefix >> sel_shift;
  for (int i = t; i < n; i += blockDim.x) {
    const unsigned long long k = order(i);
    if (k != ~0ull && (k >> sel_shift) <= sel) {
      const int slot = atomicAdd(&s_n, 1);
      a.cell_out[(size_t)f * a.out_stride + slot] = sk[i];
      if constexpr (P == OrbPoints::kMinDepth) a.cand_z[(size_t)f * a.out_stride + slot] = src_z[(size_t)f * src_stride + i];
    }
  }
  __syncthreads();
  if (t == 0) a.cell_out_count[f] = s_n;
}

// One warp per output keypoint: intensity-centroid orientation on the detector's (cell) pyramid, the cv::KeyPoint record,
// in mode 1 projectTo3D (node.cpp:900-965) + backProject (misc2.h:49-65) and the rotation (cos, sin) compute() will use.
// Detector FAST: cv::FAST's KeyPoint(x, y, 7.f, -1, score) -- no orientation; compute() steers the pattern by the angle as
// given, -1.
// kMinDepth: projectTo3D takes the keypoint's neighbourhood depth that k_frame_finalize carried over from k_min_depth
// (node.cpp:940-941) instead of the depth pixel.
// kCloud: the point is the cloud's (x, y, z, 1) at ((int)x, (int)y) as stored (node.cpp:880-889), no back-projection;
// `depth` is the cloud, cloud_stride floats per point.
template <int Detector, OrbPoints P>
__global__ void __launch_bounds__(256) k_frame_emit(OrbFrameArgs a) {
  using Kp = FrameKpOf<P>;
  constexpr bool kFast = Detector == RGBDSLAM_B200_DETECTOR_FAST;
  const int mode = P == OrbPoints::kDepthPixel ? a.mode : 1;
  const void* __restrict__ scratch = a.scratch;
  const uint8_t* __restrict__ cell_img = a.cell_img;
  const float* __restrict__ depth = a.depth;
  rgbdslam_b200_keypoint* __restrict__ kp_out = a.kp_out;
  float4* __restrict__ xyz_out = a.xyz_out;
  float2* __restrict__ trig_out = a.trig_out;
  const int* __restrict__ n_out = a.n_out;
  const int kp_stride = a.kp_stride;
  const int f = blockIdx.y;
  const int t = blockIdx.x * 8 + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (t >= n_out[f]) return;
  const int W = c_geom.W, H = c_geom.H;
  const Kp* ka = reinterpret_cast<const Kp*>(scratch) + (size_t)f * 2 * kFrameCap;
  const Kp q = (ka + kFrameCap)[reinterpret_cast<const uint16_t*>(ka)[t]];
  const OrbPlane& p = c_geom.cell[q.cell][q.level];
  float ang = -1.f;
  if constexpr (!kFast) ang = ic_angle_warp(cell_img + (size_t)f * c_geom.cell_bytes + p.off, p.w, q.lx, q.ly, lane);
  if (lane == 0) {
    rgbdslam_b200_keypoint o;
    o.x = q.x;
    o.y = q.y;
    o.size = kFast ? 7.f : __fmul_rn(31.f, p.scale);
    o.angle = ang;
    o.response = q.resp;
    o.octave = q.level;
    o.class_id = -1;
    kp_out[(size_t)f * kp_stride + t] = o;
    if (mode == 1) {
      float4 v;
      if constexpr (P == OrbPoints::kCloud) {
        const float* p = depth + ((size_t)f * W * H + (size_t)__float2int_rz(q.y) * W + __float2int_rz(q.x)) * a.cloud_stride;
        v = make_float4(p[0], p[1], p[2], 1.f);
      } else {
        float d;
        if constexpr (P == OrbPoints::kMinDepth) {
          d = q.z;
        } else {
          const int rx = (int)floorf(q.x + 0.5f), ry = (int)floorf(q.y + 0.5f);
          d = depth[(size_t)f * W * H + (size_t)ry * W + rx];
        }
        const float Z = (float)((double)d * (double)a.depth_scaling);
        v.x = __fmul_rn(__fmul_rn(__fsub_rn(q.x, a.Kinv.z), Z), a.Kinv.x);
        v.y = __fmul_rn(__fmul_rn(__fsub_rn(q.y, a.Kinv.w), Z), a.Kinv.y);
        v.z = Z;
        v.w = 1.f;
      }
      xyz_out[(size_t)f * kp_stride + t] = v;
      if (trig_out) {  // angle *= (float)(CV_PI/180.f); a = (float)cos(angle), b = (float)sin(angle)  (cv::ORB computeOrbDescriptors)
        const float ar = __fmul_rn(ang, 0.017453292519943295f);
        trig_out[(size_t)f * kp_stride + t] = make_float2((float)cos((double)ar), (float)sin((double)ar));
      }
    }
  }
}

template __global__ void k_frame_emit<RGBDSLAM_B200_DETECTOR_ORB, OrbPoints::kDepthPixel>(OrbFrameArgs);
template __global__ void k_frame_emit<RGBDSLAM_B200_DETECTOR_FAST, OrbPoints::kDepthPixel>(OrbFrameArgs);
template __global__ void k_frame_emit<RGBDSLAM_B200_DETECTOR_ORB, OrbPoints::kMinDepth>(OrbFrameArgs);
template __global__ void k_frame_emit<RGBDSLAM_B200_DETECTOR_FAST, OrbPoints::kMinDepth>(OrbFrameArgs);
template __global__ void k_frame_emit<RGBDSLAM_B200_DETECTOR_ORB, OrbPoints::kCloud>(OrbFrameArgs);
template __global__ void k_frame_emit<RGBDSLAM_B200_DETECTOR_FAST, OrbPoints::kCloud>(OrbFrameArgs);

// -------------------------------------------------------------------------------------------------
// GaussianBlur(level, 7x7, sigma 2, BORDER_REFLECT_101) as OpenCV evaluates it inside ORB: separable float filter,
// row pass accumulated left to right, column pass symmetric, round-half-even to uint8.  The multiply-adds are fused, as
// cv2 4.13's SIMD row and column filters compute them on x86-64 with FMA (RowVec_8u32f, SymmColumnVec_32f8u: v_muladd),
// except in the row pass of the columns past the last whole 32-column block, which cv2's row filter leaves to its scalar
// loop: there each product and sum is rounded.  Either rule alone differs from cv2 at a few pixels per million (DESIGN.md
// 4.5.5).
__device__ __forceinline__ int reflect101(int i, int n) {
  if (i < 0) i = -i;
  if (i >= n) i = 2 * n - 2 - i;
  return i;
}

__global__ void __launch_bounds__(256) k_blur(const uint8_t* __restrict__ src, uint8_t* __restrict__ dst, int frame_stride,
                                              int level) {
  const OrbPlane& p = c_geom.full[level];
  const int f = blockIdx.z;
  const int pw = p.w, ph = p.h;
  __shared__ float tile[22][40];  // 16 output rows + 6 halo rows, 32 output columns + 6 halo columns, as float (reflect-101 applied)
  __shared__ float rows[22][32];  // row-pass results
  const uint8_t* im = src + (size_t)f * frame_stride + p.off;
  const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;  // 32 x 8
  const int x0 = blockIdx.x * 32, y0 = blockIdx.y * 16;
  for (int i = threadIdx.x; i < 22 * 38; i += 256) {
    const int r = i / 38, c = i - r * 38;
    const int xx = reflect101(min(x0 + c - 3, pw + 2), pw), yy = reflect101(min(y0 + r - 3, ph + 2), ph);
    tile[r][c] = (float)im[yy * pw + xx];
  }
  __syncthreads();
  const bool row_tail = x0 + 32 > pw;  // the columns past the level's last whole 32-column block
  for (int r = ty; r < 22; r += 8) {
    float acc = 0.f;
    if (row_tail) {
#pragma unroll
      for (int j = 0; j < 7; j++) acc = __fadd_rn(acc, __fmul_rn(c_gauss[j], tile[r][tx + j]));
    } else {
#pragma unroll
      for (int j = 0; j < 7; j++) acc = __fmaf_rn(c_gauss[j], tile[r][tx + j], acc);  // left to right, as cv::sepFilter2D
    }
    rows[r][tx] = acc;
  }
  __syncthreads();
  const int x = x0 + tx;
  for (int r = ty; r < 16; r += 8) {
    const int y = y0 + r;
    if (x < pw && y < ph) {
      float c = __fmul_rn(c_gauss[3], rows[r + 3][tx]);
#pragma unroll
      for (int j = 1; j <= 3; j++) {
        const float pair = __fadd_rn(rows[r + 3 + j][tx], rows[r + 3 - j][tx]);
        c = __fmaf_rn(c_gauss[3 + j], pair, c);
      }
      int v = __float2int_rn(c);
      v = min(max(v, 0), 255);
      dst[(size_t)f * frame_stride + p.off + (size_t)y * pw + x] = (uint8_t)v;
    }
  }
}

// rBRIEF: one warp per keypoint, lane j produces descriptor byte j (8 tests).  Pixels outside the level are read
// from the UNBLURRED level with reflect-101 (OpenCV blurs only the level ROI of its bordered pyramid buffer).
__global__ void __launch_bounds__(256) k_describe(const uint8_t* __restrict__ pyr_raw, const uint8_t* __restrict__ pyr_blur,
                                                  int frame_stride, const rgbdslam_b200_keypoint* __restrict__ kps,
                                                  const int* __restrict__ n_kp, int kp_stride, const float2* __restrict__ trig,
                                                  uint8_t* __restrict__ desc) {
  const int f = blockIdx.y;
  const int i = blockIdx.x * 8 + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (i >= n_kp[f]) return;
  const rgbdslam_b200_keypoint kp = kps[(size_t)f * kp_stride + i];
  const OrbPlane& p = c_geom.full[kp.octave];
  const float sinv = __fdiv_rn(1.f, p.scale);
  const int cx = __float2int_rn(__fmul_rn(kp.x, sinv)), cy = __float2int_rn(__fmul_rn(kp.y, sinv));
  float a, b;
  if (trig) {  // rotation written by k_frame_emit (once per keypoint instead of once per lane)
    const float2 cs = trig[(size_t)f * kp_stride + i];
    a = cs.x;
    b = cs.y;
  } else {
    const float ang = __fmul_rn(kp.angle, 0.017453292519943295f);  // angle *= (float)(CV_PI/180.f)
    a = (float)cos((double)ang);
    b = (float)sin((double)ang);
  }
  const uint8_t* raw = pyr_raw + (size_t)f * frame_stride + p.off;
  const uint8_t* blr = pyr_blur + (size_t)f * frame_stride + p.off;
  auto pix = [&](int k, int which) -> int {
    const float px = (float)c_pattern[k][2 * which], py = (float)c_pattern[k][2 * which + 1];
    const int ix = __float2int_rn(__fsub_rn(__fmul_rn(px, a), __fmul_rn(py, b)));
    const int iy = __float2int_rn(__fadd_rn(__fmul_rn(px, b), __fmul_rn(py, a)));
    const int xx = cx + ix, yy = cy + iy;
    if (xx >= 0 && yy >= 0 && xx < p.w && yy < p.h) return blr[yy * p.w + xx];
    return raw[reflect101(yy, p.h) * p.w + reflect101(xx, p.w)];
  };
  unsigned v = 0;
#pragma unroll
  for (int t = 0; t < 8; t++) {
    const int k = lane * 8 + t;
    v |= (unsigned)(pix(k, 0) < pix(k, 1)) << t;
  }
  desc[((size_t)f * kp_stride + i) * 32 + lane] = (uint8_t)v;
}

// ================================================================================================
// launch helpers (host)
static inline dim3 plane_grid(int w, int h, int z) { return dim3((w + 31) / 32, (h + 7) / 8, z); }

cudaError_t orb_run_detect(const OrbGeom& g, const OrbTables& tab, int nframes, const uint8_t* d_gray, const uint8_t* d_mask,
                           const float* d_depth_for_mask, int detector, uint8_t* d_cell_img, uint8_t* d_cell_mask, OrbCand* d_cand,
                           int* d_cand_count, int* d_hist, int* d_mask_any, int cand_cap, cudaStream_t st, int* launches) {
  const bool fast = detector == RGBDSLAM_B200_DETECTOR_FAST;
  int maxw = 0, maxh = 0;
  for (int c = 0; c < g.ncells; c++) {
    maxw = g.cell[c][0].w > maxw ? g.cell[c][0].w : maxw;
    maxh = g.cell[c][0].h > maxh ? g.cell[c][0].h : maxh;
  }
  const int z = nframes * g.ncells;
  cudaMemsetAsync(d_cand_count, 0, sizeof(int) * z, st);
  cudaMemsetAsync(d_hist, 0, sizeof(int) * 256 * z, st);
  cudaMemsetAsync(d_mask_any, 0, sizeof(int) * z, st);
  k_cell_extract<<<plane_grid(maxw, maxh, z), 256, 0, st>>>(d_gray, d_mask, d_depth_for_mask, d_cell_img, d_cell_mask, d_mask_any);
  (*launches)++;
  const bool all_valid = d_mask == nullptr && d_depth_for_mask == nullptr;  // mask pyramid would stay 255 everywhere
  for (int l = 1; l < (fast ? 1 : kOrbLevels); l++) {  // the FAST detector works on level 0 only
    int lw = 0, lh = 0;
    for (int c = 0; c < g.ncells; c++) {
      lw = g.cell[c][l].w > lw ? g.cell[c][l].w : lw;
      lh = g.cell[c][l].h > lh ? g.cell[c][l].h : lh;
    }
    k_resize_cells<<<plane_grid(lw, lh, z), 256, 0, st>>>(d_cell_img, all_valid ? nullptr : d_cell_mask, l, tab);
    (*launches)++;
  }
  const int tiles = g_fast_tiles[fast ? RGBDSLAM_B200_DETECTOR_FAST : RGBDSLAM_B200_DETECTOR_ORB];
  if (tiles > 0) {
    const uint8_t* m = all_valid ? nullptr : d_cell_mask;
    if (fast)
      k_fast9_nms<<<dim3(tiles, z), 256, 0, st>>>(d_cell_img, m, d_cand, d_cand_count, d_hist, g_fast9_tiles_x, cand_cap);
    else
      k_fast_nms<<<dim3(tiles, z), 256, 0, st>>>(d_cell_img, m, d_cand, d_cand_count, d_hist, cand_cap);
    (*launches)++;
  }
  return cudaGetLastError();
}

cudaError_t orb_run_rgb_to_gray(int nframes, size_t px, const uint8_t* d_rgb, uint8_t* d_gray, cudaStream_t st, int* launches) {
  const size_t n = px * nframes, threads = (n + 3) / 4;
  k_rgb_to_gray<<<(unsigned)((threads + 255) / 256), 256, 0, st>>>(d_rgb, d_gray, n);
  (*launches)++;
  return cudaGetLastError();
}

cudaError_t orb_run_cloud_mask(int nframes, size_t px, const float* d_cloud, int cloud_stride, uint8_t* d_mask, cudaStream_t st,
                               int* launches) {
  const size_t n = px * nframes;
  k_cloud_mask<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(d_cloud, cloud_stride, d_mask, n);
  (*launches)++;
  return cudaGetLastError();
}

cudaError_t orb_run_depth_gather(int nframes, int w, int h, const void* d_src, bool u16, int dw, int dh, const uint16_t* d_col,
                                 const uint16_t* d_row, float* d_depth, uint8_t* d_mask, cudaStream_t st, int* launches) {
  if (u16)
    k_depth_gather<uint16_t><<<plane_grid(w, h, nframes), 256, 0, st>>>((const uint16_t*)d_src, dw, dh, d_col, d_row, d_depth, d_mask,
                                                                        w, h);
  else
    k_depth_gather<float><<<plane_grid(w, h, nframes), 256, 0, st>>>((const float*)d_src, dw, dh, d_col, d_row, d_depth, nullptr, w, h);
  (*launches)++;
  return cudaGetLastError();
}

cudaError_t orb_run_bayer_gr_to_gray(int nframes, int w, int h, const uint8_t* d_raw, uint8_t* d_gray, cudaStream_t st, int* launches) {
  k_bayer_gr_to_gray<<<plane_grid(w, h, nframes), 256, 0, st>>>(d_raw, d_gray, w, h);
  (*launches)++;
  return cudaGetLastError();
}

cudaError_t orb_run_adapt(const OrbGeom& g, int nframes, const int* d_hist, const int* d_cand_count, const int* d_mask_any,
                          double* d_state, int* d_thr, int min_features, int max_features, int max_iters, int* d_err,
                          int cand_cap, OrbThresholds mode, cudaStream_t st, int* launches) {
  if (mode == OrbThresholds::kFixed)
    k_fixed_thresholds<<<(nframes * g.ncells + 255) / 256, 256, 0, st>>>(d_cand_count, d_state, d_thr, nframes * g.ncells, g.ncells,
                                                                        d_err, cand_cap);
  else if (mode == OrbThresholds::kQuotaTable)
    k_adapt_thresholds_quota<<<1, 32 * kOrbMaxCells, 0, st>>>(d_hist, d_cand_count, d_mask_any, d_state, d_thr, nframes, g.ncells,
                                                              min_features, max_features, max_iters, d_err, cand_cap);
  else
    k_adapt_thresholds<<<1, 32 * kOrbMaxCells, 0, st>>>(d_hist, d_cand_count, d_mask_any, d_state, d_thr, nframes, g.ncells,
                                                        min_features, max_features, max_iters, d_err, cand_cap);
  (*launches)++;
  return cudaGetLastError();
}

cudaError_t orb_run_quota_counts(const OrbGeom& g, int nframes, const uint8_t* d_cell_img, const OrbCand* d_cand,
                                 const int* d_cand_count, int* d_thr_scratch, float* d_resp, int cand_cap, int* d_table,
                                 cudaStream_t st, int* launches) {
  const int z = nframes * g.ncells;
  cudaError_t e = cudaMemsetAsync(d_thr_scratch, 0, sizeof(int) * z, st);
  if (e == cudaSuccess) e = cudaMemsetAsync(d_table, 0, sizeof(int) * 256 * z, st);
  if (e != cudaSuccess) return e;
  k_harris<<<dim3((cand_cap + 255) / 256, z), 256, 0, st>>>(d_cell_img, d_cand, d_cand_count, d_thr_scratch, d_resp, cand_cap);
  k_quota_counts<<<dim3(z, kOrbLevels), 1024, 0, st>>>(d_cand, d_cand_count, d_resp, cand_cap, d_table);
  (*launches) += 2;
  return cudaGetLastError();
}

// k_frame_finalize<P> and the detector's k_frame_emit<D, P>
template <OrbPoints P>
static void launch_frames(int nframes, bool fast, const OrbFrameArgs& a, cudaStream_t st, int* launches) {
  const int max_out = a.mode == 1 && a.max_keypoints < a.kp_stride ? a.max_keypoints : a.kp_stride;
  const dim3 grid((max_out + 7) / 8, nframes);
  k_frame_finalize<P><<<nframes, 1024, 0, st>>>(a);
  if (fast)
    k_frame_emit<RGBDSLAM_B200_DETECTOR_FAST, P><<<grid, 256, 0, st>>>(a);
  else
    k_frame_emit<RGBDSLAM_B200_DETECTOR_ORB, P><<<grid, 256, 0, st>>>(a);
  (*launches) += 2;
}

cudaError_t orb_run_select(const OrbGeom& g, int nframes, int detector, OrbPoints points, const OrbCandidates& c,
                           const OrbFrameArgs& a, const OrbSurvivors* all, int* d_err, cudaStream_t st, int* launches) {
  const bool fast = detector == RGBDSLAM_B200_DETECTOR_FAST;
  const int z = nframes * g.ncells, max_per_cell = a.out_stride;
  const dim3 rgrid((c.cap + 255) / 256, z);
  const int quotas = fast ? 0 : 1;  // the FAST detector has no quotas (cv::FastFeatureDetector)
  if (fast)
    k_fast_response<<<rgrid, 256, 0, st>>>(c.cand, c.count, c.thr, c.resp, c.cap);
  else
    k_harris<<<rgrid, 256, 0, st>>>(a.cell_img, c.cand, c.count, c.thr, c.resp, c.cap);
  (*launches)++;
  if (all) {  // whole-frame detectors: no keepStrongest; k_frame_precap caps what k_frame_finalize receives
    k_cell_quota_all<<<z, 1024, 0, st>>>(c.cand, c.count, c.resp, c.cap, quotas, all->keys, all->count, all->stride);
    OrbFrameArgs pre = a;
    pre.cell_out = all->keys;
    pre.cell_out_count = all->count;
    pre.out_stride = all->stride;
    pre.cand_z = all->z;
    (*launches) += 2;
    switch (points) {
      case OrbPoints::kDepthPixel:
        k_frame_precap<OrbPoints::kDepthPixel><<<nframes, 1024, 0, st>>>(a, all->keys, all->count, all->z, all->stride, d_err);
        break;
      case OrbPoints::kMinDepth:
        k_min_depth<<<dim3((all->stride + 7) / 8, z), 256, 0, st>>>(pre, fast);
        (*launches)++;
        k_frame_precap<OrbPoints::kMinDepth><<<nframes, 1024, 0, st>>>(a, all->keys, all->count, all->z, all->stride, d_err);
        break;
      case OrbPoints::kCloud:
        k_frame_precap<OrbPoints::kCloud><<<nframes, 1024, 0, st>>>(a, all->keys, all->count, all->z, all->stride, d_err);
        break;
    }
  } else if (!quotas && c.cap == kOrbCandCap) {
    cudaError_t e = cudaFuncSetAttribute(k_cell_sort, cudaFuncAttributeMaxDynamicSharedMemorySize, kCellSortBytes);
    if (e != cudaSuccess) return e;
    k_cell_sort<<<z, 1024, kCellSortBytes, st>>>(c.cand, c.count, c.resp, c.cap, max_per_cell, a.cell_out, a.cell_out_count,
                                                 max_per_cell);
    (*launches)++;
  } else {
    k_cell_select<<<z, 1024, 0, st>>>(c.cand, c.count, c.resp, c.cap, quotas, max_per_cell, a.cell_out, a.cell_out_count,
                                      max_per_cell);
    (*launches)++;
  }
  switch (points) {
    case OrbPoints::kDepthPixel:
      launch_frames<OrbPoints::kDepthPixel>(nframes, fast, a, st, launches);
      break;
    case OrbPoints::kMinDepth:
      if (!all) {  // whole-frame detectors ran k_min_depth on the survivors, before k_frame_precap
        k_min_depth<<<dim3((max_per_cell + 7) / 8, z), 256, 0, st>>>(a, fast);
        (*launches)++;
      }
      launch_frames<OrbPoints::kMinDepth>(nframes, fast, a, st, launches);
      break;
    case OrbPoints::kCloud:
      launch_frames<OrbPoints::kCloud>(nframes, fast, a, st, launches);
      break;
  }
  return cudaGetLastError();
}

cudaError_t orb_run_describe(const OrbGeom& g, const OrbTables& tab, int nframes, int levels, const uint8_t* d_gray,
                             uint8_t* d_pyr_raw, uint8_t* d_pyr_blur, const rgbdslam_b200_keypoint* d_kp, const int* d_n,
                             int kp_stride, int max_kp, const float2* d_trig, uint8_t* d_desc, cudaStream_t st, int* launches) {
  // level 0 = the image itself
  cudaError_t e = cudaMemcpy2DAsync(d_pyr_raw, g.full_bytes, d_gray, (size_t)g.W * g.H, (size_t)g.W * g.H, nframes,
                                    cudaMemcpyDeviceToDevice, st);
  if (e != cudaSuccess) return e;
  for (int l = 1; l < levels; l++) {
    k_resize<<<plane_grid(g.full[l].w, g.full[l].h, nframes), 256, 0, st>>>(d_pyr_raw, g.full_bytes, l, tab);
    (*launches)++;
  }
  for (int l = 0; l < levels; l++) {
    const dim3 grid((g.full[l].w + 31) / 32, (g.full[l].h + 15) / 16, nframes);
    k_blur<<<grid, 256, 0, st>>>(d_pyr_raw, d_pyr_blur, g.full_bytes, l);
    (*launches)++;
  }
  k_describe<<<dim3((max_kp + 7) / 8, nframes), 256, 0, st>>>(d_pyr_raw, d_pyr_blur, g.full_bytes, d_kp, d_n, kp_stride, d_trig, d_desc);
  (*launches)++;
  return cudaGetLastError();
}

}  // namespace rb200
