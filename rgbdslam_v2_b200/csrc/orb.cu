// orb.cu -- ORB keypoint detection / description kernels for sm_90a (see orb.cuh for provenance).
//
// Node constructor path (src/node.cpp:101-240), batched over frames:
//   detector->detect(gray, kp, mask)      VideoGridAdaptedFeatureDetector (feature_adjuster.cpp:286-317) over
//                                         VideoDynamicAdaptedFeatureDetector (:185-224) over cv::ORB (:94)
//     k_cell_extract / k_resize           per-cell 8-level pyramids, chained INTER_LINEAR_EXACT; mask pyramid
//     k_fast_score / k_nms_collect        threshold-free FAST-9/16 corner score S, strict 3x3 NMS, mask + 15 px border
//                                         -> candidate list + histogram of S per (frame, cell)
//     (host) adaptive thresholds          the x0.7 / x1.3 recurrence only needs #candidates(S >= t): a histogram lookup
//     k_harris                            Harris response of the candidates that pass the final threshold
//     k_cell_select                       keepStrongest(maxTotal / cells) by |response|   (feature_adjuster.cpp:247-255)
//   removeDepthless / retainBest / compute() border filter + octave sort / projectTo3D      (node.cpp:186-210)
//     k_frame_finalize                    one CTA per frame
//   extractor->compute(gray, kp, desc)    cv::ORB::create() defaults (features.cpp:117-119)
//     k_resize / k_blur / k_describe      full-image pyramid, 7-tap float Gaussian, steered BRIEF (one warp / keypoint)
#include "orb.cuh"

#include <cuda_runtime.h>

#include <cstdlib>

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

struct FastTiling {  // tiles of the fused kernel: per level the tile grid of the LARGEST cell, prefix sums over levels
  int32_t tiles_x[kOrbLevels], tiles_y[kOrbLevels], first[kOrbLevels + 1];
};
__constant__ FastTiling c_fast_tiling;

static int g_fast_tiles = 0;  // CTAs per (frame, cell) of the fused FAST + NMS kernel
static int g_orb_legacy = -1;  // RB200_ORB_LEGACY=1: the unfused k_fast_score / k_nms_collect / k_resize detect path (cross-check)

void orb_set_legacy_detect(int on) { g_orb_legacy = on ? 1 : 0; }

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
  g_fast_tiles = ft.first[kOrbLevels];
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

// dst plane = INTER_LINEAR_EXACT resize of the previous level (8.8 fixed-point taps, round to nearest at the end).
// which: 0 = cell pyramids (plane index blockIdx.z % ncells), 1 = full-image pyramid.  tozero: THRESH_TOZERO(254)
// applied to the result (mask pyramid).
__global__ void __launch_bounds__(256) k_resize(uint8_t* __restrict__ buf, int frame_stride, int which, int level, int tozero,
                                                OrbTables tab) {
  const int per = which == 0 ? c_geom.ncells : 1;
  const int f = blockIdx.z / per, c = blockIdx.z % per;
  const OrbPlane& d = which == 0 ? c_geom.cell[c][level] : c_geom.full[level];
  const OrbPlane& s = which == 0 ? c_geom.cell[c][level - 1] : c_geom.full[level - 1];
  const int x = blockIdx.x * 32 + (threadIdx.x & 31), y = blockIdx.y * 8 + (threadIdx.x >> 5);
  if (x >= d.w || y >= d.h) return;
  const uint8_t* sp = buf + (size_t)f * frame_stride + s.off;
  const int ox = tab.ofs[d.tx + x], ax1 = tab.w1[d.tx + x], ax0 = 256 - ax1;
  const int oy = tab.ofs[d.ty + y], ay1 = tab.w1[d.ty + y], ay0 = 256 - ay1;
  const int x1 = min(ox + 1, s.w - 1), y1 = min(oy + 1, s.h - 1);
  const int h0 = sp[oy * s.w + ox] * ax0 + sp[oy * s.w + x1] * ax1;
  const int h1 = sp[y1 * s.w + ox] * ax0 + sp[y1 * s.w + x1] * ax1;
  int v = (h0 * ay0 + h1 * ay1 + (1 << 15)) >> 16;
  if (tozero && v <= 254) v = 0;
  buf[(size_t)f * frame_stride + d.off + (size_t)y * d.w + x] = (uint8_t)v;
}

// -------------------------------------------------------------------------------------------------
// FAST-9/16 corner score without a threshold: S = A - 1, A = max over the 16 arcs of 9 contiguous circle pixels
// of the minimum signed difference (centre brighter: v - p; centre darker: p - v).  A pixel is a FAST corner for
// threshold t exactly when S >= t, and its cv::FAST response is S (cornerScore<16>).
__global__ void __launch_bounds__(256) k_fast_score(const uint8_t* __restrict__ cell_img, uint8_t* __restrict__ score, int level) {
  const int f = blockIdx.z / c_geom.ncells, c = blockIdx.z % c_geom.ncells;
  const OrbPlane& p = c_geom.cell[c][level];
  const int x = blockIdx.x * 32 + (threadIdx.x & 31), y = blockIdx.y * 8 + (threadIdx.x >> 5);
  if (x >= p.w || y >= p.h) return;
  const size_t base = (size_t)f * c_geom.cell_bytes + p.off;
  int S = 0;
  if (x >= 3 && y >= 3 && x < p.w - 3 && y < p.h - 3) {
    const uint8_t* im = cell_img + base;
    const int w = p.w;
    const int v = im[y * w + x];
    const int dx[16] = {0, 1, 2, 3, 3, 3, 2, 1, 0, -1, -2, -3, -3, -3, -2, -1};
    const int dy[16] = {3, 3, 2, 1, 0, -1, -2, -3, -3, -3, -2, -1, 0, 1, 2, 3};
    int d[16];
#pragma unroll
    for (int k = 0; k < 16; k++) d[k] = v - im[(y + dy[k]) * w + x + dx[k]];
    // corner(t): 9 contiguous circle pixels all darker than v - t (d > t) or all brighter than v + t (d < -t).
    // S = largest t for which the pixel is still a corner (binary search; only corners pay for it).
    auto corner = [&](int t) -> bool {
      unsigned hi = 0, lo = 0;
#pragma unroll
      for (int k = 0; k < 16; k++) {
        hi |= (unsigned)(d[k] > t) << k;
        lo |= (unsigned)(d[k] < -t) << k;
      }
      hi |= hi << 16;  // wrap the circle
      lo |= lo << 16;
      unsigned a = hi & (hi >> 1), c2 = lo & (lo >> 1);
      a &= a >> 2; c2 &= c2 >> 2;
      a &= a >> 4; c2 &= c2 >> 4;   // runs of 8
      a &= hi >> 8; c2 &= lo >> 8;  // runs of 9
      return ((a | c2) & 0xFFFFu) != 0u;
    };
    if (corner(1)) {  // the adaptive threshold never goes below 2, scores < 2 are irrelevant
      int lo_t = 1, hi_t = 254;
      while (lo_t < hi_t) {
        const int mid = (lo_t + hi_t + 1) >> 1;
        if (corner(mid)) lo_t = mid;
        else hi_t = mid - 1;
      }
      S = lo_t;
    }
  }
  score[base + (size_t)y * p.w + x] = (uint8_t)min(S, 255);
}

// strict 3x3 non-maximum suppression on S, runByPixelsMask, runByImageBorder(15)  -> candidates + histogram
__global__ void __launch_bounds__(256) k_nms_collect(const uint8_t* __restrict__ score, const uint8_t* __restrict__ cell_mask,
                                                     int level, OrbCand* __restrict__ cand, int* __restrict__ cand_count,
                                                     int* __restrict__ hist) {
  const int f = blockIdx.z / c_geom.ncells, c = blockIdx.z % c_geom.ncells;
  const OrbPlane& p = c_geom.cell[c][level];
  const int x = blockIdx.x * 32 + (threadIdx.x & 31), y = blockIdx.y * 8 + (threadIdx.x >> 5);
  const int edge = 15;  // ORB::create(..., edgeThreshold = 15, ...)  feature_adjuster.cpp:94
  if (x < edge || y < edge || x >= p.w - edge || y >= p.h - edge) return;
  const size_t base = (size_t)f * c_geom.cell_bytes + p.off;
  const uint8_t* s = score + base;
  const int w = p.w;
  const int v = s[y * w + x];
  if (v < 2) return;  // the adaptive threshold never drops below 2 (DetectorAdjuster min_thresh)
  if (cell_mask[base + (size_t)y * w + x] == 0) return;
  const bool mx = v > s[(y - 1) * w + x - 1] && v > s[(y - 1) * w + x] && v > s[(y - 1) * w + x + 1] && v > s[y * w + x - 1] &&
                  v > s[y * w + x + 1] && v > s[(y + 1) * w + x - 1] && v > s[(y + 1) * w + x] && v > s[(y + 1) * w + x + 1];
  if (!mx) return;
  const int fc = f * c_geom.ncells + c;
  atomicAdd(&hist[fc * 256 + v], 1);
  const int slot = atomicAdd(&cand_count[fc], 1);
  if (slot < kOrbCandCap) {
    OrbCand cd;
    cd.x = (uint16_t)x;
    cd.y = (uint16_t)y;
    cd.level = (uint8_t)level;
    cd.score = (uint8_t)v;
    cd.pad_ = 0;
    cand[(size_t)fc * kOrbCandCap + slot] = cd;
  }
}

// -------------------------------------------------------------------------------------------------
// Fused FAST score + NMS for ALL pyramid levels of all (frame, cell) planes in one launch (the default detect path).
// The score is computed directly instead of by binary search over thresholds:
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

__global__ void __launch_bounds__(256) k_fast_nms(const uint8_t* __restrict__ cell_img, const uint8_t* __restrict__ cell_mask,
                                                  OrbCand* __restrict__ cand, int* __restrict__ cand_count, int* __restrict__ hist) {
  __shared__ __align__(16) uint16_t simg[kFI_H][kFI_W];
  __shared__ __align__(16) uint8_t ssc[kFS_H][kFS_W];
  int level = 0;
#pragma unroll
  for (int l = 1; l < kOrbLevels; l++)
    if ((int)blockIdx.x >= c_fast_tiling.first[l]) level = l;
  const int t = blockIdx.x - c_fast_tiling.first[level];
  const int tx = t % c_fast_tiling.tiles_x[level], ty = t / c_fast_tiling.tiles_x[level];
  const int fc = blockIdx.y;
  const int f = fc / c_geom.ncells, c = fc % c_geom.ncells;
  const int pw = c_geom.cell[c][level].w, ph = c_geom.cell[c][level].h;
  const int ox0 = kFastEdge + tx * kFT_W, oy0 = kFastEdge + ty * kFT_H;
  if (ox0 >= pw - kFastEdge || oy0 >= ph - kFastEdge) return;
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
    const int sy_last = min(kFT_H, ph - kFastEdge - oy0) + 1;
#pragma unroll
    for (int pass = 0; pass < 2; pass++) {
      const int sy = r0 + 16 * pass;  // score row (relative y = sy - 1) -> image row sy + 3
      if (sy > sy_last) continue;
      const uint32_t s01 = fast_score_pair(simg, sy + 3, 4 * q + 4);
      const uint32_t s23 = fast_score_pair(simg, sy + 3, 4 * q + 6);
      // halves hold 0..254: pack the four scores into bytes
      reinterpret_cast<uint32_t*>(ssc[sy])[q] = __byte_perm(s01, s23, 0x6420);
    }
  }
  __syncthreads();
  // strict 3x3 non-maximum suppression on S, runByPixelsMask, runByImageBorder(15) -> candidates + histogram
  for (int i = threadIdx.x; i < kFT_W * kFT_H; i += 256) {
    const int oy = i / kFT_W, ox = i - oy * kFT_W;
    const int gx = ox0 + ox, gy = oy0 + oy;
    if (gx >= pw - kFastEdge || gy >= ph - kFastEdge) continue;
    const int sx = ox + 4, sy = oy + 1;
    const int v = ssc[sy][sx];
    if (v < 2) continue;  // the adaptive threshold never drops below 2 (DetectorAdjuster min_thresh)
    const bool mxm = v > ssc[sy - 1][sx - 1] && v > ssc[sy - 1][sx] && v > ssc[sy - 1][sx + 1] && v > ssc[sy][sx - 1] &&
                     v > ssc[sy][sx + 1] && v > ssc[sy + 1][sx - 1] && v > ssc[sy + 1][sx] && v > ssc[sy + 1][sx + 1];
    if (!mxm) continue;
    if (cell_mask && cell_mask[base + (size_t)gy * pw + gx] == 0) continue;
    atomicAdd(&hist[fc * 256 + v], 1);
    const int slot = atomicAdd(&cand_count[fc], 1);
    if (slot < kOrbCandCap) {
      OrbCand cd;
      cd.x = (uint16_t)gx;
      cd.y = (uint16_t)gy;
      cd.level = (uint8_t)level;
      cd.score = (uint8_t)v;
      cd.pad_ = 0;
      cand[(size_t)fc * kOrbCandCap + slot] = cd;
    }
  }
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
// err_flag bit 0: a cell overflowed the candidate buffer.
__global__ void __launch_bounds__(32 * kOrbMaxCells) k_adapt_thresholds(const int* __restrict__ hist, const int* __restrict__ cand_count,
                                                                         const int* __restrict__ mask_any, double* __restrict__ state,
                                                                         int* __restrict__ thr_out, int nframes, int ncells,
                                                                         int min_features, int max_features, int max_iters,
                                                                         int* __restrict__ err_flag) {
  const int c = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (c >= ncells) return;
  double thresh = state[c];
  for (int f = 0; f < nframes; f++) {
    const int fc = f * ncells + c;
    int h[8];
    {
      const int4 a = reinterpret_cast<const int4*>(hist + (size_t)fc * 256)[lane * 2];
      const int4 b = reinterpret_cast<const int4*>(hist + (size_t)fc * 256)[lane * 2 + 1];
      h[0] = a.x; h[1] = a.y; h[2] = a.z; h[3] = a.w; h[4] = b.x; h[5] = b.y; h[6] = b.z; h[7] = b.w;
    }
    const int cnt = cand_count[fc];
    if (cnt > kOrbCandCap && lane == 0) atomicOr(err_flag, 1);
    const bool mask_nonzero = cnt > 0 || mask_any[fc] != 0;
    int iter = max_iters, used = 0;
    bool checked = false;
    do {
      const int t = (int)thresh;  // static_cast<int>(thresh_) feature_adjuster.cpp:94
      used = t;
      int part = 0;
#pragma unroll
      for (int k = 0; k < 8; k++) part += (lane * 8 + k >= t) ? h[k] : 0;
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) part += __shfl_xor_sync(0xffffffffu, part, o);
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
                                                float* __restrict__ resp) {
  const int fc = blockIdx.y;
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  const int n = min(cand_count[fc], kOrbCandCap);
  if (i >= n) return;
  const OrbCand cd = cand[(size_t)fc * kOrbCandCap + i];
  float r = __int_as_float(0x7fc00000);
  if (cd.score >= thr[fc]) {
    const int f = fc / c_geom.ncells, c = fc % c_geom.ncells;
    const OrbPlane& p = c_geom.cell[c][cd.level];
    r = harris_response(cell_img + (size_t)f * c_geom.cell_bytes + p.off, p.w, cd.x, cd.y);
  }
  resp[(size_t)fc * kOrbCandCap + i] = r;
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

// keepStrongest(maxPerCell) by |response| (feature_adjuster.cpp:247-255; nth_element order is unspecified in the
// reference -> canonical tie rule: (level, y, x) ascending).  One CTA per (frame, cell).
// key = [~ordered(|resp|) : 32][level:3 y:10 x:10 : 23][0 : 9]
__global__ void __launch_bounds__(1024) k_cell_select(const OrbCand* __restrict__ cand, const int* __restrict__ cand_count,
                                                      const float* __restrict__ resp, int max_per_cell,
                                                      unsigned long long* __restrict__ cell_out, int* __restrict__ cell_out_count,
                                                      int out_stride) {
  extern __shared__ unsigned long long keys[];
  __shared__ int s_n;
  const int fc = blockIdx.x;
  const int n = min(cand_count[fc], kOrbCandCap);
  if (threadIdx.x == 0) s_n = 0;
  __syncthreads();
  for (int i = threadIdx.x; i < n; i += blockDim.x) {
    const float r = resp[(size_t)fc * kOrbCandCap + i];
    if (r == r) {
      const OrbCand cd = cand[(size_t)fc * kOrbCandCap + i];
      const int slot = atomicAdd(&s_n, 1);
      const uint32_t pos = ((uint32_t)cd.level << 20) | ((uint32_t)cd.y << 10) | cd.x;
      keys[slot] = ((unsigned long long)(~f32_ordered(fabsf(r))) << 32) | ((unsigned long long)pos << 9);
      // the signed response is recovered later from the candidate position (recomputed) -- keep sign in bit 0
      keys[slot] |= (r < 0.f) ? 1ull : 0ull;
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
constexpr int kFrameCap = 4096;  // >= ncells * max_per_cell

// mode 0: detector output, cell-major, inside a cell |response| descending (canonical stand-in for the unspecified
//         nth_element order), ties by (level, y, x).
// mode 1: Node constructor: removeDepthless -> retainBest(K) by signed response (ties canonical, cut at K) ->
//         extractor border filter (31 px on cvRound'ed coordinates) -> stable sort by octave -> orientation ->
//         projectTo3D.  Final order = (octave, response descending, cell, level, y, x).
__global__ void __launch_bounds__(1024)
    k_frame_finalize(int mode, int max_keypoints, const unsigned long long* __restrict__ cell_out,
                     const int* __restrict__ cell_out_count, int out_stride, const uint8_t* __restrict__ cell_img,
                     const float* __restrict__ depth, float depth_scaling, float4 Kinv /* 1/fx, 1/fy, cx, cy */,
                     FrameKp* __restrict__ scratch /* nframes x 2 x kFrameCap */, rgbdslam_b200_keypoint* __restrict__ kp_out,
                     float4* __restrict__ xyz_out, int* __restrict__ n_out, int kp_stride) {
  __shared__ unsigned long long keys[kFrameCap];
  __shared__ int s_n, s_m;
  const int f = blockIdx.x;
  const int W = c_geom.W, H = c_geom.H;
  FrameKp* ka = scratch + (size_t)f * 2 * kFrameCap;  // gather order
  FrameKp* kc = ka + kFrameCap;                       // canonical order
  if (threadIdx.x == 0) { s_n = 0; s_m = 0; }
  __syncthreads();
  // A. gather, shift to image coordinates (pt *= scale; pt += cell origin: feature_adjuster.cpp:259-282), depth check
  for (int c = 0; c < c_geom.ncells; c++) {
    const int fc = f * c_geom.ncells + c;
    const int n = cell_out_count[fc];
    for (int i = threadIdx.x; i < n; i += blockDim.x) {
      const unsigned long long k = cell_out[(size_t)fc * out_stride + i];
      const uint32_t pos = (uint32_t)((k >> 9) & 0x7FFFFFu);
      const int level = pos >> 20, ly = (pos >> 10) & 1023, lx = pos & 1023;
      const uint32_t ord = ~(uint32_t)(k >> 32);
      float r = __uint_as_float(ord & 0x7FFFFFFFu);  // |resp| (ordered() of a non-negative float only sets bit 31)
      if (k & 1ull) r = -r;
      const float sc = c_geom.cell[c][level].scale;
      FrameKp q;
      q.x = __fadd_rn(__fmul_rn((float)lx, sc), (float)c_geom.cell_x0[c]);
      q.y = __fadd_rn(__fmul_rn((float)ly, sc), (float)c_geom.cell_y0[c]);
      q.resp = r;
      q.lx = (uint16_t)lx;
      q.ly = (uint16_t)ly;
      q.level = (uint8_t)level;
      q.cell = (uint8_t)c;
      q.flag = 0;
      bool ok = true;
      if (mode == 1) {  // removeDepthless (node.cpp:67-97)
        ok = !(q.x >= W || q.x < 0 || q.y >= H || q.y < 0);
        if (ok) {
          const int rx = (int)floorf(q.x + 0.5f), ry = (int)floorf(q.y + 0.5f);  // round(): half away from zero
          const size_t idx = (size_t)ry * W + rx;
          const float Z = idx < (size_t)W * H ? depth[(size_t)f * W * H + idx] : __int_as_float(0x7fc00000);
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
      const FrameKp q = ka[i];
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
    // C. retainBest(max_keypoints) (node.cpp:187-191): signed response descending, ties canonical, cut at K
    for (int r = threadIdx.x; r < N; r += blockDim.x)
      keys[r] = r < cnt ? (((unsigned long long)(~f32_ordered(kc[r].resp)) << 32) | (unsigned)r) : ~0ull;
    __syncthreads();
    bitonic_sort_u64(keys, N);
    const int keepK = min(cnt, max_keypoints);
    // D. extractor->compute(): runByImageBorder(31) on cvRound'ed coordinates, then stable sort by octave
    unsigned long long mine[4];  // up to 4 keys per thread (kFrameCap / 1024)
    int nm = 0;
    for (int j = threadIdx.x; j < N; j += blockDim.x) {
      unsigned long long k2 = ~0ull;
      if (j < keepK) {
        const int r = (int)(keys[j] & 0xFFFFu);
        const FrameKp q = kc[r];
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
        const FrameKp q = kc[r];
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
  if (threadIdx.x == 0) n_out[f] = n_final;
}

// One warp per output keypoint: intensity-centroid orientation on the detector's (cell) pyramid, the cv::KeyPoint record,
// in mode 1 projectTo3D (node.cpp:900-965) + backProject (misc2.h:49-65) and the rotation (cos, sin) compute() will use.
__global__ void __launch_bounds__(256)
    k_frame_emit(int mode, const FrameKp* __restrict__ scratch, const uint8_t* __restrict__ cell_img, const float* __restrict__ depth,
                 float depth_scaling, float4 Kinv, rgbdslam_b200_keypoint* __restrict__ kp_out, float4* __restrict__ xyz_out,
                 float2* __restrict__ trig_out, const int* __restrict__ n_out, int kp_stride) {
  const int f = blockIdx.y;
  const int t = blockIdx.x * 8 + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (t >= n_out[f]) return;
  const int W = c_geom.W, H = c_geom.H;
  const FrameKp* ka = scratch + (size_t)f * 2 * kFrameCap;
  const FrameKp q = (ka + kFrameCap)[reinterpret_cast<const uint16_t*>(ka)[t]];
  const OrbPlane& p = c_geom.cell[q.cell][q.level];
  const float ang = ic_angle_warp(cell_img + (size_t)f * c_geom.cell_bytes + p.off, p.w, q.lx, q.ly, lane);
  if (lane == 0) {
    rgbdslam_b200_keypoint o;
    o.x = q.x;
    o.y = q.y;
    o.size = __fmul_rn(31.f, p.scale);
    o.angle = ang;
    o.response = q.resp;
    o.octave = q.level;
    o.class_id = -1;
    kp_out[(size_t)f * kp_stride + t] = o;
    if (mode == 1) {
      const int rx = (int)floorf(q.x + 0.5f), ry = (int)floorf(q.y + 0.5f);
      const float Z = (float)((double)depth[(size_t)f * W * H + (size_t)ry * W + rx] * (double)depth_scaling);
      float4 v;
      v.x = __fmul_rn(__fmul_rn(__fsub_rn(q.x, Kinv.z), Z), Kinv.x);
      v.y = __fmul_rn(__fmul_rn(__fsub_rn(q.y, Kinv.w), Z), Kinv.y);
      v.z = Z;
      v.w = 1.f;
      xyz_out[(size_t)f * kp_stride + t] = v;
      if (trig_out) {  // angle *= (float)(CV_PI/180.f); a = (float)cos(angle), b = (float)sin(angle)  (cv::ORB computeOrbDescriptors)
        const float ar = __fmul_rn(ang, 0.017453292519943295f);
        trig_out[(size_t)f * kp_stride + t] = make_float2((float)cos((double)ar), (float)sin((double)ar));
      }
    }
  }
}

// -------------------------------------------------------------------------------------------------
// GaussianBlur(level, 7x7, sigma 2, BORDER_REFLECT_101) as OpenCV evaluates it inside ORB: separable float filter,
// row pass accumulated left to right, column pass symmetric, round-half-even to uint8.
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
  for (int r = ty; r < 22; r += 8) {
    float acc = 0.f;
#pragma unroll
    for (int j = 0; j < 7; j++) acc = __fadd_rn(acc, __fmul_rn(c_gauss[j], tile[r][tx + j]));  // left to right, as cv::sepFilter2D
    rows[r][tx] = acc;
  }
  __syncthreads();
  const int x = x0 + tx;
  for (int r = ty; r < 16; r += 8) {
    const int y = y0 + r;
    if (x < pw && y < ph) {
      float c = __fmul_rn(c_gauss[3], rows[r + 3][tx]);
#pragma unroll
      for (int j = 1; j <= 3; j++) c = __fadd_rn(c, __fmul_rn(c_gauss[3 + j], __fadd_rn(rows[r + 3 + j][tx], rows[r + 3 - j][tx])));
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
                           const float* d_depth_for_mask, uint8_t* d_cell_img, uint8_t* d_cell_mask, uint8_t* d_score, OrbCand* d_cand,
                           int* d_cand_count, int* d_hist, int* d_mask_any, cudaStream_t st, int* launches) {
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
  if (g_orb_legacy < 0) {
    const char* ev = getenv("RB200_ORB_LEGACY");
    g_orb_legacy = (ev && ev[0] == '1') ? 1 : 0;
  }
  if (!g_orb_legacy) {
    for (int l = 1; l < kOrbLevels; l++) {
      int lw = 0, lh = 0;
      for (int c = 0; c < g.ncells; c++) {
        lw = g.cell[c][l].w > lw ? g.cell[c][l].w : lw;
        lh = g.cell[c][l].h > lh ? g.cell[c][l].h : lh;
      }
      k_resize_cells<<<plane_grid(lw, lh, z), 256, 0, st>>>(d_cell_img, all_valid ? nullptr : d_cell_mask, l, tab);
      (*launches)++;
    }
    if (g_fast_tiles > 0) {
      k_fast_nms<<<dim3(g_fast_tiles, z), 256, 0, st>>>(d_cell_img, all_valid ? nullptr : d_cell_mask, d_cand, d_cand_count, d_hist);
      (*launches)++;
    }
    return cudaGetLastError();
  }
  for (int l = 0; l < kOrbLevels; l++) {
    int lw = 0, lh = 0;
    for (int c = 0; c < g.ncells; c++) {
      lw = g.cell[c][l].w > lw ? g.cell[c][l].w : lw;
      lh = g.cell[c][l].h > lh ? g.cell[c][l].h : lh;
    }
    if (l > 0) {
      k_resize<<<plane_grid(lw, lh, z), 256, 0, st>>>(d_cell_img, g.cell_bytes, 0, l, 0, tab);
      k_resize<<<plane_grid(lw, lh, z), 256, 0, st>>>(d_cell_mask, g.cell_bytes, 0, l, 1, tab);
      (*launches) += 2;
    }
    k_fast_score<<<plane_grid(lw, lh, z), 256, 0, st>>>(d_cell_img, d_score, l);
    k_nms_collect<<<plane_grid(lw, lh, z), 256, 0, st>>>(d_score, d_cell_mask, l, d_cand, d_cand_count, d_hist);
    (*launches) += 2;
  }
  return cudaGetLastError();
}

cudaError_t orb_run_adapt(const OrbGeom& g, int nframes, const int* d_hist, const int* d_cand_count, const int* d_mask_any,
                          double* d_state, int* d_thr, int min_features, int max_features, int max_iters, int* d_err,
                          cudaStream_t st, int* launches) {
  k_adapt_thresholds<<<1, 32 * kOrbMaxCells, 0, st>>>(d_hist, d_cand_count, d_mask_any, d_state, d_thr, nframes, g.ncells,
                                                      min_features, max_features, max_iters, d_err);
  (*launches)++;
  return cudaGetLastError();
}

cudaError_t orb_run_select(const OrbGeom& g, int nframes, int mode, int max_per_cell, int max_keypoints,
                           const uint8_t* d_cell_img, const OrbCand* d_cand, const int* d_cand_count, const int* d_thr,
                           float* d_resp, unsigned long long* d_cell_out, int* d_cell_out_count, const float* d_depth,
                           float depth_scaling, float4 Kinv, void* d_scratch, rgbdslam_b200_keypoint* d_kp, float4* d_xyz,
                           float2* d_trig, int* d_n, int kp_stride, cudaStream_t st, int* launches) {
  const int z = nframes * g.ncells;
  k_harris<<<dim3((kOrbCandCap + 255) / 256, z), 256, 0, st>>>(d_cell_img, d_cand, d_cand_count, d_thr, d_resp);
  static bool attr = false;
  if (!attr) {
    cudaError_t e = cudaFuncSetAttribute(k_cell_select, cudaFuncAttributeMaxDynamicSharedMemorySize, 16384 * 8);
    if (e != cudaSuccess) return e;
    attr = true;
  }
  k_cell_select<<<z, 1024, 16384 * 8, st>>>(d_cand, d_cand_count, d_resp, max_per_cell, d_cell_out, d_cell_out_count, max_per_cell);
  k_frame_finalize<<<nframes, 1024, 0, st>>>(mode, max_keypoints, d_cell_out, d_cell_out_count, max_per_cell, d_cell_img, d_depth,
                                             depth_scaling, Kinv, (FrameKp*)d_scratch, d_kp, d_xyz, d_n, kp_stride);
  const int max_out = mode == 1 ? (max_keypoints < kp_stride ? max_keypoints : kp_stride) : kp_stride;
  k_frame_emit<<<dim3((max_out + 7) / 8, nframes), 256, 0, st>>>(mode, (const FrameKp*)d_scratch, d_cell_img, d_depth, depth_scaling,
                                                                 Kinv, d_kp, d_xyz, d_trig, d_n, kp_stride);
  (*launches) += 4;
  return cudaGetLastError();
}

cudaError_t orb_run_describe(const OrbGeom& g, const OrbTables& tab, int nframes, const uint8_t* d_gray, uint8_t* d_pyr_raw,
                             uint8_t* d_pyr_blur, const rgbdslam_b200_keypoint* d_kp, const int* d_n, int kp_stride, int max_kp,
                             const float2* d_trig, uint8_t* d_desc, cudaStream_t st, int* launches) {
  // level 0 = the image itself
  cudaError_t e = cudaMemcpy2DAsync(d_pyr_raw, g.full_bytes, d_gray, (size_t)g.W * g.H, (size_t)g.W * g.H, nframes,
                                    cudaMemcpyDeviceToDevice, st);
  if (e != cudaSuccess) return e;
  for (int l = 1; l < kOrbLevels; l++) {
    k_resize<<<plane_grid(g.full[l].w, g.full[l].h, nframes), 256, 0, st>>>(d_pyr_raw, g.full_bytes, 1, l, 0, tab);
    (*launches)++;
  }
  for (int l = 0; l < kOrbLevels; l++) {
    k_blur<<<dim3((g.full[l].w + 31) / 32, (g.full[l].h + 15) / 16, nframes), 256, 0, st>>>(d_pyr_raw, d_pyr_blur, g.full_bytes, l);
    (*launches)++;
  }
  k_describe<<<dim3((max_kp + 7) / 8, nframes), 256, 0, st>>>(d_pyr_raw, d_pyr_blur, g.full_bytes, d_kp, d_n, kp_stride, d_trig, d_desc);
  (*launches)++;
  return cudaGetLastError();
}

}  // namespace rb200
