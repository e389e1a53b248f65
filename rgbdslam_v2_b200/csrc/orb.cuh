// orb.cuh -- device-side geometry of the ORB detect / describe pipeline (orb.cu).
//
// OpenCV's ORB is an un-vendored dependency of the reference (feature_adjuster.cpp:94 builds
// cv::ORB::create(10000, 1.2, 8, 15, 0, 2, HARRIS_SCORE, 31, thresh) per grid cell; features.cpp:117-119 builds the
// default cv::ORB::create() extractor).  Its published algorithm is restated here; every arithmetic detail was
// pinned against cv2 4.13 (oracle/orb_oracle.py, tests/test_orb_oracle.py): chained INTER_LINEAR_EXACT pyramid,
// FAST-9/16 corner score + 3x3 NMS, Harris response, intensity-centroid angle (fastAtan2), 7-tap float Gaussian,
// rBRIEF with the learned bit_pattern_31_.
#pragma once
#include <stdint.h>

namespace rb200 {

constexpr int kOrbLevels = 8;
constexpr int kOrbMaxCells = 16;       // detector_grid_resolution <= 4
constexpr int kOrbCandCap = 12288;     // FAST/NMS candidates per (frame, cell), all levels: the smallest buffer orb_prepare sizes
constexpr int kOrbHalfPatch = 15;
// Frames wider or taller than kOrbNarrowMax px, up to kOrbMaxSide, take a candidate buffer sized from the largest cell's area and
// need a grid whose per-cell maximum stays below cv::ORB's smallest quota (api_orb.cu).  DESIGN.md 4.5.5.
constexpr int kOrbNarrowMax = 1023;
constexpr int kOrbMaxSide = 4095;

// One image plane of a pyramid: where it lives in the packed per-frame buffer and its resize tables.
struct OrbPlane {
  int32_t w, h;
  int32_t off;         // byte offset inside the per-frame packed buffer
  int32_t tx, ty;      // offsets (in entries) into the table arrays for the resize that PRODUCES this plane
  float scale;         // layerScale (level 0: 1.0)
};

// Geometry shared by all frames of one image size.
struct OrbGeom {
  int32_t W, H;                 // full image
  int32_t ncells, grid;         // grid x grid cells (1 = no grid)
  int32_t cell_x0[kOrbMaxCells], cell_y0[kOrbMaxCells];
  OrbPlane cell[kOrbMaxCells][kOrbLevels];   // detector pyramids (one per grid cell)
  int32_t cell_bytes;           // packed bytes per frame for all cell pyramids (image; mask uses the same layout)
  OrbPlane full[kOrbLevels];    // extractor pyramid of the whole image
  int32_t full_bytes;
  int32_t n_per_level[kOrbLevels];  // ORB feature quota per level for nfeatures = 10000 (applied by k_cell_select)
};

// resize tables: for every destination column/row the first source index and the weight of the second tap (x256)
struct OrbTables {
  const int16_t* ofs;
  const uint16_t* w1;
};

struct OrbCand {   // a FAST corner that survived NMS, mask and the 15 px border filter
  uint16_t x, y;   // level coordinates
  uint8_t level;
  uint8_t score;   // FAST corner score (largest threshold for which it is still a corner)
  uint16_t pad_;
};

// cvtColor(raw, rgb, COLOR_BayerGR2RGB) (openni_listener.cpp:638-641) at pixel (x, y) of the w x h mosaic at byte `frame` of
// raw (G B on even rows, R G on odd rows), cv2 4.13's bilinear rule: an interior pixel keeps its own channel and averages the
// others over pairs, (a + b + 1) >> 1, or over the cross / diagonal quads, (a + b + c + d + 2) >> 2; rows 0 and h-1 repeat rows
// 1 and h-2, columns 0 and w-1 columns 1 and w-2.  Used by the grey conversion (orb.cu) and by the stored colour clouds (map.cu).
#ifdef __CUDACC__
__device__ __forceinline__ void bayer_gr_rgb(const uint8_t* __restrict__ raw, size_t frame, int w, int h, int x, int y, uint32_t& r,
                                             uint32_t& g, uint32_t& b) {
  const int sx = min(max(x, 1), w - 2), sy = min(max(y, 1), h - 2);
  const uint8_t* p = raw + frame + (size_t)sy * w + sx;
  const uint32_t c = p[0], up = p[-w], dn = p[w], lf = p[-1], rt = p[1];
  const uint32_t pair_v = (up + dn + 1) >> 1, pair_h = (lf + rt + 1) >> 1, cross = (up + dn + lf + rt + 2) >> 2;
  const uint32_t diag = (p[-w - 1] + p[-w + 1] + p[w - 1] + p[w + 1] + 2u) >> 2;
  if (!(sy & 1)) {
    if (!(sx & 1)) { r = pair_v; g = c; b = pair_h; }  // G, B to the sides
    else { r = diag; g = cross; b = c; }               // B
  } else {
    if (!(sx & 1)) { r = c; g = cross; b = diag; }     // R
    else { r = pair_h; g = c; b = pair_v; }            // G, R to the sides
  }
}
#endif

}  // namespace rb200
