// api_orb.cu -- C ABI of the Node constructor path (detect / describe / back-project), host orchestration.
//   rgbdslam_b200_detector_*   == createDetector("ORB" | "FAST") + its persistent adaptive-threshold state
//                                 (features.cpp:63-113, feature_adjuster.cpp:131-150, openni_listener.cpp:130-132)
//   rgbdslam_b200_orb_detect   == detector->detect(gray, keypoints, mask)             (node.cpp:160)
//   rgbdslam_b200_orb_compute  == extractor->compute(gray, keypoints, descriptors)    (node.cpp:202)
//   rgbdslam_b200_nodes_create == Node::Node(visual, depth, mask, cam_info, ...)      (node.cpp:101-240), batched; with the
//                                 CLOUD_* flags of _ex / _sharded Node::Node(visual, detector, extractor, point_cloud, mask)
//                                 (node.cpp:252-369), with VISUAL_RGB the cvtColor of a colour visual (:139-144, 275-277),
//                                 with KEEP_CLOUD the node keeps its organised cloud (pc_col, :261) for the measurement model,
//                                 with DEPTH_U16 / VISUAL_BAYER_GR the listener's conversions of its raw 16UC1 depth and
//                                 bayer_grbg8 images (openni_listener.cpp:633-659), with STORE_CLOUD the colour cloud pc_col
//                                 (createXYZRGBPointCloud, node.cpp:126-131, misc.cpp:467-556) for the map
#include <algorithm>
#include <cmath>
#include <cstring>
#include <mutex>
#include <vector>

#include "comm.h"
#include "kernels.h"
#include "orb_host.h"
#include "state.h"

namespace rb200 {

struct Detector {
  static constexpr uint32_t kMagic = 0x44455443u;  // 'DETC'
  uint32_t magic = kMagic;
  int type;                     // params.feature_detector_type when the detector was created
  double thresh[kOrbMaxCells];  // host mirror of the persistent per-cell thresholds
  DevBuf d_state;               // the same on the device: the recurrence runs there (k_adapt_thresholds)
  bool host_valid = true, dev_valid = false;
  explicit Detector(int t) : type(t) {
    // new DetectorAdjuster("ORB", 20) / DetectorAdjuster("FAST", 20)  features.cpp:92, feature_adjuster.cpp:88-91
    for (int i = 0; i < kOrbMaxCells; i++) thresh[i] = 20.0;
  }
  // cv::ORB::compute builds the pyramid up to the largest keypoint octave: FAST keypoints are all octave 0
  int describe_levels() const { return type == RGBDSLAM_B200_DETECTOR_FAST ? 1 : kOrbLevels; }
};

struct OrbCtx {
  bool ready = false;
  int W = 0, H = 0, grid = 0, max_kp = 0;
  OrbGeom g;
  std::vector<int16_t> h_ofs;
  std::vector<uint16_t> h_w1;
  DevBuf d_ofs, d_w1;
  OrbTables tab;
  int max_per_cell = 0, min_cell = 0, max_cell = 0, kp_stride = 0;
  DevBuf in_gray[2], in_mask[2], in_depth[2];  // double-buffered chunk inputs (upload of chunk k+1 under the kernels of chunk k)
  DevBuf in_rgb[2];                            // colour or Bayer input, converted into in_gray on the device
  DevBuf in_raw[2];                            // 16-bit millimetre depth, converted into in_depth (and in_mask) on the device
  PinBuf stage[2];                             // pinned staging for callers that pass pageable memory
  cudaStream_t copy_stream = nullptr;
  cudaEvent_t ev_ready[2] = {nullptr, nullptr}, ev_free[2] = {nullptr, nullptr}, ev_copied[2] = {nullptr, nullptr};
  DevBuf cell_img, cell_mask, cand, cand_count, hist, mask_any, thr, resp, cell_out, cell_out_count, cand_z, scratch, kp, xyz, n,
      pyr_raw, pyr_blur, desc, err, trig;
  // rgbdslam_b200_nodes_create_sharded: what must survive between the detection pass and the finishing pass of ALL own frames,
  // and the per-(frame, cell) tables every rank holds for ALL frames of the sequence
  DevBuf sh_gray, sh_rgb, sh_raw, sh_depth, sh_mask, sh_cell_img, sh_cand, all_hist, all_cnt, all_many, all_thr;
  const uint8_t* last_gray = nullptr;  // device pointers of frame 0 of the last call (debug hooks)
  OrbCandidates candidates() const { return {(const OrbCand*)cand.ptr, (const int*)cand_count.ptr, (const int*)thr.ptr, (float*)resp.ptr}; }
  void release() {
    DevBuf* all[] = {&d_ofs, &d_w1, &in_gray[0], &in_gray[1], &in_mask[0], &in_mask[1], &in_depth[0], &in_depth[1], &in_rgb[0],
                     &in_rgb[1], &in_raw[0], &in_raw[1], &cell_img, &cell_mask, &cand, &cand_count, &hist, &mask_any, &thr, &resp,
                     &cell_out, &cell_out_count, &cand_z, &scratch, &kp, &xyz, &n, &pyr_raw, &pyr_blur, &desc, &err, &trig, &sh_gray,
                     &sh_rgb, &sh_raw, &sh_depth, &sh_mask, &sh_cell_img, &sh_cand, &all_hist, &all_cnt, &all_many, &all_thr};
    for (DevBuf* b : all) b->release();
    stage[0].release();
    stage[1].release();
    ready = false;
  }
};
static OrbCtx g_orb;

static inline int cv_round_f(float v) { return (int)lrintf(v); }
static inline float layer_scale(int level) { return (float)std::pow((double)1.2f, (double)level); }  // ORB getScale()

// resize tables src_n -> dst_n (INTER_LINEAR_EXACT): first tap index and weight of the second tap (x256)
static void build_table(int src_n, int dst_n, std::vector<int16_t>& ofs, std::vector<uint16_t>& w1) {
  const double scale = (double)src_n / dst_n;
  for (int d = 0; d < dst_n; d++) {
    const double f = (d + 0.5) * scale - 0.5;
    int i = (int)std::floor(f);
    double fr = f - i;
    if (i < 0) { i = 0; fr = 0; }
    if (i >= src_n - 1) { i = src_n - 1; fr = 0; }
    ofs.push_back((int16_t)i);
    w1.push_back((uint16_t)std::lrint(fr * 256.0));  // cvRound: half to even
  }
}

static int orb_prepare(int W, int H) {
  State& s = g_state;
  OrbCtx& o = g_orb;
  const int grid = s.params.detector_grid_resolution > 1 ? s.params.detector_grid_resolution : 1;
  const int K = s.params.max_keypoints;
  if (o.ready && o.W == W && o.H == H && o.grid == grid && o.max_kp == K) return 0;
  if (grid * grid > kOrbMaxCells) {
    set_error("detector_grid_resolution > 4 is not supported");
    return RGBDSLAM_B200_ERR_ARG;
  }
  if (W < 96 || H < 96 || W > 1023 || H > 1023) {
    set_error("image size must be within [96, 1023] in both dimensions");
    return RGBDSLAM_B200_ERR_ARG;
  }
  o.release();
  OrbGeom& g = o.g;
  memset(&g, 0, sizeof(g));
  g.W = W; g.H = H; g.grid = grid; g.ncells = grid * grid;
  o.h_ofs.clear(); o.h_w1.clear();
  // table cache per (base length) chain
  struct Chain { int n0; int off[kOrbLevels]; };
  std::vector<Chain> chains;
  auto chain_for = [&](int n0) -> const Chain& {
    for (const Chain& c : chains) if (c.n0 == n0) return c;
    Chain c;
    c.n0 = n0;
    int prev = n0;
    c.off[0] = 0;
    for (int l = 1; l < kOrbLevels; l++) {
      const int nl = cv_round_f((float)n0 / layer_scale(l));
      c.off[l] = (int)o.h_ofs.size();
      build_table(prev, nl, o.h_ofs, o.h_w1);
      prev = nl;
    }
    chains.push_back(c);
    return chains.back();
  };
  // grid cells (feature_adjuster.cpp:286-303; edgeThreshold = 31: feature_adjuster.h:110)
  const int edge = 31;
  int off = 0;
  for (int i = 0; i < grid; i++)
    for (int j = 0; j < grid; j++) {
      const int c = j + i * grid;
      int y0 = 0, y1 = H, x0 = 0, x1 = W;
      if (grid > 1) {
        y0 = std::max((i * H) / grid - edge, 0);
        y1 = std::min(H, ((i + 1) * H) / grid + edge);
        x0 = std::max((j * W) / grid - edge, 0);
        x1 = std::min(W, ((j + 1) * W) / grid + edge);
      }
      g.cell_x0[c] = x0;
      g.cell_y0[c] = y0;
      const int w0 = x1 - x0, h0 = y1 - y0;
      const Chain cx = chain_for(w0), cy = chain_for(h0);
      for (int l = 0; l < kOrbLevels; l++) {
        OrbPlane& p = g.cell[c][l];
        p.scale = layer_scale(l);
        p.w = l == 0 ? w0 : cv_round_f((float)w0 / p.scale);
        p.h = l == 0 ? h0 : cv_round_f((float)h0 / p.scale);
        p.off = off;
        p.tx = cx.off[l];
        p.ty = cy.off[l];
        off += (p.w * p.h + 15) / 16 * 16;
        if (p.w < 40 || p.h < 40) {
          set_error("image too small for an 8-level ORB pyramid per grid cell");
          return RGBDSLAM_B200_ERR_ARG;
        }
      }
    }
  g.cell_bytes = off;
  {
    const Chain cx = chain_for(W), cy = chain_for(H);
    int foff = 0;
    for (int l = 0; l < kOrbLevels; l++) {
      OrbPlane& p = g.full[l];
      p.scale = layer_scale(l);
      p.w = l == 0 ? W : cv_round_f((float)W / p.scale);
      p.h = l == 0 ? H : cv_round_f((float)H / p.scale);
      p.off = foff;
      p.tx = cx.off[l];
      p.ty = cy.off[l];
      foff += (p.w * p.h + 15) / 16 * 16;
    }
    g.full_bytes = foff;
  }
  {  // ORB per-level quotas for nfeatures = 10000 (only used to detect a binding retainBest)
    const float factor = 1.f / 1.2f;
    float nd = 10000 * (1 - factor) / (1 - (float)std::pow((double)factor, (double)kOrbLevels));
    int sum = 0;
    for (int l = 0; l < kOrbLevels - 1; l++) {
      g.n_per_level[l] = cv_round_f(nd);
      sum += g.n_per_level[l];
      nd *= factor;
    }
    g.n_per_level[kOrbLevels - 1] = std::max(10000 - sum, 0);
  }
  int umax[kOrbHalfPatch + 2];
  {
    const int hp = kOrbHalfPatch;
    const int vmax = (int)std::floor(hp * std::sqrt(2.f) / 2 + 1), vmin = (int)std::ceil(hp * std::sqrt(2.f) / 2);
    for (int v = 0; v <= hp + 1; v++) umax[v] = 0;
    for (int v = 0; v <= vmax; ++v) umax[v] = (int)std::lrint(std::sqrt((double)hp * hp - v * v));
    for (int v = hp, v0 = 0; v >= vmin; --v) {
      while (umax[v0] == umax[v0 + 1]) ++v0;
      umax[v] = v0;
      ++v0;
    }
  }
  // adjustedGridWrapper (features.cpp:43-60)
  const int mn = K, mx = (int)(K * 1.5);
  if (grid > 1) {
    o.min_cell = (int)std::lround(mn / (float)g.ncells);
    o.max_cell = (int)std::lround(mx / (float)g.ncells);
    o.max_per_cell = mx / g.ncells;  // maxTotalKeypoints / (gridRows*gridCols), feature_adjuster.cpp:292
  } else {
    o.min_cell = mn;
    o.max_cell = mx;
    o.max_per_cell = kOrbFrameCap;  // no keepStrongest without the grid wrapper
  }
  if (o.max_per_cell * g.ncells > kOrbFrameCap && grid > 1) {
    set_error("max_keypoints too large for the per-frame staging buffer (1.5 * max_keypoints <= 4096)");
    return RGBDSLAM_B200_ERR_ARG;
  }
  o.kp_stride = std::min(kOrbFrameCap, o.max_per_cell * g.ncells);
  o.W = W; o.H = H; o.grid = grid; o.max_kp = K;
  int rc;
  if ((rc = o.d_ofs.ensure(o.h_ofs.size() * 2 + 16)) || (rc = o.d_w1.ensure(o.h_w1.size() * 2 + 16))) return rc;
  cudaStream_t st = s.stream;
  cudaError_t e = cudaMemcpyAsync(o.d_ofs.ptr, o.h_ofs.data(), o.h_ofs.size() * 2, cudaMemcpyHostToDevice, st);
  if (e == cudaSuccess) e = cudaMemcpyAsync(o.d_w1.ptr, o.h_w1.data(), o.h_w1.size() * 2, cudaMemcpyHostToDevice, st);
  if (e == cudaSuccess) e = orb_upload_constants(g, umax, st);
  if (e == cudaSuccess) e = cudaStreamSynchronize(st);
  if (e != cudaSuccess) return cuda_fail(e, "orb_prepare upload");
  o.tab.ofs = (const int16_t*)o.d_ofs.ptr;
  o.tab.w1 = (const uint16_t*)o.d_w1.ptr;
  o.ready = true;
  return 0;
}

constexpr int kOrbChunk = 64;  // frames per pass of nodes_create for grey + depth-image input

// The recipe of a call: what one frame brings (from the flags of nodes_create*, include/rgbdslam_b200.h) and how its keypoints
// become nodes (from the parameters).  A default FrameInput is orb_detect's: the detector output of a grey image (mode 0).
struct FrameInput {
  int mode = 0;                               // 0: detector output, 1: Node constructor
  bool rgb = false, bayer = false, mask_from_depth = false, mask_from_cloud = false;
  bool depth_u16 = false, mask_from_u16 = false;  // 16-bit millimetres; its mask is written into the mask buffer (k_depth_u16)
  bool caller_mask = false;                   // the caller's mask is uploaded (not replaced by one derived on the device)
  int cloud_stride = 0;                       // floats per cloud point (4: PointXYZ, 8: PointXYZRGB); 0 = depth image
  size_t gray_bytes = 0, depth_bytes = 0;     // per frame, as the caller passes them: the visual image, the depth image or cloud
  size_t plane_bytes = 0;                     // per frame on the device: the float depth image or the cloud
  OrbPoints points = OrbPoints::kDepthPixel;
  float depth_scaling = 1.f;
  float4 Kinv = {0.f, 0.f, 0.f, 0.f};         // projectTo3D intrinsics (node.cpp:913-916): float(1./fx), float(1./fy), cx, cy
  FrameInput() = default;
  FrameInput(int flags, size_t px, const rgbdslam_b200_params& p, const float* K4, const uint8_t* mask) {
    mode = 1;
    rgb = (flags & RGBDSLAM_B200_VISUAL_RGB) != 0;
    bayer = (flags & RGBDSLAM_B200_VISUAL_BAYER_GR) != 0;
    depth_u16 = (flags & RGBDSLAM_B200_DEPTH_U16) != 0;
    const bool from_depth = (flags & RGBDSLAM_B200_MASK_FROM_DEPTH) != 0;
    mask_from_depth = from_depth && !depth_u16;  // the float rule, applied by k_cell_extract
    mask_from_u16 = from_depth && depth_u16;
    mask_from_cloud = (flags & RGBDSLAM_B200_MASK_FROM_CLOUD) != 0;
    caller_mask = mask && !from_depth && !mask_from_cloud;
    cloud_stride = (flags & RGBDSLAM_B200_CLOUD_XYZRGB) ? 8 : (flags & RGBDSLAM_B200_CLOUD_XYZ) ? 4 : 0;
    gray_bytes = rgb ? 3 * px : px;
    depth_bytes = cloud_stride ? px * cloud_stride * 4 : depth_u16 ? px * 2 : px * 4;
    plane_bytes = cloud_stride ? depth_bytes : px * 4;
    // getMinDepthInNeighborhood (node.cpp:82-83, 940-941) is a depth-image rule: the point-cloud constructor does not read it
    points = cloud_stride ? OrbPoints::kCloud : p.use_feature_min_depth ? OrbPoints::kMinDepth : OrbPoints::kDepthPixel;
    if (!cloud_stride) {  // the point-cloud constructor takes its points from the cloud: no intrinsics
      depth_scaling = (float)p.depth_scaling_factor;
      Kinv = make_float4((float)(1. / (double)K4[0]), (float)(1. / (double)K4[1]), K4[2], K4[3]);
    }
  }
  bool mask_buffer() const { return caller_mask || mask_from_cloud || mask_from_u16; }  // a device mask per frame
  bool raw_visual() const { return rgb || bayer; }  // the visual is uploaded into in_rgb / sh_rgb and converted into grey
  // frames per chunk: the input and staging buffers hold about as many bytes as kOrbChunk grey + depth-image frames (a
  // 640x480 XYZRGB cloud is 9.8 MB, against 1.5 MB), and never more than kOrbChunk frames, which bounds the per-frame work
  // buffers (16-bit depth would allow 106); the chunk size does not change any result
  int chunk(int nframes, size_t px) const {
    const size_t cap = std::max<size_t>(1, (size_t)kOrbChunk * 5 * px / (gray_bytes + depth_bytes));
    return (int)std::min<size_t>((size_t)std::min(std::max(nframes, 1), kOrbChunk), cap);
  }
};

static int orb_ensure_streams() {
  OrbCtx& o = g_orb;
  if (o.copy_stream) return 0;
  cudaError_t e = cudaStreamCreateWithFlags(&o.copy_stream, cudaStreamNonBlocking);
  for (int i = 0; i < 2 && e == cudaSuccess; i++) {
    e = cudaEventCreateWithFlags(&o.ev_ready[i], cudaEventDisableTiming);
    if (e == cudaSuccess) e = cudaEventCreateWithFlags(&o.ev_free[i], cudaEventDisableTiming);
    if (e == cudaSuccess) e = cudaEventCreateWithFlags(&o.ev_copied[i], cudaEventDisableTiming);
  }
  if (e != cudaSuccess) return cuda_fail(e, "orb streams / events");
  return 0;
}

// work buffers for F frames per pass; nbuf input buffers (1: synchronous single-frame entry points, 2: nodes_create)
// depth_bytes: per frame (0 = a w*h float depth image); visual_bytes / raw_bytes: per frame of the colour or Bayer input
// buffers / of the 16-bit depth input buffers (0 = none)
static int orb_ensure_buffers(int F, int nbuf, bool want_mask, size_t depth_bytes = 0, size_t visual_bytes = 0, size_t raw_bytes = 0) {
  OrbCtx& o = g_orb;
  const OrbGeom& g = o.g;
  const size_t px = (size_t)g.W * g.H, z = (size_t)F * g.ncells;
  if (depth_bytes == 0) depth_bytes = px * 4;
  int rc;
  for (int b = 0; b < nbuf; b++)
    if ((rc = o.in_gray[b].ensure(px * F)) || (want_mask && (rc = o.in_mask[b].ensure(px * F))) ||
        (rc = o.in_depth[b].ensure(depth_bytes * F)) || (visual_bytes && (rc = o.in_rgb[b].ensure(visual_bytes * F))) ||
        (raw_bytes && (rc = o.in_raw[b].ensure(raw_bytes * F))))
      return rc;
  if ((rc = o.cell_img.ensure((size_t)g.cell_bytes * F)) || (rc = o.cell_mask.ensure((size_t)g.cell_bytes * F)) ||
      (rc = o.cand.ensure(z * kOrbCandCap * sizeof(OrbCand))) ||
      (rc = o.cand_count.ensure(z * 4)) || (rc = o.hist.ensure(z * 256 * 4)) || (rc = o.mask_any.ensure(z * 4)) ||
      (rc = o.thr.ensure(z * 4)) || (rc = o.resp.ensure(z * kOrbCandCap * 4)) ||
      (rc = o.cell_out.ensure(z * (size_t)o.max_per_cell * 8)) || (rc = o.cell_out_count.ensure(z * 4)) ||
      (rc = o.cand_z.ensure(z * (size_t)o.max_per_cell * 4)) || (rc = o.scratch.ensure((size_t)F * 2 * kOrbFrameCap * kOrbFrameKpBytes)) ||
      (rc = o.kp.ensure((size_t)F * o.kp_stride * sizeof(rgbdslam_b200_keypoint))) ||
      (rc = o.xyz.ensure((size_t)F * o.kp_stride * 16)) || (rc = o.n.ensure((size_t)F * 4)) ||
      (rc = o.pyr_raw.ensure((size_t)g.full_bytes * F)) || (rc = o.pyr_blur.ensure((size_t)g.full_bytes * F)) ||
      (rc = o.desc.ensure((size_t)F * o.kp_stride * 32)) || (rc = o.err.ensure(16)) ||
      (rc = o.trig.ensure((size_t)F * o.kp_stride * 8)))
    return rc;
  return 0;
}

static Detector* get_detector(uint64_t h) {
  Detector* d = (Detector*)(uintptr_t)h;
  if (!d || d->magic != Detector::kMagic) {
    set_error("invalid detector handle");
    return nullptr;
  }
  return d;
}

// the detector's thresholds live on the device while frames are being processed; the host mirror is refreshed on demand
static int detector_to_device(Detector* det, cudaStream_t st) {
  int rc;
  if ((rc = det->d_state.ensure(sizeof(double) * kOrbMaxCells))) return rc;
  if (!det->dev_valid) {
    cudaError_t e = cudaMemcpyAsync(det->d_state.ptr, det->thresh, sizeof(double) * kOrbMaxCells, cudaMemcpyHostToDevice, st);
    if (e != cudaSuccess) return cuda_fail(e, "detector state upload");
    det->dev_valid = true;
  }
  return 0;
}
static int detector_to_host(Detector* det) {
  if (det->host_valid) return 0;
  cudaError_t e = cudaMemcpy(det->thresh, det->d_state.ptr, sizeof(double) * kOrbMaxCells, cudaMemcpyDeviceToHost);
  if (e != cudaSuccess) return cuda_fail(e, "detector state download");
  det->host_valid = true;
  return 0;
}

// detection stage for F frames resident at d_gray / d_mask (or the mask derived from d_depth_for_mask): candidates,
// histograms, and the adaptive-threshold recurrence of the F frames in order -- all queued on `st`, no host round trip
static int orb_detect_stage(Detector* det, int F, const uint8_t* d_gray, const uint8_t* d_mask, const float* d_depth_for_mask,
                            cudaStream_t st, int* launches) {
  State& s = g_state;
  OrbCtx& o = g_orb;
  const OrbGeom& g = o.g;
  int rc;
  if ((rc = detector_to_device(det, st))) return rc;
  cudaError_t e = orb_run_detect(g, o.tab, F, d_gray, d_mask, d_depth_for_mask, det->type, (uint8_t*)o.cell_img.ptr,
                                 (uint8_t*)o.cell_mask.ptr,
                                 (OrbCand*)o.cand.ptr, (int*)o.cand_count.ptr, (int*)o.hist.ptr,
                                 (int*)o.mask_any.ptr, st, launches);
  if (e != cudaSuccess) return cuda_fail(e, "orb detect kernels");
  e = orb_run_adapt(g, F, (const int*)o.hist.ptr, (const int*)o.cand_count.ptr, (const int*)o.mask_any.ptr, (double*)det->d_state.ptr,
                    (int*)o.thr.ptr, o.min_cell, o.max_cell, s.params.adjuster_max_iterations, (int*)o.err.ptr, st, launches);
  if (e != cudaSuccess) return cuda_fail(e, "orb threshold kernel");
  det->host_valid = false;
  return 0;
}

static int orb_check_err_flag(int flag) {
  if (flag & 1) {
    set_error("ORB / FAST candidate buffer overflow (more than 12288 FAST corners in one grid cell)");
    return RGBDSLAM_B200_ERR_STATE;
  }
  return 0;
}

static bool is_pinned(const void* p) {
  cudaPointerAttributes a;
  if (cudaPointerGetAttributes(&a, p) != cudaSuccess) {
    cudaGetLastError();
    return false;
  }
  return a.type == cudaMemoryTypeHost;
}

// Argument checks shared by nodes_create_ex and nodes_create_sharded (before any device work).
static int check_nodes_args(const char* what, const Detector* det, int nframes, const float* K4, const uint64_t* node_handles,
                            int flags) {
  constexpr int kAll = RGBDSLAM_B200_MASK_FROM_DEPTH | RGBDSLAM_B200_VISUAL_RGB | RGBDSLAM_B200_CLOUD_XYZRGB | RGBDSLAM_B200_CLOUD_XYZ |
                       RGBDSLAM_B200_MASK_FROM_CLOUD | RGBDSLAM_B200_KEEP_CLOUD | RGBDSLAM_B200_DEPTH_U16 |
                       RGBDSLAM_B200_VISUAL_BAYER_GR | RGBDSLAM_B200_STORE_CLOUD | RGBDSLAM_B200_ENCODING_RGB;
  const bool cloud = (flags & (RGBDSLAM_B200_CLOUD_XYZRGB | RGBDSLAM_B200_CLOUD_XYZ)) != 0;
  const char* bad = nullptr;
  if (flags & ~kAll) bad = "unknown flag bits";
  else if ((flags & RGBDSLAM_B200_CLOUD_XYZRGB) && (flags & RGBDSLAM_B200_CLOUD_XYZ)) bad = "CLOUD_XYZRGB and CLOUD_XYZ are exclusive";
  else if ((flags & RGBDSLAM_B200_MASK_FROM_CLOUD) && !cloud) bad = "MASK_FROM_CLOUD needs CLOUD_XYZRGB or CLOUD_XYZ";
  else if ((flags & RGBDSLAM_B200_MASK_FROM_DEPTH) && cloud) bad = "MASK_FROM_DEPTH needs a depth image, not a cloud (MASK_FROM_CLOUD)";
  else if ((flags & RGBDSLAM_B200_KEEP_CLOUD) && !cloud) bad = "KEEP_CLOUD needs CLOUD_XYZRGB or CLOUD_XYZ";
  else if ((flags & RGBDSLAM_B200_DEPTH_U16) && cloud) bad = "DEPTH_U16 describes a depth image, not a cloud";
  else if ((flags & RGBDSLAM_B200_VISUAL_BAYER_GR) && (flags & RGBDSLAM_B200_VISUAL_RGB))
    bad = "VISUAL_BAYER_GR and VISUAL_RGB are exclusive";
  else if ((flags & RGBDSLAM_B200_VISUAL_BAYER_GR) && cloud) bad = "VISUAL_BAYER_GR needs a depth image, not a cloud";
  else if ((flags & RGBDSLAM_B200_ENCODING_RGB) && !(flags & RGBDSLAM_B200_STORE_CLOUD)) bad = "ENCODING_RGB needs STORE_CLOUD";
  if (bad) {
    set_error(std::string(what) + ": " + bad);
    return RGBDSLAM_B200_ERR_ARG;
  }
  // the point-cloud constructor takes its points from the cloud: no intrinsics
  if (!det || nframes < 0 || (nframes > 0 && ((!K4 && !cloud) || !node_handles))) {
    set_error(std::string(what) + ": bad arguments");
    return RGBDSLAM_B200_ERR_ARG;
  }
  return 0;
}

// The nodes of one nodes_create* call share one device allocation (no per-node cudaMalloc), every region 256-byte aligned:
// [desc nodes x K x 32][xyz nodes x K x 16][n nodes x 4][kp kp_frames x K x 28]
struct NodeBatch {
  NodeSlab* slab = nullptr;
  int K = 0;  // feature rows per node
  uint8_t* desc = nullptr;
  float4* xyz = nullptr;
  int* n = nullptr;
  size_t n_bytes = 0;
  rgbdslam_b200_keypoint* kp = nullptr;
  // Node::pc_col of every node in one more allocation (pc.slab; none when the call keeps no cloud), pc_node_words 4-byte words
  // per node: depth-image input [z] at the skip-step raster, cloud input [x | y | z] at w x h, each plus [colour] for
  // STORE_CLOUD.  pc holds frame 0's planes.
  NodeCloud pc;
  size_t pc_node_words = 0;
};

static int batch_alloc(NodeBatch& nb, int nodes, int kp_frames, int K) {
  auto up = [](size_t v) { return (v + 255) / 256 * 256; };
  const size_t b_desc = up((size_t)nodes * K * 32), b_xyz = up((size_t)nodes * K * 16), b_n = up((size_t)nodes * 4);
  const size_t b_kp = up((size_t)kp_frames * K * sizeof(rgbdslam_b200_keypoint));
  nb.slab = new NodeSlab();
  cudaError_t e = cudaMalloc(&nb.slab->base, b_desc + b_xyz + b_n + b_kp);
  if (e != cudaSuccess) {
    delete nb.slab;
    nb.slab = nullptr;
    return cuda_fail(e, "cudaMalloc(node slab)");
  }
  nb.K = K;
  nb.desc = (uint8_t*)nb.slab->base;
  nb.xyz = (float4*)(nb.desc + b_desc);
  nb.n = (int*)((uint8_t*)nb.xyz + b_xyz);
  nb.n_bytes = b_n;
  nb.kp = (rgbdslam_b200_keypoint*)((uint8_t*)nb.n + b_n);
  return 0;
}

// Failure after batch_alloc: waits for the work already queued on both streams, frees what the batch owns, returns code.
static int batch_fail(NodeBatch& nb, int code) {
  cudaStreamSynchronize(g_orb.copy_stream);
  cudaStreamSynchronize(g_state.stream);
  cudaFree(nb.slab->base);
  delete nb.slab;
  if (nb.pc.slab) {
    cudaFree(nb.pc.slab->base);
    delete nb.pc.slab;
  }
  return code;
}

// Frame input of a nodes_create* call: the caller's buffers are copied from directly when they are pinned, else through the two
// pinned staging buffers (chunk frames each).
static int setup_staging(const uint8_t* gray, const float* depth, const uint8_t* mask, size_t px, const FrameInput& in, int chunk,
                         bool* pinned) {
  OrbCtx& o = g_orb;
  *pinned = is_pinned(gray) && is_pinned(depth) && (!mask || is_pinned(mask));
  if (*pinned) return 0;
  const size_t bytes = (in.gray_bytes + in.depth_bytes + (mask ? px : 0)) * chunk;
  int rc;
  if ((rc = o.stage[0].ensure(bytes)) || (rc = o.stage[1].ensure(bytes))) return rc;
  return 0;
}

// Host -> device copy of the F frames of chunk ci (visual image, depth image or cloud, optional mask) into dg / dd / dm on the
// copy stream, through staging buffer ci & 1 unless pinned.  The copy stream first waits for `after` (if given); the compute
// stream waits for the copy.
static int upload_chunk(int ci, int F, int chunk, size_t px, const FrameInput& in, bool pinned, const uint8_t* hg, const float* hd,
                        const uint8_t* hm, uint8_t* dg, void* dd, uint8_t* dm, cudaEvent_t after) {
  OrbCtx& o = g_orb;
  const int b = ci & 1;
  const size_t gb = in.gray_bytes, db = in.depth_bytes;
  cudaStream_t cs = o.copy_stream;
  if (!pinned) {  // the previous copy out of this staging buffer must have finished
    if (ci >= 2) RB200_CUDA(cudaEventSynchronize(o.ev_copied[b]));
    uint8_t* sp = (uint8_t*)o.stage[b].ptr;
    memcpy(sp, hg, gb * F);
    memcpy(sp + gb * chunk, hd, db * F);
    if (hm) memcpy(sp + (gb + db) * chunk, hm, px * F);
    hg = sp;
    hd = (const float*)(sp + gb * chunk);
    if (hm) hm = sp + (gb + db) * chunk;
  }
  if (after) RB200_CUDA(cudaStreamWaitEvent(cs, after, 0));
  RB200_CUDA(cudaMemcpyAsync(dg, hg, gb * F, cudaMemcpyHostToDevice, cs));
  RB200_CUDA(cudaMemcpyAsync(dd, hd, db * F, cudaMemcpyHostToDevice, cs));
  if (hm) RB200_CUDA(cudaMemcpyAsync(dm, hm, px * F, cudaMemcpyHostToDevice, cs));
  RB200_CUDA(cudaEventRecord(o.ev_ready[b], cs));
  RB200_CUDA(cudaEventRecord(o.ev_copied[b], cs));
  RB200_CUDA(cudaStreamWaitEvent(g_state.stream, o.ev_ready[b], 0));
  return 0;
}

// The input kernels of a chunk of F frames: cvtColor of the colour or Bayer visuals drgb into dg, the conversion of the 16-bit
// depth images draw into dd (and their mask into dm), calculateDepthMask of the clouds dd into dm.
static cudaError_t chunk_inputs(const FrameInput& in, int F, size_t px, const uint8_t* drgb, uint8_t* dg, const uint16_t* draw,
                                float* dd, uint8_t* dm, cudaStream_t st, int* launches) {
  cudaError_t e = cudaSuccess;
  if (in.rgb) e = orb_run_rgb_to_gray(F, px, drgb, dg, st, launches);
  if (in.bayer) e = orb_run_bayer_gr_to_gray(F, g_orb.g.W, g_orb.g.H, drgb, dg, st, launches);
  if (e == cudaSuccess && in.depth_u16) e = orb_run_depth_u16(F, px, draw, dd, in.mask_from_u16 ? dm : nullptr, st, launches);
  if (e == cudaSuccess && in.mask_from_cloud) e = orb_run_cloud_mask(F, px, dd, in.cloud_stride, dm, st, launches);
  return e;
}

// Where the features of a chunk go: `stride` rows per frame (slab rows f0... of a nodes_create* call).
struct FeatureRows {
  rgbdslam_b200_keypoint* kp;
  float4* xyz;
  int* n;
  uint8_t* desc;  // mode 1
  int stride;
};

// Harris / keepStrongest / finalize of F detected frames (cell pyramids cell_img, candidates c, depth images or clouds dd)
// into `out`; in mode 1 also extractor->compute() on the grey images dg.
static int select_describe(const Detector* det, const FrameInput& in, int F, const uint8_t* cell_img, const OrbCandidates& c,
                           const float* dd, const uint8_t* dg, const FeatureRows& out, cudaStream_t st, int* launches) {
  OrbCtx& o = g_orb;
  OrbFrameArgs a;
  a.cell_out = (unsigned long long*)o.cell_out.ptr;
  a.cell_out_count = (int*)o.cell_out_count.ptr;
  a.out_stride = o.max_per_cell;
  a.depth = dd;
  a.cloud_stride = in.cloud_stride;
  a.cand_z = (float*)o.cand_z.ptr;
  a.cell_img = cell_img;
  a.depth_scaling = in.depth_scaling;
  a.Kinv = in.Kinv;
  a.scratch = o.scratch.ptr;
  a.kp_out = out.kp;
  a.xyz_out = out.xyz;
  a.trig_out = (float2*)o.trig.ptr;
  a.n_out = out.n;
  a.kp_stride = out.stride;
  a.max_keypoints = g_state.params.max_keypoints;
  a.mode = in.mode;
  cudaError_t e = orb_run_select(o.g, F, det->type, in.points, c, a, st, launches);
  if (e != cudaSuccess) return cuda_fail(e, "orb select kernels");
  if (in.mode == 1) {
    e = orb_run_describe(o.g, o.tab, F, det->describe_levels(), dg, (uint8_t*)o.pyr_raw.ptr, (uint8_t*)o.pyr_blur.ptr, out.kp, out.n,
                         out.stride, out.stride, a.trig_out, out.desc, st, launches);
    if (e != cudaSuccess) return cuda_fail(e, "orb describe kernels");
  }
  return 0;
}

// End of a nodes_create* call: waits for it, checks the device error flag and hands out one node per frame -- features of
// frame f at slab row f * K, 2-D keypoints only for frames [kp_first, kp_first + kp_frames).  Frees the batch on failure.
static int batch_publish(NodeBatch& nb, int nframes, int kp_first, int kp_frames, const int32_t* ids, uint64_t* node_handles,
                         int32_t* n_features, const char* what) {
  OrbCtx& o = g_orb;
  cudaStream_t st = g_state.stream;
  std::vector<int> n(nframes);
  int flag = 0;
  cudaError_t e = cudaMemcpyAsync(n.data(), nb.n, 4 * (size_t)nframes, cudaMemcpyDeviceToHost, st);
  if (e == cudaSuccess) e = cudaMemcpyAsync(&flag, o.err.ptr, 4, cudaMemcpyDeviceToHost, st);
  if (e == cudaSuccess) e = cudaStreamSynchronize(st);
  if (e == cudaSuccess) e = cudaStreamSynchronize(o.copy_stream);
  if (e != cudaSuccess) return batch_fail(nb, cuda_fail(e, what));
  if (int rc = orb_check_err_flag(flag)) return batch_fail(nb, rc);
  const int K = nb.K, Kpad = ((K > 0 ? K : 1) + 255) / 256 * 256;
  for (int f = 0; f < nframes; f++) {
    NodeDev* nd = new NodeDev();
    nd->magic = NodeDev::kMagic;
    nd->id = ids ? ids[f] : f;
    nd->n = n[f];
    nd->n_pad = Kpad;
    nd->desc = nb.desc + (size_t)f * K * 32;
    nd->xyz = nb.xyz + (size_t)f * K;
    nd->kp = (f >= kp_first && f < kp_first + kp_frames) ? nb.kp + (size_t)(f - kp_first) * K : nullptr;
    nd->slab = nb.slab;
    nb.slab->refs++;
    if (nb.pc.slab) {
      NodeCloud& c = nd->pc;
      c = nb.pc;
      const size_t off = nb.pc_node_words * f;
      for (float** plane : {&c.x, &c.y, &c.z})
        if (*plane) *plane += off;
      if (c.rgb) c.rgb += off;
      nb.pc.slab->refs++;
    }
    node_handles[f] = (uint64_t)(uintptr_t)nd;
    if (n_features) n_features[f] = n[f];
  }
  return 0;
}

}  // namespace rb200

using namespace rb200;

extern "C" {

int rgbdslam_b200_detector_create(uint64_t* detector) {
  if (!detector) {
    set_error("detector_create: null output");
    return RGBDSLAM_B200_ERR_ARG;
  }
  int type;
  {
    std::lock_guard<std::mutex> lk(g_state.mu);
    type = g_state.params.feature_detector_type;  // validated by rgbdslam_b200_init; 0 (ORB) before it
  }
  *detector = (uint64_t)(uintptr_t) new Detector(type);
  return 0;
}
int rgbdslam_b200_detector_destroy(uint64_t detector) {
  std::lock_guard<std::mutex> lk(g_state.mu);
  Detector* d = get_detector(detector);
  if (!d) return RGBDSLAM_B200_ERR_ARG;
  if (g_state.inited) {
    cudaSetDevice(g_state.device);
    cudaStreamSynchronize(g_state.stream);
  }
  d->d_state.release();
  d->magic = 0;
  delete d;
  return 0;
}
int rgbdslam_b200_detector_thresholds(uint64_t detector, double* thresholds16, int set) {
  std::lock_guard<std::mutex> lk(g_state.mu);
  Detector* d = get_detector(detector);
  if (!d) return RGBDSLAM_B200_ERR_ARG;
  if (!thresholds16) {
    set_error("detector_thresholds: null thresholds");
    return RGBDSLAM_B200_ERR_ARG;
  }
  if (!d->host_valid) {
    int rc = check_inited();
    if (rc) return rc;
    cudaError_t e = cudaStreamSynchronize(g_state.stream);
    if (e != cudaSuccess) return cuda_fail(e, "detector_thresholds");
    if ((rc = detector_to_host(d))) return rc;
  }
  for (int i = 0; i < kOrbMaxCells; i++) {
    if (set) d->thresh[i] = thresholds16[i];
    else thresholds16[i] = d->thresh[i];
  }
  if (set) d->dev_valid = false;
  return 0;
}

int rgbdslam_b200_orb_detect(uint64_t detector, const uint8_t* gray, const uint8_t* mask, int w, int h,
                             rgbdslam_b200_keypoint* kp_out, int capacity, int* n_out) {
  RB200_ENTER_INITED();
  Detector* det = get_detector(detector);
  if (!det || !gray || !kp_out || !n_out || capacity < 0) {
    set_error("orb_detect: bad arguments");
    return RGBDSLAM_B200_ERR_ARG;
  }
  int rc;
  if ((rc = orb_prepare(w, h)) || (rc = orb_ensure_buffers(1, 1, true))) return rc;
  OrbCtx& o = g_orb;
  cudaStream_t st = g_state.stream;
  const size_t px = (size_t)w * h;
  cudaError_t e = cudaMemsetAsync(o.err.ptr, 0, 4, st);
  if (e == cudaSuccess) e = cudaMemcpyAsync(o.in_gray[0].ptr, gray, px, cudaMemcpyHostToDevice, st);
  if (e == cudaSuccess && mask) e = cudaMemcpyAsync(o.in_mask[0].ptr, mask, px, cudaMemcpyHostToDevice, st);
  if (e != cudaSuccess) return cuda_fail(e, "orb_detect upload");
  o.last_gray = (const uint8_t*)o.in_gray[0].ptr;
  int launches = 0;
  if ((rc = orb_detect_stage(det, 1, (const uint8_t*)o.in_gray[0].ptr, mask ? (const uint8_t*)o.in_mask[0].ptr : nullptr, nullptr, st,
                             &launches)))
    return rc;
  const FeatureRows rows = {(rgbdslam_b200_keypoint*)o.kp.ptr, (float4*)o.xyz.ptr, (int*)o.n.ptr, nullptr, o.kp_stride};
  if ((rc = select_describe(det, FrameInput(), 1, (const uint8_t*)o.cell_img.ptr, o.candidates(), nullptr, nullptr, rows, st,
                            &launches)))
    return rc;
  int n = 0, flag = 0;
  e = cudaMemcpyAsync(&n, o.n.ptr, 4, cudaMemcpyDeviceToHost, st);
  if (e == cudaSuccess) e = cudaMemcpyAsync(&flag, o.err.ptr, 4, cudaMemcpyDeviceToHost, st);
  if (e == cudaSuccess) e = cudaStreamSynchronize(st);
  if (e != cudaSuccess) return cuda_fail(e, "orb_detect download count");
  if ((rc = orb_check_err_flag(flag))) return rc;
  *n_out = n;
  const int m = n < capacity ? n : capacity;
  if (m > 0) {
    e = cudaMemcpyAsync(kp_out, o.kp.ptr, sizeof(rgbdslam_b200_keypoint) * m, cudaMemcpyDeviceToHost, st);
    if (e == cudaSuccess) e = cudaStreamSynchronize(st);
    if (e != cudaSuccess) return cuda_fail(e, "orb_detect download keypoints");
  }
  g_state.launches += launches;
  return 0;
}

int rgbdslam_b200_orb_compute(const uint8_t* gray, int w, int h, const rgbdslam_b200_keypoint* kp_in, int n_in,
                              rgbdslam_b200_keypoint* kp_out, uint8_t* desc_out, int* n_out) {
  RB200_ENTER_INITED();
  if (!gray || n_in < 0 || (n_in > 0 && (!kp_in || !kp_out || !desc_out)) || !n_out) {
    set_error("orb_compute: bad arguments");
    return RGBDSLAM_B200_ERR_ARG;
  }
  int rc;
  if ((rc = orb_prepare(w, h)) || (rc = orb_ensure_buffers(1, 1, true))) return rc;
  OrbCtx& o = g_orb;
  // cv::ORB::compute: runByImageBorder(31) on cvRound'ed coordinates, then group by octave (stable)
  std::vector<rgbdslam_b200_keypoint> kept;
  kept.reserve(n_in);
  for (int i = 0; i < n_in; i++) {
    const rgbdslam_b200_keypoint& k = kp_in[i];
    if (k.octave < 0 || k.octave >= kOrbLevels) {
      set_error("orb_compute: keypoint octave outside [0,8)");
      return RGBDSLAM_B200_ERR_ARG;
    }
    const long rx = lrintf(k.x), ry = lrintf(k.y);
    if (rx >= 31 && rx < w - 31 && ry >= 31 && ry < h - 31) kept.push_back(k);
  }
  std::stable_sort(kept.begin(), kept.end(),
                   [](const rgbdslam_b200_keypoint& a, const rgbdslam_b200_keypoint& b) { return a.octave < b.octave; });
  const int n = (int)kept.size();
  *n_out = n;
  if (n == 0) return 0;
  DevBuf dk, dd;  // keypoint counts are caller-sized here, not bounded by kp_stride
  if ((rc = dk.ensure(sizeof(rgbdslam_b200_keypoint) * (size_t)n)) || (rc = dd.ensure(32 * (size_t)n))) { dk.release(); dd.release(); return rc; }
  cudaStream_t st = g_state.stream;
  int launches = 0;
  cudaError_t e = cudaMemcpyAsync(o.in_gray[0].ptr, gray, (size_t)w * h, cudaMemcpyHostToDevice, st);
  if (e == cudaSuccess) e = cudaMemcpyAsync(dk.ptr, kept.data(), sizeof(rgbdslam_b200_keypoint) * (size_t)n, cudaMemcpyHostToDevice, st);
  if (e == cudaSuccess) e = cudaMemcpyAsync(o.n.ptr, &n, 4, cudaMemcpyHostToDevice, st);
  if (e == cudaSuccess)
    e = orb_run_describe(o.g, o.tab, 1, kOrbLevels, (const uint8_t*)o.in_gray[0].ptr, (uint8_t*)o.pyr_raw.ptr, (uint8_t*)o.pyr_blur.ptr,
                         (const rgbdslam_b200_keypoint*)dk.ptr, (const int*)o.n.ptr, n, n, nullptr, (uint8_t*)dd.ptr, st, &launches);
  if (e == cudaSuccess) e = cudaMemcpyAsync(desc_out, dd.ptr, 32 * (size_t)n, cudaMemcpyDeviceToHost, st);
  if (e == cudaSuccess) e = cudaStreamSynchronize(st);
  dk.release();
  dd.release();
  if (e != cudaSuccess) return cuda_fail(e, "orb_compute");
  memcpy(kp_out, kept.data(), sizeof(rgbdslam_b200_keypoint) * (size_t)n);
  g_state.launches += launches;
  return 0;
}

// Node::Node for nframes frames in order.  Pipeline per chunk of kOrbChunk frames:
//   copy stream    : host -> device of the chunk's gray / depth / mask into one of two input buffers (straight from the caller's
//                    buffers when they are pinned, else through pinned staging filled by this thread)
//   compute stream : detect kernels -> threshold recurrence (device) -> Harris / keepStrongest / finalize -> describe, writing
//                    straight into the slab that holds all nodes of the call (no per-node allocation, no device->device copy)
// The only host synchronisation is the download of the feature counts at the end.
int rgbdslam_b200_nodes_create_ex(uint64_t detector, int nframes, const uint8_t* gray, const float* depth, const uint8_t* mask,
                                  int w, int h, const float* K4, const int32_t* ids, int flags, uint64_t* node_handles,
                                  int32_t* n_features) {
  RB200_ENTER_INITED();
  Detector* det = get_detector(detector);
  int rc;
  if ((rc = check_nodes_args("nodes_create", det, nframes, K4, node_handles, flags))) return rc;
  if (nframes > 0 && (!gray || !depth)) {
    set_error("nodes_create: null image buffers");
    return RGBDSLAM_B200_ERR_ARG;
  }
  if (nframes == 0) return 0;
  State& s = g_state;
  const size_t px = (size_t)w * h;
  const FrameInput in(flags, px, s.params, K4, mask);
  const bool store = (flags & RGBDSLAM_B200_STORE_CLOUD) != 0, model = s.params.observability_threshold > 0.0;
  // a stored cloud of cloud input is the kept cloud plus colour: the measurement model reads it as it reads KEEP_CLOUD's
  const bool keep_cloud = (flags & RGBDSLAM_B200_KEEP_CLOUD) != 0 || (store && in.cloud_stride);
  const int pc_step = s.params.cloud_creation_skip_step > 0 ? s.params.cloud_creation_skip_step : 1;
  if (store && !in.cloud_stride && (w % pc_step != 0 || h % pc_step != 0)) {
    // the reference warns that this "will most likely crash" (misc.cpp:479-481): its index arithmetic reads the wrong pixels
    set_error("nodes_create: STORE_CLOUD needs a cloud_creation_skip_step that divides the image width and height");
    return RGBDSLAM_B200_ERR_ARG;
  }
  if (in.cloud_stride && !keep_cloud && model) {
    set_error("nodes_create: the environment measurement model needs the point cloud on the node (observability_threshold > 0): "
              "pass RGBDSLAM_B200_KEEP_CLOUD");
    return RGBDSLAM_B200_ERR_STATE;
  }
  if (!in.caller_mask) mask = nullptr;
  if ((rc = orb_prepare(w, h)) || (rc = orb_ensure_streams())) return rc;
  OrbCtx& o = g_orb;
  const int chunk = in.chunk(nframes, px);
  if ((rc = orb_ensure_buffers(chunk, 2, in.mask_buffer(), in.plane_bytes, in.raw_visual() ? in.gray_bytes : 0,
                               in.depth_u16 ? in.depth_bytes : 0)))
    return rc;
  cudaStream_t st = s.stream;
  const int K = std::min(o.kp_stride, s.params.max_keypoints);  // features per node (finalize mode 1 emits <= max_keypoints)
  NodeBatch nb;
  if ((rc = batch_alloc(nb, nframes, nframes, K))) return rc;
  if (store || keep_cloud || model) {  // Node::pc_col (node.cpp:126-131, 261) of every frame, allocated before any work is queued
    NodeCloud& c = nb.pc;
    c.step = in.cloud_stride ? 0 : pc_step;
    c.w = in.cloud_stride ? w : (w + pc_step - 1) / pc_step;  // ceil(cols / skip), misc.cpp:482-483
    c.h = in.cloud_stride ? h : (h + pc_step - 1) / pc_step;
    // kept clouds: the camera the model projects into, depth_camera_fx ... cy, 0 when unset (misc.cpp:56-63)
    for (int k = 0; k < 4; k++) c.K[k] = K4 ? K4[k] : 0.f;
    const size_t P = (size_t)c.w * c.h;
    nb.pc_node_words = (P * ((in.cloud_stride ? 3 : 1) + (store ? 1 : 0)) + 63) / 64 * 64;
    c.slab = new NodeSlab();
    cudaError_t e = cudaMalloc(&c.slab->base, 4 * nb.pc_node_words * nframes);
    if (e != cudaSuccess) {
      delete c.slab;
      c.slab = nullptr;
      return batch_fail(nb, cuda_fail(e, "cudaMalloc(node clouds)"));
    }
    float* planes = (float*)c.slab->base;
    if (in.cloud_stride) {
      c.x = planes;
      c.y = planes + P;
      planes += 2 * P;
    }
    c.z = planes;
    if (store) c.rgb = (uint32_t*)(planes + P);
  }
  bool pinned = false;
  if ((rc = setup_staging(gray, depth, mask, px, in, chunk, &pinned))) return batch_fail(nb, rc);
  cudaError_t e = cudaMemsetAsync(o.err.ptr, 0, 4, st);
  // the copy stream must not run ahead of work already queued on the compute stream that still reads the input buffers
  if (e == cudaSuccess) e = cudaEventRecord(o.ev_free[0], st);
  if (e == cudaSuccess) e = cudaEventRecord(o.ev_free[1], st);
  if (e != cudaSuccess) return batch_fail(nb, cuda_fail(e, "nodes_create setup"));
  int launches = 0, ci = 0;
  for (int f0 = 0; f0 < nframes; f0 += chunk, ci++) {
    const int F = std::min(chunk, nframes - f0), b = ci & 1;
    uint8_t* dg = (uint8_t*)o.in_gray[b].ptr;
    float* dd = (float*)o.in_depth[b].ptr;
    uint8_t* drgb = (uint8_t*)o.in_rgb[b].ptr;
    uint16_t* draw = (uint16_t*)o.in_raw[b].ptr;
    uint8_t* dm = in.mask_buffer() ? (uint8_t*)o.in_mask[b].ptr : nullptr;
    if ((rc = upload_chunk(ci, F, chunk, px, in, pinned, gray + in.gray_bytes * f0, (const float*)((const uint8_t*)depth + in.depth_bytes * f0),
                           mask ? mask + px * f0 : nullptr, in.raw_visual() ? drgb : dg, in.depth_u16 ? (void*)draw : dd,
                           mask ? dm : nullptr, o.ev_free[b])))
      return batch_fail(nb, rc);
    if (f0 == 0) o.last_gray = dg;
    if ((e = chunk_inputs(in, F, px, drgb, dg, draw, dd, dm, st, &launches)) != cudaSuccess)
      return batch_fail(nb, cuda_fail(e, "nodes_create input kernels"));
    if ((rc = orb_detect_stage(det, F, dg, dm, in.mask_from_depth ? dd : nullptr, st, &launches))) return batch_fail(nb, rc);
    const FeatureRows rows = {nb.kp + (size_t)f0 * K, nb.xyz + (size_t)f0 * K, nb.n + f0, nb.desc + (size_t)f0 * K * 32, K};
    if ((rc = select_describe(det, in, F, (const uint8_t*)o.cell_img.ptr, o.candidates(), dd, dg, rows, st, &launches)))
      return batch_fail(nb, rc);
    if (nb.pc.slab) {  // createXYZRGBPointCloud of the chunk's frames from the buffers it holds (misc.cpp:467-556, node.cpp:261)
      const size_t words = nb.pc_node_words;
      if (in.cloud_stride) {
        e = launch_store_cloud_points(F, dd, in.cloud_stride, (int)px, store, nb.pc.x + words * f0, words, st);
      } else {
        const int vis = in.bayer ? 2 : in.rgb ? 1 : 0;
        e = launch_store_depth_cloud(F, dd, store ? (vis ? drgb : dg) : nullptr, vis, (flags & RGBDSLAM_B200_ENCODING_RGB) == 0, w,
                                     h, pc_step, s.params.depth_scaling_factor, s.params.minimum_depth, nb.pc.z + words * f0, words,
                                     st);
      }
      if (e != cudaSuccess) return batch_fail(nb, cuda_fail(e, "store_cloud kernel"));
      launches += 1;
    }
    e = cudaEventRecord(o.ev_free[b], st);
    if (e != cudaSuccess) return batch_fail(nb, cuda_fail(e, "nodes_create events"));
  }
  if ((rc = batch_publish(nb, nframes, 0, nframes, ids, node_handles, n_features, "nodes_create finish"))) return rc;
  s.launches += launches;
  return 0;
}

// Frame-sharded Node construction: see include/rgbdslam_b200.h.  Two passes over the rank's own frames around ONE exchange of
// the score histograms; then one exchange of the finished features.
int rgbdslam_b200_nodes_create_sharded(uint64_t detector, uint64_t comm_handle, int total_frames, const uint8_t* gray,
                                       const float* depth, const uint8_t* mask, int w, int h, const float* K4, const int32_t* ids,
                                       int flags, uint64_t* node_handles, int32_t* n_features) {
  RB200_ENTER_INITED();
  if (flags & (RGBDSLAM_B200_KEEP_CLOUD | RGBDSLAM_B200_STORE_CLOUD)) {
    set_error("nodes_create_sharded: KEEP_CLOUD and STORE_CLOUD are not supported (the clouds are not exchanged between ranks)");
    return RGBDSLAM_B200_ERR_ARG;
  }
  Comm* cm = get_comm(comm_handle);
  if (!cm) return RGBDSLAM_B200_ERR_ARG;
  Detector* det = get_detector(detector);
  int rc;
  if ((rc = check_nodes_args("nodes_create_sharded", det, total_frames, K4, node_handles, flags))) return rc;
  if (total_frames == 0) return 0;
  State& s = g_state;
  if (s.params.observability_threshold > 0.0) {
    set_error("nodes_create_sharded: the environment measurement model needs every node's depth cloud on every rank (not exchanged)");
    return RGBDSLAM_B200_ERR_STATE;
  }
  const int world = cm->world, rank = cm->rank;
  const int per = (total_frames + world - 1) / world;
  const int f0 = std::min(rank * per, total_frames), f1 = std::min((rank + 1) * per, total_frames);
  const int own = f1 - f0, Wp = world * per;
  if (own > 0 && (!gray || !depth)) {
    set_error("nodes_create_sharded: null image buffers");
    return RGBDSLAM_B200_ERR_ARG;
  }
  const size_t px = (size_t)w * h;
  const FrameInput in(flags, px, s.params, K4, mask);
  if (!in.caller_mask) mask = nullptr;
  if ((rc = orb_prepare(w, h)) || (rc = orb_ensure_streams())) return rc;
  OrbCtx& o = g_orb;
  const OrbGeom& g = o.g;
  const int chunk = in.chunk(own, px);
  if ((rc = orb_ensure_buffers(chunk, 0, false))) return rc;
  const size_t nc = (size_t)g.ncells;
  const size_t own_ = (size_t)std::max(own, 1);
  if ((rc = o.sh_gray.ensure(px * own_)) || (rc = o.sh_depth.ensure(in.plane_bytes * own_)) ||
      (in.mask_buffer() && (rc = o.sh_mask.ensure(px * own_))) || (in.raw_visual() && (rc = o.sh_rgb.ensure(in.gray_bytes * own_))) ||
      (in.depth_u16 && (rc = o.sh_raw.ensure(in.depth_bytes * own_))) ||
      (rc = o.sh_cell_img.ensure((size_t)g.cell_bytes * own_)) || (rc = o.sh_cand.ensure(own_ * nc * kOrbCandCap * sizeof(OrbCand))) ||
      (rc = o.all_hist.ensure((size_t)Wp * nc * 256 * 4)) || (rc = o.all_cnt.ensure((size_t)Wp * nc * 4)) ||
      (rc = o.all_many.ensure((size_t)Wp * nc * 4)) || (rc = o.all_thr.ensure((size_t)Wp * nc * 4)))
    return rc;
  cudaStream_t st = s.stream, cs = o.copy_stream;
  const int K = std::min(o.kp_stride, s.params.max_keypoints);
  NodeBatch nb;  // descriptors, points and counts of all Wp frames; 2-D keypoints of the own frames
  if ((rc = batch_alloc(nb, Wp, (int)own_, K))) return rc;
  bool pinned = true;
  if (own > 0 && (rc = setup_staging(gray, depth, mask, px, in, chunk, &pinned))) return batch_fail(nb, rc);
  int* hist_all = (int*)o.all_hist.ptr;
  int* cnt_all = (int*)o.all_cnt.ptr;
  int* many_all = (int*)o.all_many.ptr;
  int* thr_all = (int*)o.all_thr.ptr;
  cudaError_t e = cudaMemsetAsync(o.err.ptr, 0, 4, st);
  if (e == cudaSuccess) e = cudaMemsetAsync(nb.n, 0, nb.n_bytes, st);
  // frames of the padding (Wp > total_frames) and of ranks without frames must read as "no candidates"
  if (e == cudaSuccess) e = cudaMemsetAsync(hist_all, 0, (size_t)Wp * nc * 256 * 4, st);
  if (e == cudaSuccess) e = cudaMemsetAsync(cnt_all, 0, (size_t)Wp * nc * 4, st);
  if (e == cudaSuccess) e = cudaMemsetAsync(many_all, 0, (size_t)Wp * nc * 4, st);
  if (e == cudaSuccess) e = cudaEventRecord(o.ev_free[0], st);  // uploads start after everything queued so far
  if (e == cudaSuccess) e = cudaStreamWaitEvent(cs, o.ev_free[0], 0);
  if (e != cudaSuccess) return batch_fail(nb, cuda_fail(e, "nodes_create_sharded setup"));
  int launches = 0, ci = 0;
  // ---- pass A: upload + pyramids + FAST / NMS candidates + score histograms of the own frames
  for (int c0 = 0; c0 < own; c0 += chunk, ci++) {
    const int F = std::min(chunk, own - c0);
    uint8_t* dg = (uint8_t*)o.sh_gray.ptr + px * c0;
    uint8_t* drgb = in.raw_visual() ? (uint8_t*)o.sh_rgb.ptr + in.gray_bytes * c0 : nullptr;
    uint16_t* draw = in.depth_u16 ? (uint16_t*)o.sh_raw.ptr + px * c0 : nullptr;
    float* dd = (float*)((uint8_t*)o.sh_depth.ptr + in.plane_bytes * c0);
    uint8_t* dm = in.mask_buffer() ? (uint8_t*)o.sh_mask.ptr + px * c0 : nullptr;
    if ((rc = upload_chunk(ci, F, chunk, px, in, pinned, gray + in.gray_bytes * c0, (const float*)((const uint8_t*)depth + in.depth_bytes * c0),
                           mask ? mask + px * c0 : nullptr, in.raw_visual() ? drgb : dg, in.depth_u16 ? (void*)draw : dd,
                           mask ? dm : nullptr, nullptr)))
      return batch_fail(nb, rc);
    if (c0 == 0) o.last_gray = dg;
    if ((e = chunk_inputs(in, F, px, drgb, dg, draw, dd, dm, st, &launches)) != cudaSuccess)
      return batch_fail(nb, cuda_fail(e, "nodes_create_sharded input kernels"));
    const size_t gf = (size_t)(f0 + c0);  // global index of the chunk's first frame
    e = orb_run_detect(g, o.tab, F, dg, dm, in.mask_from_depth ? dd : nullptr, det->type,
                       (uint8_t*)o.sh_cell_img.ptr + (size_t)g.cell_bytes * c0, (uint8_t*)o.cell_mask.ptr, (OrbCand*)o.sh_cand.ptr + (size_t)c0 * nc * kOrbCandCap,
                       cnt_all + gf * nc, hist_all + gf * nc * 256, many_all + gf * nc, st, &launches);
    if (e != cudaSuccess) return batch_fail(nb, cuda_fail(e, "orb detect kernels"));
  }
  // ---- the exchange that makes the frames independent: every rank gets every frame's score histograms, replays the
  //      threshold recurrence of the whole sequence (feature_adjuster.cpp:131-150, 185-224) and keeps its own frames' thresholds
  if (world > 1) {
    ncclResult_t r = g_nccl.AllGather(hist_all + (size_t)rank * per * nc * 256, hist_all, (size_t)per * nc * 256 * 4, 0, cm->comm, st);
    if (r == 0) r = g_nccl.AllGather(cnt_all + (size_t)rank * per * nc, cnt_all, (size_t)per * nc * 4, 0, cm->comm, st);
    if (r == 0) r = g_nccl.AllGather(many_all + (size_t)rank * per * nc, many_all, (size_t)per * nc * 4, 0, cm->comm, st);
    if (r != 0) return batch_fail(nb, nccl_fail(r, "ncclAllGather(histograms)"));
  }
  if ((rc = detector_to_device(det, st))) return batch_fail(nb, rc);
  e = orb_run_adapt(g, total_frames, hist_all, cnt_all, many_all, (double*)det->d_state.ptr, thr_all, o.min_cell, o.max_cell,
                    s.params.adjuster_max_iterations, (int*)o.err.ptr, st, &launches);
  if (e != cudaSuccess) return batch_fail(nb, cuda_fail(e, "orb threshold kernel"));
  det->host_valid = false;
  // ---- pass B: Harris / keepStrongest / finalize / describe of the own frames, straight into the slab
  for (int c0 = 0; c0 < own; c0 += chunk) {
    const int F = std::min(chunk, own - c0);
    const size_t gf = (size_t)(f0 + c0);
    const uint8_t* dg = (const uint8_t*)o.sh_gray.ptr + px * c0;
    const float* dd = (const float*)((const uint8_t*)o.sh_depth.ptr + in.plane_bytes * c0);
    const uint8_t* cimg = (const uint8_t*)o.sh_cell_img.ptr + (size_t)g.cell_bytes * c0;
    const OrbCandidates c = {(const OrbCand*)o.sh_cand.ptr + (size_t)c0 * nc * kOrbCandCap, cnt_all + gf * nc, thr_all + gf * nc,
                             (float*)o.resp.ptr};
    const FeatureRows rows = {nb.kp + (size_t)c0 * K, nb.xyz + gf * K, nb.n + gf, nb.desc + gf * K * 32, K};
    if ((rc = select_describe(det, in, F, cimg, c, dd, dg, rows, st, &launches))) return batch_fail(nb, rc);
  }
  // ---- every rank gets every node's features (48 KB per 1000-keypoint frame over NVLink)
  if (world > 1) {
    ncclResult_t r = g_nccl.AllGather(nb.desc + (size_t)rank * per * K * 32, nb.desc, (size_t)per * K * 32, 0, cm->comm, st);
    if (r == 0) r = g_nccl.AllGather((uint8_t*)(nb.xyz + (size_t)rank * per * K), nb.xyz, (size_t)per * K * 16, 0, cm->comm, st);
    if (r == 0) r = g_nccl.AllGather((uint8_t*)(nb.n + (size_t)rank * per), nb.n, (size_t)per * 4, 0, cm->comm, st);
    if (r != 0) return batch_fail(nb, nccl_fail(r, "ncclAllGather(features)"));
  }
  if ((rc = batch_publish(nb, total_frames, f0, own, ids, node_handles, n_features, "nodes_create_sharded finish"))) return rc;
  s.launches += launches;
  return 0;
}

int rgbdslam_b200_nodes_create(uint64_t detector, int nframes, const uint8_t* gray, const float* depth, const uint8_t* mask,
                               int w, int h, const float* K4, const int32_t* ids, uint64_t* node_handles, int32_t* n_features) {
  return rgbdslam_b200_nodes_create_ex(detector, nframes, gray, depth, mask, w, h, K4, ids, 0, node_handles, n_features);
}

/* Debug/inspection hook (used by tools/debug_orb.py and the tests): the FAST/NMS candidates of grid cell `cell` of
 * frame 0 of the last detect / nodes_create call: 8-byte records {u16 x, u16 y, u8 level, u8 score, u16 0} and their
 * responses as the detector of that call defines them -- Harris (ORB) or the corner score (FAST); NaN = below the cell's
 * final threshold. */
int rgbdslam_b200_orb_debug_candidates(int cell, void* cand_out, float* resp_out, int capacity, int* n_out, int* thr_out) {
  RB200_ENTER_INITED();
  OrbCtx& o = g_orb;
  if (!o.ready || cell < 0 || cell >= o.g.ncells || !n_out) {
    set_error("orb_debug_candidates: no detection has run / bad cell");
    return RGBDSLAM_B200_ERR_STATE;
  }
  int n = 0, thr = 0;
  cudaStream_t st = g_state.stream;
  cudaMemcpyAsync(&n, (const int*)o.cand_count.ptr + cell, 4, cudaMemcpyDeviceToHost, st);
  cudaMemcpyAsync(&thr, (const int*)o.thr.ptr + cell, 4, cudaMemcpyDeviceToHost, st);
  cudaError_t e = cudaStreamSynchronize(st);
  if (e != cudaSuccess) return cuda_fail(e, "orb_debug_candidates");
  *n_out = n;
  if (thr_out) *thr_out = thr;
  const int m = std::min(std::min(n, capacity), kOrbCandCap);
  if (m > 0 && cand_out) cudaMemcpyAsync(cand_out, (const OrbCand*)o.cand.ptr + (size_t)cell * kOrbCandCap, 8 * (size_t)m, cudaMemcpyDeviceToHost, st);
  if (m > 0 && resp_out) cudaMemcpyAsync(resp_out, (const float*)o.resp.ptr + (size_t)cell * kOrbCandCap, 4 * (size_t)m, cudaMemcpyDeviceToHost, st);
  e = cudaStreamSynchronize(st);
  if (e != cudaSuccess) return cuda_fail(e, "orb_debug_candidates copy");
  return 0;
}

int rgbdslam_b200_orb_debug_plane(int which, int cell, int level, uint8_t* out, int capacity, int* w_out, int* h_out) {
  RB200_ENTER_INITED();
  OrbCtx& o = g_orb;
  if (which < 0 || which == 2 || which > 4) {
    set_error("orb_debug_plane: which must be 0, 1, 3 or 4 (the FAST score map is never stored: scores stay in shared memory)");
    return RGBDSLAM_B200_ERR_ARG;
  }
  if (!o.ready || level < 0 || level >= kOrbLevels || !w_out || !h_out || (which <= 1 && (cell < 0 || cell >= o.g.ncells))) {
    set_error("orb_debug_plane: no detection has run / bad level or cell");
    return RGBDSLAM_B200_ERR_ARG;
  }
  const OrbPlane* p;
  const uint8_t* base;
  if (which <= 1) {
    p = &o.g.cell[cell][level];
    base = (const uint8_t*)(which == 0 ? o.cell_img.ptr : o.cell_mask.ptr);
  } else {
    p = &o.g.full[level];
    base = (const uint8_t*)(which == 3 ? o.pyr_raw.ptr : o.pyr_blur.ptr);
  }
  *w_out = p->w;
  *h_out = p->h;
  if (out && capacity >= p->w * p->h) {
    cudaError_t e = cudaMemcpyAsync(out, base + p->off, (size_t)p->w * p->h, cudaMemcpyDeviceToHost, g_state.stream);
    if (e == cudaSuccess) e = cudaStreamSynchronize(g_state.stream);
    if (e != cudaSuccess) return cuda_fail(e, "orb_debug_plane");
  }
  return 0;
}

int rgbdslam_b200_node_download_keypoints(uint64_t node_handle, rgbdslam_b200_keypoint* kp_out) {
  RB200_ENTER_INITED();
  NodeDev* nd = get_node(node_handle);
  if (!nd) return RGBDSLAM_B200_ERR_ARG;
  if (!kp_out) {
    set_error("node_download_keypoints: null output");
    return RGBDSLAM_B200_ERR_ARG;
  }
  if (!nd->kp) {
    set_error("node has no keypoints (it was created from features)");
    return RGBDSLAM_B200_ERR_STATE;
  }
  if (nd->n == 0) return 0;
  cudaError_t e = cudaMemcpyAsync(kp_out, nd->kp, sizeof(rgbdslam_b200_keypoint) * (size_t)nd->n, cudaMemcpyDeviceToHost, g_state.stream);
  if (e == cudaSuccess) e = cudaStreamSynchronize(g_state.stream);
  if (e != cudaSuccess) return cuda_fail(e, "node_download_keypoints");
  return 0;
}

}  // extern "C"
