// api.cu -- the extern "C" boundary declared in include/rgbdslam_b200.h.
// Host-side orchestration only: device memory, streams, workspaces, launches.  There is no CPU
// compute path in this file: every entry point that computes anything requires a CUDA device.
#include <cuda_runtime.h>

#include <cmath>
#include <cstdio>
#include <cstring>
#include <mutex>
#include <string>
#include <functional>
#include <vector>

#include "kernels.h"
#include "posegraph.h"
#include "state.h"

namespace rb200 {

static thread_local std::string t_last_error;
State g_state;

void set_error(const std::string& s) { t_last_error = s; }

int cuda_fail(cudaError_t e, const char* what) {
  char buf[512];
  snprintf(buf, sizeof(buf), "CUDA error in %s: %s (%s)", what, cudaGetErrorString(e), cudaGetErrorName(e));
  set_error(buf);
  return RGBDSLAM_B200_ERR_CUDA;
}

int DevBuf::ensure(size_t bytes) {
  if (bytes <= cap) return 0;
  if (ptr) cudaFree(ptr);
  ptr = nullptr;
  cap = 0;
  size_t want = bytes + bytes / 4 + 256;
  cudaError_t e = cudaMalloc(&ptr, want);
  if (e != cudaSuccess) return cuda_fail(e, "cudaMalloc(workspace)");
  cap = want;
  return 0;
}
void DevBuf::release() {
  if (ptr) cudaFree(ptr);
  ptr = nullptr;
  cap = 0;
}
int PinBuf::ensure(size_t bytes) {
  if (bytes <= cap) return 0;
  if (ptr) cudaFreeHost(ptr);
  ptr = nullptr;
  cap = 0;
  size_t want = bytes + bytes / 4 + 256;
  cudaError_t e = cudaMallocHost(&ptr, want);
  if (e != cudaSuccess) return cuda_fail(e, "cudaMallocHost(staging)");
  cap = want;
  return 0;
}
void PinBuf::release() {
  if (ptr) cudaFreeHost(ptr);
  ptr = nullptr;
  cap = 0;
}

static void make_dev_params(const rgbdslam_b200_params& p, double z0, DevParams& d) {
  d.min_matches = p.min_matches;
  d.max_matches = p.max_matches;
  d.ransac_iterations = p.ransac_iterations;
  d.pad_ = 0;
  d.max_dist_m = (float)p.max_dist_for_inliers;              // node.cpp:1105 (const float max_dist_m)
  d.sq_max_dist = (double)(d.max_dist_m * d.max_dist_m);     // node.cpp:1152 (float product promoted)
  d.sigma_depth = p.sigma_depth;
  if (p.depth_cov_z0 < 0) {
    d.cov_z_const = -1.0;
  } else {
    const double sd = p.sigma_depth * z0 * z0;  // misc2.h:20-35, first-call static cache
    d.cov_z_const = sd * sd;
  }
  // misc.cpp:702-709
  const double cam_angle_x = 58.0 / 180.0 * M_PI, cam_angle_y = 45.0 / 180.0 * M_PI;
  const double rsx = 3 * tan(cam_angle_x / 640), rsy = 3 * tan(cam_angle_y / 480);
  d.raster_cov_x = rsx * rsx;
  d.raster_cov_y = rsy * rsy;
}

int check_inited() {
  if (!g_state.inited) {
    set_error("rgbdslam_b200_init() has not been called");
    return RGBDSLAM_B200_ERR_STATE;
  }
  cudaError_t e = cudaSetDevice(g_state.device);
  if (e != cudaSuccess) return cuda_fail(e, "cudaSetDevice");
  return 0;
}

NodeDev* get_node(uint64_t h) {
  NodeDev* nd = (NodeDev*)(uintptr_t)h;
  if (!nd || nd->magic != NodeDev::kMagic) {
    set_error("invalid node handle");
    return nullptr;
  }
  return nd;
}

Workspace* get_slot(int slot) {
  if (slot < 0 || slot >= kSlots) {
    set_error("slot out of range [0,8)");
    return nullptr;
  }
  return &g_state.ws[slot];
}

// blocks until everything queued on the slot (and its edge all-gather) has finished
static int drain_slot(Workspace& w, const char* what) {
  cudaError_t e = cudaStreamSynchronize(w.stream);
  if (e == cudaSuccess && w.gather_pending) e = cudaEventSynchronize(w.ev_gather);
  if (e != cudaSuccess) return cuda_fail(e, what);
  w.pending = false;
  w.gather_pending = false;
  return 0;
}

// the timing events of the slot describe one match_pairs* call that has finished
static int check_finished_call(const Workspace& w, const char* what) {
  if (!w.timing_valid || w.pending) {
    set_error(std::string(what) + ": no finished match_pairs call on this slot (call match_pairs_wait first)");
    return RGBDSLAM_B200_ERR_STATE;
  }
  return 0;
}

static int push_dev_params() {
  State& s = g_state;
  make_dev_params(s.params, s.z0, s.dp);
  cudaError_t e = set_dev_params(s.dp, s.stream);
  if (e != cudaSuccess) return cuda_fail(e, "set_dev_params");
  // the constant upload reads s.dp asynchronously from pageable memory -> staged by the runtime; safe.
  return 0;
}

static inline int pad256(int n) { return ((n > 0 ? n : 1) + 255) / 256 * 256; }

// RootSIFT + bf16 tiles + norms of a set of SIFT nodes.
static int prepare_sift_nodes(Workspace& w, const std::vector<SiftJob>& jobs, int siftgpu = 0) {
  State& s = g_state;
  if (jobs.empty()) return 0;
  int rc;
  if ((rc = w.d_jobs.ensure(sizeof(SiftJob) * jobs.size()))) return rc;
  if ((rc = w.h_jobs.ensure(sizeof(SiftJob) * jobs.size()))) return rc;
  int max_pad = 0;
  for (const SiftJob& j : jobs) max_pad = j.n_pad > max_pad ? j.n_pad : max_pad;
  memcpy(w.h_jobs.ptr, jobs.data(), sizeof(SiftJob) * jobs.size());
  cudaError_t e = cudaMemcpyAsync(w.d_jobs.ptr, w.h_jobs.ptr, sizeof(SiftJob) * jobs.size(), cudaMemcpyHostToDevice, w.stream);
  if (e != cudaSuccess) return cuda_fail(e, "upload sift jobs");
  e = launch_sift_prepare((const SiftJob*)w.d_jobs.ptr, (int)jobs.size(), max_pad, s.params.use_root_sift ? 1 : 0, siftgpu, w.stream);
  if (e != cudaSuccess) return cuda_fail(e, "sift_prepare kernel");
  s.launches += 1;
  return 0;
}

// The pair table of a newer / older node pair.
static PairDesc make_pair(const NodeDev& a, const NodeDev& b) {
  PairDesc pd{};
  pd.q_desc = (const uint32_t*)a.desc;
  pd.t_desc = (const uint32_t*)b.desc;
  pd.q_xyz = a.xyz;
  pd.t_xyz = b.xyz;
  pd.nq = a.n;
  pd.nt = b.n;
  pd.id_q = a.id;
  pd.id_t = b.id;
  pd.q_i8 = a.desc_i8;
  pd.t_i8 = b.desc_i8;
  pd.q_f32 = a.desc_f32;
  pd.t_f32 = b.desc_f32;
  pd.t_norm = b.norms;
  pd.sift_kind = a.sift_kind;
  pd.q_kp = a.kp;
  pd.t_kp = b.kp;
  pd.q_cloud = a.pc.view();
  pd.t_cloud = b.pc.view();
  return pd;
}

// pair table -> w.d_pairs, through the slot's pinned staging (the copy may still be in flight when this returns)
static int upload_pairs(Workspace& w, const PairDesc* pairs, int npairs) {
  int rc;
  if ((rc = w.d_pairs.ensure(sizeof(PairDesc) * npairs)) || (rc = w.h_pairs.ensure(sizeof(PairDesc) * npairs))) return rc;
  memcpy(w.h_pairs.ptr, pairs, sizeof(PairDesc) * npairs);
  cudaError_t e = cudaMemcpyAsync(w.d_pairs.ptr, w.h_pairs.ptr, sizeof(PairDesc) * npairs, cudaMemcpyHostToDevice, w.stream);
  if (e != cudaSuccess) return cuda_fail(e, "upload pair table");
  return 0;
}

// Work items of the tensor-core match kernels (128- or 256-query blocks of every pair), staged on the stream.
// Returns the item count in *n_items.
// kind: 0 = ORB Hamming, 1 = SIFT bf16 scores (exact 2-NN matcher), 2 = SiftGPU matcher (u8 dots; one item set with the
// newer node's rows as queries and one with the roles swapped -- the row and the column pass of GetSiftMatch)
static int stage_match_items(Workspace& w, const PairDesc* h_pairs, int npairs, int stride, int kind, int* n_items) {
  State& s = g_state;
  *n_items = 0;
  const bool sift = kind != 0;
  if (!sift && s.hamming_path == 0) return 0;
  int rc;
  if (sift) {
    if ((rc = w.d_top4.ensure(sizeof(int4) * (size_t)npairs * stride))) return rc;
    if ((rc = w.d_knn.ensure(sizeof(float4) * (size_t)npairs * stride))) return rc;
  }
  // work items: 256 queries of one pair against 128-row train tiles (every tensor-core kernel).  The ORB kernel gets the 32-byte
  // descriptors themselves (its binary GEMM's operands); the float-descriptor matchers read the bf16 / u8 operand tiles their
  // nodes keep resident.
  const bool raw = kind == 0;
  const int mblk = 256, nblk = 128;
  std::vector<HamItem> items;
  items.reserve((size_t)npairs * 8);
  for (int p = 0; p < npairs; p++) {
    const PairDesc& pd = h_pairs[p];
    for (int pass = 0; pass < (kind == 2 ? 2 : 1); pass++) {
      const int8_t* a = pass ? pd.t_i8 : pd.q_i8;
      const int8_t* b = pass ? pd.q_i8 : pd.t_i8;
      if (raw) {
        a = reinterpret_cast<const int8_t*>(pd.q_desc);
        b = reinterpret_cast<const int8_t*>(pd.t_desc);
      }
      const int na = pass ? pd.nt : pd.nq, nb = pass ? pd.nq : pd.nt;
      // bruteForceSearchORB never looks at the last train row (features.cpp:174); the float matchers search every row
      const int nsearch = sift ? nb : (nb - 1 > 0 ? nb - 1 : 0);
      for (int m0 = 0; m0 < na; m0 += mblk) {
        HamItem it;
        it.a = a + (size_t)m0 * (raw ? 32 : 256);
        it.b = b;
        if (!sift) it.out = reinterpret_cast<int2*>(w.d_best.ptr) + (size_t)p * stride + m0;
        else if (pass == 0) it.out = reinterpret_cast<int2*>(reinterpret_cast<int4*>(w.d_top4.ptr) + (size_t)p * stride + m0);
        else it.out = reinterpret_cast<int2*>(reinterpret_cast<int4*>(w.d_knn.ptr) + (size_t)p * stride + m0);
        it.nq_valid = na - m0 < mblk ? na - m0 : mblk;
        it.nsearch = nsearch;
        it.n_btiles = (nsearch + nblk - 1) / nblk;
        it.pad_ = pass;  // SiftGPU: tie rule of RowMatch_Kernel (0) / ColMatch_Kernel (1)
        it.bnorm = kind == 1 ? pd.t_norm : nullptr;
        items.push_back(it);
      }
    }
  }
  if (items.empty()) return 0;
  if ((rc = w.d_items.ensure(sizeof(HamItem) * items.size()))) return rc;
  if ((rc = w.h_items.ensure(sizeof(HamItem) * items.size()))) return rc;
  memcpy(w.h_items.ptr, items.data(), sizeof(HamItem) * items.size());
  cudaError_t e = cudaMemcpyAsync(w.d_items.ptr, w.h_items.ptr, sizeof(HamItem) * items.size(), cudaMemcpyHostToDevice, w.stream);
  if (e != cudaSuccess) return cuda_fail(e, "upload match items");
  *n_items = (int)items.size();
  return 0;
}

// SIFT matching stage: bf16 tensor-core scores -> exact fp32 2-NN among the 4 best -> (optionally) ratio/uniqueness.
static int launch_sift_knn(Workspace& w, const PairDesc* d_pairs, int npairs, int max_nq, int stride, int n_items) {
  State& s = g_state;
  cudaEventRecord(w.ev[kEvMatchBegin], w.stream);
  if (n_items > 0) {
    cudaError_t e = launch_l2_tc256((const HamItem*)w.d_items.ptr, n_items, s.sm_count, w.stream);
    if (e != cudaSuccess) return cuda_fail(e, "l2 tensor-core kernel");
    s.launches += 1;
  }
  cudaEventRecord(w.ev[kEvMatchEnd], w.stream);
  cudaError_t e = launch_l2_refine(d_pairs, npairs, max_nq, (const int4*)w.d_top4.ptr, stride, (float4*)w.d_knn.ptr, w.stream);
  if (e != cudaSuccess) return cuda_fail(e, "l2 refine kernel");
  s.launches += 1;
  return 0;
}

// Hamming stage dispatcher (counts the launch); records kEvMatchBegin / kEvMatchEnd immediately around the kernel.
static int launch_hamming(Workspace& w, const PairDesc* d_pairs, int npairs, int max_nq, int stride, int n_items) {
  State& s = g_state;
  cudaError_t e = cudaSuccess;
  cudaEventRecord(w.ev[kEvMatchBegin], w.stream);
  if (s.hamming_path == 0) {
    e = launch_hamming_simt(d_pairs, npairs, max_nq, (int2*)w.d_best.ptr, stride, w.stream);
  } else if (n_items > 0) {
    if (!w.d_claim.ptr) {  // zeroed once; from then on every launch leaves the ticket where the next one expects it
      if (int rc = w.d_claim.ensure(sizeof(unsigned long long))) return rc;
      e = cudaMemsetAsync(w.d_claim.ptr, 0, sizeof(unsigned long long), w.stream);
      if (e != cudaSuccess) return cuda_fail(e, "zero the match kernel's claim counter");
      w.claim = ClaimCounter{(unsigned long long*)w.d_claim.ptr, 0};
    }
    e = launch_hamming_tc_b1((const HamItem*)w.d_items.ptr, n_items, s.sm_count, w.claim, w.stream);
  } else {
    cudaEventRecord(w.ev[kEvMatchEnd], w.stream);
    return 0;
  }
  cudaEventRecord(w.ev[kEvMatchEnd], w.stream);
  if (e != cudaSuccess) return cuda_fail(e, "hamming kernel");
  s.launches += 1;
  return 0;
}

// Every precondition of run_pairs that the pair table decides.  Runs before anything of the call is queued, so a rejected
// call leaves nothing behind on its slot.
static int check_pairs(const std::vector<PairDesc>& h_pairs, int64_t first_pair, bool sync) {
  const State& s = g_state;
  if (h_pairs.empty()) return 0;
  bool any_sift = false, any_orb = false;
  for (const PairDesc& pd : h_pairs) {
    if (pd.nq > kMaxFeatures || pd.nt > kMaxFeatures) {
      set_error("node has more than 4096 features");
      return RGBDSLAM_B200_ERR_ARG;
    }
    (pd.q_f32 ? any_sift : any_orb) = true;
  }
  if (any_sift && any_orb) {
    set_error("match_pairs: ORB and SIFT pairs cannot be mixed in one call");
    return RGBDSLAM_B200_ERR_ARG;
  }
  const bool siftgpu = h_pairs[0].q_f32 && h_pairs[0].sift_kind == 1;
  for (const PairDesc& pd : h_pairs)
    if (any_sift && (pd.sift_kind == 1) != siftgpu) {
      set_error("match_pairs: SiftGPU-matcher nodes and ratio-matcher nodes cannot be mixed in one call");
      return RGBDSLAM_B200_ERR_ARG;
    }
  for (const PairDesc& pd : h_pairs)
    if (any_sift && pd.nq > 0 && (!pd.q_i8 || !pd.t_i8)) {
      set_error("internal: tensor-core match path without tiled operands");
      return RGBDSLAM_B200_ERR_STATE;
    }
  if (s.params.depth_cov_z0 == 0.0 && s.z0 == 0.0 && (first_pair != 0 || s.comm_count > 0 || !sync)) {
    // every rank / in-flight slot would latch a different z0 (and rewrite constant memory under running kernels)
    set_error("depth_cov_z0 == 0 (latch like the reference) is only possible in a synchronous single-process call with "
              "first_pair_index 0: set params.depth_cov_z0 for sharded or pipelined use");
    return RGBDSLAM_B200_ERR_STATE;
  }
  if (s.params.g2o_transformation_refinement > 0)
    for (const PairDesc& pd : h_pairs)
      if ((pd.nq > 0 && !pd.q_kp) || (pd.nt > 0 && !pd.t_kp)) {
        set_error("g2o_transformation_refinement > 0 needs nodes with 2-D keypoints (nodes_create or node_set_keypoints)");
        return RGBDSLAM_B200_ERR_STATE;
      }
  if (s.params.observability_threshold > 0.0)
    for (const PairDesc& pd : h_pairs)
      if (!pd.q_cloud.z || !pd.t_cloud.z) {
        set_error("observability_threshold > 0 needs nodes with a depth cloud (nodes_create or node_set_depth) that "
                  "rgbdslam_b200_reduce_clouds has not voxel-filtered, rgbdslam_b200_octomap_filter_clouds has not left "
                  "without a raster and rgbdslam_b200_transform_clouds has not moved into the map frame");
        return RGBDSLAM_B200_ERR_STATE;
      } else if (!pd.q_cloud.x != !pd.t_cloud.x) {
        // the reference never holds both kinds in one process (topic_points is global): there is no rule to restate
        set_error("observability_threshold > 0: a pair mixes a node that keeps its point cloud (KEEP_CLOUD) with a depth-image node");
        return RGBDSLAM_B200_ERR_STATE;
      }
  return 0;
}

// Core of match_pairs*: h_pairs (device pointers inside, accepted by check_pairs) -> results on the host, on slot w.
static int run_pairs(Workspace& w, const std::vector<PairDesc>& h_pairs, uint64_t seed, int64_t first_pair,
                     rgbdslam_b200_pair_result* results, rgbdslam_b200_dmatch* all_matches,
                     rgbdslam_b200_dmatch* inlier_matches, bool sync = true,
                     const std::function<int()>& after_tables = nullptr) {
  State& s = g_state;
  const int npairs = (int)h_pairs.size();
  if (npairs == 0) return 0;
  int max_nq = 0;
  for (const PairDesc& pd : h_pairs) max_nq = pd.nq > max_nq ? pd.nq : max_nq;
  const bool any_sift = h_pairs[0].q_f32 != nullptr;
  const bool siftgpu = any_sift && h_pairs[0].sift_kind == 1;
  int max_rows = max_nq;
  if (siftgpu)
    for (const PairDesc& pd : h_pairs) max_rows = pd.nt > max_rows ? pd.nt : max_rows;  // the column pass is indexed by train row
  const int stride = (max_rows + 127) / 128 * 128 + 128;
  const int maxM = s.params.max_matches;
  const int H = s.params.ransac_iterations;
  int rc;
  if ((rc = w.d_best.ensure(sizeof(int2) * (size_t)npairs * stride))) return rc;
  if ((rc = w.d_matches.ensure(sizeof(rgbdslam_b200_dmatch) * (size_t)npairs * maxM))) return rc;
  if ((rc = w.d_inliers.ensure(sizeof(rgbdslam_b200_dmatch) * (size_t)npairs * maxM))) return rc;
  // + kMaxMatchesCap rows of slack: the scoring loop reads whole 32-row words past a pair's last match (masked out)
  if ((rc = w.d_mfrom.ensure(sizeof(float4) * ((size_t)npairs * maxM + kMaxMatchesCap)))) return rc;
  if ((rc = w.d_mto.ensure(sizeof(float4) * ((size_t)npairs * maxM + kMaxMatchesCap)))) return rc;
  if ((rc = w.d_nall.ensure(sizeof(int32_t) * npairs))) return rc;
  if ((rc = w.d_hyp.ensure(sizeof(HypResult) * (size_t)npairs * (H > 0 ? H : 1)))) return rc;
  if ((rc = w.d_results.ensure(sizeof(rgbdslam_b200_pair_result) * npairs))) return rc;
  if ((rc = w.d_cen.ensure(sizeof(float) * 8 * (size_t)npairs))) return rc;
  if ((rc = w.d_nextn.ensure(sizeof(int32_t) * (size_t)npairs))) return rc;

  cudaStream_t st = w.stream;
  cudaError_t e;
  if ((rc = upload_pairs(w, h_pairs.data(), npairs))) return rc;
  const PairDesc* d_pairs = (const PairDesc*)w.d_pairs.ptr;
  int n_items = 0;
  if ((rc = stage_match_items(w, h_pairs.data(), npairs, stride, any_sift ? (siftgpu ? 2 : 1) : 0, &n_items))) return rc;
  // every table of this call is on its way; now the bulk uploads + operand expansion of the host-feature path
  if (after_tables && (rc = after_tables())) return rc;

  cudaEventRecord(w.ev[kEvTables], st);
  if (siftgpu) {
    cudaEventRecord(w.ev[kEvMatchBegin], st);
    if (n_items > 0) {
      e = launch_siftgpu_tc256((const HamItem*)w.d_items.ptr, n_items, s.sm_count, st);
      if (e != cudaSuccess) return cuda_fail(e, "siftgpu tensor-core kernel");
      s.launches += 1;
    }
    cudaEventRecord(w.ev[kEvMatchEnd], st);
    e = launch_select_siftgpu(d_pairs, npairs, (const int4*)w.d_top4.ptr, (const int4*)w.d_knn.ptr, stride, maxM,
                              (rgbdslam_b200_dmatch*)w.d_matches.ptr, (float4*)w.d_mfrom.ptr, (float4*)w.d_mto.ptr,
                              (int32_t*)w.d_nall.ptr, st);
    if (e != cudaSuccess) return cuda_fail(e, "select_siftgpu kernel");
    s.launches += 1;
  } else if (any_sift) {
    if ((rc = launch_sift_knn(w, d_pairs, npairs, max_nq, stride, n_items))) return rc;
    e = launch_select_sift(d_pairs, npairs, (const float4*)w.d_knn.ptr, stride, s.params.nn_distance_ratio, maxM,
                           (rgbdslam_b200_dmatch*)w.d_matches.ptr, (float4*)w.d_mfrom.ptr, (float4*)w.d_mto.ptr,
                           (int32_t*)w.d_nall.ptr, st);
    if (e != cudaSuccess) return cuda_fail(e, "select_sift kernel");
    s.launches += 1;
  } else {
    if ((rc = launch_hamming(w, d_pairs, npairs, max_nq, stride, n_items))) return rc;
    e = launch_select_matches(d_pairs, npairs, (const int2*)w.d_best.ptr, stride, seed, first_pair,
                              (rgbdslam_b200_dmatch*)w.d_matches.ptr, (float4*)w.d_mfrom.ptr, (float4*)w.d_mto.ptr,
                              (int32_t*)w.d_nall.ptr, st);
    if (e != cudaSuccess) return cuda_fail(e, "select_matches kernel");
    s.launches += 1;
  }

  if (s.params.depth_cov_z0 == 0.0 && s.z0 == 0.0) {
    // Emulate the function-static of depth_covariance (misc2.h:30-35): latch the z of the first
    // correspondence errorFunction2 would see -- first pair that reaches RANSAC, first sorted match with
    // non-zero, non-NaN depth on both sides (node.cpp:994, misc.cpp:711-716).  check_pairs made sure this is a
    // synchronous single-process call.
    std::vector<int32_t> nall(npairs);
    e = cudaMemcpyAsync(nall.data(), w.d_nall.ptr, sizeof(int32_t) * npairs, cudaMemcpyDeviceToHost, st);
    if (e == cudaSuccess) e = cudaStreamSynchronize(st);
    if (e != cudaSuccess) return cuda_fail(e, "z0 latch (n_all)");
    for (int p = 0; p < npairs && s.z0 == 0.0; p++) {
      if (nall[p] <= s.params.min_matches) continue;
      std::vector<float4> f(nall[p]), t(nall[p]);
      cudaMemcpyAsync(f.data(), (float4*)w.d_mfrom.ptr + (size_t)p * maxM, sizeof(float4) * nall[p],
                      cudaMemcpyDeviceToHost, st);
      cudaMemcpyAsync(t.data(), (float4*)w.d_mto.ptr + (size_t)p * maxM, sizeof(float4) * nall[p],
                      cudaMemcpyDeviceToHost, st);
      e = cudaStreamSynchronize(st);
      if (e != cudaSuccess) return cuda_fail(e, "z0 latch (points)");
      for (int i = 0; i < nall[p]; i++) {
        if (f[i].z == 0.f || t[i].z == 0.f) continue;
        if (std::isnan(f[i].z) || std::isnan(t[i].z)) continue;
        s.z0 = (double)f[i].z;
        break;
      }
    }
    if (s.z0 != 0.0 && (rc = push_dev_params())) return rc;
  }

  int hyp_launches = 0;
  e = launch_ransac_hypotheses(npairs, H, maxM, seed, first_pair, (const float4*)w.d_mfrom.ptr,
                               (const float4*)w.d_mto.ptr, (const int32_t*)w.d_nall.ptr, (HypResult*)w.d_hyp.ptr,
                               (float*)w.d_cen.ptr, (int32_t*)w.d_nextn.ptr, st, &hyp_launches);
  if (e != cudaSuccess) return cuda_fail(e, "ransac_hyp kernel");
  e = launch_ransac_select(d_pairs, npairs, H, maxM, (const float4*)w.d_mfrom.ptr, (const float4*)w.d_mto.ptr,
                           (const int32_t*)w.d_nall.ptr, (const rgbdslam_b200_dmatch*)w.d_matches.ptr,
                           (const HypResult*)w.d_hyp.ptr, (rgbdslam_b200_pair_result*)w.d_results.ptr,
                           (rgbdslam_b200_dmatch*)w.d_inliers.ptr, st);
  if (e != cudaSuccess) return cuda_fail(e, "ransac_select kernel");
  s.launches += 1 + hyp_launches;
  if (s.params.g2o_transformation_refinement > 0) {  // node.cpp:1225-1268
    e = launch_refine_g2o(d_pairs, npairs, maxM, s.params.g2o_transformation_refinement, (const float4*)w.d_mfrom.ptr,
                          (const float4*)w.d_mto.ptr, (const int32_t*)w.d_nall.ptr,
                          (const rgbdslam_b200_dmatch*)w.d_matches.ptr, (rgbdslam_b200_pair_result*)w.d_results.ptr,
                          (rgbdslam_b200_dmatch*)w.d_inliers.ptr, st);
    if (e != cudaSuccess) return cuda_fail(e, "refine_g2o kernel");
    s.launches += 1;
  }
  if (s.params.observability_threshold > 0.0) {  // node.cpp:1340-1342
    bool depth_pairs = false, cloud_pairs = false;
    for (const PairDesc& pd : h_pairs) (pd.q_cloud.x ? cloud_pairs : depth_pairs) = true;
    int emm_launches = 0;
    e = launch_emm_pairs(d_pairs, npairs, depth_pairs, cloud_pairs, s.params.cloud_creation_skip_step, s.params.emm_skip_step,
                         s.dp.cov_z_const, s.params.sigma_depth, s.params.observability_threshold,
                         (rgbdslam_b200_pair_result*)w.d_results.ptr, st, &emm_launches);
    if (e != cudaSuccess) return cuda_fail(e, "emm kernel");
    s.launches += emm_launches;
  }
  cudaEventRecord(w.ev[kEvStagesEnd], st);

  if (results) {
    e = cudaMemcpyAsync(results, w.d_results.ptr, sizeof(rgbdslam_b200_pair_result) * npairs, cudaMemcpyDeviceToHost, st);
    if (e != cudaSuccess) return cuda_fail(e, "download results");
  }
  if (all_matches) {
    e = cudaMemcpyAsync(all_matches, w.d_matches.ptr, sizeof(rgbdslam_b200_dmatch) * (size_t)npairs * maxM,
                        cudaMemcpyDeviceToHost, st);
    if (e != cudaSuccess) return cuda_fail(e, "download all_matches");
  }
  if (inlier_matches) {
    e = cudaMemcpyAsync(inlier_matches, w.d_inliers.ptr, sizeof(rgbdslam_b200_dmatch) * (size_t)npairs * maxM,
                        cudaMemcpyDeviceToHost, st);
    if (e != cudaSuccess) return cuda_fail(e, "download inlier_matches");
  }
  cudaEventRecord(w.ev[kEvDownloaded], st);
  w.timing_valid = true;
  w.pending = true;
  if (sync) {
    e = cudaStreamSynchronize(st);
    if (e != cudaSuccess) return cuda_fail(e, "match_pairs synchronize");
    w.pending = false;
  }
  return 0;
}

void release_slab(NodeSlab* slab) {
  if (slab && --slab->refs == 0) {
    cudaFree(slab->base);
    delete slab;
  }
}

// frees everything a (possibly half-built) node owns
void free_node(NodeDev* nd) {
  nd->magic = 0;
  if (nd->slab) {
    release_slab(nd->slab);
  } else {
    if (nd->desc) cudaFree(nd->desc);
    if (nd->xyz) cudaFree(nd->xyz);
    if (nd->desc_i8) cudaFree(nd->desc_i8);
    if (nd->kp) cudaFree(nd->kp);
  }
  release_slab(nd->pc.slab);
  if (nd->desc_f32) cudaFree(nd->desc_f32);
  if (nd->norms) cudaFree(nd->norms);
  delete nd;
}

}  // namespace rb200

using namespace rb200;

extern "C" {

void rgbdslam_b200_default_params(rgbdslam_b200_params* p) {
  if (!p) return;
  memset(p, 0, sizeof(*p));
  p->max_keypoints = 600;
  p->min_matches = 20;
  p->max_matches = 300;
  p->ransac_iterations = 200;
  p->max_dist_for_inliers = 3.0;
  p->sigma_depth = 0.01;
  p->depth_cov_z0 = 0.0;
  p->depth_scaling_factor = 1.0;
  p->detector_grid_resolution = 3;
  p->adjuster_max_iterations = 5;
  p->min_translation_meter = 0.0;
  p->min_rotation_degree = 0.0;
  p->max_translation_meter = 1e10;
  p->max_rotation_degree = 360.0;
  p->nn_distance_ratio = 0.95;
  p->use_root_sift = 1;
  p->g2o_transformation_refinement = 0;
  p->observability_threshold = -0.6;
  p->emm_skip_step = 8;
  p->cloud_creation_skip_step = 2;
  p->minimum_depth = 0.1f;
}

const char* rgbdslam_b200_last_error(void) { return t_last_error.c_str(); }

int rgbdslam_b200_init(int device, const rgbdslam_b200_params* p) {
  std::lock_guard<std::mutex> lk(g_state.mu);
  State& s = g_state;
  rgbdslam_b200_params prm;
  if (p) prm = *p;
  else rgbdslam_b200_default_params(&prm);
  if (prm.max_matches < 1 || prm.max_matches > RGBDSLAM_B200_MAX_MATCHES_CAP || prm.min_matches < 0 ||
      prm.ransac_iterations < 0 || prm.ransac_iterations > 10000) {
    set_error("invalid parameters (max_matches must be in [1,512], ransac_iterations in [0,10000])");
    return RGBDSLAM_B200_ERR_ARG;
  }
  if (!(prm.sigma_depth > 0.0) || !(prm.max_dist_for_inliers > 0.0)) {
    set_error("invalid parameters (sigma_depth and max_dist_for_inliers must be positive)");
    return RGBDSLAM_B200_ERR_ARG;
  }
  if (prm.observability_threshold > 0.0 && (prm.emm_skip_step <= 0 || prm.cloud_creation_skip_step <= 0)) {
    // the reference treats emm__skip_step < 0 as "accept" (misc.cpp:828-832); the kernels divide by both steps
    set_error("invalid parameters (observability_threshold > 0 needs emm_skip_step >= 1 and cloud_creation_skip_step >= 1)");
    return RGBDSLAM_B200_ERR_ARG;
  }
  if (prm.use_feature_min_depth > 1) {  // a bool in the reference (parameter_server.cpp:90)
    set_error("invalid parameters (use_feature_min_depth must be 0 or 1)");
    return RGBDSLAM_B200_ERR_ARG;
  }
  if (prm.allow_features_without_depth_) {
    // optional branch of the path that is not built (node.cpp:1120-1125): fail loudly
    set_error("allow_features_without_depth is not supported (reference default: false)");
    return RGBDSLAM_B200_ERR_ARG;
  }
  if (prm.feature_detector_type != RGBDSLAM_B200_DETECTOR_ORB && prm.feature_detector_type != RGBDSLAM_B200_DETECTOR_FAST) {
    // parameter_server.cpp:80; SIFT / SURF need OpenCV's non-free module and are not built
    set_error("invalid parameters (feature_detector_type must be RGBDSLAM_B200_DETECTOR_ORB (0) or RGBDSLAM_B200_DETECTOR_FAST (1))");
    return RGBDSLAM_B200_ERR_ARG;
  }
  int count = 0;
  cudaError_t e = cudaGetDeviceCount(&count);
  if (e != cudaSuccess) return cuda_fail(e, "cudaGetDeviceCount (no CUDA device: this library has no CPU fallback)");
  if (device < 0 || device >= count) {
    set_error("device index out of range");
    return RGBDSLAM_B200_ERR_ARG;
  }
  RB200_CUDA(cudaSetDevice(device));
  cudaDeviceProp prop;
  RB200_CUDA(cudaGetDeviceProperties(&prop, device));
  if (prop.major != 9 || prop.minor != 0) {
    set_error(std::string("this build targets sm_90a (H100); device is ") + prop.name);
    return RGBDSLAM_B200_ERR_CUDA;
  }
  if (!s.inited) {
    RB200_CUDA(cudaStreamCreateWithFlags(&s.own_stream, cudaStreamNonBlocking));
    RB200_CUDA(cudaEventCreate(&s.epoch));
    for (int k = 0; k < kSlots; k++) {
      for (cudaEvent_t& ev : s.ws[k].ev) RB200_CUDA(cudaEventCreate(&ev));
      RB200_CUDA(cudaEventCreateWithFlags(&s.ws[k].ev_gather, cudaEventDisableTiming));
      if (k > 0) RB200_CUDA(cudaStreamCreateWithFlags(&s.ws[k].stream, cudaStreamNonBlocking));
    }
    s.stream = s.own_stream;
    s.ws[0].stream = s.stream;
    s.launches = 0;
  }
  s.device = device;
  s.sm_count = prop.multiProcessorCount;
  s.params = prm;
  s.z0 = prm.depth_cov_z0 > 0 ? prm.depth_cov_z0 : 0.0;
  s.inited = true;
  s.ws[0].timing_valid = false;
  int rc = push_dev_params();
  if (rc) return rc;
  RB200_CUDA(cudaStreamSynchronize(s.stream));
  return 0;
}

int rgbdslam_b200_shutdown(void) {
  std::lock_guard<std::mutex> lk(g_state.mu);
  State& s = g_state;
  if (!s.inited) return 0;
  cudaSetDevice(s.device);
  cudaDeviceSynchronize();
  s.release_workspaces();
  posegraph_release();
  landmark_ba_release();
  for (int k = 0; k < kSlots; k++) {
    for (cudaEvent_t ev : s.ws[k].ev) cudaEventDestroy(ev);
    cudaEventDestroy(s.ws[k].ev_gather);
    if (k > 0) cudaStreamDestroy(s.ws[k].stream);
  }
  cudaStreamDestroy(s.own_stream);
  cudaEventDestroy(s.epoch);
  s.inited = false;
  return 0;
}

int rgbdslam_b200_set_stream(void* cuda_stream) {
  RB200_ENTER_INITED();
  g_state.stream = cuda_stream ? (cudaStream_t)cuda_stream : g_state.own_stream;
  g_state.ws[0].stream = g_state.stream;
  return push_dev_params();  // constant memory is per-context, but keep ordering on the new stream
}

int rgbdslam_b200_synchronize(void) {
  RB200_ENTER_INITED();
  RB200_CUDA(cudaStreamSynchronize(g_state.stream));
  return 0;
}

int rgbdslam_b200_node_set_keypoints(uint64_t node_handle, const rgbdslam_b200_keypoint* keypoints) {
  RB200_ENTER_INITED();
  NodeDev* nd = get_node(node_handle);
  if (!nd) return RGBDSLAM_B200_ERR_ARG;
  if (nd->n > 0 && !keypoints) {
    set_error("node_set_keypoints: null keypoints");
    return RGBDSLAM_B200_ERR_ARG;
  }
  if (nd->n == 0) return 0;
  cudaError_t e = cudaSuccess;
  if (!nd->kp) e = cudaMalloc(&nd->kp, sizeof(rgbdslam_b200_keypoint) * (size_t)nd->n);
  if (e == cudaSuccess)
    e = cudaMemcpyAsync(nd->kp, keypoints, sizeof(rgbdslam_b200_keypoint) * (size_t)nd->n, cudaMemcpyHostToDevice, g_state.stream);
  if (e == cudaSuccess) e = cudaStreamSynchronize(g_state.stream);
  if (e != cudaSuccess) return cuda_fail(e, "node_set_keypoints");
  return 0;
}

int rgbdslam_b200_node_set_depth(uint64_t node_handle, const float* depth_m, int w, int h, const float K4[4]) {
  RB200_ENTER_INITED();
  NodeDev* nd = get_node(node_handle);
  if (!nd) return RGBDSLAM_B200_ERR_ARG;
  if (!depth_m || !K4 || w <= 0 || h <= 0) {
    set_error("node_set_depth: bad arguments");
    return RGBDSLAM_B200_ERR_ARG;
  }
  NodeCloud& c = nd->pc;
  if (c.x) {
    set_error("node_set_depth: the node keeps the organised cloud it was built from (KEEP_CLOUD)");
    return RGBDSLAM_B200_ERR_STATE;
  }
  if (c.rgb) {
    set_error("node_set_depth: the node keeps the colour cloud it was built from (STORE_CLOUD)");
    return RGBDSLAM_B200_ERR_STATE;
  }
  State& s = g_state;
  int rc;
  if ((rc = s.d_f32_a.ensure(sizeof(float) * (size_t)w * h))) return rc;
  RB200_CUDA(cudaMemcpyAsync(s.d_f32_a.ptr, depth_m, sizeof(float) * (size_t)w * h, cudaMemcpyHostToDevice, s.stream));
  const int step = s.params.cloud_creation_skip_step > 0 ? s.params.cloud_creation_skip_step : 1;
  const int cw = (w + step - 1) / step, ch = (h + step - 1) / step;  // ceil(cols / skip), misc.cpp:482-483
  if (!(c.slab && c.slab->refs == 1 && c.w == cw && c.h == ch)) {  // else the node alone owns a z-plane of this raster
    NodeSlab* slab = new NodeSlab();
    cudaError_t e = cudaMalloc(&slab->base, sizeof(float) * (size_t)cw * ch);
    if (e != cudaSuccess) {
      delete slab;
      return cuda_fail(e, "cudaMalloc(cloud)");
    }
    slab->refs = 1;
    release_slab(c.slab);
    c.slab = slab;
    c.z = (float*)slab->base;
    c.w = cw;
    c.h = ch;
  }
  c.step = step;
  for (int k = 0; k < 4; k++) c.K[k] = K4[k];
  RB200_CUDA(launch_store_depth_cloud(1, (const float*)s.d_f32_a.ptr, nullptr, 0, false, w, h, step, s.params.depth_scaling_factor,
                                      s.params.minimum_depth, c.z, (size_t)cw * ch, s.stream));
  s.launches += 1;
  RB200_CUDA(cudaStreamSynchronize(s.stream));
  return 0;
}

int rgbdslam_b200_observation_likelihood(uint64_t newer, uint64_t older, const float T[16], uint32_t counts[4]) {
  RB200_ENTER_INITED();
  NodeDev* a = get_node(newer);
  NodeDev* b = a ? get_node(older) : nullptr;
  if (!b) return RGBDSLAM_B200_ERR_ARG;
  if (!T || !counts) {
    set_error("observation_likelihood: bad arguments");
    return RGBDSLAM_B200_ERR_ARG;
  }
  if (!a->pc.z || !b->pc.z) {
    set_error("observation_likelihood: both nodes need a depth cloud (nodes_create with observability_threshold > 0 or STORE_CLOUD, "
              "or node_set_depth)");
    return RGBDSLAM_B200_ERR_STATE;
  }
  if (a->pc.unorganised || b->pc.unorganised) {
    set_error("observation_likelihood: a voxel-filtered (rgbdslam_b200_reduce_clouds) or occupancy-filtered "
              "(rgbdslam_b200_octomap_filter_clouds) cloud has no raster for the measurement model");
    return RGBDSLAM_B200_ERR_STATE;
  }
  if (a->pc.transformed || b->pc.transformed) {
    set_error("observation_likelihood: a cloud moved into the map frame (rgbdslam_b200_transform_clouds) holds no camera points");
    return RGBDSLAM_B200_ERR_STATE;
  }
  if (!a->pc.x != !b->pc.x) {
    set_error("observation_likelihood: a node that keeps its point cloud (KEEP_CLOUD) and a depth-image node cannot be compared");
    return RGBDSLAM_B200_ERR_STATE;
  }
  State& s = g_state;
  if (s.params.depth_cov_z0 == 0.0 && s.z0 == 0.0) {
    // the reference latches depth_covariance's static on its first call (misc2.h:30-35); here that happens in the first
    // match_pairs call that reaches RANSAC
    set_error("observation_likelihood: depth covariance not latched yet (depth_cov_z0 == 0): run match_pairs first or set depth_cov_z0");
    return RGBDSLAM_B200_ERR_STATE;
  }
  int rc;
  if ((rc = s.d_f32_b.ensure(128))) return rc;
  cudaError_t e = cudaMemcpyAsync(s.d_f32_b.ptr, T, 64, cudaMemcpyHostToDevice, s.stream);
  if (e == cudaSuccess)
    e = launch_emm_single(a->pc.view(), b->pc.view(), (const float*)s.d_f32_b.ptr, s.params.cloud_creation_skip_step,
                          s.params.emm_skip_step, s.dp.cov_z_const, s.params.sigma_depth, (unsigned*)((char*)s.d_f32_b.ptr + 64), s.stream);
  if (e == cudaSuccess) e = cudaMemcpyAsync(counts, (char*)s.d_f32_b.ptr + 64, 16, cudaMemcpyDeviceToHost, s.stream);
  if (e == cudaSuccess) e = cudaStreamSynchronize(s.stream);
  if (e != cudaSuccess) return cuda_fail(e, "observation_likelihood");
  s.launches += 1;
  return 0;
}

int rgbdslam_b200_set_sift_matcher(int matcher) {
  std::lock_guard<std::mutex> lk(g_state.mu);
  if (matcher < 0 || matcher > 1) {
    set_error("set_sift_matcher: 0 = exact 2-NN ratio matcher (FLANN branch), 1 = SiftGPU matcher");
    return RGBDSLAM_B200_ERR_ARG;
  }
  g_state.sift_matcher = matcher;
  return 0;
}

int rgbdslam_b200_set_hamming_path(int path) {
  std::lock_guard<std::mutex> lk(g_state.mu);
  if (path < 0 || path > 1) {
    set_error("set_hamming_path: 0 = SIMT popcount (cross-check), 1 = wgmma binary AND-popcount GEMM (default)");
    return RGBDSLAM_B200_ERR_ARG;
  }
  g_state.hamming_path = path;
  return 0;
}

int rgbdslam_b200_get_params(rgbdslam_b200_params* p) {
  std::lock_guard<std::mutex> lk(g_state.mu);
  if (!p) {
    set_error("get_params: null output");
    return RGBDSLAM_B200_ERR_ARG;
  }
  if (!g_state.inited) {
    set_error("rgbdslam_b200_init() has not been called");
    return RGBDSLAM_B200_ERR_STATE;
  }
  *p = g_state.params;
  return 0;
}

int64_t rgbdslam_b200_launch_count(void) { return g_state.launches; }
double rgbdslam_b200_depth_cov_z0(void) { return g_state.z0; }

int rgbdslam_b200_last_timing(float* hamming_ms, float* total_device_ms) {
  return rgbdslam_b200_last_timing_slot(0, hamming_ms, total_device_ms);
}

int rgbdslam_b200_slot_stage_times(int slot, float* ms6) {
  RB200_ENTER_INITED();
  Workspace* w = get_slot(slot);
  if (!w) return RGBDSLAM_B200_ERR_ARG;
  if (!ms6) {
    set_error("slot_stage_times: null output");
    return RGBDSLAM_B200_ERR_ARG;
  }
  if (int rc = check_finished_call(*w, "slot_stage_times")) return rc;
  const cudaEvent_t* ev = w->ev;
  for (int i = 0; i < 6; i++) ms6[i] = 0.f;
  if (w->host_path) {
    RB200_CUDA(cudaEventElapsedTime(&ms6[0], ev[kEvSubmit], ev[kEvUploaded]));  // host -> device copies
    RB200_CUDA(cudaEventElapsedTime(&ms6[1], ev[kEvUploaded], ev[kEvTables]));  // int8 expansion + pair table
  }
  RB200_CUDA(cudaEventElapsedTime(&ms6[2], ev[kEvMatchBegin], ev[kEvMatchEnd]));    // Hamming kernel
  RB200_CUDA(cudaEventElapsedTime(&ms6[3], ev[kEvMatchEnd], ev[kEvStagesEnd]));     // match selection + RANSAC
  RB200_CUDA(cudaEventElapsedTime(&ms6[4], ev[kEvStagesEnd], ev[kEvDownloaded]));   // device -> host copies
  RB200_CUDA(cudaEventElapsedTime(&ms6[5], ev[w->host_path ? kEvSubmit : kEvTables], ev[kEvDownloaded]));  // whole call
  return 0;
}

int rgbdslam_b200_timeline_epoch(void) {
  RB200_ENTER_INITED();
  RB200_CUDA(cudaEventRecord(g_state.epoch, g_state.own_stream));
  RB200_CUDA(cudaEventSynchronize(g_state.epoch));
  return 0;
}

int rgbdslam_b200_slot_timeline(int slot, float* ms7) {
  RB200_ENTER_INITED();
  Workspace* w = get_slot(slot);
  if (!w) return RGBDSLAM_B200_ERR_ARG;
  if (!ms7) {
    set_error("slot_timeline: null output");
    return RGBDSLAM_B200_ERR_ARG;
  }
  if (int rc = check_finished_call(*w, "slot_timeline")) return rc;
  for (int i = kEvSubmit; i <= kEvDownloaded; i++) {
    ms7[i] = -1.f;
    if (!w->host_path && i <= kEvUploaded) continue;
    cudaError_t e = cudaEventElapsedTime(&ms7[i], g_state.epoch, w->ev[i]);
    if (e != cudaSuccess) return cuda_fail(e, "slot_timeline (call rgbdslam_b200_timeline_epoch first)");
  }
  return 0;
}

int rgbdslam_b200_last_timing_slot(int slot, float* hamming_ms, float* total_device_ms) {
  RB200_ENTER_INITED();
  Workspace* w = get_slot(slot);
  if (!w) return RGBDSLAM_B200_ERR_ARG;
  if (int rc = check_finished_call(*w, "last_timing_slot")) return rc;
  float a = 0, b = 0;
  RB200_CUDA(cudaEventElapsedTime(&a, w->ev[kEvMatchBegin], w->ev[kEvMatchEnd]));
  RB200_CUDA(cudaEventElapsedTime(&b, w->ev[kEvTables], w->ev[kEvStagesEnd]));
  if (hamming_ms) *hamming_ms = a;
  if (total_device_ms) *total_device_ms = b;
  return 0;
}

int rgbdslam_b200_brute_force_orb(const uint64_t* q, int nq, const uint64_t* t, int nt, int32_t* idx, int32_t* hd) {
  RB200_ENTER_INITED();
  if (nq < 0 || nt < 0 || (nq > 0 && (!q || !idx || !hd)) || (nt > 0 && !t)) {
    set_error("brute_force_orb: bad arguments");
    return RGBDSLAM_B200_ERR_ARG;
  }
  if (nq == 0) return 0;
  if (nq > kMaxFeatures || nt > kMaxFeatures) {
    set_error("brute_force_orb: more than 4096 descriptors");
    return RGBDSLAM_B200_ERR_ARG;
  }
  Workspace& w = g_state.ws[0];
  const int stride = (nq + 127) / 128 * 128 + 128;
  int rc;
  if ((rc = w.d_feat_a.ensure(32 * (size_t)nq)) || (rc = w.d_feat_b.ensure(32 * (size_t)(nt > 0 ? nt : 1))) ||
      (rc = w.d_best.ensure(sizeof(int2) * (size_t)stride)))
    return rc;
  RB200_CUDA(cudaMemcpyAsync(w.d_feat_a.ptr, q, 32 * (size_t)nq, cudaMemcpyHostToDevice, w.stream));
  if (nt > 0) RB200_CUDA(cudaMemcpyAsync(w.d_feat_b.ptr, t, 32 * (size_t)nt, cudaMemcpyHostToDevice, w.stream));
  PairDesc pd{};
  pd.q_desc = (const uint32_t*)w.d_feat_a.ptr;
  pd.t_desc = (const uint32_t*)w.d_feat_b.ptr;
  pd.nq = nq;
  pd.nt = nt;
  int n_items = 0;
  if ((rc = upload_pairs(w, &pd, 1)) || (rc = stage_match_items(w, &pd, 1, stride, 0, &n_items)) ||
      (rc = launch_hamming(w, (const PairDesc*)w.d_pairs.ptr, 1, nq, stride, n_items)))
    return rc;
  std::vector<int2> h(nq);
  RB200_CUDA(cudaMemcpyAsync(h.data(), w.d_best.ptr, sizeof(int2) * nq, cudaMemcpyDeviceToHost, w.stream));
  RB200_CUDA(cudaStreamSynchronize(w.stream));
  for (int i = 0; i < nq; i++) {
    hd[i] = h[i].x;
    idx[i] = h[i].y;
  }
  return 0;
}

int rgbdslam_b200_node_create_from_features(int32_t id, const uint8_t* desc, const float* xyz1, int n,
                                            uint64_t* node_handle) {
  RB200_ENTER_INITED();
  if (!node_handle || n < 0 || n > kMaxFeatures || (n > 0 && (!desc || !xyz1))) {
    set_error("node_create_from_features: bad arguments (0 <= n <= 4096)");
    return RGBDSLAM_B200_ERR_ARG;
  }
  NodeDev* nd = new NodeDev();
  nd->magic = NodeDev::kMagic;
  nd->id = id;
  nd->n = n;
  nd->n_pad = pad256(n);
  const size_t nalloc = (size_t)(n > 0 ? n : 1);
  cudaError_t e = cudaMalloc(&nd->desc, 32 * nalloc);
  if (e == cudaSuccess) e = cudaMalloc(&nd->xyz, 16 * nalloc);
  if (e != cudaSuccess) {
    free_node(nd);
    return cuda_fail(e, "cudaMalloc(node)");
  }
  if (n > 0) {
    cudaStream_t st = g_state.stream;
    e = cudaMemcpyAsync(nd->desc, desc, 32 * (size_t)n, cudaMemcpyHostToDevice, st);
    if (e == cudaSuccess) e = cudaMemcpyAsync(nd->xyz, xyz1, 16 * (size_t)n, cudaMemcpyHostToDevice, st);
    if (e == cudaSuccess) e = cudaStreamSynchronize(st);
    if (e != cudaSuccess) {
      free_node(nd);
      return cuda_fail(e, "node upload");
    }
  }
  *node_handle = (uint64_t)(uintptr_t)nd;
  return 0;
}

int rgbdslam_b200_node_num_features(uint64_t node_handle, int* n) {
  NodeDev* nd = get_node(node_handle);
  if (!nd) return RGBDSLAM_B200_ERR_ARG;
  if (!n) {
    set_error("node_num_features: null output");
    return RGBDSLAM_B200_ERR_ARG;
  }
  *n = nd->n;
  return 0;
}

int rgbdslam_b200_node_download(uint64_t node_handle, uint8_t* desc, float* xyz1) {
  RB200_ENTER_INITED();
  NodeDev* nd = get_node(node_handle);
  if (!nd) return RGBDSLAM_B200_ERR_ARG;
  if (nd->n == 0) return 0;
  cudaStream_t st = g_state.stream;
  cudaError_t e = cudaSuccess;
  if (desc && nd->desc) e = cudaMemcpyAsync(desc, nd->desc, 32 * (size_t)nd->n, cudaMemcpyDeviceToHost, st);
  if (e == cudaSuccess && xyz1) e = cudaMemcpyAsync(xyz1, nd->xyz, 16 * (size_t)nd->n, cudaMemcpyDeviceToHost, st);
  if (e == cudaSuccess) e = cudaStreamSynchronize(st);
  if (e != cudaSuccess) return cuda_fail(e, "node download");
  return 0;
}

int rgbdslam_b200_node_destroy(uint64_t node_handle) {
  std::lock_guard<std::mutex> lk(g_state.mu);
  NodeDev* nd = get_node(node_handle);
  if (!nd) return RGBDSLAM_B200_ERR_ARG;
  if (g_state.inited) {
    cudaSetDevice(g_state.device);
    cudaStreamSynchronize(g_state.stream);
  }
  free_node(nd);
  return 0;
}

static int match_pairs_impl(int slot, bool sync, const uint64_t* newer, const uint64_t* older, int npairs, uint64_t seed,
                            int64_t first_pair_index, rgbdslam_b200_pair_result* results,
                            rgbdslam_b200_dmatch* all_matches, rgbdslam_b200_dmatch* inlier_matches) {
  RB200_ENTER_INITED();
  Workspace* w = get_slot(slot);
  if (!w) return RGBDSLAM_B200_ERR_ARG;
  if (npairs < 0 || (npairs > 0 && (!newer || !older || !results))) {
    set_error("match_pairs: bad arguments");
    return RGBDSLAM_B200_ERR_ARG;
  }
  std::vector<PairDesc> pairs(npairs);
  for (int i = 0; i < npairs; i++) {
    NodeDev* a = get_node(newer[i]);
    NodeDev* b = a ? get_node(older[i]) : nullptr;
    if (!b) return RGBDSLAM_B200_ERR_ARG;
    if ((a->desc_f32 != nullptr) != (b->desc_f32 != nullptr) || a->sift_kind != b->sift_kind) {
      set_error("match_pairs: nodes of different descriptor / matcher kinds paired");
      return RGBDSLAM_B200_ERR_ARG;
    }
    pairs[i] = make_pair(*a, *b);
  }
  int rc;
  if ((rc = check_pairs(pairs, first_pair_index, sync))) return rc;
  // the slot's pinned staging is about to be reused: its previous call must have finished
  if (w->pending && (rc = drain_slot(*w, "drain slot"))) return rc;
  w->host_path = false;
  return run_pairs(*w, pairs, seed, first_pair_index, results, all_matches, inlier_matches, sync);
}

int rgbdslam_b200_match_pairs(const uint64_t* newer, const uint64_t* older, int npairs, uint64_t seed,
                              int64_t first_pair_index, rgbdslam_b200_pair_result* results,
                              rgbdslam_b200_dmatch* all_matches, rgbdslam_b200_dmatch* inlier_matches) {
  return match_pairs_impl(0, true, newer, older, npairs, seed, first_pair_index, results, all_matches, inlier_matches);
}

int rgbdslam_b200_match_pairs_submit(int slot, const uint64_t* newer, const uint64_t* older, int npairs, uint64_t seed,
                                     int64_t first_pair_index, rgbdslam_b200_pair_result* results,
                                     rgbdslam_b200_dmatch* all_matches, rgbdslam_b200_dmatch* inlier_matches) {
  return match_pairs_impl(slot, false, newer, older, npairs, seed, first_pair_index, results, all_matches, inlier_matches);
}

int rgbdslam_b200_match_pairs_wait(int slot) {
  RB200_ENTER_INITED();
  Workspace* w = get_slot(slot);
  if (!w) return RGBDSLAM_B200_ERR_ARG;
  return drain_slot(*w, "match_pairs_wait");
}

static int match_pairs_host_impl(int slot, bool sync, const uint8_t* desc_newer, const float* xyz_newer, const int32_t* n_newer,
                                 const uint8_t* desc_older, const float* xyz_older, const int32_t* n_older,
                                 const int32_t* id_newer, const int32_t* id_older, int npairs, uint64_t seed,
                                 int64_t first_pair_index, rgbdslam_b200_pair_result* results,
                                 rgbdslam_b200_dmatch* all_matches, rgbdslam_b200_dmatch* inlier_matches) {
  RB200_ENTER_INITED();
  Workspace* w = get_slot(slot);
  if (!w) return RGBDSLAM_B200_ERR_ARG;
  if (npairs < 0 || (npairs > 0 && (!n_newer || !n_older || !results))) {
    set_error("match_pairs_host: bad arguments");
    return RGBDSLAM_B200_ERR_ARG;
  }
  if (npairs == 0) return 0;
  size_t tot_n = 0, tot_o = 0;
  for (int i = 0; i < npairs; i++) {
    if (n_newer[i] < 0 || n_older[i] < 0 || n_newer[i] > kMaxFeatures || n_older[i] > kMaxFeatures) {
      set_error("match_pairs_host: feature count out of range [0,4096]");
      return RGBDSLAM_B200_ERR_ARG;
    }
    tot_n += n_newer[i];
    tot_o += n_older[i];
  }
  if ((tot_n && (!desc_newer || !xyz_newer)) || (tot_o && (!desc_older || !xyz_older))) {
    set_error("match_pairs_host: null feature buffer");
    return RGBDSLAM_B200_ERR_ARG;
  }
  // the pair table points into the slot's feature buffers, which are only (re)allocated below: check it with null bases
  std::vector<PairDesc> pairs(npairs);
  for (int i = 0; i < npairs; i++) {
    pairs[i].nq = n_newer[i];
    pairs[i].nt = n_older[i];
    pairs[i].id_q = id_newer ? id_newer[i] : i;
    pairs[i].id_t = id_older ? id_older[i] : i;
  }
  int rc;
  if ((rc = check_pairs(pairs, first_pair_index, sync))) return rc;
  if (w->pending && (rc = drain_slot(*w, "drain slot"))) return rc;
  if ((rc = w->d_feat_a.ensure(32 * (tot_n + 1))) || (rc = w->d_feat_b.ensure(32 * (tot_o + 1))) ||
      (rc = w->d_xyz_a.ensure(16 * (tot_n + 1))) || (rc = w->d_xyz_b.ensure(16 * (tot_o + 1))))
    return rc;
  cudaStream_t st = w->stream;
  cudaEventRecord(w->ev[kEvSubmit], st);
  w->host_path = true;
  size_t on = 0, oo = 0;
  for (PairDesc& pd : pairs) {
    pd.q_desc = (const uint32_t*)((const uint8_t*)w->d_feat_a.ptr + 32 * on);
    pd.t_desc = (const uint32_t*)((const uint8_t*)w->d_feat_b.ptr + 32 * oo);
    pd.q_xyz = (const float4*)w->d_xyz_a.ptr + on;
    pd.t_xyz = (const float4*)w->d_xyz_b.ptr + oo;
    on += pd.nq;
    oo += pd.nt;
  }
  auto bulk_uploads = [&]() -> int {
    if (tot_n) {
      RB200_CUDA(cudaMemcpyAsync(w->d_feat_a.ptr, desc_newer, 32 * tot_n, cudaMemcpyHostToDevice, st));
      RB200_CUDA(cudaMemcpyAsync(w->d_xyz_a.ptr, xyz_newer, 16 * tot_n, cudaMemcpyHostToDevice, st));
    }
    if (tot_o) {
      RB200_CUDA(cudaMemcpyAsync(w->d_feat_b.ptr, desc_older, 32 * tot_o, cudaMemcpyHostToDevice, st));
      RB200_CUDA(cudaMemcpyAsync(w->d_xyz_b.ptr, xyz_older, 16 * tot_o, cudaMemcpyHostToDevice, st));
    }
    cudaEventRecord(w->ev[kEvUploaded], st);
    return 0;
  };
  return run_pairs(*w, pairs, seed, first_pair_index, results, all_matches, inlier_matches, sync, bulk_uploads);
}

int rgbdslam_b200_match_pairs_host(const uint8_t* desc_newer, const float* xyz_newer, const int32_t* n_newer,
                                   const uint8_t* desc_older, const float* xyz_older, const int32_t* n_older,
                                   const int32_t* id_newer, const int32_t* id_older, int npairs, uint64_t seed,
                                   int64_t first_pair_index, rgbdslam_b200_pair_result* results,
                                   rgbdslam_b200_dmatch* all_matches, rgbdslam_b200_dmatch* inlier_matches) {
  return match_pairs_host_impl(0, true, desc_newer, xyz_newer, n_newer, desc_older, xyz_older, n_older, id_newer, id_older, npairs,
                               seed, first_pair_index, results, all_matches, inlier_matches);
}

int rgbdslam_b200_match_pairs_host_submit(int slot, const uint8_t* desc_newer, const float* xyz_newer, const int32_t* n_newer,
                                          const uint8_t* desc_older, const float* xyz_older, const int32_t* n_older,
                                          const int32_t* id_newer, const int32_t* id_older, int npairs, uint64_t seed,
                                          int64_t first_pair_index, rgbdslam_b200_pair_result* results,
                                          rgbdslam_b200_dmatch* all_matches, rgbdslam_b200_dmatch* inlier_matches) {
  return match_pairs_host_impl(slot, false, desc_newer, xyz_newer, n_newer, desc_older, xyz_older, n_older, id_newer, id_older,
                               npairs, seed, first_pair_index, results, all_matches, inlier_matches);
}

int rgbdslam_b200_node_create_from_sift(int32_t id, const float* desc128, const float* xyz1, int n, uint64_t* node_handle) {
  RB200_ENTER_INITED();
  if (!node_handle || n < 0 || n > kMaxFeatures || (n > 0 && (!desc128 || !xyz1))) {
    set_error("node_create_from_sift: bad arguments (0 <= n <= 4096)");
    return RGBDSLAM_B200_ERR_ARG;
  }
  State& s = g_state;
  NodeDev* nd = new NodeDev();
  nd->magic = NodeDev::kMagic;
  nd->id = id;
  nd->n = n;
  nd->n_pad = pad256(n);
  const size_t na = (size_t)(n > 0 ? n : 1);
  int rc;
  if ((rc = s.d_f32_a.ensure(512 * na))) { delete nd; return rc; }
  cudaError_t e = cudaMalloc(&nd->desc_f32, 512 * na);
  if (e == cudaSuccess) e = cudaMalloc(&nd->xyz, 16 * na);
  if (e == cudaSuccess) e = cudaMalloc(&nd->desc_i8, 256 * (size_t)nd->n_pad);
  if (e == cudaSuccess) e = cudaMalloc(&nd->norms, 4 * (size_t)nd->n_pad);
  if (e != cudaSuccess) {
    free_node(nd);
    return cuda_fail(e, "cudaMalloc(sift node)");
  }
  cudaStream_t st = s.stream;
  if (n > 0) {
    e = cudaMemcpyAsync(s.d_f32_a.ptr, desc128, 512 * (size_t)n, cudaMemcpyHostToDevice, st);
    if (e == cudaSuccess) e = cudaMemcpyAsync(nd->xyz, xyz1, 16 * (size_t)n, cudaMemcpyHostToDevice, st);
    if (e != cudaSuccess) {
      free_node(nd);
      return cuda_fail(e, "sift node upload");
    }
  }
  std::vector<SiftJob> jobs(1);
  jobs[0] = {(const float*)s.d_f32_a.ptr, nd->desc_f32, (uint16_t*)nd->desc_i8, nd->norms, n, nd->n_pad};
  nd->sift_kind = s.sift_matcher;
  if ((rc = prepare_sift_nodes(s.ws[0], jobs, nd->sift_kind))) {
    free_node(nd);
    return rc;
  }
  e = cudaStreamSynchronize(st);
  if (e != cudaSuccess) {
    free_node(nd);
    return cuda_fail(e, "sift node prepare");
  }
  *node_handle = (uint64_t)(uintptr_t)nd;
  return 0;
}

int rgbdslam_b200_knn2_l2(const float* q, int nq, const float* t, int nt, int32_t* idx2, float* dist2) {
  RB200_ENTER_INITED();
  if (nq < 0 || nt < 0 || nq > kMaxFeatures || nt > kMaxFeatures || (nq > 0 && (!q || !idx2 || !dist2)) || (nt > 0 && !t)) {
    set_error("knn2_l2: bad arguments (at most 4096 rows)");
    return RGBDSLAM_B200_ERR_ARG;
  }
  if (nq == 0) return 0;
  State& s = g_state;
  Workspace& w = s.ws[0];
  const int pq = pad256(nq), pt = pad256(nt);
  const int stride = (nq + 127) / 128 * 128 + 128;
  int rc;
  if ((rc = s.d_f32_a.ensure(512 * (size_t)nq)) || (rc = s.d_f32_b.ensure(512 * (size_t)(nt > 0 ? nt : 1))) ||
      (rc = s.d_root_a.ensure(512 * (size_t)pq)) || (rc = s.d_root_b.ensure(512 * (size_t)pt)) ||
      (rc = s.d_i8_a.ensure(256 * (size_t)pq)) || (rc = s.d_i8_b.ensure(256 * (size_t)pt)) ||
      (rc = s.d_norm_a.ensure(4 * (size_t)pq)) || (rc = s.d_norm_b.ensure(4 * (size_t)pt)))
    return rc;
  RB200_CUDA(cudaMemcpyAsync(s.d_f32_a.ptr, q, 512 * (size_t)nq, cudaMemcpyHostToDevice, w.stream));
  if (nt > 0) RB200_CUDA(cudaMemcpyAsync(s.d_f32_b.ptr, t, 512 * (size_t)nt, cudaMemcpyHostToDevice, w.stream));
  std::vector<SiftJob> jobs(2);
  jobs[0] = {(const float*)s.d_f32_a.ptr, (float*)s.d_root_a.ptr, (uint16_t*)s.d_i8_a.ptr, (float*)s.d_norm_a.ptr, nq, pq};
  jobs[1] = {(const float*)s.d_f32_b.ptr, (float*)s.d_root_b.ptr, (uint16_t*)s.d_i8_b.ptr, (float*)s.d_norm_b.ptr, nt, pt};
  if ((rc = prepare_sift_nodes(w, jobs))) return rc;
  PairDesc pd{};
  pd.nq = nq;
  pd.nt = nt;
  pd.q_i8 = (const int8_t*)s.d_i8_a.ptr;
  pd.t_i8 = (const int8_t*)s.d_i8_b.ptr;
  pd.q_f32 = (const float*)s.d_root_a.ptr;
  pd.t_f32 = (const float*)s.d_root_b.ptr;
  pd.t_norm = (const float*)s.d_norm_b.ptr;
  int n_items = 0;
  if ((rc = upload_pairs(w, &pd, 1)) || (rc = stage_match_items(w, &pd, 1, stride, 1, &n_items)) ||
      (rc = launch_sift_knn(w, (const PairDesc*)w.d_pairs.ptr, 1, nq, stride, n_items)))
    return rc;
  std::vector<float4> h(nq);
  RB200_CUDA(cudaMemcpyAsync(h.data(), w.d_knn.ptr, sizeof(float4) * nq, cudaMemcpyDeviceToHost, w.stream));
  RB200_CUDA(cudaStreamSynchronize(w.stream));
  for (int i = 0; i < nq; i++) {
    memcpy(&idx2[2 * i], &h[i].x, 4);
    memcpy(&idx2[2 * i + 1], &h[i].y, 4);
    dist2[2 * i] = h[i].z;
    dist2[2 * i + 1] = h[i].w;
  }
  return 0;
}

}  // extern "C"
