/*
 * rgbdslam_b200.h -- C ABI of the B200-native RGB-D SLAM front-end hot path.
 *
 * Drop-in boundary for felixendres/rgbdslam_v2 (SURVEY.md section 8b).  The
 * reference has no FFI layer; its hot path is reached through C++ member calls
 * (Node ctor, Node::matchNodePair, bruteForceSearchORB,
 * GraphManager::optimizeGraph).  Every entry point below cites the reference
 * interface it replaces (paths relative to the reference tree).  The C++ shim
 * classes in include/rgbdslam_b200/ (Node, MatchingResult, LoadedEdge3D ...)
 * keep those call sites compiling unchanged and forward to this ABI.
 *
 * Conventions
 *  - plain C: pointers + sizes, POD structs, no exceptions, no torch types.
 *  - every function returns 0 on success, non-zero on error;
 *    rgbdslam_b200_last_error() returns a thread-local message.
 *  - caller owns all host buffers.  Device memory is owned by the library
 *    (node handles, workspaces) unless a function name ends in _device, in
 *    which case the pointers are device pointers owned by the caller.
 *  - there is NO CPU fallback: without a CUDA device every compute call fails
 *    with RGBDSLAM_B200_ERR_CUDA.
 */
#ifndef RGBDSLAM_B200_H
#define RGBDSLAM_B200_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define RGBDSLAM_B200_OK 0
#define RGBDSLAM_B200_ERR_ARG 1
#define RGBDSLAM_B200_ERR_CUDA 2
#define RGBDSLAM_B200_ERR_STATE 3
#define RGBDSLAM_B200_ERR_NCCL 4

#define RGBDSLAM_B200_MAX_MATCHES_CAP 512 /* hard upper bound for params.max_matches */

/* Layout-compatible with cv::KeyPoint (7 x 4 B): node.h:167 feature_locations_2d_. */
typedef struct rgbdslam_b200_keypoint {
  float x, y;     /* pt */
  float size;     /* 31 * 1.2^octave for ORB */
  float angle;    /* degrees */
  float response; /* Harris response */
  int32_t octave;
  int32_t class_id;
} rgbdslam_b200_keypoint;

/* Layout-compatible with cv::DMatch (4 x 4 B): matching_result.h:35-36. */
typedef struct rgbdslam_b200_dmatch {
  int32_t queryIdx; /* index into the newer node's features   */
  int32_t trainIdx; /* index into the older node's features   */
  int32_t imgIdx;   /* always -1 (cv::DMatch default)         */
  float distance;   /* hd/256 + jitter (node.cpp:573)         */
} rgbdslam_b200_dmatch;

/*
 * Hot-path parameters = the ParameterServer defaults the path reads
 * (src/parameter_server.cpp, SURVEY.md appendix A).
 */
typedef struct rgbdslam_b200_params {
  int32_t max_keypoints;        /* 600   parameter_server.cpp:83  */
  int32_t min_matches;          /* 20    :85                      */
  int32_t max_matches;          /* 300   :86  (<= MAX_MATCHES_CAP) */
  int32_t ransac_iterations;    /* 200   :101                     */
  double max_dist_for_inliers;  /* 3.0   :100 (Mahalanobis)       */
  double sigma_depth;           /* 0.01  :46                      */
  /*
   * depth_covariance() in misc2.h:30-35 caches its FIRST result in a function
   * static: cov_z is the constant (sigma_depth*z0^2)^2 of the first depth it
   * ever sees.  depth_cov_z0 > 0 : use this z0 (deterministic emulation).
   * depth_cov_z0 == 0 : latch z0 like the reference does -- from the first
   * scored match of the first pair of the first match_pairs call.
   * depth_cov_z0 < 0 : per-point covariance (sigma*z^2)^2 (quirk switched off).
   */
  double depth_cov_z0;
  double depth_scaling_factor;  /* 1.0   :34                      */
  int32_t detector_grid_resolution; /* 3 :87                      */
  int32_t adjuster_max_iterations;  /* 5 :89                      */
  double min_translation_meter; /* 0     :98                      */
  double min_rotation_degree;   /* 0     :99                      */
  double max_translation_meter; /* 1e10  :96                      */
  double max_rotation_degree;   /* 360   :97                      */
  double nn_distance_ratio;     /* 0.95  :160 (SIFT path)         */
  int32_t use_root_sift;        /* 1     :92                      */
  int32_t g2o_transformation_refinement; /* 0 :103 -- Gauss-Newton iterations of the pairwise refinement (node.cpp:1225-1268,
                                          * transformation_estimation.cpp:126-170); needs nodes with 2-D keypoints */
  /* Environment measurement model (node.cpp:1340-1342, misc.cpp:814-969, 1136-1148): > 0 enables it; an accepted RANSAC
   * transformation is kept only if inliers / (inliers + outliers) > threshold and inliers / (inl + outl + occluded) > 0.25.
   * Needs nodes with a depth cloud (rgbdslam_b200_nodes_create keeps one when this is > 0, or rgbdslam_b200_node_set_depth). */
  double observability_threshold; /* -0.6 :114 (off) */
  int32_t emm_skip_step;          /* 8    :112       */
  int32_t cloud_creation_skip_step; /* 2  :36        */
  float minimum_depth;            /* 0.1  :39        */
  /* Optional branches of the path that are NOT built; rgbdslam_b200_init fails with ERR_ARG when either is set:
   * use_feature_min_depth (parameter_server.cpp:90; node.cpp:85, misc.cpp:774-791) and allow_features_without_depth
   * (:115; node.cpp:1120-1125).  Both default to false in the reference. */
  uint8_t use_feature_min_depth_, allow_features_without_depth_;
  uint8_t reserved_[2];
} rgbdslam_b200_params;

/*
 * One frame pair = MatchingResult (matching_result.h:24-46) + LoadedEdge3D
 * (edge.h:24-32) without the two std::vector<cv::DMatch>, which are returned in
 * separate arrays (params.max_matches entries per pair).
 */
typedef struct rgbdslam_b200_pair_result {
  int32_t id1, id2;        /* edge.id1 = older id, edge.id2 = newer id; -1,-1 = no transformation (node.cpp:1420) */
  int32_t n_all_matches;   /* all_matches.size()   after keepStrongestMatches */
  int32_t n_inliers;       /* inlier_matches.size() */
  float rmse;              /* MatchingResult::rmse (Mahalanobis RMS of the inliers) */
  int32_t valid_iterations;/* RANSAC iterations that produced a refined model (node.cpp:1170) */
  float ransac_trafo[16];  /* Eigen::Matrix4f, column-major; maps newer-frame points into the older frame */
  double info_scale;       /* edge.informationMatrix = I6 * info_scale, = n_inliers / rmse^2 (node.cpp:1335) */
  int32_t used_identity;   /* 1 if the identity last-resort hypothesis was taken (node.cpp:1192-1215) */
  /* MatchingResult::inlier_points / outlier_points / occluded_points / all_points (matching_result.h:40-42): filled by the
   * environment measurement model when params.observability_threshold > 0, else 0 */
  uint32_t inlier_points, outlier_points, occluded_points, all_points;
  int32_t reserved_;
} rgbdslam_b200_pair_result;

/* ---- library state ------------------------------------------------------- */

/* Fill *p with the reference defaults (parameter_server.cpp:22-173). */
void rgbdslam_b200_default_params(rgbdslam_b200_params* p);

/* Select CUDA device + parameters.  Replaces ParameterServer::instance() for this path. */
int rgbdslam_b200_init(int device, const rgbdslam_b200_params* p);
int rgbdslam_b200_shutdown(void);
/* The parameter set the library currently runs with (what ParameterServer::instance()->get<>() would return). */
int rgbdslam_b200_get_params(rgbdslam_b200_params* p);

/* Run all subsequent work of the synchronous calls (slot 0) on this cudaStream_t.  NULL = the library's own non-blocking
 * stream -- note that the legacy default stream has handle 0 too, so it cannot be selected: work a caller queues on the
 * default stream is NOT ordered against the library unless it passes a real stream here. */
int rgbdslam_b200_set_stream(void* cuda_stream);
/* Block until all work queued by the library has finished. */
int rgbdslam_b200_synchronize(void);

/* Which kernel computes the Hamming brute-force stage: 0 = SIMT popcount kernel (cross-check); 1 (default) = wgmma s8
 * tensor-core GEMM with arg-max epilogue, the 32-byte descriptors expanded to int8 operands inside the kernel.  Both are exact
 * and give identical results (DESIGN.md 4.1); other values are rejected. */
int rgbdslam_b200_set_hamming_path(int path);

const char* rgbdslam_b200_last_error(void);
/* Number of kernels launched by this library since init (for bench gpu_launches). */
int64_t rgbdslam_b200_launch_count(void);
/* The z0 currently latched for depth_covariance (0 if not latched yet). */
double rgbdslam_b200_depth_cov_z0(void);

/* ---- brute-force ORB search ----------------------------------------------
 * == bruteForceSearchORB (src/features.cpp:168-182) applied to nq query rows,
 * i.e. the loop node.cpp:567-575 without the hd>=128 filter.  Quirk kept: only
 * train rows [0, nt-2] are examined (features.cpp:174); lowest index wins ties;
 * nt <= 1 gives hd = 257, idx = -1.  q/t are host buffers of nq*4 / nt*4 uint64. */
int rgbdslam_b200_brute_force_orb(const uint64_t* q, int nq, const uint64_t* t, int nt,
                                  int32_t* idx, int32_t* hd);

/* ---- nodes ---------------------------------------------------------------
 * A node handle owns the device copy of what Node keeps per frame
 * (node.h:167-174): descriptors (N x 32 B), 3-D points (N x Vector4f). */

/* Upload precomputed ORB features (host buffers).  desc: n*32 B, xyz1: n*4 float. */
int rgbdslam_b200_node_create_from_features(int32_t id, const uint8_t* desc, const float* xyz1, int n,
                                            uint64_t* node_handle);
int rgbdslam_b200_node_num_features(uint64_t node_handle, int* n);
/* Download (any pointer may be NULL). */
int rgbdslam_b200_node_download(uint64_t node_handle, uint8_t* desc, float* xyz1);
/* == Node::~Node (node.cpp:371). */
/* Give a node its point cloud (Node::pc_col) for the environment measurement model: the depth image in metres (row-major
 * w x h float, NaN = no measurement) and K4 = (fx, fy, cx, cy).  Only the z-plane of createXYZRGBPointCloud
 * (misc.cpp:467-556) at every params.cloud_creation_skip_step-th pixel is kept on the device. */
int rgbdslam_b200_node_set_depth(uint64_t node_handle, const float* depth_m, int w, int h, const float K4[4]);
/* == pairwiseObservationLikelihood(newer, older, mr) (node.cpp:1520-1554) for an explicit transformation T (Eigen::Matrix4f,
 * column-major, newer -> older frame): counts[4] = inlier, outlier, occluded, all points. */
int rgbdslam_b200_observation_likelihood(uint64_t newer, uint64_t older, const float T[16], uint32_t counts[4]);
/* Attach the 2-D keypoints (feature_locations_2d_, n entries) to a node created from features: only the pairwise g2o
 * refinement reads them (edgeToFeature, transformation_estimation.cpp:91-124).  Nodes built from images carry theirs. */
int rgbdslam_b200_node_set_keypoints(uint64_t node_handle, const rgbdslam_b200_keypoint* keypoints);
int rgbdslam_b200_node_destroy(uint64_t node_handle);

/* ---- SIFT-128 float descriptors (feature_extractor_type SIFT / SURF / SIFTGPU) -----------
 * Node with 128-d float descriptors.  squareroot_descriptor_space (RootSIFT, node.cpp:1557-1571) is applied when
 * params.use_root_sift != 0 (node.cpp:233-239).  Such nodes are matched by rgbdslam_b200_match_pairs with the float
 * branch of Node::featureMatching (node.cpp:610-667): 2-NN, ratio test against nn_distance_ratio, first-come
 * uniqueness of trainIdx, distance = ratio.  The reference's approximate FLANN kd-tree search (4 trees, 16 checks,
 * node.cpp:493-514,1573-1581) is replaced by an EXACT 2-NN: bf16 tensor-core score matrix, 4 best candidates per
 * query re-ranked with exact fp32 distances. */
int rgbdslam_b200_node_create_from_sift(int32_t id, const float* desc128, const float* xyz1, int n, uint64_t* node_handle);
/* == Node::knnSearch(query, indices, dists, 2, ...) (node.cpp:1573-1581) with exact search: idx2 / dist2 hold 2
 * entries per query row (squared L2 distances, as cv::flann returns them).  RootSIFT applied per params. */
int rgbdslam_b200_knn2_l2(const float* q, int nq, const float* t, int nt, int32_t* idx2, float* dist2);

/* Matcher used by float-descriptor nodes CREATED AFTER the call (parameter `matcher_type`, parameter_server.cpp:82):
 *   0 (default)  exact 2-NN + ratio / uniqueness test -- the FLANN branch, src/node.cpp:610-667;
 *   1            the SiftGPU matcher, src/node.cpp:553-557 -> SiftGPUWrapper::match (src/sift_gpu_wrapper.cpp:169-227):
 *                descriptors quantised to unsigned 8 bit (external/SiftGPU/src/SiftGPU/SiftMatchCU.cpp:87-101), integer
 *                dot-product matrix, acos distance < 0.9, ratio < 0.9, mutual best match (ProgramCU.cu:1405-1478,
 *                1689-1784, SiftMatchCU.cpp:139-176), DMatch.distance = float L2 of the raw rows.  Bit-exact restatement;
 *                the nodes keep the raw rows (no RootSIFT).  Both nodes of a pair must be of the same kind. */
int rgbdslam_b200_set_sift_matcher(int matcher);

/* ---- frame-pair matching --------------------------------------------------
 * == Node::matchNodePair (node.cpp:1305-1429) for npairs independent pairs
 * (the QtConcurrent::blockingMapped fan-out of graph_manager.cpp:548 as one
 * batched launch): featureMatching ORB branch (node.cpp:561-576,674) ->
 * getRelativeTransformationTo (node.cpp:1074-1277) -> edge (node.cpp:1335-1339).
 * The reference draws from global rand(); this ABI takes an explicit seed and
 * uses a counter-based generator keyed by (seed, pair_index[, hypothesis]).
 * pair_index = first_pair_index + position in the batch, so sharded callers
 * reproduce the single-call results.
 * all_matches / inlier_matches: npairs * params.max_matches entries (may be NULL). */
int rgbdslam_b200_match_pairs(const uint64_t* newer, const uint64_t* older, int npairs,
                              uint64_t seed, int64_t first_pair_index,
                              rgbdslam_b200_pair_result* results,
                              rgbdslam_b200_dmatch* all_matches,
                              rgbdslam_b200_dmatch* inlier_matches);

/* Same, but the nodes are given as host feature buffers (upload inside the call):
 * desc_* : concatenated descriptors, xyz_* : concatenated points; n_*[i] features
 * of pair i.  This is the "host buffers in, host results out" path used for the
 * end-to-end measurement. */
int rgbdslam_b200_match_pairs_host(const uint8_t* desc_newer, const float* xyz_newer, const int32_t* n_newer,
                                   const uint8_t* desc_older, const float* xyz_older, const int32_t* n_older,
                                   const int32_t* id_newer, const int32_t* id_older, int npairs,
                                   uint64_t seed, int64_t first_pair_index,
                                   rgbdslam_b200_pair_result* results,
                                   rgbdslam_b200_dmatch* all_matches,
                                   rgbdslam_b200_dmatch* inlier_matches);

/* Pipelined variants: up to 8 independent slots (own CUDA stream + workspace each).  submit() only enqueues the
 * uploads, kernels and result downloads and returns; wait(slot) blocks until that slot's results are in the output
 * buffers (which must stay valid -- pinned memory recommended).  Successive batches submitted to different slots
 * overlap on the GPU (host->device copies of batch k+1 with the kernels of batch k; the latency-bound RANSAC phases
 * of several batches with each other).  slot 0 shares the stream of the synchronous calls.  Results are identical
 * to the synchronous calls. */
int rgbdslam_b200_match_pairs_submit(int slot, const uint64_t* newer, const uint64_t* older, int npairs, uint64_t seed,
                                     int64_t first_pair_index, rgbdslam_b200_pair_result* results,
                                     rgbdslam_b200_dmatch* all_matches, rgbdslam_b200_dmatch* inlier_matches);
int rgbdslam_b200_match_pairs_host_submit(int slot, const uint8_t* desc_newer, const float* xyz_newer, const int32_t* n_newer,
                                          const uint8_t* desc_older, const float* xyz_older, const int32_t* n_older,
                                          const int32_t* id_newer, const int32_t* id_older, int npairs, uint64_t seed,
                                          int64_t first_pair_index, rgbdslam_b200_pair_result* results,
                                          rgbdslam_b200_dmatch* all_matches, rgbdslam_b200_dmatch* inlier_matches);
int rgbdslam_b200_match_pairs_wait(int slot);

/* Timing hook: CUDA-event duration (ms) of the dominant kernel (Hamming match)
 * and of the whole device part of the last match_pairs* call. */
int rgbdslam_b200_last_timing(float* hamming_ms, float* total_device_ms);
int rgbdslam_b200_last_timing_slot(int slot, float* hamming_ms, float* total_device_ms);
/* CUDA-event stage times (ms) of the last finished call on a slot: [0] host->device copies, [1] float-descriptor operand
 * preparation (0 for ORB: descriptors are expanded inside the match kernel), [2] Hamming kernel, [3] match selection + RANSAC, [4] device->host copies, [5] whole call on the stream. */
int rgbdslam_b200_slot_stage_times(int slot, float* ms6);
/* Pipeline diagnostics: timeline_epoch() marks t = 0 on the device; slot_timeline() returns, for the last finished
 * call on a slot, the device time (ms since the epoch) of [0] submit, [1] uploads done, [2] operand expansion done,
 * [3] match kernel start, [4] match kernel end, [5] RANSAC end, [6] downloads done ([0], [1] = -1 for handle calls). */
int rgbdslam_b200_timeline_epoch(void);
int rgbdslam_b200_slot_timeline(int slot, float* ms7);

/* ---- Node construction from images -------------------------------------------
 * The reference builds one detector / extractor pair and shares it between all Node constructors
 * (openni_listener.cpp:130-132); the detector carries the adaptive FAST threshold of every grid cell across
 * frames (feature_adjuster.cpp:131-150, .h:17).  A detector handle holds exactly that state. */
/* == createDetector("ORB") (features.cpp:63-113): thresholds start at 20 (features.cpp:92). */
int rgbdslam_b200_detector_create(uint64_t* detector);
int rgbdslam_b200_detector_destroy(uint64_t detector);
/* read (set = 0) or overwrite (set = 1) the 16 per-cell thresholds (cell = col + row * grid). */
int rgbdslam_b200_detector_thresholds(uint64_t detector, double* thresholds16, int set);

/* == detector->detect(gray, keypoints, mask) (node.cpp:160): VideoGridAdaptedFeatureDetector
 * (feature_adjuster.cpp:286-317) over VideoDynamicAdaptedFeatureDetector (:185-224) over
 * cv::ORB::create(10000, 1.2, 8, 15, 0, 2, HARRIS_SCORE, 31, int(thresh)) (:94).  gray/mask: w*h bytes (mask may be
 * NULL).  Output order: cell-major, |response| descending inside a cell (the reference's nth_element order is
 * unspecified).  *n_out = number found; at most `capacity` are written. */
int rgbdslam_b200_orb_detect(uint64_t detector, const uint8_t* gray, const uint8_t* mask, int w, int h,
                             rgbdslam_b200_keypoint* kp_out, int capacity, int* n_out);

/* == extractor->compute(gray, keypoints, descriptors) (node.cpp:202) with cv::ORB::create() defaults
 * (features.cpp:117-119): keypoints closer than 31 px (cvRound'ed) to the border are dropped, the rest is stably
 * re-ordered by octave; kp_out (n_in entries) receives the surviving keypoints, desc_out n_out x 32 bytes. */
int rgbdslam_b200_orb_compute(const uint8_t* gray, int w, int h, const rgbdslam_b200_keypoint* kp_in, int n_in,
                              rgbdslam_b200_keypoint* kp_out, uint8_t* desc_out, int* n_out);

/* == Node::Node(visual, depth, detection_mask, cam_info, header, detector, extractor) (node.cpp:101-240) for nframes
 * frames IN ORDER (the detector state makes frames sequentially dependent): detect -> removeDepthless (:186) ->
 * retainBest(max_keypoints) (:187-191) -> compute (:202) -> projectTo3D (:210).  gray / mask: nframes*w*h bytes,
 * depth: nframes*w*h floats (metres, NaN = invalid), K4 = fx, fy, cx, cy.  Feature order inside a node:
 * (octave, response descending, cell, y, x). */
int rgbdslam_b200_nodes_create(uint64_t detector, int nframes, const uint8_t* gray, const float* depth, const uint8_t* mask,
                               int w, int h, const float* K4, const int32_t* ids, uint64_t* node_handles, int32_t* n_features);
/* The same with options.  RGBDSLAM_B200_MASK_FROM_DEPTH: the detection mask is what the caller of the reference's constructor
 * builds from the depth image -- depthToCV8UC1 (misc.cpp:414-418: depth.convertTo(mono8, CV_8UC1, 100, 0), NaN -> 0; handed
 * over as `depth_mono8_img`, openni_listener.cpp:779) -- computed on the device, `mask` is ignored (saves 1/6 of the upload).
 * Host buffers may be pinned (copied straight from, asynchronously) or pageable (staged through pinned memory); the upload
 * of a chunk of frames overlaps the kernels of the previous chunk; all nodes of a call share one device allocation. */
#define RGBDSLAM_B200_MASK_FROM_DEPTH 1
int rgbdslam_b200_nodes_create_ex(uint64_t detector, int nframes, const uint8_t* gray, const float* depth, const uint8_t* mask,
                                  int w, int h, const float* K4, const int32_t* ids, int flags, uint64_t* node_handles,
                                  int32_t* n_features);
/* The same for a sequence whose frames are SHARDED over the ranks of a communicator (one process per GPU; BASELINE config C4):
 * rank r passes only its own frames [r * per, min((r + 1) * per, total_frames)), per = ceil(total_frames / world), in order.
 * The reference's detector makes frames sequentially dependent -- the adaptive FAST threshold of every grid cell persists
 * from frame to frame (feature_adjuster.cpp:131-150) -- but only through the number of corners above a threshold: ranks
 * detect their frames without a threshold (corner score histograms), all-gather the histograms (NCCL), EVERY rank replays the
 * threshold recurrence of the whole sequence (:185-224) and finishes its own frames with exactly the thresholds one process
 * would have used; the finished features (descriptors, 3-D points, counts) are all-gathered so that every rank holds every
 * node.  node_handles / n_features / ids: total_frames entries.  Bit-identical to rgbdslam_b200_nodes_create_ex on one GPU
 * (2-D keypoints, which only the pairwise g2o refinement reads, stay on the rank that built the node).  Collective: every
 * rank of the communicator must call it with the same total_frames and parameters. */
int rgbdslam_b200_nodes_create_sharded(uint64_t detector, uint64_t comm_handle, int total_frames, const uint8_t* gray,
                                       const float* depth, const uint8_t* mask, int w, int h, const float* K4, const int32_t* ids,
                                       int flags, uint64_t* node_handles, int32_t* n_features);
/* Inspection hook: FAST/NMS candidates {u16 x, u16 y, u8 level, u8 score, u16 0} and Harris responses (NaN = below
 * the cell's final threshold) of grid cell `cell` in frame 0 of the last detect / nodes_create call. */
int rgbdslam_b200_orb_debug_candidates(int cell, void* cand_out, float* resp_out, int capacity, int* n_out, int* thr_out);
/* Inspection hook: one plane of frame 0 of the last call.  which: 0 cell image, 1 cell mask, 2 FAST score map
 * (cell pyramids); 3 raw / 4 blurred extractor pyramid (cell ignored). */
int rgbdslam_b200_orb_debug_plane(int which, int cell, int level, uint8_t* out, int capacity, int* w_out, int* h_out);
/* Inspection hook: 1 = detect with the unfused kernels (FAST score by threshold search into a global score map -- the one
 * orb_debug_plane(2, ...) returns --, separate NMS and resize passes), 0 = the default fused kernels.  Identical results. */
int rgbdslam_b200_orb_debug_detect_path(int unfused);
/* feature_locations_2d_ (node.h:167) of a node built by nodes_create. */
int rgbdslam_b200_node_download_keypoints(uint64_t node_handle, rgbdslam_b200_keypoint* kp_out);

/* ---- multi-GPU exchange ---------------------------------------------------------
 * Frame pairs are independent (the QtConcurrent fan-out of graph_manager.cpp:548 has no cross-pair state): ranks
 * process disjoint pair ranges (first_pair_index keeps the random streams global) and all-gather the fixed-size edge
 * records ONCE over NCCL before the replicated pose-graph solve.  One process per GPU; rank 0 obtains the unique id
 * and distributes it to the other ranks out of band (e.g. torch.distributed / MPI / a file). */
int rgbdslam_b200_comm_unique_id(uint8_t* id128);
int rgbdslam_b200_comm_init(int rank, int world, const uint8_t* id128, uint64_t* comm_handle);
int rgbdslam_b200_comm_destroy(uint64_t comm_handle);
/* local: n_per_rank records of this rank (host); all: world * n_per_rank records, rank-major (host). */
int rgbdslam_b200_allgather_edges(uint64_t comm_handle, const rgbdslam_b200_pair_result* local, int n_per_rank,
                                  rgbdslam_b200_pair_result* all);
/* The same exchange for a batch still in flight on a pipeline slot: queued behind the slot's kernels on the communicator's
 * own stream, straight from the device-side edge records (no host round trip); rgbdslam_b200_match_pairs_wait(slot) also
 * waits for it.  Call right after match_pairs*_submit(slot, ...); all ranks must use the same slot order.  `all` (host)
 * receives world * n_per_rank records ordered by rank. */
int rgbdslam_b200_allgather_slot_edges(uint64_t comm, int slot, int n_per_rank, rgbdslam_b200_pair_result* all);

/* ---- pose-graph solve --------------------------------------------------------
 * == GraphManager::optimizeGraph(double iter, bool nonthreaded) -> optimizeGraphImpl
 * (src/graph_manager.cpp:900-1066) on the optimizer createOptimizer builds (:107-201):
 * Levenberg-Marquardt, 6x6 pose blocks, block-Jacobi PCG (backend_solver "pcg"), EdgeSE3 with the shared Huber
 * kernel (graph_manager.h:382, delta 1.0), fixed vertices per fixationOfVertices (:911-937).
 *   poses : nv x 7 doubles (tx ty tz qx qy qz qw), in = current estimates (vertex = v1 * T,
 *           graph_manager.cpp:858), out = optimised estimates
 *   fixed : nv bytes, 1 = setFixed(true)            ij : ne x 2 vertex indices (edge.id1, edge.id2)
 *   meas  : ne x 7 (LoadedEdge3D::transform)         info : ne x 36 row-major (LoadedEdge3D::informationMatrix)
 *   stop  : optimizer_iterations semantics (graph_manager.cpp:998-1014): >= 1 iteration budget,
 *           (0,1) relative chi2 improvement per chunk of 5 iterations
 * Returns chi2 = optimizer_->chi2() (sum e' Omega e), the number of LM iterations and of PCG iterations.
 * backend_solver (graph_manager.cpp:126-180): only the reference default "pcg" is built -- cholmod / csparse / dense solve
 * the same linear systems to a tighter residual, so they are not selectable here (SURVEY 8b's `solver` argument dropped).
 * Non-finite information entries are rejected with ERR_ARG. */
int rgbdslam_b200_posegraph_optimize(int nv, double* poses, const uint8_t* fixed, int ne, const int32_t* ij,
                                     const double* meas, const double* info, double stop, double huber_delta,
                                     double* chi2, int* iters, int* cg_iters);
/* Pre-size the solver's cached device buffers for graphs of up to nv vertices / ne edges (they only ever grow).  The reference
 * lets g2o allocate as the graph grows (graph_manager.cpp:811-898); a caller that knows the size of its session takes the
 * allocations out of its first large solve. */
int rgbdslam_b200_posegraph_reserve(int nv, int ne);
/* Host glue (no device work): what GraphManager::nodeComparisons + addEdgeToG2O (graph_manager.cpp:550-583, 636-655,
 * 811-898) do with the MatchingResults of a new node, for an OFFLINE candidate list (SURVEY.md 8e: no Dijkstra feedback).
 * pairs: n_pairs x (newer, older) frame indices grouped by ascending newer frame, results aligned with them.  Per new frame:
 * every valid result becomes an edge (older -> newer, measurement = ransac_trafo, information = I6 * info_scale); the vertex
 * estimate is v_older * T of the first edge and is replaced whenever a later edge has strictly more inliers; without an edge
 * to the predecessor a constant-position edge (identity, information I6 / const_edge_dt) is appended.  Vertex 0 is fixed.
 * Outputs: poses7 n_frames x 7, fixed n_frames, ij / meas7 / info36 with capacity n_pairs + n_frames edges. */
int rgbdslam_b200_graph_from_pairs(int n_frames, int n_pairs, const int32_t* pairs, const rgbdslam_b200_pair_result* results,
                                   double const_edge_dt, double* poses7, uint8_t* fixed, int32_t* ij, double* meas7, double* info36,
                                   int* n_edges, int* n_const_edges);
/* computeActiveErrors + chi2 (graph_manager.cpp:1002-1003); per_edge_chi2 (ne doubles, may be NULL) is what
 * pruneEdgesWithErrorAbove (graph_manager.cpp:1106-1246) thresholds. */
int rgbdslam_b200_posegraph_chi2(int nv, const double* poses, int ne, const int32_t* ij, const double* meas,
                                 const double* info, double huber_delta, double* chi2, double* per_edge_chi2);

/* Bundle adjustment over camera poses AND 3-D landmarks (the reference's DO_FEATURE_OPTIMIZATION build: src/landmark.cpp:97-187
 * creates a VertexPointXYZ per landmark and an EdgeSE3PointXYZDepth per observation, optimizeGraphImpl includes them when
 * optimize_landmarks is set, src/graph_manager.cpp:963-967).  Observation o: landmark obs_point[o] seen by camera obs_cam[o]
 * at pixel (u, v) with depth d (obs_uvd, 3 doubles), information diag(obs_info3[o]) -- the reference uses
 * point_information_matrix(d) = diag(1, 1, 1 / depth_covariance(d)) (misc2.h:37-47) -- pin-hole K4 = (fx, fy, cx, cy)
 * (ParameterCamera, graph_manager.cpp:189-192).  Optional pose-pose edges (ij / meas7 / info36, as posegraph_optimize) share
 * the Huber kernel of width huber_delta; projection edges have no robust kernel (landmark.cpp:176).  Runs `iterations`
 * Levenberg-Marquardt iterations (optimizer_->optimize(n)); every step eliminates the landmarks by the Schur complement and
 * solves the reduced camera system with a block-Jacobi PCG on the GPU.  poses7 (n_cams x 7: t, q) and points3 (n_points x 3,
 * world frame) are updated in place; chi2_* include the robustified pose-edge terms. */
int rgbdslam_b200_landmark_ba(int n_cams, double* poses7, const uint8_t* fixed, int n_points, double* points3, int n_obs,
                              const int32_t* obs_cam, const int32_t* obs_point, const double* obs_uvd, const double* obs_info3,
                              const double* K4, int n_edges, const int32_t* ij, const double* meas7, const double* info36,
                              int iterations, double huber_delta, double* chi2_before, double* chi2_after, int* lm_iterations,
                              int* pcg_iterations);

#ifdef __cplusplus
}
#endif
#endif /* RGBDSLAM_B200_H */
