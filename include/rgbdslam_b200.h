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
 *  - there is NO CPU fallback: without a CUDA device rgbdslam_b200_init fails
 *    with RGBDSLAM_B200_ERR_CUDA, and every later call that needs the library
 *    returns RGBDSLAM_B200_ERR_STATE.
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
  float size;     /* 31 * 1.2^octave for ORB, 7 for FAST */
  float angle;    /* degrees; -1 for FAST (no orientation) */
  float response; /* Harris response (ORB) / corner score (FAST) */
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
   * Needs nodes with a depth cloud (rgbdslam_b200_nodes_create keeps one when this is > 0 or with RGBDSLAM_B200_STORE_CLOUD, or
   * rgbdslam_b200_node_set_depth), or point-cloud nodes built with RGBDSLAM_B200_KEEP_CLOUD or STORE_CLOUD; a pair must not mix
   * the two kinds.  A depth cloud's z is (float)((double)depth * depth_scaling_factor), NaN where !(z >= minimum_depth). */
  double observability_threshold; /* -0.6 :114 (off) */
  int32_t emm_skip_step;          /* 8    :112       */
  int32_t cloud_creation_skip_step; /* 2  :36        */
  float minimum_depth;            /* 0.1  :39        */
  /* use_feature_min_depth (parameter_server.cpp:90, default 0): 1 = the Node constructor takes as a keypoint's depth the
   * nearest point of its neighbourhood, getMinDepthInNeighborhood(depth, kp.pt, kp.size) (misc.cpp:774-791), in removeDepthless
   * (node.cpp:82-83) and projectTo3D (:940-941): the minimum of the raw depth image over [int(y - r), int(y + r)) x
   * [int(x - r), int(x + r)) clipped to the image, r = int((size - 1) / 2) (15 .. 55 for ORB octaves 0 .. 7, 3 for FAST).
   * NaN pixels are ignored; a window without a number, or whose minimum is 0, gives NaN (the keypoint is dropped).  The
   * parameters current at a nodes_create* call decide.  rgbdslam_b200_init rejects values other than 0 and 1 with ERR_ARG.
   * allow_features_without_depth (:115; node.cpp:1120-1125) is NOT built: init fails with ERR_ARG when it is set (reference
   * default false). */
  uint8_t use_feature_min_depth, allow_features_without_depth_;
  /* feature_detector_type (parameter_server.cpp:80): the detector rgbdslam_b200_detector_create makes --
   * RGBDSLAM_B200_DETECTOR_ORB (default) or RGBDSLAM_B200_DETECTOR_FAST; rgbdslam_b200_init rejects other values with ERR_ARG.
   * SIFT / SURF (non-free in OpenCV) are not built. */
  uint8_t feature_detector_type;
  uint8_t reserved_;
} rgbdslam_b200_params;
#define RGBDSLAM_B200_DETECTOR_ORB 0
#define RGBDSLAM_B200_DETECTOR_FAST 1

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

/* Which kernel computes the Hamming brute-force stage: 0 = SIMT popcount kernel (cross-check); 1 (default) = wgmma binary
 * tensor-core GEMM (AND-popcount of the raw 32-byte descriptors) with arg-max epilogue.  Both are exact
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
 * (misc.cpp:467-556) at every params.cloud_creation_skip_step-th pixel is kept on the device; it replaces a z-plane the node
 * had.  A node that keeps the cloud it was built from (RGBDSLAM_B200_KEEP_CLOUD or RGBDSLAM_B200_STORE_CLOUD) returns
 * ERR_STATE before any device work. */
int rgbdslam_b200_node_set_depth(uint64_t node_handle, const float* depth_m, int w, int h, const float K4[4]);
/* == pairwiseObservationLikelihood(newer, older, mr) (node.cpp:1520-1554) for an explicit transformation T (Eigen::Matrix4f,
 * column-major, newer -> older frame): counts[4] = inlier, outlier, occluded, all points.  Both nodes have a depth cloud, or
 * both keep their organised cloud (RGBDSLAM_B200_KEEP_CLOUD); a mixed pair returns ERR_STATE. */
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
 * preparation (0 for ORB: the match kernel reads the descriptors themselves), [2] Hamming kernel, [3] match selection + RANSAC, [4] device->host copies, [5] whole call on the stream. */
int rgbdslam_b200_slot_stage_times(int slot, float* ms6);
/* Pipeline diagnostics: timeline_epoch() marks t = 0 on the device; slot_timeline() returns, for the last finished
 * call on a slot, the device time (ms since the epoch) of [0] submit, [1] uploads done, [2] operand expansion done,
 * [3] match kernel start, [4] match kernel end, [5] RANSAC end, [6] downloads done ([0], [1] = -1 for handle calls). */
int rgbdslam_b200_timeline_epoch(void);
int rgbdslam_b200_slot_timeline(int slot, float* ms7);

/* ---- Node construction from images -------------------------------------------
 * The reference builds one detector / extractor pair and shares it between all Node constructors
 * (openni_listener.cpp:130-132); the detector carries the adaptive FAST threshold of every grid cell across
 * frames (feature_adjuster.cpp:131-150, .h:17).  A detector handle holds exactly that state, and its type. */
/* == createDetector(feature_detector_type) (features.cpp:63-113) for the type in the current parameters (ORB before
 * rgbdslam_b200_init): "ORB" = DetectorAdjuster("ORB", 20), "FAST" = DetectorAdjuster("FAST", 20) (feature_adjuster.cpp:85-150)
 * under the same dynamic + grid wrappers; thresholds start at 20 (features.cpp:92).  Every call that takes the handle runs
 * the detector of the handle's type, whatever the parameters say later, so ORB and FAST detectors can be used side by side. */
int rgbdslam_b200_detector_create(uint64_t* detector);
int rgbdslam_b200_detector_destroy(uint64_t detector);
/* read (set = 0) or overwrite (set = 1) the 16 per-cell thresholds (cell = col + row * grid). */
int rgbdslam_b200_detector_thresholds(uint64_t detector, double* thresholds16, int set);

/* == detector->detect(gray, keypoints, mask) (node.cpp:160): VideoGridAdaptedFeatureDetector
 * (feature_adjuster.cpp:286-317) over VideoDynamicAdaptedFeatureDetector (:185-224) over
 * cv::ORB::create(10000, 1.2, 8, 15, 0, 2, HARRIS_SCORE, 31, int(thresh)) (:94) for an ORB detector, or over
 * cv::FastFeatureDetector::create(int(thresh)) (FAST-9/16 with non-max suppression, :88-91) for a FAST detector: integer
 * positions in [3, n-4] of each cell, size 7, angle -1, octave 0, response = corner score.  gray/mask: w*h bytes (mask may
 * be NULL).  Output order: cell-major, |response| descending inside a cell, ties by (octave, y, x) (the reference's
 * nth_element order is unspecified).  *n_out = number found; at most `capacity` are written.  The detector is the one the
 * parameters name (see rgbdslam_b200_nodes_create); at most 4096 keypoints per call: a whole-frame detector (grid <= 1 or
 * adjuster_max_iterations <= 0) that returns more fails with ERR_STATE.  The Node constructor has no such limit. */
int rgbdslam_b200_orb_detect(uint64_t detector, const uint8_t* gray, const uint8_t* mask, int w, int h,
                             rgbdslam_b200_keypoint* kp_out, int capacity, int* n_out);

/* == extractor->compute(gray, keypoints, descriptors) (node.cpp:202) with cv::ORB::create() defaults
 * (features.cpp:117-119): keypoints closer than 31 px (cvRound'ed) to the border are dropped, the rest is stably
 * re-ordered by octave; kp_out (n_in entries) receives the surviving keypoints, desc_out n_out x 32 bytes. */
int rgbdslam_b200_orb_compute(const uint8_t* gray, int w, int h, const rgbdslam_b200_keypoint* kp_in, int n_in,
                              rgbdslam_b200_keypoint* kp_out, uint8_t* desc_out, int* n_out);

/* == Node::Node(visual, depth, detection_mask, cam_info, header, detector, extractor) (node.cpp:101-240) for nframes
 * frames IN ORDER (the detector state makes frames sequentially dependent): detect -> removeDepthless (:186) ->
 * retainBest(max_keypoints) (:187-191) -> compute (:202) -> projectTo3D (:210), with the ORB or FAST detector of the
 * handle and the ORB extractor (FAST keypoints keep angle -1: compute() does not orient given keypoints).
 * gray / mask: nframes*w*h bytes, depth: nframes*w*h floats (metres, NaN = invalid), K4 = fx, fy, cx, cy.  Feature order
 * inside a node: (octave, response descending, cell, y, x).  A keypoint's depth is the pixel at its rounded position, or with
 * params.use_feature_min_depth the minimum over its neighbourhood (see rgbdslam_b200_params), for _ex and _sharded too.
 * Frame size limits (every entry point that takes w and h, every input kind of _ex and _sharded; ERR_ARG before any device
 * work): 96 <= w, h <= 4095, and each grid cell at least 40 px per side at pyramid level 7, so the smallest side that builds
 * is 142 px without a grid, 222 with detector_grid_resolution 2, 333 with 3 (the default), 444 with 4.  Above 1023 px in
 * either dimension the detector needs detector_grid_resolution >= 2, adjuster_max_iterations > 0 and
 * round(1.5 * max_keypoints / cells) < 606 (the smallest per-level quota of the reference's cv::ORB: every 3x3 setting
 * qualifies, 2x2 up to max_keypoints 1614).  The detector is createDetector's (features.cpp:101-112): the grid adjuster
 * (grid > 1, iterations > 0), the whole-frame adjuster (grid <= 1, iterations > 0, no keepStrongest) or, with
 * adjuster_max_iterations <= 0, one whole-frame detection at the handle's cell-0 threshold, which never changes.  The ORB
 * detector applies cv::ORB's per-level quotas everywhere, in the adjuster's counts too.  A grid cell holds at most 12288 FAST
 * candidates up to 1023 px and a cell above 1023 px proportionally more (ERR_STATE when exceeded); a whole-frame cell, or
 * one whose maximum reaches 606, holds every FAST / NMS maximum its pixels can have. */
int rgbdslam_b200_nodes_create(uint64_t detector, int nframes, const uint8_t* gray, const float* depth, const uint8_t* mask,
                               int w, int h, const float* K4, const int32_t* ids, uint64_t* node_handles, int32_t* n_features);
/* The same with options.  RGBDSLAM_B200_MASK_FROM_DEPTH: the detection mask is what the caller of the reference's constructor
 * builds from the depth image -- depthToCV8UC1 (misc.cpp:414-418: depth.convertTo(mono8, CV_8UC1, 100, 0), NaN -> 0; handed
 * over as `depth_mono8_img`, openni_listener.cpp:779) -- computed on the device, `mask` is ignored (saves 1/6 of the upload).
 * Host buffers may be pinned (copied straight from, asynchronously) or pageable (staged through pinned memory); the upload
 * of a chunk of frames overlaps the kernels of the previous chunk; all nodes of a call share one device allocation.
 *
 * RGBDSLAM_B200_VISUAL_RGB: `gray` holds nframes*w*h*3 bytes of colour (CV_8UC3), converted on the device as both reference
 * constructors do, cvtColor(visual, gray, CV_RGB2GRAY) (node.cpp:139-144, 275-277): channel 0 is weighted as R whatever the
 * real channel order (a bgr8 image is converted with R and B swapped, as in the reference), with OpenCV 4's arithmetic
 * (R * 9798 + G * 19235 + B * 3735 + 2^14) >> 15.  For depth-image and cloud input alike.
 *
 * RGBDSLAM_B200_CLOUD_XYZRGB / RGBDSLAM_B200_CLOUD_XYZ: the point-cloud constructor, Node(visual, detector, extractor,
 * point_cloud, detection_mask) (node.cpp:252-369; openni_listener.cpp:754 for registered Kinect clouds, stereo cameras and PCD
 * replay).  `depth` points to nframes organised w x h clouds of pcl::PointXYZRGB (32 bytes per point, the default point_type)
 * or pcl::PointXYZ (16 bytes, RGB_IS_4TH_DIM) (parameter_server.h:33-42): x, y, z at byte offsets 0, 4, 8.  Per frame: detect
 * (the same detector and per-cell threshold state), then projectTo3D (:855-898) on the detector output in its order
 * (cell-major, |response| descending inside a cell, ties by (octave, y, x)) with NO removeDepthless and NO retainBest: a
 * keypoint is kept when the cloud point at ((int)x, (int)y) -- truncated, not rounded -- has no NaN coordinate, and the point
 * is (x, y, z, 1) as stored (no intrinsics, no depth_scaling_factor); the first max_keypoints kept keypoints are the node's.
 * Then compute(): the 31 px border filter and the stable octave sort.  Feature order inside a node: (octave, cell, |response|
 * descending, y, x).  Unlike the reference, each 3-D point moves with its keypoint through compute() (the reference pairs
 * descriptor i with another keypoint's point once compute() drops or re-orders keypoints, and its asserts at node.cpp:317-318
 * fail).  maximum_depth (parameter_server.cpp:38) is fixed at its default, +inf: no point is too far and a +inf z is kept.
 * K4 may be NULL; use_feature_min_depth and depth_scaling_factor are not read.  params.observability_threshold > 0 (the
 * environment measurement model, which needs a cloud per node) returns ERR_STATE for cloud input without KEEP_CLOUD or STORE_CLOUD.
 *
 * RGBDSLAM_B200_KEEP_CLOUD (with a cloud bit only): the node keeps its organised cloud, the reference's pc_col (node.cpp:261,
 * kept when store_pointclouds or emm__skip_step is set, :344-350): x, y and z planes at full resolution on the device, 12 bytes
 * per point (3.7 MB at 640 x 480), de-interleaved from the uploaded cloud by one kernel launch per chunk.  The environment measurement model then runs on
 * these clouds as observationLikelihood (misc.cpp:814-969) does when clouds are the input (topic_points set): every
 * emm_skip_step-th point of the full-resolution cloud, x / y / z as stored, cloud_creation_skip_step not applied (no division
 * of the intrinsics, no sigma scaling); a point with a non-finite coordinate is left untransformed, as
 * pcl::transformPointCloud does on a cloud that is not dense (a +inf z stays +inf and is judged); round() as x86-64 evaluates
 * it (NaN -> INT_MIN, outside the raster); a direction whose two clouds differ in width contributes nothing (:844-847).  K4
 * is here the camera the model projects into, the reference's depth_camera_fx / fy / cx / cy (misc.cpp:56-63); NULL means
 * (0, 0, 0, 0), what the reference uses when those parameters are unset (the cloud constructor never sets cam_info): every
 * finite point then projects to pixel (0, 0).  The node's features, and the detector thresholds, are those of the same call
 * without the flag.  Rejected with ERR_ARG by rgbdslam_b200_nodes_create_sharded (clouds are not exchanged).
 *
 * RGBDSLAM_B200_MASK_FROM_CLOUD: the detection mask is calculateDepthMask of the cloud (openni_listener.cpp:520-534, the
 * stereo and PCD callers), computed on the device and `mask` ignored: static_cast<uchar>(z * 50.0) as x86-64 compilers emit
 * it (truncation to int32, 0x80000000 when out of range, low byte), 0 for NaN -- so the mask is 0 below ~0.02 m, in a band at
 * every multiple of 5.12 m and for +-inf.
 *
 * RGBDSLAM_B200_DEPTH_U16 (depth-image input only): `depth` points to nframes*w*h uint16_t millimetres, 0 = no depth (16UC1,
 * the default topic_image_depth .../sw_registered/image_rect_raw), converted on the device as the listener does before it
 * builds the Node (noCloudCallback, openni_listener.cpp:633-659): depth = convertTo(CV_32FC1, 0.001), (float)d * 0.001f -- a
 * hole becomes 0 m, not NaN, so removeDepthless keeps a keypoint there, and with use_feature_min_depth a neighbourhood that
 * touches a hole has minimum 0, which drops the keypoint.  depth_scaling_factor, use_feature_min_depth and projectTo3D then act
 * on these metres, and so does the environment measurement model.  With MASK_FROM_DEPTH the mask is depthToCV8UC1 of the
 * 16-bit image (misc.cpp:414-425): convertTo(CV_8UC1, 0.05, -25) = saturate_cast<uchar>(fmaf(d, 0.05f, -25.f)), non-zero iff
 * d >= 510 -- nothing closer than 0.51 m is detected, unlike the float rule above, which accepts depths from ~5 mm.  Without it
 * the caller's mask, or none, as for float depth.  The upload moves 2 bytes per depth pixel.
 *
 * RGBDSLAM_B200_VISUAL_BAYER_GR (depth-image input only): `gray` holds nframes*w*h raw bayer_grbg8 bytes (G B on even rows,
 * R G on odd rows), converted as the listener and the Node do: cvtColor(COLOR_BayerGR2RGB) (openni_listener.cpp:638-641, cv2
 * 4.13's bilinear rule, borders repeating the nearest interior row / column), rounded to u8, then CV_RGB2GRAY as for
 * VISUAL_RGB.  Every frame of the call is converted (the listener hands its first Bayer frame over raw: pass that one without
 * the flag to do the same).
 *
 * RGBDSLAM_B200_STORE_CLOUD: every node keeps its colour point cloud, the reference's pc_col (store_pointclouds, node.cpp:126-131,
 * 261), for rgbdslam_b200_node_download_cloud and rgbdslam_b200_render_cloud (rgbdslam_b200/map.h).  Depth-image input: createXYZRGBPointCloud(depth,
 * visual, cam_info) (misc.cpp:467-556) at every params.cloud_creation_skip_step-th pixel -- z = (float)((double)depth *
 * depth_scaling_factor), NaN where !(z >= minimum_depth); x / y are not stored, they follow from the pixel and K4 -- and the
 * packed colour word of the visual the Node receives (the grey image, the three-channel image, or the debayered RGB image of
 * VISUAL_BAYER_GR): channel 0 is blue (encoding_bgr, the reference default) or red (RGBDSLAM_B200_ENCODING_RGB), alpha 0, and
 * point 0 keeps colour 0 (misc.cpp:537).  8 bytes per point (614 kB per 640 x 480 node at skip step 2).  The skip step must
 * divide w and h.  Cloud input: the node keeps its organised cloud as KEEP_CLOUD does (also without that flag) plus the colour
 * word of each point (the float at byte 16 of PointXYZRGB, data[3] of PointXYZ), 16 bytes per point.  The stored cloud is the
 * node's only cloud: the environment measurement model reads it, also when it is switched on after the node was built.  The
 * planes of all nodes of a call share one device allocation, made before any work is queued, and are written by one kernel
 * launch per chunk from the buffers the chunk already holds.  Features, detector thresholds and measurement-model counts are
 * those of the same call without the flag.
 *
 * Rejected with ERR_ARG before any device work: unknown bits, CLOUD_XYZRGB with CLOUD_XYZ, MASK_FROM_CLOUD without a cloud
 * bit, MASK_FROM_DEPTH with a cloud bit, KEEP_CLOUD without a cloud bit, DEPTH_U16 or VISUAL_BAYER_GR with a cloud bit,
 * VISUAL_BAYER_GR with VISUAL_RGB, ENCODING_RGB without STORE_CLOUD, STORE_CLOUD on depth-image input whose w or h the skip step
 * does not divide. */
#define RGBDSLAM_B200_MASK_FROM_DEPTH 1
#define RGBDSLAM_B200_VISUAL_RGB 2
#define RGBDSLAM_B200_CLOUD_XYZRGB 4
#define RGBDSLAM_B200_CLOUD_XYZ 8
#define RGBDSLAM_B200_MASK_FROM_CLOUD 16
#define RGBDSLAM_B200_KEEP_CLOUD 128
#define RGBDSLAM_B200_DEPTH_U16 256
#define RGBDSLAM_B200_VISUAL_BAYER_GR 512
/* bits 32, 64, 1024 and 2048 stay unassigned: they have always been rejected as unknown */
#define RGBDSLAM_B200_STORE_CLOUD 4096
#define RGBDSLAM_B200_ENCODING_RGB 8192
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
 * rank of the communicator must call it with the same total_frames and parameters.  KEEP_CLOUD and STORE_CLOUD are rejected
 * with ERR_ARG (clouds are not exchanged). */
int rgbdslam_b200_nodes_create_sharded(uint64_t detector, uint64_t comm_handle, int total_frames, const uint8_t* gray,
                                       const float* depth, const uint8_t* mask, int w, int h, const float* K4, const int32_t* ids,
                                       int flags, uint64_t* node_handles, int32_t* n_features);
/* Inspection hook: FAST/NMS candidates {u16 x, u16 y, u8 level, u8 score, u16 0} and their responses -- Harris for an
 * ORB detector, the corner score for a FAST detector; NaN = below the cell's final threshold -- of grid cell `cell` in
 * frame 0 of the last detect / nodes_create call. */
int rgbdslam_b200_orb_debug_candidates(int cell, void* cand_out, float* resp_out, int capacity, int* n_out, int* thr_out);
/* Inspection hook: one plane of frame 0 of the last call.  which: 0 cell image, 1 cell mask (cell pyramids); 3 raw /
 * 4 blurred extractor pyramid (cell ignored).  2 (the FAST score map, which the detector never stores) and any other
 * value return ERR_ARG. */
int rgbdslam_b200_orb_debug_plane(int which, int cell, int level, uint8_t* out, int capacity, int* w_out, int* h_out);
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
