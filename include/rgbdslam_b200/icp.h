/*
 * rgbdslam_b200/icp.h -- C ABI of the ICP fallback of Node::matchNodePair (node.cpp:1356-1377, compiled in the reference with
 * USE_PCL_ICP): icpAlignment(filterCloud(source->pc_col), filterCloud(target->pc_col), Identity) (icp.cpp:20-89).  The
 * conventions of ../rgbdslam_b200.h hold; the call needs an initialised library.  The clouds are the nodes' stored clouds of
 * map.h (RGBDSLAM_B200_STORE_CLOUD, RGBDSLAM_B200_KEEP_CLOUD, the measurement model's depth clouds, voxel-reduced clouds).
 */
#ifndef RGBDSLAM_B200_ICP_H
#define RGBDSLAM_B200_ICP_H

#include "../rgbdslam_b200.h"

#ifdef __cplusplus
extern "C" {
#endif

typedef struct rgbdslam_b200_icp_result {
  float T[16];                /* getFinalTransformation(), column-major like pair_result.ransac_trafo; identity unless converged */
  int32_t converged;          /* hasConverged() */
  int32_t iterations;         /* nr_iterations_ */
  int32_t criterion;          /* 0 fewer than 3 correspondences, 1 iterations, 2 transform, 3 absolute MSE, 4 relative MSE */
  int32_t n_source, n_target; /* points after filterCloud */
  int32_t n_correspondences;  /* of the last iteration */
  double mse;                 /* calculateMSE of the last completed iteration, 0 when none completed */
} rgbdslam_b200_icp_result;

/* == icpAlignment(filterCloud(source[k]), filterCloud(target[k]), Identity) for the n pairs k, on the device.  T maps the
 * source cloud onto the target cloud.  The rules, every operation in float unless noted:
 *   - filterCloud(cloud, desired = max_cloud_size) (icp.cpp:20-45): the indices of the points whose z is not NaN, in storage
 *     order (a z of +-inf is kept); float step = n / (float)desired, at least 1; for (float i = 0; i < n; i += step) the point
 *     of index (unsigned)i is kept.  The float loop may keep desired + 1 points.
 *   - pcl::IterativeClosestPoint<PointXYZRGB, PointXYZRGB> (PCL 1.7) with max correspondence distance 0.05, 50 iterations,
 *     transformation epsilon 1e-8 and Euclidean fitness epsilon 1.  One iteration:
 *     1. for each source point in order, the nearest target point, d = ((dx dx + dy dy) + dz dz); the pair is kept when
 *        (double)d <= 0.05 * 0.05 (in double).  The lowest target index wins a tie.  A point with a non-finite coordinate
 *        takes no part, on either side;
 *     2. fewer than 3 correspondences: stop, not converged (criterion 0);
 *     3. T_inc = Umeyama without scaling: the means (sums times 1 / (float)n), sigma = (1 / n) * dst_demean src_demean^T,
 *        a 3 x 3 Jacobi SVD, S_3 = -1 when det U det V < 0, R = U S V^T, t = dst_mean - R src_mean.  The float sums run in a
 *        fixed order: 256 partial sums, partial j adding the terms of source points j, j + 256, ... in order from +0, then a
 *        pairwise tree (p[j] += p[j + s], s = 128 ... 1).  The SVD is the two-sided cyclic Jacobi method of Eigen's
 *        JacobiSVD, with correctly rounded operations throughout;
 *     4. every finite source point moves to ((r0 x + r1 y) + r2 z) + t; final = T_inc final;
 *     5. DefaultConvergenceCriteria with prev_mse = DBL_MAX at the start, tested in this order: iterations >= 50 (criterion 1);
 *        0.5 * (double)(((R00 + R11) + R22) - 1) >= 1 - 1e-8 and (double)((t0 t0 + t1 t1) + t2 t2) <= 1e-8 (criterion 2);
 *        mse = (sum in double of the kept d, in source order) / n, |mse - prev| < 1e-12 (criterion 3);
 *        |mse - prev| / prev < 1 (criterion 4, PCL 1.7's relative MSE threshold: so ICP normally stops after 2 iterations);
 *        otherwise prev = mse and the next iteration runs.
 * A node may appear in several pairs and on both sides (also as its own partner); it is filtered once per call.  The call
 * changes no node.  A cloud without a usable point is no error: that pair reports criterion 0 and identity.  The result does
 * not depend on which other pairs share the call.
 * ERR_ARG before any device work: n < 0, max_cloud_size < 1, a NULL array with n > 0, an unknown handle.  ERR_STATE before any
 * device work: a node without a stored cloud. */
int rgbdslam_b200_icp_align(int n, const uint64_t* source, const uint64_t* target, int max_cloud_size,
                            rgbdslam_b200_icp_result* out);

#ifdef __cplusplus
}
#endif
#endif /* RGBDSLAM_B200_ICP_H */
