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
  int32_t iterations;         /* nr_iterations_: ICP iterations */
  int32_t criterion;          /* 0 fewer than the method's minimum (3 for icp, 4 for icp_nl), 1 iterations, 2 transform,
                                 3 absolute MSE, 4 relative MSE */
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

/* icp_method (parameter_server.cpp:110, icp.cpp:50-58): "icp" is IterativeClosestPoint, "icp_nl" IterativeClosestPointNonLinear */
#define RGBDSLAM_B200_ICP_METHOD_ICP 0
#define RGBDSLAM_B200_ICP_METHOD_ICP_NL 1

/* rgbdslam_b200_icp_align with the estimator chosen by method; rgbdslam_b200_icp_align(...) == _ex(..., METHOD_ICP).
 * METHOD_ICP_NL is pcl::IterativeClosestPointNonLinear<PointXYZRGB, PointXYZRGB> (PCL 1.7, float): the loop, filterCloud, the
 * correspondences, the move, final = T_inc final, the MSE and the convergence test are those above, except:
 *   - fewer than 4 correspondences stop ICP, not converged (criterion 0);
 *   - T_inc comes from TransformationEstimationLM over the correspondences in source order: x in R^6 from 0, read through
 *     WarpPointRigid6D as (tx, ty, tz, qx, qy, qz); q.q = (qx qx + qz qz) + qy qy (the order of Eigen's SSE reduction of a
 *     Vector4 with w = 0), w = sqrt(1 - q.q), q is not renormalised (PCL 1.7.2), the rotation is Quaternion::
 *     toRotationMatrix's formula; q.q > 1 makes w and every residual NaN, and every comparison with NaN is false, as written;
 *   - residual i = sqrt((dx dx + dz dz) + dy dy) of warp(src_i) - tgt_i, warp(p) = ((r0 x + r1 y) + r2 z) + t;
 *   - Eigen's LevenbergMarquardt<NumericalDiff<.>, float>::minimize with the defaults (factor 100, maxfev 400,
 *     ftol = xtol = sqrt(FLT_EPSILON), gtol 0): forward differences h = sqrt(FLT_EPSILON) |x_j| (sqrt(FLT_EPSILON) when 0),
 *     column (f(x + h e_j) - f(x)) / h; NumericalDiff's f(x) equals the current residual vector bit for bit, so it is reused,
 *     and every Jacobian counts 7 evaluations against maxfev.  With 4 or 5 correspondences Eigen refuses (fewer rows than
 *     parameters): T_inc is the identity and the transform criterion (2) ends ICP;
 *   - ColPivHouseholderQR as in Eigen 3.2 (and 3.3-beta1, ROS kinetic's): squared column norms, the chosen column's
 *     squared norm recomputed over its rows >= k, downdated by subtracting the squared new row-k entries, pivot ties to the
 *     first maximum, no stop at a small pivot (only the count of nonzero pivots), rank() = the diagonal entries among them
 *     above |max pivot| * 6 FLT_EPSILON; Householder vectors as makeHouseholderInPlace (tail squared norm <= FLT_MIN: tau 0);
 *     Q^T f applies H_0 first; lmpar2 and qrsolv (MINPACK's order: the rotated diagonal is solved, then R's restored);
 *   - stableNorm as Eigen 3.3 (blocks of 4096 in index order, scale updated per block); blueNorm as Eigen with float's
 *     constants (b1 2^-63, b2 2^52, s1m 2^63, s2m 2^-76, relerr sqrt(FLT_EPSILON));
 *   - sums over the m correspondences (stableNorm's and blueNorm's sums of squares, column norms, Householder tails and dot
 *     products, Q^T f) run in the fixed order above: 256 partials, partial j adding the rows j, j + 256, ... in order from +0
 *     (rows outside the operated range add nothing), then the pairwise tree; a stableNorm block of 4096 rows is summed the
 *     same way on its own.  Sums of six values (the norms of 6-vectors) take that order too: ((v0 + v4) + v2) + ((v1 + v5)
 *     + v3).  Other 6-term dot products add their products in index order starting from the first; triangular solves run as
 *     Eigen's column-major (back substitution, a zero right-hand side skipped) and row-major (dot product, then divide) ones;
 *   - mixed literals follow C++ promotion: actred = 1. - (fnorm1 / fnorm)^2 is a double subtraction rounded to float;
 *     std::max / std::min are (a < b) ? b : a and (b < a) ? b : a.
 * The LM's status and function evaluations are not reported.  The arguments are checked as above, and a method that is
 * neither ICP nor ICP_NL is ERR_ARG, before any device work. */
int rgbdslam_b200_icp_align_ex(int n, const uint64_t* source, const uint64_t* target, int max_cloud_size, int method,
                               rgbdslam_b200_icp_result* out);

#ifdef __cplusplus
}
#endif
#endif /* RGBDSLAM_B200_ICP_H */
