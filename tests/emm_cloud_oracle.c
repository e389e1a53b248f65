/*
 * emm_cloud_oracle.c -- CPU oracle of the environment measurement model on the organised clouds that point-cloud nodes keep
 * (RGBDSLAM_B200_KEEP_CLOUD).  TEST INFRASTRUCTURE ONLY, built by tests/emm_cloud_exact.py with -ffp-contract=off (the
 * reference is built without FMA contraction) and run on x86-64, where round()'s conversion is cvttsd2si.
 *
 *   emm_cloud_observation_likelihood   observationLikelihood (misc.cpp:814-969, one direction) with clouds as input
 *                                      (topic_points set: cloud_creation_skip_step 1, intrinsics not divided, sigma not scaled)
 *   emm_cloud_pairwise_observation     pairwiseObservationLikelihood (node.cpp:1520-1554)
 * pcl::transformPointCloud (PCL 1.7, not vendored) on a cloud that is not dense: the input is copied, a point with a
 * non-finite coordinate stays untransformed, the others become the float affine map R p + t.  Eigen's Matrix4f::inverse() of
 * the affine transformation is restated as the float cofactor inverse.
 */
#include <math.h>
#include <stddef.h>
#include <stdint.h>

/* depth_covariance (misc2.h:20-35) with its function-static latched at z0 when z0 > 0, per point otherwise */
static double depth_cov(double sigma_depth, double z0, double z) {
  double zz = z0 > 0 ? z0 : z;
  double sd = sigma_depth * zz * zz;
  return sd * sd;
}

static int round_ref(float d) { return (int)floor(d + 0.5); } /* misc.cpp:804-807 */

static double cdf(double x, double mu, double sigma) { return 0.5 * (1 + erf((x - mu) / (sigma * 1.41421))); } /* :809-812 */

/* T: column-major Matrix4f (new -> old).  Clouds: w x h row-major points of `stride` floats, x / y / z at 0 / 1 / 2.
 * K = fx, fy, cx, cy of the camera the model projects into (depth_camera_*).  counts += inl, outl, occl, all */
void emm_cloud_observation_likelihood(double sigma_depth, double z0, const float* T, const float* new_pc, int nw, int nh,
                                      const float* old_pc, int ow, int oh, int stride, const float* K, int skip_step,
                                      uint32_t counts[4]) {
  if (ow != nw) return; /* misc.cpp:844-847 */
  const float fx = K[0], fy = K[1], cx = K[2], cy = K[3];
  uint32_t good_points = 0, bad_points = 0, occluded_points = 0, all = 0;
  for (int new_ry = 0; new_ry < nh; new_ry += skip_step)
    for (int new_rx = 0; new_rx < nw; new_rx += skip_step, all++) {
      const float* q = new_pc + ((size_t)new_ry * nw + new_rx) * stride;
      float x = q[0], y = q[1], z = q[2], px = x, py = y, pz = z;
      if (isfinite(x) && isfinite(y) && isfinite(z)) {
        px = T[0] * x + T[4] * y + T[8] * z + T[12];
        py = T[1] * x + T[5] * y + T[9] * z + T[13];
        pz = T[2] * x + T[6] * y + T[10] * z + T[14];
      }
      if (pz != pz) continue;
      if (pz < 0) continue;
      int old_rx_center = round_ref((px / pz) * fx + cx);
      int old_ry_center = round_ref((py / pz) * fy + cy);
      if (old_rx_center >= ow || old_rx_center < 0 || old_ry_center >= oh || old_ry_center < 0) continue;
      int nbhd = 2;
      int good_point = 0, occluded_point = 0, bad_point = 0;
      int startx = old_rx_center - nbhd > 0 ? old_rx_center - nbhd : 0;
      int starty = old_ry_center - nbhd > 0 ? old_ry_center - nbhd : 0;
      int endx = ow < old_rx_center + nbhd + 1 ? ow : old_rx_center + nbhd + 1;
      int endy = oh < old_ry_center + nbhd + 1 ? oh : old_ry_center + nbhd + 1;
      for (int old_ry = starty; old_ry < endy; old_ry += 2)
        for (int old_rx = startx; old_rx < endx; old_rx += 2) {
          float oz = old_pc[((size_t)old_ry * ow + old_rx) * stride + 2];
          if (oz != oz) continue;
          double old_sigma = 1 * depth_cov(sigma_depth, z0, oz);
          double new_sigma = 1 * depth_cov(sigma_depth, z0, pz);
          double joint_sigma = old_sigma + new_sigma;
          double p_new_in_front = cdf(oz, pz, sqrt(joint_sigma));
          if (p_new_in_front < 0.001) occluded_point = 1;
          else if (p_new_in_front < 0.999) good_point = 1;
          else bad_point = 1;
        }
      if (good_point) good_points++;
      else if (occluded_point) occluded_points++;
      else if (bad_point) bad_points++;
    }
  counts[0] += good_points;
  counts[1] += bad_points;
  counts[2] += occluded_points;
  counts[3] += all;
}

static void affine_inverse_f(const float* T, float* Ti) { /* column-major in / out */
  float R[9];
  for (int r = 0; r < 3; r++)
    for (int c = 0; c < 3; c++) R[3 * r + c] = T[4 * c + r];
  float c00 = R[4] * R[8] - R[5] * R[7], c01 = R[5] * R[6] - R[3] * R[8], c02 = R[3] * R[7] - R[4] * R[6];
  float det = R[0] * c00 + R[1] * c01 + R[2] * c02, id = 1.0f / det;
  float Ri[9] = {c00 * id, (R[2] * R[7] - R[1] * R[8]) * id, (R[1] * R[5] - R[2] * R[4]) * id,
                 c01 * id, (R[0] * R[8] - R[2] * R[6]) * id, (R[2] * R[3] - R[0] * R[5]) * id,
                 c02 * id, (R[1] * R[6] - R[0] * R[7]) * id, (R[0] * R[4] - R[1] * R[3]) * id};
  for (int r = 0; r < 3; r++) {
    for (int c = 0; c < 3; c++) Ti[4 * c + r] = Ri[3 * r + c];
    Ti[12 + r] = -(Ri[3 * r] * T[12] + Ri[3 * r + 1] * T[13] + Ri[3 * r + 2] * T[14]);
  }
  Ti[3] = Ti[7] = Ti[11] = 0.f;
  Ti[15] = 1.f;
}

/* z0 > 0: depth covariance latched at z0; otherwise per point */
void emm_cloud_pairwise_observation(double sigma_depth, double z0, const float* T, const float* newer_pc, int nw, int nh,
                                    const float* newerK, const float* older_pc, int ow, int oh, const float* olderK, int stride,
                                    int skip_step, uint32_t counts[4]) {
  counts[0] = counts[1] = counts[2] = counts[3] = 0;
  emm_cloud_observation_likelihood(sigma_depth, z0, T, newer_pc, nw, nh, older_pc, ow, oh, stride, olderK, skip_step, counts);
  float Ti[16];
  affine_inverse_f(T, Ti);
  emm_cloud_observation_likelihood(sigma_depth, z0, Ti, older_pc, ow, oh, newer_pc, nw, nh, stride, newerK, skip_step, counts);
}
