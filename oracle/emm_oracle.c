/*
 * emm_oracle.c -- CPU ORACLE of the environment measurement model (SURVEY.md 8f rank 3).  TEST INFRASTRUCTURE ONLY.
 *
 *   oracle_create_cloud_z                createXYZRGBPointCloud   src/misc.cpp:467-556 (z-plane; x / y follow from backProject,
 *                                                                  src/misc2.h:49-65)
 *   oracle_observation_likelihood        observationLikelihood    src/misc.cpp:814-969 (one direction)
 *   oracle_pairwise_observation          pairwiseObservationLikelihood  src/node.cpp:1520-1554
 *   oracle_observation_criterion_met     observation_criterion_met      src/misc.cpp:1136-1148
 * pcl::transformPointCloud (PCL 1.7, not vendored) is the float affine map R p + t.  Eigen's Matrix4f::inverse() of the
 * affine transformation is restated as the float cofactor inverse.  Parity unpinned (no fixtures in the reference).
 */
#include <math.h>
#include <stddef.h>
#include <stdint.h>

typedef struct {
  int32_t min_matches, max_matches, ransac_iterations, pad_;
  double max_dist_for_inliers, sigma_depth, depth_cov_z0;
} oracle_params;

static double depth_cov(const oracle_params* p, double z) { /* misc2.h:20-35 incl. the static cache */
  double zz = p->depth_cov_z0 > 0 ? p->depth_cov_z0 : z;
  double sd = p->sigma_depth * zz * zz;
  return sd * sd;
}

void oracle_create_cloud_z(const float* depth, int w, int h, int step, double scaling, float min_depth, float* cloud_z) {
  int cw = (w + step - 1) / step, ch = (h + step - 1) / step;
  for (int ry = 0; ry < ch; ry++)
    for (int rx = 0; rx < cw; rx++) {
      int u = rx * step, v = ry * step;
      float z = NAN;
      if (u < w && v < h) {
        float Z = (float)((double)depth[(size_t)v * w + u] * scaling); /* double depth_scaling (misc.cpp:502, 522) */
        if (Z >= min_depth) z = Z;
      }
      cloud_z[(size_t)ry * cw + rx] = z;
    }
}

static int round_ref(float d) { return (int)floor(d + 0.5); } /* misc.cpp:804-807 */

static double cdf(double x, double mu, double sigma) { return 0.5 * (1 + erf((x - mu) / (sigma * 1.41421))); } /* :809-812 */

/* T: column-major Matrix4f (new -> old).  K = fx, fy, cx, cy of the full-resolution cameras. counts += inl, outl, occl, all */
void oracle_observation_likelihood(const oracle_params* p, const float* T, const float* new_z, int ncw, int nch, const float* newK,
                                   const float* old_z, int ocw, int och, const float* oldK, int cloud_step, int skip_step,
                                   uint32_t counts[4]) {
  const float nfxinv = (float)(1. / newK[0]), nfyinv = (float)(1. / newK[1]), ncx = newK[2], ncy = newK[3];
  float fx = oldK[0] / cloud_step, fy = oldK[1] / cloud_step, cx = oldK[2] / cloud_step, cy = oldK[3] / cloud_step;
  uint32_t good_points = 0, bad_points = 0, occluded_points = 0, all = 0;
  for (int new_ry = 0; new_ry < nch; new_ry += skip_step)
    for (int new_rx = 0; new_rx < ncw; new_rx += skip_step, all++) {
      float Z = new_z[(size_t)new_ry * ncw + new_rx];
      float u = (float)(new_rx * cloud_step), v = (float)(new_ry * cloud_step);
      float x, y, z;
      if (isnan(Z)) {
        x = (u - ncx) * 1.0 * nfxinv; y = (v - ncy) * 1.0 * nfyinv; z = Z;
      } else {
        x = (u - ncx) * Z * nfxinv; y = (v - ncy) * Z * nfyinv; z = Z;
      }
      float px = T[0] * x + T[4] * y + T[8] * z + T[12];
      float py = T[1] * x + T[5] * y + T[9] * z + T[13];
      float pz = T[2] * x + T[6] * y + T[10] * z + T[14];
      if (pz != pz) continue;
      if (pz < 0) continue;
      int old_rx_center = round_ref((px / pz) * fx + cx);
      int old_ry_center = round_ref((py / pz) * fy + cy);
      if (old_rx_center >= ocw || old_rx_center < 0 || old_ry_center >= och || old_ry_center < 0) continue;
      int nbhd = 2;
      int good_point = 0, occluded_point = 0, bad_point = 0;
      int startx = old_rx_center - nbhd > 0 ? old_rx_center - nbhd : 0;
      int starty = old_ry_center - nbhd > 0 ? old_ry_center - nbhd : 0;
      int endx = ocw < old_rx_center + nbhd + 1 ? ocw : old_rx_center + nbhd + 1;
      int endy = och < old_ry_center + nbhd + 1 ? och : old_ry_center + nbhd + 1;
      for (int old_ry = starty; old_ry < endy; old_ry += 2)
        for (int old_rx = startx; old_rx < endx; old_rx += 2) {
          float oz = old_z[(size_t)old_ry * ocw + old_rx];
          if (oz != oz) continue;
          double old_sigma = cloud_step * depth_cov(p, oz);
          double new_sigma = cloud_step * depth_cov(p, pz);
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

void oracle_pairwise_observation(const oracle_params* p, const float* T, const float* newer_z, int ncw, int nch, const float* newerK,
                                 const float* older_z, int ocw, int och, const float* olderK, int cloud_step, int skip_step,
                                 uint32_t counts[4]) {
  counts[0] = counts[1] = counts[2] = counts[3] = 0;
  oracle_observation_likelihood(p, T, newer_z, ncw, nch, newerK, older_z, ocw, och, olderK, cloud_step, skip_step, counts);
  float Ti[16];
  affine_inverse_f(T, Ti);
  oracle_observation_likelihood(p, Ti, older_z, ocw, och, olderK, newer_z, ncw, nch, newerK, cloud_step, skip_step, counts);
}

int oracle_observation_criterion_met(uint32_t inliers, uint32_t outliers, uint32_t all, double obs_thresh, double* quality) {
  if (obs_thresh < 0) return 1;
  *quality = inliers / (double)(inliers + outliers);
  double certainty = inliers / (double)all;
  return (*quality > obs_thresh) && (certainty > 0.25);
}
