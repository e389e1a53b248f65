/* octomap_filter_oracle.c -- plain-C restatement of ColorOctomapServer::occupancyFilter (DESIGN.md 4.15) over the pointer
 * octree of octomap_oracle.c, which it includes, so that one library holds both the map and the filter:
 *   - om_occupancy_filter: the keep decision of every point of a cloud, the reference's loops and libm's exp as they are.
 *   - om_sensor_transform: q * v + t as the filter forms it.
 * Compile with -ffp-contract=off. */
#include "octomap_oracle.c"

/* coordToKey: (int)floor as x86-64's cvttsd2si converts it (INT_MIN for NaN, +-inf and out of range), + 32768, to key_type */
static uint16_t coord_to_key(const Map* m, double c) { return (uint16_t)((unsigned)(int)floor(m->rf * c) + 32768u); }
static double key_to_coord(const Map* m, uint16_t k) { return ((double)((int)k - 32768) + 0.5) * m->res; }

/* q * v + t.head<3>(): Eigen's _transformVector, uv = q.vec().cross(v); uv += uv; v + q.w() * uv + q.vec().cross(uv) */
void om_sensor_transform(const float* q, const float* t, const float* v, float* in) {
  float uv[3] = {q[1] * v[2] - q[2] * v[1], q[2] * v[0] - q[0] * v[2], q[0] * v[1] - q[1] * v[0]};
  for (int c = 0; c < 3; c++) uv[c] += uv[c];
  const float cr[3] = {q[1] * uv[2] - q[2] * uv[1], q[2] * uv[0] - q[0] * uv[2], q[0] * uv[1] - q[1] * uv[0]};
  for (int c = 0; c < 3; c++) in[c] = v[c] + q[3] * uv[c] + cr[c] + t[c];
}

/* xyz (n x 3 float) the cloud's points as stored, q (x, y, z, w) and t its sensor_orientation_ / sensor_origin_;
 * keep[i] = 1 for a kept point.  Returns the count. */
long om_occupancy_filter(void* p, const float* xyz, long n, const float* q, const float* t, double thr, uint8_t* keep) {
  const Map* m = (const Map*)p;
  long kept = 0;
  for (long i = 0; i < n; i++) {
    keep[i] = 0;
    float in[3];
    om_sensor_transform(q, t, xyz + 3 * i, in);
    if (isnan(in[2])) continue;
    const int radius = 1;
    int x_a = coord_to_key(m, in[0]) - radius, x_b = coord_to_key(m, in[0]) + radius;
    int y_a = coord_to_key(m, in[1]) - radius, y_b = coord_to_key(m, in[1]) + radius;
    int z_a = coord_to_key(m, in[2]) - radius, z_b = coord_to_key(m, in[2]) + radius;
    double sum_of_occupancy = 0, sum_of_weights = 0;
    /* the reference's loops: y_a and z_a are never reset */
    for (; x_a <= x_b; ++x_a) {
      for (; y_a <= y_b; ++y_a) {
        for (; z_a <= z_b; ++z_a) {
          const uint16_t key[3] = {(uint16_t)x_a, (uint16_t)y_a, (uint16_t)z_a};
          const Node* node = search(m, key);
          if (node != NULL) {
            double dx = key_to_coord(m, (uint16_t)x_a) - in[0];
            double dy = key_to_coord(m, (uint16_t)y_a) - in[1];
            double dz = key_to_coord(m, (uint16_t)z_a) - in[2];
            double weight = dx * dx + dy * dy + dz * dz;
            double weighted_occ = (1. - (1. / (1. + exp((double)node->lo)))) / weight;
            sum_of_weights += weight;
            sum_of_occupancy += weighted_occ;
          }
        }
      }
    }
    if (sum_of_occupancy < thr * sum_of_weights) {
      keep[i] = 1;
      kept++;
    }
  }
  return kept;
}
