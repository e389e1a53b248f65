/* Plain-C oracle of the voxel filter of a node's stored cloud, written the way pcl::VoxelGrid<PointXYZRGB>::applyFilter
 * (PCL 1.7, downsample_all_data_, no filter field, min_points_per_voxel_ 0) goes about it: bounds of the finite points, the
 * int64 guard, min_b / div_b / divb_mul, an index vector of (voxel index, point index), a sort, and a walk over the runs that
 * sums x, y, z, r, g, b in float and scales by the float reciprocal of the count (Eigen 3.2's operator/=(Scalar)).  PCL's
 * std::sort leaves the order inside a voxel open; here the point index breaks ties, which is the raster order the library
 * fixes.  Built with -ffp-contract=off: no operation is fused. */
#include <math.h>
#include <stdint.h>
#include <stdlib.h>

typedef struct {
  unsigned idx, point;
} index_pair;

static int by_idx_then_point(const void* a, const void* b) {
  const index_pair *p = (const index_pair*)a, *q = (const index_pair*)b;
  if (p->idx != q->idx) return p->idx < q->idx ? -1 : 1;
  return p->point < q->point ? -1 : p->point > q->point;
}

static int finite3(float x, float y, float z) { return isfinite(x) && isfinite(y) && isfinite(z); }

/* Returns the number of output points, or -1 when the leaf size is too small for the cloud (the input is the output). */
long voxel_grid_filter(const float* x, const float* y, const float* z, const uint32_t* rgb, long n, float leaf, float* ox, float* oy,
                       float* oz, uint32_t* orgb) {
  const float inv = 1.0f / leaf;
  float mn[3] = {INFINITY, INFINITY, INFINITY}, mx[3] = {-INFINITY, -INFINITY, -INFINITY};
  long used = 0;
  for (long i = 0; i < n; i++) { /* getMinMax3D */
    if (!finite3(x[i], y[i], z[i])) continue;
    const float p[3] = {x[i], y[i], z[i]};
    for (int a = 0; a < 3; a++) {
      if (p[a] < mn[a]) mn[a] = p[a];
      if (p[a] > mx[a]) mx[a] = p[a];
    }
    used++;
  }
  if (used == 0) return 0;
  int64_t guard = 1, cells = 1;
  int min_b[3], div_b[3];
  for (int a = 0; a < 3; a++) {
    const float extent = (mx[a] - mn[a]) * inv;
    guard *= (int64_t)extent + 1;
    min_b[a] = (int)floorf(mn[a] * inv);
    div_b[a] = (int)floorf(mx[a] * inv) - min_b[a] + 1;
    cells *= div_b[a];
    if (guard > INT32_MAX || cells > INT32_MAX) return -1; /* "Leaf size is too small for the input dataset" */
  }
  const int mul[3] = {1, div_b[0], div_b[0] * div_b[1]};
  index_pair* v = (index_pair*)malloc(sizeof(index_pair) * (size_t)used);
  long m = 0;
  for (long i = 0; i < n; i++) {
    if (!finite3(x[i], y[i], z[i])) continue;
    const int i0 = (int)(floorf(x[i] * inv) - (float)min_b[0]);
    const int i1 = (int)(floorf(y[i] * inv) - (float)min_b[1]);
    const int i2 = (int)(floorf(z[i] * inv) - (float)min_b[2]);
    v[m].idx = (unsigned)(i0 * mul[0] + i1 * mul[1] + i2 * mul[2]);
    v[m++].point = (unsigned)i;
  }
  qsort(v, (size_t)used, sizeof(index_pair), by_idx_then_point);
  long out = 0;
  for (long first = 0; first < used;) {
    long last = first;
    float c[6] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
    for (; last < used && v[last].idx == v[first].idx; last++) {
      const unsigned i = v[last].point;
      c[0] += x[i];
      c[1] += y[i];
      c[2] += z[i];
      c[3] += (float)((rgb[i] >> 16) & 255u); /* pcl::RGB: b, g, r, a in memory */
      c[4] += (float)((rgb[i] >> 8) & 255u);
      c[5] += (float)(rgb[i] & 255u);
    }
    const float scale = 1.0f / (float)(last - first);
    for (int a = 0; a < 6; a++) c[a] *= scale;
    ox[out] = c[0];
    oy[out] = c[1];
    oz[out] = c[2];
    orgb[out] = ((uint32_t)(int)c[3] << 16) | ((uint32_t)(int)c[4] << 8) | (uint32_t)(int)c[5];
    out++;
    first = last;
  }
  free(v);
  return out;
}
