/* map_cloud_oracle.c -- plain-C restatement of the reference's colour cloud and map steps, for tests/map_cloud_exact.py.
 * Built with -O2 -ffp-contract=off, so every float operation is rounded on its own as on an x86-64 build without -mfma.
 *   map_create_cloud      createXYZRGBPointCloud (misc.cpp:467-556), with its running colour / depth index arithmetic
 *   map_transform_append  transformAndAppendPointCloud (misc.cpp:183-238) of one cloud of 32-byte PointXYZRGB records
 */
#include <math.h>
#include <stdint.h>
#include <string.h>

typedef struct {
  float x, y, z;
  uint32_t w;  /* data[3] */
  uint32_t rgb;
  uint32_t pad[3];
} point32;
typedef struct {
  float x, y, z;
  uint32_t w;
} point16;

/* depth: w x h float metres, visual: w x h x ch bytes (ch 1 or 3), K4 = fx, fy, cx, cy.  out: (h / step) x (w / step) records of
 * point_bytes (32: PointXYZRGB, 16: PointXYZ with the colour in data[3]).  Every point starts default-constructed (PCL 1.7:
 * x = y = z = 0, data[3] = 1, colour 0). */
void map_create_cloud(const float* depth, const uint8_t* visual, int w, int h, int ch, const float* K4, int step, double scaling,
                      float min_depth, int bgr, int point_bytes, void* out) {
  const float fxinv = (float)(1.0 / (double)K4[0]), fyinv = (float)(1.0 / (double)K4[1]), cx = K4[2], cy = K4[3];
  const int cw = (int)ceilf(w / (float)step), chh = (int)ceilf(h / (float)step);
  const int red = ch == 3 && bgr ? 2 : 0, blue = ch == 3 && bgr ? 0 : 2;
  const unsigned pix_step = ch * (w / cw), row_step = ch * (h / chh - 1) * w;
  const unsigned dpix_step = w / cw, drow_step = (h / chh - 1) * w;
  const long total = (long)w * h;
  int color_idx = 0, depth_idx = 0;
  long n = 0;
  for (int v = 0; v < h; v += step, color_idx += row_step, depth_idx += drow_step)
    for (int u = 0; u < w; u += step, color_idx += pix_step, depth_idx += dpix_step, n++) {
      if (n >= (long)cw * chh) break;
      float x = 0.f, y = 0.f, z = 0.f;
      uint32_t w3 = 0x3f800000u, rgb = 0;
      const float Z = (float)(depth[depth_idx] * scaling);
      if (!(Z >= min_depth)) {
        x = (float)((u - cx) * 1.0 * fxinv);
        y = (float)((v - cy) * 1.0 * fyinv);
        z = NAN;
      } else {
        const float uf = (float)u, vf = (float)v;
        x = (uf - cx) * Z * fxinv;
        y = (vf - cy) * Z * fyinv;
        z = Z;
      }
      if (color_idx > 0 && color_idx < total * (long)pix_step) {
        uint8_t r, g, b;
        if (ch == 3) {
          r = visual[color_idx + red];
          g = visual[color_idx + 1];
          b = visual[color_idx + blue];
        } else {
          r = g = b = visual[color_idx];
        }
        rgb = (uint32_t)b | ((uint32_t)g << 8) | ((uint32_t)r << 16);  /* b, g, r, a bytes; alpha 0 */
        w3 = point_bytes == 16 ? rgb : w3;
      }
      if (point_bytes == 32) {
        point32* p = (point32*)out + n;
        memset(p, 0, sizeof(*p));
        p->x = x, p->y = y, p->z = z, p->w = w3, p->rgb = rgb;
      } else {
        point16* p = (point16*)out + n;
        p->x = x, p->y = y, p->z = z, p->w = w3;
      }
    }
}

/* One cloud of n records appended to an empty aggregate: returns the number of output records.  T: row-major 3 x 4 double,
 * cast to float entry by entry; R p summed as (r0 p0 + r1 p1) + r2 p2. */
long map_transform_append(const point32* in, long n, const double* T, float max_depth, int preserve, point32* out) {
  float R[12];
  for (int k = 0; k < 12; k++) R[k] = (float)T[k];
  long j = 0;
  for (long i = 0; i < n; i++) {
    const point32 p = in[i];
    if (!preserve) out[j] = p;
    else out[i] = p;  /* the untransformed copy of cloud_to_append_to += cloud_in */
    point32* o = preserve ? &out[i] : &out[j];
    if (max_depth >= 0) {
      const float dx = 0.f - p.x, dy = 0.f - p.y, dz = 0.f - p.z;
      if (dx * dx + dy * dy + dz * dz > max_depth * max_depth) {
        o->x = o->y = o->z = NAN;
        if (preserve) j++;
        continue;
      }
    }
    if (isnan(p.x) || isnan(p.y) || isnan(p.z)) {
      if (preserve) j++;
      continue;
    }
    const float a0 = R[0] * p.x, a1 = R[1] * p.y, a2 = R[2] * p.z;
    const float b0 = R[4] * p.x, b1 = R[5] * p.y, b2 = R[6] * p.z;
    const float c0 = R[8] * p.x, c1 = R[9] * p.y, c2 = R[10] * p.z;
    o->x = ((a0 + a1) + a2) + R[3];
    o->y = ((b0 + b1) + b2) + R[7];
    o->z = ((c0 + c1) + c2) + R[11];
    j++;
  }
  return j;
}
