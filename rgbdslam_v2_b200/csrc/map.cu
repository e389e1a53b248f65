// map.cu -- the nodes' colour point clouds and the registered map (RGBDSLAM_B200_STORE_CLOUD, rgbdslam_b200_render_cloud):
//   k_store_depth_cloud   createXYZRGBPointCloud (misc.cpp:467-556) for every frame of a Node-constructor chunk: the z-plane
//                         at the cloud_creation_skip_step raster and, for STORE_CLOUD, the packed colour words (x / y follow
//                         from the pixel)
//   k_store_cloud_points  pc_col of the point-cloud constructor (node.cpp:261): x / y / z planes and, for STORE_CLOUD, the
//                         colour words
// These two build every node cloud: the measurement model (emm.cu) and the map read the same planes.
//   k_map_count           transformAndAppendPointCloud (misc.cpp:183-238): the points each 1024-point block keeps
//   k_map_scan            exclusive scan of the block counts (output offsets, in node order then raster order)
//   k_map_scatter         the kept points of the blocks that overlap one staging piece, transformed, as PCL records
// The float point chain is written with explicit _rn intrinsics: nvcc would otherwise contract it into FMAs, which the
// reference (x86-64 without -mfma) does not do.
#include "kernels.h"
#include "orb.cuh"

namespace rb200 {

constexpr uint32_t kOneF = 0x3f800000u;  // 1.0f: data[3] of a default-constructed pcl::PointXYZ / PointXYZRGB (PCL 1.7)

__device__ __forceinline__ float map_nan() { return __int_as_float(0x7fc00000); }

// The raster is ceil(w / step) x ceil(h / step) (misc.cpp:482-483): point (rx, ry) is pixel (rx * step, ry * step).  Visual
// (NULL: no colour plane) of a depth-image frame: vis_kind 0 grey (w*h bytes), 1 three-channel (3*w*h bytes), 2 Bayer GRBG
// mosaic (w*h bytes, debayered as the listener does before it builds the Node).  Channel c0 is blue under encoding_bgr
// (misc.cpp:487-489, RGBValue :453-464: the word holds b, g, r, a in memory), red without it; alpha is 0.  Point 0 keeps
// colour word 0: its color_idx is 0, which fails `color_idx > 0` (:537).  The reference's colour index only matches the pixel
// when step divides w and h, which the caller requires for colour.
__global__ void __launch_bounds__(256) k_store_depth_cloud(const float* __restrict__ depth, const uint8_t* __restrict__ visual,
                                                           int vis_kind, int bgr, int w, int h, int step, int cw, int ch,
                                                           double scaling, float min_depth, float* __restrict__ out,
                                                           size_t node_words) {
  const int i = blockIdx.x * 256 + threadIdx.x;
  const int P = cw * ch;
  if (i >= P) return;
  const size_t f = blockIdx.y, px = (size_t)w * h;
  const int u = (i % cw) * step, v = (i / cw) * step;
  const size_t pix = (size_t)v * w + u;
  // Z = depth * depth_scaling: a float times a double, one double product rounded to float (misc.cpp:502, 522)
  const float Z = __double2float_rn(__dmul_rn((double)depth[f * px + pix], scaling));
  float* z = out + f * node_words;
  z[i] = Z >= min_depth ? Z : map_nan();  // !(Z >= minimum_depth), NaN included (:525-530)
  if (!visual) return;
  uint32_t word = 0;
  if (i > 0) {
    uint32_t c0, c1, c2;
    if (vis_kind == 0) {
      c0 = c1 = c2 = visual[f * px + pix];
    } else if (vis_kind == 1) {
      const uint8_t* p = visual + 3 * (f * px + pix);
      c0 = p[0];
      c1 = p[1];
      c2 = p[2];
    } else {
      bayer_gr_rgb(visual, f * px, w, h, u, v, c0, c1, c2);
    }
    word = bgr ? (c0 | (c1 << 8) | (c2 << 16)) : (c2 | (c1 << 8) | (c0 << 16));
  }
  reinterpret_cast<uint32_t*>(z + P)[i] = word;
}

cudaError_t launch_store_depth_cloud(int nframes, const float* d_depth, const uint8_t* d_visual, int vis_kind, bool bgr, int w, int h,
                                     int step, double scaling, float min_depth, float* out, size_t node_words, cudaStream_t st) {
  const int cw = (w + step - 1) / step, ch = (h + step - 1) / step;
  k_store_depth_cloud<<<dim3((cw * ch + 255) / 256, nframes), 256, 0, st>>>(d_depth, d_visual, vis_kind, bgr ? 1 : 0, w, h, step, cw,
                                                                             ch, scaling, min_depth, out, node_words);
  return cudaGetLastError();
}

// Organised clouds of `stride` floats per point (8: PointXYZRGB, colour word at byte 16; 4: PointXYZ with RGB_IS_4TH_DIM,
// colour in data[3]) -> per node [x | y | z] planes of n points each, and the colour plane when rgb.
__global__ void __launch_bounds__(256) k_store_cloud_points(const float* __restrict__ cloud, int stride, int n, int rgb,
                                                            float* __restrict__ out, size_t node_words) {
  const int i = blockIdx.x * 256 + threadIdx.x;
  if (i >= n) return;
  const size_t f = blockIdx.y;
  const float* p = cloud + (f * n + i) * stride;
  float* o = out + f * node_words;
  o[i] = p[0];
  o[n + i] = p[1];
  o[2 * (size_t)n + i] = p[2];
  if (rgb) o[3 * (size_t)n + i] = p[stride == 8 ? 4 : 3];
}

cudaError_t launch_store_cloud_points(int nframes, const float* d_cloud, int stride, int n, bool rgb, float* out, size_t node_words,
                                      cudaStream_t st) {
  k_store_cloud_points<<<dim3((n + 255) / 256, nframes), 256, 0, st>>>(d_cloud, stride, n, rgb ? 1 : 0, out, node_words);
  return cudaGetLastError();
}

// ---- the registered map -------------------------------------------------------------------------------------------------

__device__ __forceinline__ float dot3_map(float a0, float b0, float a1, float b1, float a2, float b2) {  // (a0 b0 + a1 b1) + a2 b2
  return __fadd_rn(__fadd_rn(__fmul_rn(a0, b0), __fmul_rn(a1, b1)), __fmul_rn(a2, b2));
}

struct MapOut {
  float x, y, z;
  uint32_t rgb, w16;  // colour word; data[3] of a 16-byte record
};

// Point i of node nd as transformAndAppendPointCloud sees it: returns whether it goes to the output, and what goes there.
__device__ __forceinline__ bool map_point(const MapNode& nd, int i, const MapArgs& a, MapOut& o) {
  float x, y, z;
  o.rgb = nd.rgb[i];
  if (nd.step > 0) {  // depth-image node: x / y of createXYZRGBPointCloud from the pixel
    z = nd.z[i];
    // for a NaN z the reference forms (u - cx) * 1.0 * fxinv in double: the product of two floats is exact there, so it is the
    // rounded float product of the 1 m ray
    const float2 xy = depth_point_xy((float)((i % nd.cw) * nd.step), (float)((i / nd.cw) * nd.step), z, nd.cx, nd.cy, nd.fxinv,
                                     nd.fyinv);
    x = xy.x;
    y = xy.y;
    o.w16 = i == 0 ? kOneF : o.rgb;  // point 0 keeps the default-constructed data[3]
  } else {
    x = nd.x[i];
    y = nd.y[i];
    z = nd.z[i];
    o.w16 = o.rgb;
  }
  // squaredEuclideanDistance(p, origin) > max_Depth^2 (PCL: ((dx dx + dy dy) + dz dz), dx = 0 - x)
  if (a.filter && __fadd_rn(__fadd_rn(__fmul_rn(x, x), __fmul_rn(y, y)), __fmul_rn(z, z)) > a.maxd2) {
    o.x = o.y = o.z = map_nan();
    return a.preserve != 0;
  }
  if (isnan(x) || isnan(y) || isnan(z)) {  // left as it is (+-inf is not NaN and is transformed)
    o.x = x;
    o.y = y;
    o.z = z;
    return a.preserve != 0;
  }
  if (a.transform) {  // p_out = rot * p_in + trans (Matrix4f of pcl_ros::transformAsMatrix)
    o.x = __fadd_rn(dot3_map(nd.m[0], x, nd.m[1], y, nd.m[2], z), nd.m[3]);
    o.y = __fadd_rn(dot3_map(nd.m[4], x, nd.m[5], y, nd.m[6], z), nd.m[7]);
    o.z = __fadd_rn(dot3_map(nd.m[8], x, nd.m[9], y, nd.m[10], z), nd.m[11]);
  } else {
    o.x = x;
    o.y = y;
    o.z = z;
  }
  return true;
}

constexpr int kMapThreads = 256;

__global__ void __launch_bounds__(kMapThreads) k_map_count(const MapNode* __restrict__ nodes, const int2* __restrict__ blocks, MapArgs a,
                                                           int* __restrict__ counts) {
  __shared__ int warp_sum[kMapThreads / 32];
  const int2 blk = blocks[blockIdx.x];
  const MapNode& nd = nodes[blk.x];
  const int P = nd.cw * nd.ch;
  int c = 0;
#pragma unroll
  for (int k = 0; k < kMapBlockPoints / kMapThreads; k++) {
    const int i = blk.y + k * kMapThreads + threadIdx.x;
    MapOut o;
    if (i < P && map_point(nd, i, a, o)) c++;
  }
#pragma unroll
  for (int s = 16; s > 0; s >>= 1) c += __shfl_xor_sync(0xffffffffu, c, s);
  if ((threadIdx.x & 31) == 0) warp_sum[threadIdx.x >> 5] = c;
  __syncthreads();
  if (threadIdx.x == 0) {
    int t = 0;
    for (int w = 0; w < kMapThreads / 32; w++) t += warp_sum[w];
    counts[blockIdx.x] = t;
  }
}

// One CTA: offs[b] = sum of counts[0, b), offs[n] = total.
__global__ void __launch_bounds__(1024) k_map_scan(const int* __restrict__ counts, int n, long long* __restrict__ offs) {
  __shared__ long long warp_sum[32];
  __shared__ long long carry;
  if (threadIdx.x == 0) carry = 0;
  __syncthreads();
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  for (int base = 0; base < n; base += 1024) {
    const int b = base + threadIdx.x;
    const long long c = b < n ? counts[b] : 0;
    long long incl = c;
#pragma unroll
    for (int s = 1; s < 32; s <<= 1) {
      const long long t = __shfl_up_sync(0xffffffffu, incl, s);
      if (lane >= s) incl += t;
    }
    if (lane == 31) warp_sum[wid] = incl;
    __syncthreads();
    if (wid == 0) {
      long long ws = warp_sum[lane];
#pragma unroll
      for (int s = 1; s < 32; s <<= 1) {
        const long long t = __shfl_up_sync(0xffffffffu, ws, s);
        if (lane >= s) ws += t;
      }
      warp_sum[lane] = ws;  // inclusive over warps
    }
    __syncthreads();
    const long long before = carry + (wid > 0 ? warp_sum[wid - 1] : 0);
    if (b < n) offs[b] = before + incl - c;
    __syncthreads();
    if (threadIdx.x == 0) carry += warp_sum[31];
    __syncthreads();
  }
  if (threadIdx.x == 0) offs[n] = carry;
}

// Blocks [b0, b0 + gridDim.x): the kept points whose output index lies in [lo, hi) go to out[index - lo] as PCL records --
// 32 bytes (PointXYZRGB: x, y, z, 1.0f, colour, 12 zero bytes) or 16 bytes (PointXYZ: x, y, z, data[3] = colour).
__global__ void __launch_bounds__(kMapThreads) k_map_scatter(const MapNode* __restrict__ nodes, const int2* __restrict__ blocks,
                                                             const long long* __restrict__ offs, int b0, long long lo, long long hi,
                                                             MapArgs a, uint4* __restrict__ out) {
  __shared__ int warp_cnt[kMapThreads / 32];
  const int b = b0 + blockIdx.x;
  const int2 blk = blocks[b];
  const MapNode& nd = nodes[blk.x];
  const int P = nd.cw * nd.ch;
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  long long next = offs[b];
#pragma unroll 1
  for (int k = 0; k < kMapBlockPoints / kMapThreads; k++) {
    const int i = blk.y + k * kMapThreads + threadIdx.x;
    MapOut o;
    const bool keep = i < P && map_point(nd, i, a, o);
    const unsigned bal = __ballot_sync(0xffffffffu, keep);
    if (lane == 0) warp_cnt[wid] = __popc(bal);
    __syncthreads();
    int before = 0, total = 0;
#pragma unroll
    for (int w = 0; w < kMapThreads / 32; w++) {
      const int c = warp_cnt[w];
      before += w < wid ? c : 0;
      total += c;
    }
    const long long g = next + before + __popc(bal & ((1u << lane) - 1u));
    if (keep && g >= lo && g < hi) {
      const size_t r = (size_t)(g - lo);
      if (a.point_bytes == 32) {
        out[2 * r] = make_uint4(__float_as_uint(o.x), __float_as_uint(o.y), __float_as_uint(o.z), kOneF);
        out[2 * r + 1] = make_uint4(o.rgb, 0u, 0u, 0u);
      } else {
        out[r] = make_uint4(__float_as_uint(o.x), __float_as_uint(o.y), __float_as_uint(o.z), o.w16);
      }
    }
    next += total;
    __syncthreads();
  }
}

cudaError_t launch_map_count(const MapNode* d_nodes, const int2* d_blocks, int nblocks, const MapArgs& a, int* d_counts,
                             cudaStream_t st) {
  if (nblocks <= 0) return cudaSuccess;
  k_map_count<<<nblocks, kMapThreads, 0, st>>>(d_nodes, d_blocks, a, d_counts);
  return cudaGetLastError();
}

cudaError_t launch_map_scan(const int* d_counts, int nblocks, long long* d_offs, cudaStream_t st) {
  k_map_scan<<<1, 1024, 0, st>>>(d_counts, nblocks, d_offs);
  return cudaGetLastError();
}

cudaError_t launch_map_scatter(const MapNode* d_nodes, const int2* d_blocks, const long long* d_offs, int b0, int b1, long long lo,
                               long long hi, const MapArgs& a, void* d_out, cudaStream_t st) {
  if (b1 <= b0) return cudaSuccess;
  k_map_scatter<<<b1 - b0, kMapThreads, 0, st>>>(d_nodes, d_blocks, d_offs, b0, lo, hi, a, (uint4*)d_out);
  return cudaGetLastError();
}

}  // namespace rb200
