// map.cuh -- the one reader of a node's stored cloud (Node::pc_col): point i of a MapNode as transformAndAppendPointCloud
// sees it.  Shared by the map kernels (map.cu) and the voxel filter (voxel.cu).
#pragma once
#include "kernels.h"

namespace rb200 {

constexpr uint32_t kOneF = 0x3f800000u;  // 1.0f: data[3] of a default-constructed pcl::PointXYZ / PointXYZRGB (PCL 1.7)

__device__ __forceinline__ float map_nan() { return __int_as_float(0x7fc00000); }

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
    o.w16 = i == 0 && nd.point0_one ? kOneF : o.rgb;
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

}  // namespace rb200
