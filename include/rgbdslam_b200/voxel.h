/*
 * rgbdslam_b200/voxel.h -- C ABI of the voxel filter of the stored colour clouds: Node::reducePointCloud (node.cpp:1448-1460),
 * the reference's parameter voxelfilter_size (parameter_server.cpp:159).  The conventions of ../rgbdslam_b200.h hold; the call
 * needs an initialised library.  The clouds are those of map.h, and a reduced cloud is read by the calls of map.h unchanged.
 */
#ifndef RGBDSLAM_B200_VOXEL_H
#define RGBDSLAM_B200_VOXEL_H

#include "../rgbdslam_b200.h"

#ifdef __cplusplus
extern "C" {
#endif

/* == Node::reducePointCloud(voxelfilter_size) (node.cpp:1448-1460) for n nodes built with RGBDSLAM_B200_STORE_CLOUD: each
 * node's pc_col is replaced, on the device, by what pcl::VoxelGrid<PointXYZRGB> (PCL 1.7, setLeafSize(v, v, v), all fields
 * downsampled, no filter field) makes of it -- one point per occupied voxel, the centroid of the voxel's points and the mean of
 * their colours.  The rule, with leaf = (float)voxelfilter_size and inv = 1.0f / leaf, every operation in float unless noted:
 *   - a point takes part when x, y and z are all finite; min_p / max_p are the per-axis bounds of those points;
 *   - min_b = (int)floor(min_p * inv), max_b likewise, div_b = max_b - min_b + 1 per axis; a point's voxel index is
 *     ix + iy * div_b.x + iz * div_b.x * div_b.y with ix = (int)(floor(x * inv) - (float)min_b.x);
 *   - when ((int64)((max_p.x - min_p.x) * inv) + 1) * (the same for y) * (for z), or div_b.x * div_b.y * div_b.z, exceeds
 *     INT32_MAX the leaf size is too small for the cloud (PCL warns and copies its input): that node keeps its cloud as it is
 *     and reports -1, the other nodes of the call are reduced;
 *   - the output holds one point per occupied voxel in ascending voxel index.  x, y, z and the r, g, b bytes of the colour
 *     word (bytes 2, 1, 0) are each summed in float over the voxel's points in raster order -- PCL's sort leaves that order
 *     open, this is the library's fixed choice -- and multiplied by 1.0f / n; the colour word is (r << 16) | (g << 8) | b of
 *     the means truncated to integers, alpha 0.
 * The reduced cloud is unorganised, *w = the number of voxels and *h = 1 in rgbdslam_b200_node_download_cloud (0 x 1 when no
 * point was finite); its 32-byte records have data[3] = 1.0f and its 16-byte records carry the colour word in data[3], as a
 * point-cloud node's.  rgbdslam_b200_render_cloud reads reduced and unreduced nodes alike.  A reduced node may be reduced
 * again.  Its cloud no longer feeds the environment measurement model (the reference refuses the combination,
 * parameter_server.cpp:233): rgbdslam_b200_match_pairs* with observability_threshold > 0 and
 * rgbdslam_b200_observation_likelihood return ERR_STATE for it.  Features, keypoints and everything else of the node stay.
 * n_points (may be NULL) receives each node's new point count, or -1.  Deterministic; the result does not depend on how
 * many nodes one call reduces.  The old cloud's device memory is freed once every node of the nodes_create call that made it
 * has been reduced or destroyed.
 * ERR_ARG before any device work: n < 0, a voxelfilter_size that is not finite or not > 0 as a float (the reference warns and
 * does nothing), an unknown handle, a handle listed twice.  ERR_STATE before any device work: a node without a stored colour
 * cloud.  When the call fails no node is changed. */
int rgbdslam_b200_reduce_clouds(int n, const uint64_t* nodes, double voxelfilter_size, int32_t* n_points);

#ifdef __cplusplus
}
#endif
#endif /* RGBDSLAM_B200_VOXEL_H */
