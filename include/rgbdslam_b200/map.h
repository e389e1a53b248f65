/*
 * rgbdslam_b200/map.h -- C ABI of the stored colour clouds and the registered map: Node::pc_col (node.cpp:126-131, 261) of the
 * nodes built with RGBDSLAM_B200_STORE_CLOUD (rgbdslam_b200_nodes_create_ex, ../rgbdslam_b200.h) and
 * GraphManager::saveAllCloudsToFile (graph_mgr_io.cpp:502-583).  The conventions of ../rgbdslam_b200.h hold; both calls
 * need an initialised library.
 * The voxel filter of these clouds (Node::reducePointCloud) is declared in voxel.h and their in-place transform
 * (transform_individual_clouds) in cloud_transform.h; both calls read a reduced or transformed cloud as they read any other.
 */
#ifndef RGBDSLAM_B200_MAP_H
#define RGBDSLAM_B200_MAP_H

#include "../rgbdslam_b200.h"

#ifdef __cplusplus
extern "C" {
#endif

/* Node::pc_col of a node built with RGBDSLAM_B200_STORE_CLOUD as the organised cloud the reference holds: *w x *h records in
 * raster order (depth-image nodes: w / skip step x h / skip step; point-cloud nodes: the input's size).  point_bytes 32:
 * pcl::PointXYZRGB -- x, y, z, data[3] = 1.0f, the colour word, 12 zero bytes; 16: pcl::PointXYZ with the colour word in data[3]
 * (RGB_IS_4TH_DIM).  A depth-image point without depth is x = (u - cx) / fx, y = (v - cy) / fy, z = NaN (misc.cpp:525-530);
 * point 0 of a depth-image node has colour word 0 and data[3] = 1.0f, what PCL 1.7's default constructors leave.  out may be
 * NULL (only *w, *h).  ERR_STATE for a node without a stored cloud, ERR_ARG for point_bytes other than 16 or 32. */
int rgbdslam_b200_node_download_cloud(uint64_t node_handle, int point_bytes, void* out, int* w, int* h);
/* == transformAndAppendPointCloud(*node->pc_col, aggregate, transform, maximum_depth) (misc.cpp:183-238) for n nodes in the
 * order given, the loop of GraphManager::saveAllCloudsToFile (graph_mgr_io.cpp:502-583) without its node selection.
 * transforms12: n row-major 3 x 4 doubles, cast entry by entry to float as pcl_ros::transformAsMatrix does; used16 (may be
 * NULL) receives the n float matrices used (Eigen::Matrix4f, column-major).  maximum_depth is taken as a float; when it is >= 0
 * a point whose untransformed squared distance ((x^2 + y^2) + z^2, float) exceeds its square is dropped, or with preserve_raster
 * (preserve_raster_on_save) kept with x = y = z = NaN; otherwise a point with a NaN coordinate is dropped, or kept unchanged
 * with preserve_raster; every other point (+-inf included) becomes R p + t in float, R p summed as (r0 p0 + r1 p1) + r2 p2.
 * Records as rgbdslam_b200_node_download_cloud, in node order then raster order; deterministic.  *n_out = the number of
 * records.  out == NULL: only the count.  Otherwise out (host, pinned or pageable) must hold `capacity` records: with fewer
 * the call returns ERR_ARG with *n_out set and writes nothing.  ERR_ARG before any device work for point_bytes other than 16
 * or 32 or a non-finite transform entry, ERR_STATE for a node without a stored cloud. */
int rgbdslam_b200_render_cloud(int n, const uint64_t* nodes, const double* transforms12, double maximum_depth, int preserve_raster,
                               int point_bytes, void* out, int64_t capacity, int64_t* n_out, float* used16);

#ifdef __cplusplus
}
#endif
#endif /* RGBDSLAM_B200_MAP_H */
