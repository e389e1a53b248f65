/*
 * rgbdslam_b200/cloud_transform.h -- C ABI of the in-place transform of the stored colour clouds: the
 * transform_individual_clouds step of GraphManager::saveIndividualCloudsToFile (graph_mgr_io.cpp:372-374), the reference's
 * parameter transform_individual_clouds (parameter_server.cpp:67).  The conventions of ../rgbdslam_b200.h hold; the call needs
 * an initialised library.  The clouds are those of map.h, and a transformed cloud is read by the calls of map.h unchanged.
 */
#ifndef RGBDSLAM_B200_CLOUD_TRANSFORM_H
#define RGBDSLAM_B200_CLOUD_TRANSFORM_H

#include "../rgbdslam_b200.h"

#ifdef __cplusplus
extern "C" {
#endif

/* == pcl::transformPointCloud(*pc_col, *pc_col, m) (PCL 1.7) for n nodes built with RGBDSLAM_B200_STORE_CLOUD, node k by
 * m = transforms12[k] (row-major 3 x 4 doubles, each entry cast to float: v->estimate().matrix().cast<float>()).  The clouds
 * are not dense, so a point with a non-finite x, y or z (NaN or +-inf) is left as it is, and every other point becomes, per
 * row r, ((m_r0 x + m_r1 y) + m_r2 z) + m_r3 in float without FMA contraction.  Colour words, data[3] and the raster (w x h,
 * organised or not) stay; a depth-image point without depth keeps x = (u - cx) / fx, y = (v - cy) / fy, z = NaN.
 * The node keeps the transformed cloud: rgbdslam_b200_node_download_cloud, rgbdslam_b200_render_cloud,
 * rgbdslam_b200_reduce_clouds, rgbdslam_b200_octomap_insert and rgbdslam_b200_octomap_filter_clouds read it as they read any
 * stored cloud, and a second call transforms it again.  Its points are no longer camera points: the environment measurement
 * model (rgbdslam_b200_match_pairs* with observability_threshold > 0, rgbdslam_b200_observation_likelihood) and
 * rgbdslam_b200_icp_align(_ex) return ERR_STATE for a node it has transformed.  Deterministic; the result does not depend on
 * how many nodes one call transforms.  The old cloud's device memory is freed once every node of the call that made it has
 * let go of it.
 * ERR_ARG before any device work: n < 0, an unknown handle, a handle listed twice, a non-finite transform entry.  ERR_STATE
 * before any device work: a node without a stored colour cloud.  When the call fails no node is changed. */
int rgbdslam_b200_transform_clouds(int n, const uint64_t* nodes, const double* transforms12);

#ifdef __cplusplus
}
#endif
#endif /* RGBDSLAM_B200_CLOUD_TRANSFORM_H */
