/*
 * rgbdslam_b200/octomap.h -- C ABI of the colour OctoMap built from the nodes' stored clouds: GraphManager::saveOctomap /
 * renderToOctomap (graph_mgr_io.cpp:253-329) over ColorOctomapServer::insertCloudCallback (ColorOctomapServer.cpp), i.e.
 * octomap::ColorOcTree::insertPointCloud(cloud, origin, max_range, lazy_eval = true), averageNodeColor for every point,
 * updateInnerOccupancy, and ColorOcTree::write (the .ot format).  The conventions of ../rgbdslam_b200.h hold; every call but
 * default_params needs an initialised library.  The clouds are those of map.h, reduced (voxel.h) or not.
 *
 * The map is a handle owning device memory: the leaves (16-level keys, float log-odds, colour) in Morton order.  The rules,
 * restated from octomap 1.6-1.8 (DESIGN.md 4.14):
 *   - a point is map_point of its node (map.h's transform, no depth filter); one with a non-finite coordinate contributes
 *     nothing.  The ray origin is the transform's translation column.
 *   - key(c) = (int)floor((1 / res) * (double)c) + 32768, rejected outside [0, 65536) (NaN and +-inf included).
 *   - the cells of a ray are OcTreeBaseImpl::computeRayKeys (Amanatides & Woo in double with float direction and length).
 *   - per node (scan): with max_range < 0 or |p - origin| <= max_range the ray's cells are free and key(p) occupied, otherwise
 *     the ray to origin + normalized(p - origin) * (float)max_range is all free; a key both free and occupied is occupied;
 *     each key of the scan gets one update: l = clamp(l + logodds(hit or miss)) in float, a new leaf starting at 0.
 *   - then every point with finite coordinates, in point order, folds its colour into the leaf at key(p) if that leaf exists:
 *     (prev + new) / 2 per channel in int, or the new colour when the leaf's is unset -- (255, 255, 255) counts as unset.
 *   - inner nodes: log-odds the maximum over the children, colour the int mean of the children whose colour is set (else
 *     (255, 255, 255)).  Nothing is pruned.
 * Nodes are inserted one after another in the order given; how many one call takes changes nothing.
 */
#ifndef RGBDSLAM_B200_OCTOMAP_H
#define RGBDSLAM_B200_OCTOMAP_H

#include "../rgbdslam_b200.h"

#ifdef __cplusplus
extern "C" {
#endif

/* The ColorOctomapServer::reset parameters (parameter_server.cpp:56-65); occupancy_threshold does not change the file. */
typedef struct rgbdslam_b200_octomap_params {
  double resolution;    /* octomap_resolution, metres: > 0 */
  double prob_hit;      /* octomap_prob_hit: in (0, 1) */
  double prob_miss;     /* octomap_prob_miss: in (0, 1) */
  double clamping_min;  /* octomap_clamping_min: in (0, 1), <= clamping_max */
  double clamping_max;  /* octomap_clamping_max: in (0, 1) */
} rgbdslam_b200_octomap_params;

/* The reference's defaults: 0.05, 0.9, 0.4, 0.001, 0.999.  Needs no library. */
void rgbdslam_b200_octomap_default_params(rgbdslam_b200_octomap_params* p);
/* An empty map.  ERR_ARG for a parameter out of its range (above) or a null argument. */
int rgbdslam_b200_octomap_create(const rgbdslam_b200_octomap_params* p, uint64_t* map);
/* Inserts n nodes' stored clouds in order.  transforms12: n row-major 3 x 4 floats, node -> map (the pose chain of
 * updateCloudOrigin and pcl_ros::transformPointCloud, formed by the caller); max_range: maximum_depth, < 0 or +inf for none.
 * ERR_ARG before any device work for a bad handle, a non-finite matrix entry or a NaN max_range; ERR_STATE for a node without
 * a stored cloud; the map is then unchanged.  A failure during device work (ERR_CUDA, e.g. out of memory) leaves the map
 * holding some prefix of the call's nodes, possibly with part of one node's update: clear or destroy it then. */
int rgbdslam_b200_octomap_insert(uint64_t map, int n, const uint64_t* nodes, const float* transforms12, double max_range);
/* The .ot file (AbstractOcTree::write) into out: *n_bytes = its size.  out == NULL: only the size.  Otherwise out must hold
 * `capacity` bytes: with fewer the call returns ERR_ARG with *n_bytes set and writes nothing. */
int rgbdslam_b200_octomap_write(uint64_t map, void* out, int64_t capacity, int64_t* n_bytes);
/* *nodes = the tree's node count, the root included (0 for an empty map); *leaves = its leaves at full depth. */
int rgbdslam_b200_octomap_stats(uint64_t map, int64_t* nodes, int64_t* leaves);
/* ColorOctomapServer::reset without new parameters: the map becomes empty and every device buffer it holds is freed. */
int rgbdslam_b200_octomap_clear(uint64_t map);
int rgbdslam_b200_octomap_destroy(uint64_t map);
/* Node::clearPointCloud (octomap_clear_raycasted_clouds): the node drops its stored cloud (Node::pc_col, also the cloud the
 * measurement model and ICP read) and its device memory is freed with the last node of its allocation that lets it go.
 * Features and keypoints stay.  A node without a cloud is left as it is. */
int rgbdslam_b200_node_clear_cloud(uint64_t node_handle);

/* ColorOctomapServer::occupancyFilter(pc_col, pc_col, occupancy_threshold) (ColorOctomapServer.cpp:132-185) for n nodes, in
 * place: GraphManager::occupancyFilterClouds (graph_manager.cpp:1372-1381).  sensor7: per node qx qy qz qw ox oy oz, the
 * cloud's sensor_orientation_ / sensor_origin_ (updateCloudOrigin; PCL's default is 0 0 0 1 0 0 0).  n_points may be NULL,
 * else it receives each node's new point count.  The rule (DESIGN.md 4.15), for each point p of the cloud in storage order --
 * p as node_download_cloud returns it:
 *   1. in = q * p + t in float, q * p Eigen's _transformVector: uv = q.vec() x p; uv += uv; v = p + q.w() * uv + q.vec() x uv,
 *      each component left to right without contraction, then + t.
 *   2. in.z NaN: the point is dropped.
 *   3. k = coordToKey(in.c) per axis, unchecked: (uint16)((int)floor((1 / res) * (double)c) + 32768), (int) as x86-64
 *      converts (INT_MIN for NaN, +-inf and out of range).
 *   4. a = k - 1 per axis: the reference's nested loops never reset y_a and z_a, so only the cells (ax, ay, az + d), d = 0, 1,
 *      2, are visited, every key taken back to uint16 (-1 is 65535).
 *   5. for each visited cell that is a leaf of the map: d. = keyToCoord(key.) - (double)in., w = (dx dx + dy dy) + dz dz,
 *      occ = 1 - 1 / (1 + exp((double)lo)) as glibc computes it; sum_occ += occ / w, sum_w += w (double).
 *   6. the point is kept iff sum_occ < threshold * sum_w: a point with no visited leaf (e.g. every point of an empty map) is
 *      dropped.
 * Kept points keep their records, in order.  A node that keeps every point keeps its cloud as it is (same raster, no copy);
 * any other becomes an unorganised n x 1 cloud (0 x 1 when nothing is kept) that render_cloud, octomap_insert, reduce_clouds,
 * icp_align and this call read, and that the measurement model refuses (ERR_STATE) for want of a raster.  How many nodes one
 * call takes changes nothing.  ERR_ARG before any device work for a bad map or node handle, a node listed twice, a non-finite
 * sensor7 entry or a NaN threshold; ERR_STATE for a node without a stored cloud.  A failed call changes no node. */
int rgbdslam_b200_octomap_filter_clouds(uint64_t map, int n, const uint64_t* nodes, const float* sensor7, double occupancy_threshold,
                                        int32_t* n_points);

#ifdef __cplusplus
}
#endif
#endif /* RGBDSLAM_B200_OCTOMAP_H */
