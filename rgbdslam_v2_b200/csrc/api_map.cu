// api_map.cu -- C ABI of the stored colour clouds and the registered map, host orchestration:
//   rgbdslam_b200_node_download_cloud  == Node::pc_col (node.cpp:126-131, 261) as an organised cloud
//   rgbdslam_b200_render_cloud         == transformAndAppendPointCloud (misc.cpp:183-238) of many nodes, the loop of
//                                         GraphManager::saveAllCloudsToFile (graph_mgr_io.cpp:502-583)
// Both run count -> scan -> scatter (map.cu) and move the records to the host through a two-piece device staging ring: the copy
// of piece k runs on its own stream while piece k + 1 is computed.
#include <algorithm>
#include <cmath>
#include <cstring>
#include <vector>

#include "../../include/rgbdslam_b200/map.h"
#include "kernels.h"
#include "state.h"

namespace rb200 {

constexpr long long kMapPiecePoints = 1 << 21;  // records per staging piece (64 MB of 32-byte records)

struct MapCtx {
  cudaStream_t copy_stream = nullptr;
  cudaEvent_t ev_done[2] = {nullptr, nullptr}, ev_copied[2] = {nullptr, nullptr};
  DevBuf nodes, blocks, counts, offs, stage[2];
};
static MapCtx g_map;

static int map_ensure_streams() {
  MapCtx& m = g_map;
  if (m.copy_stream) return 0;
  cudaError_t e = cudaStreamCreateWithFlags(&m.copy_stream, cudaStreamNonBlocking);
  for (int i = 0; i < 2 && e == cudaSuccess; i++) {
    e = cudaEventCreateWithFlags(&m.ev_done[i], cudaEventDisableTiming);
    if (e == cudaSuccess) e = cudaEventCreateWithFlags(&m.ev_copied[i], cudaEventDisableTiming);
  }
  if (e != cudaSuccess) return cuda_fail(e, "map streams / events");
  return 0;
}

// The stored cloud of nd as the map kernels read it, with transform T (row-major 3 x 4 float; may be NULL).
static MapNode map_node(const NodeDev* nd, const float* T) {
  const NodeCloud& c = nd->pc;
  MapNode m;
  memset(&m, 0, sizeof(m));
  m.x = c.x;
  m.y = c.y;
  m.z = c.z;
  m.rgb = c.rgb;
  m.cw = c.w;
  m.ch = c.h;
  m.step = c.step;
  m.fxinv = (float)(1.0 / (double)c.K[0]);  // getCameraIntrinsicsInverseFocalLength (misc.cpp:64-69); unused by organised clouds
  m.fyinv = (float)(1.0 / (double)c.K[1]);
  m.cx = c.K[2];
  m.cy = c.K[3];
  if (T) memcpy(m.m, T, sizeof(m.m));
  return m;
}

// Count, scan and (unless out is NULL) scatter the records of `nodes` into the host buffer out (capacity records).
static int map_emit(const std::vector<MapNode>& nodes, const MapArgs& a, void* out, int64_t capacity, int64_t* n_out) {
  MapCtx& m = g_map;
  State& s = g_state;
  cudaStream_t st = s.stream;
  int rc;
  if ((rc = map_ensure_streams())) return rc;
  std::vector<int2> blocks;
  for (size_t k = 0; k < nodes.size(); k++) {
    const int P = nodes[k].cw * nodes[k].ch;
    for (int first = 0; first < P; first += kMapBlockPoints) blocks.push_back(make_int2((int)k, first));
  }
  const int nb = (int)blocks.size();
  std::vector<long long> offs(nb + 1);
  if ((rc = m.nodes.ensure(sizeof(MapNode) * std::max<size_t>(nodes.size(), 1))) ||
      (rc = m.blocks.ensure(sizeof(int2) * std::max(nb, 1))) || (rc = m.counts.ensure(4 * (size_t)std::max(nb, 1))) ||
      (rc = m.offs.ensure(8 * (size_t)(nb + 1))))
    return rc;
  int launches = 0;
  if (!nodes.empty()) RB200_CUDA(cudaMemcpyAsync(m.nodes.ptr, nodes.data(), sizeof(MapNode) * nodes.size(), cudaMemcpyHostToDevice, st));
  if (nb > 0) RB200_CUDA(cudaMemcpyAsync(m.blocks.ptr, blocks.data(), sizeof(int2) * nb, cudaMemcpyHostToDevice, st));
  const MapNode* d_nodes = (const MapNode*)m.nodes.ptr;
  const int2* d_blocks = (const int2*)m.blocks.ptr;
  long long* d_offs = (long long*)m.offs.ptr;
  RB200_CUDA(launch_map_count(d_nodes, d_blocks, nb, a, (int*)m.counts.ptr, st));
  RB200_CUDA(launch_map_scan((const int*)m.counts.ptr, nb, d_offs, st));
  launches += (nb > 0) + 1;
  RB200_CUDA(cudaMemcpyAsync(offs.data(), d_offs, 8 * (size_t)(nb + 1), cudaMemcpyDeviceToHost, st));
  RB200_CUDA(cudaStreamSynchronize(st));
  const long long total = offs[nb];
  *n_out = total;
  s.launches += launches;
  if (!out) return 0;
  if (capacity < total) {
    set_error("render_cloud: capacity " + std::to_string(capacity) + " < " + std::to_string(total) + " records");
    return RGBDSLAM_B200_ERR_ARG;
  }
  const size_t pb = (size_t)a.point_bytes;
  const long long npieces = (total + kMapPiecePoints - 1) / kMapPiecePoints;
  for (int b = 0; b < 2 && b < npieces; b++)
    if ((rc = m.stage[b].ensure(pb * (size_t)kMapPiecePoints))) return rc;
  // scatter of piece p into staging buffer p & 1, after the copy out of that buffer (piece p - 2) has finished
  auto scatter = [&](long long p) -> int {
    const int buf = (int)(p & 1);
    const long long lo = p * kMapPiecePoints, hi = std::min(total, lo + kMapPiecePoints);
    // the blocks whose outputs overlap [lo, hi): from the one holding lo to the first that starts at or after hi
    const int b0 = (int)(std::upper_bound(offs.begin(), offs.begin() + nb, lo) - offs.begin()) - 1;
    const int b1 = (int)(std::lower_bound(offs.begin(), offs.begin() + nb, hi) - offs.begin());
    if (p >= 2) RB200_CUDA(cudaStreamWaitEvent(st, m.ev_copied[buf], 0));
    RB200_CUDA(launch_map_scatter(d_nodes, d_blocks, d_offs, std::max(b0, 0), b1, lo, hi, a, m.stage[buf].ptr, st));
    RB200_CUDA(cudaEventRecord(m.ev_done[buf], st));
    s.launches += 1;
    return 0;
  };
  if (npieces > 0 && (rc = scatter(0))) return rc;
  for (long long p = 0; p < npieces; p++) {
    // queue the next piece's kernel before this piece's copy: a copy into pageable memory returns only when it is done
    if (p + 1 < npieces && (rc = scatter(p + 1))) return rc;
    const int buf = (int)(p & 1);
    const long long lo = p * kMapPiecePoints, hi = std::min(total, lo + kMapPiecePoints);
    RB200_CUDA(cudaStreamWaitEvent(m.copy_stream, m.ev_done[buf], 0));
    RB200_CUDA(cudaMemcpyAsync((uint8_t*)out + pb * (size_t)lo, m.stage[buf].ptr, pb * (size_t)(hi - lo), cudaMemcpyDeviceToHost,
                               m.copy_stream));
    RB200_CUDA(cudaEventRecord(m.ev_copied[buf], m.copy_stream));
  }
  RB200_CUDA(cudaStreamSynchronize(m.copy_stream));
  RB200_CUDA(cudaStreamSynchronize(st));
  return 0;
}

}  // namespace rb200

using namespace rb200;

extern "C" {

int rgbdslam_b200_node_download_cloud(uint64_t node_handle, int point_bytes, void* out, int* w, int* h) {
  RB200_ENTER_INITED();
  NodeDev* nd = get_node(node_handle);
  if (!nd) return RGBDSLAM_B200_ERR_ARG;
  if ((point_bytes != 16 && point_bytes != 32) || !w || !h) {
    set_error("node_download_cloud: point_bytes must be 16 or 32, w and h non-null");
    return RGBDSLAM_B200_ERR_ARG;
  }
  if (!nd->pc.rgb) {
    set_error("node_download_cloud: the node has no stored cloud (nodes_create_ex with RGBDSLAM_B200_STORE_CLOUD)");
    return RGBDSLAM_B200_ERR_STATE;
  }
  *w = nd->pc.w;
  *h = nd->pc.h;
  if (!out) return 0;
  const MapArgs a{0.f, 0, 1, 0, point_bytes};  // every point, as stored
  int64_t n = 0;
  return map_emit(std::vector<MapNode>(1, map_node(nd, nullptr)), a, out, (int64_t)nd->pc.w * nd->pc.h, &n);
}

int rgbdslam_b200_render_cloud(int n, const uint64_t* nodes, const double* transforms12, double maximum_depth, int preserve_raster,
                               int point_bytes, void* out, int64_t capacity, int64_t* n_out, float* used16) {
  RB200_ENTER_INITED();
  if (n < 0 || (n > 0 && (!nodes || !transforms12)) || !n_out || (out && capacity < 0)) {
    set_error("render_cloud: bad arguments");
    return RGBDSLAM_B200_ERR_ARG;
  }
  if (point_bytes != 16 && point_bytes != 32) {
    set_error("render_cloud: point_bytes must be 16 (PointXYZ) or 32 (PointXYZRGB)");
    return RGBDSLAM_B200_ERR_ARG;
  }
  for (size_t i = 0; i < (size_t)n * 12; i++)
    if (!std::isfinite(transforms12[i])) {
      set_error("render_cloud: transform " + std::to_string(i / 12) + " has a non-finite entry");
      return RGBDSLAM_B200_ERR_ARG;
    }
  std::vector<MapNode> table(n);
  for (int k = 0; k < n; k++) {
    NodeDev* nd = get_node(nodes[k]);
    if (!nd) return RGBDSLAM_B200_ERR_ARG;
    if (!nd->pc.rgb) {
      set_error("render_cloud: node " + std::to_string(k) + " has no stored cloud (nodes_create_ex with RGBDSLAM_B200_STORE_CLOUD)");
      return RGBDSLAM_B200_ERR_STATE;
    }
    float T[12];  // pcl_ros::transformAsMatrix: every double entry of the tf::Transform cast to float
    for (int j = 0; j < 12; j++) T[j] = (float)transforms12[(size_t)k * 12 + j];
    table[k] = map_node(nd, T);
    if (used16) {  // Eigen::Matrix4f, column-major
      float* M = used16 + (size_t)k * 16;
      for (int r = 0; r < 3; r++)
        for (int c = 0; c < 4; c++) M[4 * c + r] = T[4 * r + c];
      M[3] = M[7] = M[11] = 0.f;
      M[15] = 1.f;
    }
  }
  // transformAndAppendPointCloud takes max_Depth as a float and filters when it is >= 0 (misc.cpp:206-208)
  const float maxd = (float)maximum_depth;
  const MapArgs a{maxd * maxd, maxd >= 0.f ? 1 : 0, preserve_raster ? 1 : 0, 1, point_bytes};
  return map_emit(table, a, out, capacity, n_out);
}

}  // extern "C"
