// api_map.cu -- C ABI of the stored colour clouds and the registered map, host orchestration:
//   rgbdslam_b200_node_download_cloud  == Node::pc_col (node.cpp:126-131, 261) as an organised cloud
//   rgbdslam_b200_render_cloud         == transformAndAppendPointCloud (misc.cpp:183-238) of many nodes, the loop of
//                                         GraphManager::saveAllCloudsToFile (graph_mgr_io.cpp:502-583)
//   rgbdslam_b200_reduce_clouds        == Node::reducePointCloud (node.cpp:1448-1460) of many nodes (voxel.cu)
//   rgbdslam_b200_transform_clouds     == pcl::transformPointCloud(*pc_col, *pc_col, m) of many nodes, the
//                                         transform_individual_clouds step of saveIndividualCloudsToFile (graph_mgr_io.cpp:372-374)
//   rgbdslam_b200_icp_align(_ex)       == icpAlignment(filterCloud(..), filterCloud(..)) (icp.cpp:20-89) of many pairs (icp.cu,
//                                         icp_nl.cu)
// The first two run count -> scan -> scatter (map.cu) and move the records to the host through a two-piece device staging
// ring: the copy of piece k runs on its own stream while piece k + 1 is computed.
#include <algorithm>
#include <cmath>
#include <cstdlib>
#include <cstring>
#include <unordered_map>
#include <vector>

#include "../../include/rgbdslam_b200/cloud_transform.h"
#include "../../include/rgbdslam_b200/icp.h"
#include "../../include/rgbdslam_b200/map.h"
#include "../../include/rgbdslam_b200/voxel.h"
#include "kernels.h"
#include "state.h"

namespace rb200 {

constexpr long long kMapPiecePoints = 1 << 21;  // records per staging piece (64 MB of 32-byte records)

struct MapCtx {
  cudaStream_t copy_stream = nullptr;
  cudaEvent_t ev_done[2] = {nullptr, nullptr}, ev_copied[2] = {nullptr, nullptr};
  DevBuf nodes, blocks, counts, offs, stage[2];
  DevBuf first;  // transform_clouds: each node's first point in its chunk's slab
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
MapNode map_node(const NodeDev* nd, const float* T) {
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
  m.point0_one = c.point0_one ? 1 : 0;
  m.fxinv = (float)(1.0 / (double)c.K[0]);  // getCameraIntrinsicsInverseFocalLength (misc.cpp:64-69); unused by organised clouds
  m.fyinv = (float)(1.0 / (double)c.K[1]);
  m.cx = c.K[2];
  m.cy = c.K[3];
  if (T) memcpy(m.m, T, sizeof(m.m));
  return m;
}

int stored_cloud_nodes(const char* call, int n, const uint64_t* handles, bool distinct, std::vector<NodeDev*>* nds) {
  nds->resize(n);
  for (int k = 0; k < n; k++) {
    if (!((*nds)[k] = get_node(handles[k]))) return RGBDSLAM_B200_ERR_ARG;
    if (!(*nds)[k]->pc.rgb) {
      set_error(std::string(call) + ": node " + std::to_string(k) +
                " has no stored cloud (nodes_create_ex with RGBDSLAM_B200_STORE_CLOUD)");
      return RGBDSLAM_B200_ERR_STATE;
    }
  }
  if (!distinct) return 0;
  std::vector<uint64_t> sorted(handles, handles + n);
  std::sort(sorted.begin(), sorted.end());
  if (std::adjacent_find(sorted.begin(), sorted.end()) != sorted.end()) {
    set_error(std::string(call) + ": a node is listed twice");
    return RGBDSLAM_B200_ERR_ARG;
  }
  return 0;
}

std::vector<int2> map_blocks(const std::vector<MapNode>& nodes, std::vector<int>* first) {
  std::vector<int2> blocks;
  if (first) first->resize(nodes.size() + 1);
  for (size_t k = 0; k < nodes.size(); k++) {
    if (first) (*first)[k] = (int)blocks.size();
    const int P = nodes[k].cw * nodes[k].ch;
    for (int f = 0; f < P; f += kMapBlockPoints) blocks.push_back(make_int2((int)k, f));
  }
  if (first) first->back() = (int)blocks.size();
  return blocks;
}

long long chunk_limit(long long limit, const char* env_name) {
  const char* env = std::getenv(env_name);
  return env ? std::max(1ll, std::atoll(env)) : limit;
}

// Each node takes its new cloud and lets go of its old allocation; slabs no node took are freed.
static void adopt_clouds(const std::vector<CloudResult>& results, const std::vector<NodeSlab*>& slabs) {
  for (const CloudResult& r : results) {
    release_slab(r.nd->pc.slab);
    r.nd->pc = r.pc;
    r.pc.slab->refs++;
  }
  for (NodeSlab* sl : slabs)
    if (sl->refs == 0) {  // a chunk whose nodes all kept their clouds
      cudaFree(sl->base);
      delete sl;
    }
}

// After a failure: frees the call's new slabs (after the stream has drained).
static void drop_slabs(const std::vector<NodeSlab*>& slabs) {
  cudaStreamSynchronize(g_state.stream);
  for (NodeSlab* sl : slabs) {
    cudaFree(sl->base);
    delete sl;
  }
}

int rebuild_clouds(const std::vector<NodeDev*>& nds, long long limit, const CloudChunk& chunk) {
  const int n = (int)nds.size();
  std::vector<CloudResult> results;
  std::vector<NodeSlab*> slabs;
  int rc = 0;
  for (int k0 = 0; k0 < n && rc == 0;) {  // chunks of whole nodes, at least one
    int k1 = k0;
    long long points = 0;
    do points += (long long)nds[k1]->pc.w * nds[k1]->pc.h;
    while (++k1 < n && points + (long long)nds[k1]->pc.w * nds[k1]->pc.h <= limit);
    rc = chunk(k0, k1, points, results, slabs);
    k0 = k1;
  }
  if (rc) {  // no node is changed
    drop_slabs(slabs);
    return rc;
  }
  adopt_clouds(results, slabs);
  return 0;
}

NodeSlab* new_slab(long long points, const char* what, std::vector<NodeSlab*>& slabs) {
  NodeSlab* slab = new NodeSlab();
  cudaError_t e = cudaMalloc(&slab->base, 16 * (size_t)std::max(points, 1ll));
  if (e != cudaSuccess) {
    delete slab;
    cuda_fail(e, what);
    return nullptr;
  }
  slabs.push_back(slab);
  return slab;
}

NodeCloud slab_cloud(const NodeCloud& c, NodeSlab* slab, long long first, long long count) {
  NodeCloud r = c;
  r.x = (float*)slab->base + 4 * first;
  r.y = r.x + count;
  r.z = r.y + count;
  r.rgb = (uint32_t*)(r.z + count);
  r.step = 0;
  r.slab = slab;
  return r;
}

// Count, scan and (unless out is NULL) scatter the records of `nodes` into the host buffer out (capacity records).
static int map_emit(const std::vector<MapNode>& nodes, const MapArgs& a, void* out, int64_t capacity, int64_t* n_out) {
  MapCtx& m = g_map;
  State& s = g_state;
  cudaStream_t st = s.stream;
  int rc;
  if ((rc = map_ensure_streams())) return rc;
  const std::vector<int2> blocks = map_blocks(nodes, nullptr);
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

// ---- the voxel filter ------------------------------------------------------------------------------------------------------

constexpr long long kVoxChunkPoints = 1 << 23;  // points of the nodes reduced together: 24 bytes of work buffers per point

struct VoxCtx {
  DevBuf segs, bounds, grid, key[2], idx[2], hist, heads;
  void release() {
    DevBuf* all[] = {&segs, &bounds, &grid, &key[0], &key[1], &idx[0], &idx[1], &hist, &heads};
    for (DevBuf* b : all) b->release();
  }
};

// Reduces nodes [k0, k1) of the call, whose clouds hold `points` points in all, into one new slab.  Appends a CloudResult per
// reduced node and writes n_points[k] (-1: the leaf size is too small for node k, which keeps its cloud).
static int vox_chunk(VoxCtx& v, const std::vector<NodeDev*>& nds, int k0, int k1, long long points, float inv_leaf,
                     std::vector<CloudResult>& results, std::vector<NodeSlab*>& slabs, int32_t* n_points) {
  MapCtx& m = g_map;
  State& s = g_state;
  cudaStream_t st = s.stream;
  const int nn = k1 - k0;
  std::vector<MapNode> nodes(nn);
  for (int k = 0; k < nn; k++) nodes[k] = map_node(nds[k0 + k], nullptr);
  std::vector<int> first_block;
  const std::vector<int2> blocks = map_blocks(nodes, &first_block);
  std::vector<VoxSeg> segs(nn);
  for (int k = 0, pt = 0; k < nn; k++) {
    const int P = nodes[k].cw * nodes[k].ch;
    segs[k] = VoxSeg{pt, P, first_block[k], first_block[k + 1] - first_block[k]};
    pt += P;
  }
  const int nb = (int)blocks.size();
  const size_t np = (size_t)std::max<long long>(points, 1);
  int rc;
  if ((rc = m.nodes.ensure(sizeof(MapNode) * nn)) || (rc = m.blocks.ensure(sizeof(int2) * std::max(nb, 1))) ||
      (rc = m.counts.ensure(4 * (size_t)std::max(nb, 1))) || (rc = m.offs.ensure(8 * (size_t)(nb + 1))) ||
      (rc = v.segs.ensure(sizeof(VoxSeg) * nn)) || (rc = v.bounds.ensure(24 * (size_t)nn)) ||
      (rc = v.grid.ensure(sizeof(VoxGrid) * nn)) || (rc = v.hist.ensure(1024 * (size_t)std::max(nb, 1))) ||
      (rc = v.heads.ensure(sizeof(int2) * np)))
    return rc;
  for (int b = 0; b < 2; b++)
    if ((rc = v.key[b].ensure(4 * np)) || (rc = v.idx[b].ensure(4 * np))) return rc;
  VoxBufs b;
  b.nodes = (const MapNode*)m.nodes.ptr;
  b.blocks = (const int2*)m.blocks.ptr;
  b.segs = (const VoxSeg*)v.segs.ptr;
  b.bmin = (uint32_t*)v.bounds.ptr;
  b.bmax = b.bmin + 3 * (size_t)nn;
  b.grid = (VoxGrid*)v.grid.ptr;
  for (int i = 0; i < 2; i++) {
    b.key[i] = (uint32_t*)v.key[i].ptr;
    b.idx[i] = (uint32_t*)v.idx[i].ptr;
  }
  b.hist = (int*)v.hist.ptr;
  b.counts = (int*)m.counts.ptr;
  b.offs = (long long*)m.offs.ptr;
  b.heads = (int2*)v.heads.ptr;
  RB200_CUDA(cudaMemcpyAsync(m.nodes.ptr, nodes.data(), sizeof(MapNode) * nn, cudaMemcpyHostToDevice, st));
  RB200_CUDA(cudaMemcpyAsync(v.segs.ptr, segs.data(), sizeof(VoxSeg) * nn, cudaMemcpyHostToDevice, st));
  if (nb > 0) RB200_CUDA(cudaMemcpyAsync(m.blocks.ptr, blocks.data(), sizeof(int2) * nb, cudaMemcpyHostToDevice, st));
  int launches = 0;
  RB200_CUDA(launch_vox_keys(b, nn, nb, inv_leaf, st, &launches));
  // the grids decide how many radix passes the chunk needs: enough bytes to hold its largest cell count, so that every voxel
  // index sorts below the key of the points that take no part
  std::vector<VoxGrid> grid(nn);
  RB200_CUDA(cudaMemcpyAsync(grid.data(), v.grid.ptr, sizeof(VoxGrid) * nn, cudaMemcpyDeviceToHost, st));
  RB200_CUDA(cudaStreamSynchronize(st));
  s.launches += launches;
  int passes = 1;
  for (const VoxGrid& g : grid)
    while (passes < 4 && ((long long)g.cells >> (8 * passes)) != 0) passes++;
  launches = 0;
  RB200_CUDA(launch_vox_sort(b, nn, nb, passes, st, &launches));
  std::vector<long long> offs(nb + 1);
  RB200_CUDA(cudaMemcpyAsync(offs.data(), b.offs, 8 * (size_t)(nb + 1), cudaMemcpyDeviceToHost, st));
  RB200_CUDA(cudaStreamSynchronize(st));
  s.launches += launches;
  const long long nvox = offs[nb];
  NodeSlab* slab = new_slab(nvox, "cudaMalloc(reduced clouds)", slabs);
  if (!slab) return RGBDSLAM_B200_ERR_CUDA;
  RB200_CUDA(launch_vox_centroids(b, passes, nvox, (float*)slab->base, st));
  RB200_CUDA(cudaStreamSynchronize(st));  // the work buffers are the next chunk's
  s.launches += nvox > 0;
  for (int k = 0; k < nn; k++) {
    if (grid[k].too_small) {
      n_points[k0 + k] = -1;
      continue;
    }
    const long long first = offs[first_block[k]], count = offs[first_block[k + 1]] - first;
    CloudResult r{nds[k0 + k], slab_cloud(nds[k0 + k]->pc, slab, first, count)};
    r.pc.w = (int32_t)count;
    r.pc.h = 1;
    r.pc.unorganised = true;
    r.pc.point0_one = false;
    results.push_back(r);
    n_points[k0 + k] = (int32_t)count;
  }
  return 0;
}

// ---- transform_individual_clouds -------------------------------------------------------------------------------------------

constexpr long long kXfChunkPoints = 1 << 24;  // points of the nodes transformed together: one slab of 16 bytes per point

// Transforms nodes [k0, k1) of the call, whose clouds hold `points` points in all, into one new slab and appends a CloudResult
// per node.  The new planes keep the raster; a depth-image node's x / y are stored from now on.
static int xf_chunk(const std::vector<NodeDev*>& nds, const double* transforms12, int k0, int k1, long long points,
                    std::vector<CloudResult>& results, std::vector<NodeSlab*>& slabs) {
  MapCtx& m = g_map;
  State& s = g_state;
  cudaStream_t st = s.stream;
  const int nn = k1 - k0;
  std::vector<MapNode> nodes(nn);
  std::vector<long long> first(nn);
  long long pt = 0;
  for (int k = 0; k < nn; k++) {
    float T[12];  // Eigen's Matrix4d::cast<float>(): every double entry rounded to float
    for (int j = 0; j < 12; j++) T[j] = (float)transforms12[(size_t)(k0 + k) * 12 + j];
    nodes[k] = map_node(nds[k0 + k], T);
    first[k] = pt;
    pt += nodes[k].cw * nodes[k].ch;
  }
  const std::vector<int2> blocks = map_blocks(nodes, nullptr);
  const int nb = (int)blocks.size();
  int rc;
  if ((rc = m.nodes.ensure(sizeof(MapNode) * nn)) || (rc = m.blocks.ensure(sizeof(int2) * std::max(nb, 1))) ||
      (rc = m.first.ensure(sizeof(long long) * nn)))
    return rc;
  NodeSlab* slab = new_slab(points, "cudaMalloc(transformed clouds)", slabs);
  if (!slab) return RGBDSLAM_B200_ERR_CUDA;
  RB200_CUDA(cudaMemcpyAsync(m.nodes.ptr, nodes.data(), sizeof(MapNode) * nn, cudaMemcpyHostToDevice, st));
  RB200_CUDA(cudaMemcpyAsync(m.first.ptr, first.data(), sizeof(long long) * nn, cudaMemcpyHostToDevice, st));
  if (nb > 0) RB200_CUDA(cudaMemcpyAsync(m.blocks.ptr, blocks.data(), sizeof(int2) * nb, cudaMemcpyHostToDevice, st));
  RB200_CUDA(launch_transform_clouds((const MapNode*)m.nodes.ptr, (const int2*)m.blocks.ptr, nb, (const long long*)m.first.ptr,
                                     (float*)slab->base, st));
  RB200_CUDA(cudaStreamSynchronize(st));  // the work buffers are the next chunk's
  s.launches += nb > 0;
  for (int k = 0; k < nn; k++) {
    NodeDev* nd = nds[k0 + k];
    CloudResult r{nd, slab_cloud(nd->pc, slab, first[k], (long long)nodes[k].cw * nodes[k].ch)};
    r.pc.point0_one = nd->pc.step > 0 || nd->pc.point0_one;
    r.pc.transformed = true;
    results.push_back(r);
  }
  return 0;
}

// ---- the ICP fallback of matchNodePair -------------------------------------------------------------------------------------

constexpr long long kIcpChunkPoints = 1 << 24;  // raster points of the nodes one filter launch treats: 4 bytes of scratch each

struct IcpCtx {
  DevBuf nodes, pairs, targets, scratch, pts, nf, nfin, key[2], idx[2], work, corr, dist, results;
};
static IcpCtx g_icp;

// Room for the points filterCloud keeps of a cloud of P points: at most desired + 1 with an exact step, and the float sum
// i += step may run behind by up to about desired^2 * 2^-24 steps.
static int icp_capacity(int P, int desired) {
  const long long d = desired;
  return (int)std::min<long long>(P, d + 2 + d * (d + 4) / (1ll << 23));
}

static int icp_run(const std::vector<NodeDev*>& nds, std::vector<IcpPair>& pairs, int desired, int method,
                   rgbdslam_b200_icp_result* out) {
  IcpCtx& c = g_icp;
  State& s = g_state;
  cudaStream_t st = s.stream;
  const int U = (int)nds.size(), n = (int)pairs.size();
  std::vector<IcpNode> nodes(U);
  std::vector<int> first_of_chunk;  // the node each filter launch starts at
  long long f = 0, scratch = 0, chunk = 0, max_chunk = 1;
  for (int u = 0; u < U; u++) {
    IcpNode& x = nodes[u];
    x.src = map_node(nds[u], nullptr);
    if (!x.src.rgb) x.src.rgb = reinterpret_cast<const uint32_t*>(x.src.z);  // map_point reads a colour word ICP never uses
    x.P = x.src.cw * x.src.ch;
    x.cap = icp_capacity(x.P, desired);
    x.f0 = f;
    f += x.cap;
    if (u == 0 || chunk + x.P > kIcpChunkPoints) {
      first_of_chunk.push_back(u);
      chunk = 0;
    }
    x.scratch0 = chunk;
    chunk += x.P;
    max_chunk = std::max(max_chunk, chunk);
  }
  first_of_chunk.push_back(U);
  scratch = max_chunk;
  const long long plane = std::max(f, 1ll);
  std::vector<char> is_target(U, 0);
  std::vector<int> targets;
  long long w = 0;
  for (IcpPair& p : pairs) {
    if (!is_target[p.t]) targets.push_back(p.t);
    is_target[p.t] = 1;
    p.w0 = w;
    w += nodes[p.s].cap;
  }
  const long long wplane = std::max(w, 1ll);
  int rc;
  if ((rc = c.nodes.ensure(sizeof(IcpNode) * U)) || (rc = c.pairs.ensure(sizeof(IcpPair) * n)) ||
      (rc = c.targets.ensure(sizeof(int) * targets.size())) || (rc = c.scratch.ensure(sizeof(int) * scratch)) ||
      (rc = c.pts.ensure(3 * sizeof(float) * plane)) || (rc = c.nf.ensure(sizeof(int) * U)) || (rc = c.nfin.ensure(sizeof(int) * U)) ||
      (rc = c.work.ensure(icp_work_planes(method) * sizeof(float) * wplane)) || (rc = c.corr.ensure(sizeof(int) * wplane)) ||
      (rc = c.dist.ensure(sizeof(float) * wplane)) || (rc = c.results.ensure(sizeof(rgbdslam_b200_icp_result) * n)))
    return rc;
  for (int b = 0; b < 2; b++)
    if ((rc = c.key[b].ensure(sizeof(unsigned long long) * plane)) || (rc = c.idx[b].ensure(sizeof(int) * plane))) return rc;
  RB200_CUDA(cudaMemcpyAsync(c.nodes.ptr, nodes.data(), sizeof(IcpNode) * U, cudaMemcpyHostToDevice, st));
  RB200_CUDA(cudaMemcpyAsync(c.pairs.ptr, pairs.data(), sizeof(IcpPair) * n, cudaMemcpyHostToDevice, st));
  RB200_CUDA(cudaMemcpyAsync(c.targets.ptr, targets.data(), sizeof(int) * targets.size(), cudaMemcpyHostToDevice, st));
  const IcpNode* d_nodes = (const IcpNode*)c.nodes.ptr;
  float* pts = (float*)c.pts.ptr;
  int* nf = (int*)c.nf.ptr;
  int launches = 0;
  for (size_t k = 0; k + 1 < first_of_chunk.size(); k++) {
    const int u0 = first_of_chunk[k], u1 = first_of_chunk[k + 1];
    RB200_CUDA(launch_icp_filter(d_nodes + u0, u1 - u0, desired, (int*)c.scratch.ptr, pts, plane, nf + u0, st));
    launches++;
  }
  unsigned long long* key[2] = {(unsigned long long*)c.key[0].ptr, (unsigned long long*)c.key[1].ptr};
  int* idx[2] = {(int*)c.idx[0].ptr, (int*)c.idx[1].ptr};
  RB200_CUDA(launch_icp_cells(d_nodes, (const int*)c.targets.ptr, (int)targets.size(), pts, plane, nf, key, idx, (int*)c.nfin.ptr, st));
  RB200_CUDA(launch_icp_align(method, (const IcpPair*)c.pairs.ptr, n, d_nodes, pts, plane, nf, key[0], idx[0], (const int*)c.nfin.ptr,
                              (float*)c.work.ptr, wplane, (int*)c.corr.ptr, (float*)c.dist.ptr, (rgbdslam_b200_icp_result*)c.results.ptr, st));
  launches += 2;
  std::vector<int> kept(U);
  RB200_CUDA(cudaMemcpyAsync(kept.data(), nf, sizeof(int) * U, cudaMemcpyDeviceToHost, st));
  RB200_CUDA(cudaMemcpyAsync(out, c.results.ptr, sizeof(rgbdslam_b200_icp_result) * n, cudaMemcpyDeviceToHost, st));
  RB200_CUDA(cudaStreamSynchronize(st));
  s.launches += launches;
  for (int u = 0; u < U; u++)
    if (kept[u] > nodes[u].cap) {
      set_error("icp_align: filterCloud kept " + std::to_string(kept[u]) + " points, more than the " + std::to_string(nodes[u].cap) +
                " allowed for");
      return RGBDSLAM_B200_ERR_CUDA;
    }
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
  std::vector<NodeDev*> nds;
  int rc;
  if ((rc = check_finite("render_cloud", "transform", n, 12, transforms12)) ||
      (rc = stored_cloud_nodes("render_cloud", n, nodes, false, &nds)))
    return rc;
  std::vector<MapNode> table(n);
  for (int k = 0; k < n; k++) {
    float T[12];  // pcl_ros::transformAsMatrix: every double entry of the tf::Transform cast to float
    for (int j = 0; j < 12; j++) T[j] = (float)transforms12[(size_t)k * 12 + j];
    table[k] = map_node(nds[k], T);
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

int rgbdslam_b200_reduce_clouds(int n, const uint64_t* nodes, double voxelfilter_size, int32_t* n_points) {
  RB200_ENTER_INITED();
  const float leaf = (float)voxelfilter_size;
  if (n < 0 || (n > 0 && !nodes) || !std::isfinite(voxelfilter_size) || !(leaf > 0.f) || !std::isfinite(leaf)) {
    set_error("reduce_clouds: n >= 0, nodes non-null and a finite voxelfilter_size > 0 (as a float) are needed");
    return RGBDSLAM_B200_ERR_ARG;
  }
  std::vector<NodeDev*> nds;
  int rc;
  if ((rc = stored_cloud_nodes("reduce_clouds", n, nodes, true, &nds))) return rc;
  const float inv_leaf = 1.0f / leaf;
  std::vector<int32_t> counts(n);
  VoxCtx v;
  rc = rebuild_clouds(nds, chunk_limit(kVoxChunkPoints, "RB200_VOX_CHUNK_POINTS"),
                      [&](int k0, int k1, long long points, auto& results, auto& slabs) {
                        return vox_chunk(v, nds, k0, k1, points, inv_leaf, results, slabs, counts.data());
                      });
  v.release();
  if (rc) return rc;
  if (n_points) std::copy(counts.begin(), counts.end(), n_points);
  return 0;
}

int rgbdslam_b200_transform_clouds(int n, const uint64_t* nodes, const double* transforms12) {
  RB200_ENTER_INITED();
  if (n < 0 || (n > 0 && (!nodes || !transforms12))) {
    set_error("transform_clouds: n >= 0 and non-null nodes and transforms are needed");
    return RGBDSLAM_B200_ERR_ARG;
  }
  std::vector<NodeDev*> nds;
  int rc;
  if ((rc = check_finite("transform_clouds", "transform", n, 12, transforms12)) ||
      (rc = stored_cloud_nodes("transform_clouds", n, nodes, true, &nds)))
    return rc;
  return rebuild_clouds(nds, kXfChunkPoints, [&](int k0, int k1, long long points, auto& results, auto& slabs) {
    return xf_chunk(nds, transforms12, k0, k1, points, results, slabs);
  });
}

int rgbdslam_b200_icp_align(int n, const uint64_t* source, const uint64_t* target, int max_cloud_size,
                            rgbdslam_b200_icp_result* out) {
  return rgbdslam_b200_icp_align_ex(n, source, target, max_cloud_size, RGBDSLAM_B200_ICP_METHOD_ICP, out);
}

int rgbdslam_b200_icp_align_ex(int n, const uint64_t* source, const uint64_t* target, int max_cloud_size, int method,
                               rgbdslam_b200_icp_result* out) {
  RB200_ENTER_INITED();
  if (n < 0 || max_cloud_size < 1 || (n > 0 && (!source || !target || !out))) {
    set_error("icp_align: n >= 0, max_cloud_size >= 1 and non-null source, target and out are needed");
    return RGBDSLAM_B200_ERR_ARG;
  }
  if (method != RGBDSLAM_B200_ICP_METHOD_ICP && method != RGBDSLAM_B200_ICP_METHOD_ICP_NL) {
    set_error("icp_align: method must be RGBDSLAM_B200_ICP_METHOD_ICP or RGBDSLAM_B200_ICP_METHOD_ICP_NL");
    return RGBDSLAM_B200_ERR_ARG;
  }
  std::vector<NodeDev*> nds;  // the distinct nodes of the call, in order of first appearance
  std::unordered_map<uint64_t, int> slot;
  std::vector<IcpPair> pairs(n);
  for (int k = 0; k < 2 * n; k++) {
    const uint64_t h = (k & 1 ? target : source)[k >> 1];
    auto it = slot.find(h);
    int u;
    if (it != slot.end()) {
      u = it->second;
    } else {
      NodeDev* nd = get_node(h);
      if (!nd) return RGBDSLAM_B200_ERR_ARG;
      u = (int)nds.size();
      slot.emplace(h, u);
      nds.push_back(nd);
    }
    (k & 1 ? pairs[k >> 1].t : pairs[k >> 1].s) = u;
  }
  for (size_t u = 0; u < nds.size(); u++)
    if (!nds[u]->pc.z) {
      set_error("icp_align: a node has no stored cloud (nodes_create_ex with RGBDSLAM_B200_STORE_CLOUD or KEEP_CLOUD)");
      return RGBDSLAM_B200_ERR_STATE;
    } else if (nds[u]->pc.transformed) {
      set_error("icp_align: a cloud moved into the map frame (rgbdslam_b200_transform_clouds) holds no camera points");
      return RGBDSLAM_B200_ERR_STATE;
    }
  if (n == 0) return 0;
  return icp_run(nds, pairs, max_cloud_size, method, out);
}

}  // extern "C"
