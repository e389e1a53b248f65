// voxel.cu -- the voxel filter of the nodes' stored clouds, Node::reducePointCloud (node.cpp:1448-1460): pcl::VoxelGrid with a
// cubic leaf replaces pc_col by one centroid (position and colour) per occupied voxel, in ascending voxel index.  For a chunk
// of whole nodes whose points lie back to back:
//   k_vox_bounds     getMinMax3D: per-axis float minimum / maximum of each node's finite points
//   k_vox_grid       per node min_b, the index multipliers, the cell count, and PCL's "leaf size is too small" decision
//   k_vox_keys       per point its voxel index (0xffffffff when a coordinate is not finite) and its raster index
//   k_vox_hist / k_vox_offsets / k_vox_scatter
//                    one pass of a stable 8-bit LSD radix sort inside every node's segment.  Stability makes "sorted by voxel
//                    index" mean "raster order inside a voxel", which fixes the order of the centroid sums.
//   k_vox_heads      the first point of every voxel's run, counted per block; after the map's scan, listed per voxel
//   k_vox_centroids  one thread per voxel walks its run in order and writes the centroid
// Points are read through map_point (map.cuh), the one reader of a stored cloud.  Every float operation is an explicit _rn
// intrinsic: PCL on x86-64 without -mfma does not contract.
#include "kernels.h"
#include "map.cuh"

namespace rb200 {

constexpr int kVoxThreads = 256;
constexpr int kVoxRounds = kMapBlockPoints / kVoxThreads;
constexpr uint32_t kVoxNoKey = 0xffffffffu;

// The points as stored: no depth filter, no transform, every raster position.
__device__ __forceinline__ MapArgs vox_args() { return MapArgs{0.f, 0, 1, 0, 32}; }

__device__ __forceinline__ bool vox_finite(const MapOut& o) { return isfinite(o.x) && isfinite(o.y) && isfinite(o.z); }

// Order-preserving image of a float in the unsigned integers (for atomicMin / atomicMax), and back.
__device__ __forceinline__ uint32_t vox_ordered(float f) {
  const uint32_t b = __float_as_uint(f);
  return b ^ ((b >> 31) ? 0xffffffffu : 0x80000000u);
}
__device__ __forceinline__ float vox_unordered(uint32_t k) { return __uint_as_float(k ^ ((k >> 31) ? 0x80000000u : 0xffffffffu)); }

// bmin starts as 0xffffffff and bmax as 0 (no finite float has either image); a node without a finite point keeps them.
__global__ void __launch_bounds__(kVoxThreads) k_vox_bounds(const MapNode* __restrict__ nodes, const int2* __restrict__ blocks,
                                                            uint32_t* __restrict__ bmin, uint32_t* __restrict__ bmax) {
  __shared__ float red[6][kVoxThreads / 32];
  const int2 blk = blocks[blockIdx.x];
  const MapNode& nd = nodes[blk.x];
  const int P = nd.cw * nd.ch;
  const MapArgs a = vox_args();
  float v[6] = {INFINITY, INFINITY, INFINITY, -INFINITY, -INFINITY, -INFINITY};
#pragma unroll
  for (int k = 0; k < kVoxRounds; k++) {
    const int i = blk.y + k * kVoxThreads + threadIdx.x;
    MapOut o;
    if (i >= P) continue;
    map_point(nd, i, a, o);
    if (!vox_finite(o)) continue;
    v[0] = fminf(v[0], o.x), v[1] = fminf(v[1], o.y), v[2] = fminf(v[2], o.z);
    v[3] = fmaxf(v[3], o.x), v[4] = fmaxf(v[4], o.y), v[5] = fmaxf(v[5], o.z);
  }
#pragma unroll
  for (int c = 0; c < 6; c++) {
#pragma unroll
    for (int s = 16; s > 0; s >>= 1) {
      const float t = __shfl_xor_sync(0xffffffffu, v[c], s);
      v[c] = c < 3 ? fminf(v[c], t) : fmaxf(v[c], t);
    }
    if ((threadIdx.x & 31) == 0) red[c][threadIdx.x >> 5] = v[c];
  }
  __syncthreads();
  if (threadIdx.x < 6) {
    const int c = threadIdx.x;
    float r = red[c][0];
    for (int w = 1; w < kVoxThreads / 32; w++) r = c < 3 ? fminf(r, red[c][w]) : fmaxf(r, red[c][w]);
    if (c < 3 && r != INFINITY) atomicMin(&bmin[3 * blk.x + c], vox_ordered(r));
    if (c >= 3 && r != -INFINITY) atomicMax(&bmax[3 * blk.x + c - 3], vox_ordered(r));
  }
}

// pcl::VoxelGrid::applyFilter up to the index loop (PCL 1.7 voxel_grid.hpp): the int64 guard on (max_p - min_p) * inv, then
// min_b / max_b / div_b / divb_mul.  The cloud is also left alone when div_b.x * div_b.y * div_b.z itself passes INT32_MAX,
// which the guard can miss by one cell per axis: PCL's int index would overflow there.
__global__ void k_vox_grid(int nnodes, const uint32_t* __restrict__ bmin, const uint32_t* __restrict__ bmax, float inv,
                           VoxGrid* __restrict__ grid) {
  const int k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= nnodes) return;
  VoxGrid g;
  g.min_b[0] = g.min_b[1] = g.min_b[2] = 0;
  g.mul[0] = g.mul[1] = g.mul[2] = 0;
  g.cells = 0;
  g.too_small = 0;
  if (bmax[3 * k] != 0u) {
    long long guard = 1, cells = 1;
    int div[3];
#pragma unroll
    for (int c = 0; c < 3; c++) {
      const float mn = vox_unordered(bmin[3 * k + c]), mx = vox_unordered(bmax[3 * k + c]);
      const long long d = (long long)__fmul_rn(__fsub_rn(mx, mn), inv) + 1;
      g.min_b[c] = (int)floorf(__fmul_rn(mn, inv));
      const long long db = (long long)(int)floorf(__fmul_rn(mx, inv)) - g.min_b[c] + 1;
      // both products only grow (every factor is >= 1), so a running test against INT32_MAX equals the test of the full product
      guard = guard > INT32_MAX || d > INT32_MAX ? (long long)INT32_MAX + 1 : guard * d;
      cells = cells > INT32_MAX || db > INT32_MAX ? (long long)INT32_MAX + 1 : cells * db;
      div[c] = (int)db;
    }
    if (guard > INT32_MAX || cells > INT32_MAX) {
      g.too_small = 1;
    } else {
      g.mul[0] = 1;
      g.mul[1] = div[0];
      g.mul[2] = div[0] * div[1];
      g.cells = (int)cells;
    }
  }
  grid[k] = g;
}

__global__ void __launch_bounds__(kVoxThreads) k_vox_keys(const MapNode* __restrict__ nodes, const int2* __restrict__ blocks,
                                                          const VoxSeg* __restrict__ segs, const VoxGrid* __restrict__ grid, float inv,
                                                          uint32_t* __restrict__ key, uint32_t* __restrict__ idx) {
  const int2 blk = blocks[blockIdx.x];
  const MapNode& nd = nodes[blk.x];
  const VoxGrid g = grid[blk.x];
  const int P = nd.cw * nd.ch, pt0 = segs[blk.x].pt0;
  const MapArgs a = vox_args();
#pragma unroll
  for (int k = 0; k < kVoxRounds; k++) {
    const int i = blk.y + k * kVoxThreads + threadIdx.x;
    if (i >= P) continue;
    MapOut o;
    map_point(nd, i, a, o);
    uint32_t kk = kVoxNoKey;
    if (g.cells > 0 && vox_finite(o)) {
      const int ix = (int)__fsub_rn(floorf(__fmul_rn(o.x, inv)), (float)g.min_b[0]);
      const int iy = (int)__fsub_rn(floorf(__fmul_rn(o.y, inv)), (float)g.min_b[1]);
      const int iz = (int)__fsub_rn(floorf(__fmul_rn(o.z, inv)), (float)g.min_b[2]);
      kk = (uint32_t)ix * (uint32_t)g.mul[0] + (uint32_t)iy * (uint32_t)g.mul[1] + (uint32_t)iz * (uint32_t)g.mul[2];
    }
    key[pt0 + i] = kk;
    idx[pt0 + i] = (uint32_t)i;
  }
}

// ---- one radix pass: digit = (key >> shift) & 255 --------------------------------------------------------------------------

__global__ void __launch_bounds__(kVoxThreads) k_vox_hist(const uint32_t* __restrict__ key, int shift, const int2* __restrict__ blocks,
                                                          const VoxSeg* __restrict__ segs, int* __restrict__ hist) {
  __shared__ int h[256];
  const int2 blk = blocks[blockIdx.x];
  const VoxSeg sg = segs[blk.x];
  h[threadIdx.x] = 0;
  __syncthreads();
#pragma unroll
  for (int k = 0; k < kVoxRounds; k++) {
    const int i = blk.y + k * kVoxThreads + threadIdx.x;
    if (i < sg.npts) atomicAdd(&h[(key[sg.pt0 + i] >> shift) & 255u], 1);
  }
  __syncthreads();
  hist[blockIdx.x * 256 + threadIdx.x] = h[threadIdx.x];
}

// One CTA per node, thread d owns digit d: the counts of the node's blocks become output positions, digit-major then block
// order, from the node's first point.
__global__ void __launch_bounds__(256) k_vox_offsets(const VoxSeg* __restrict__ segs, int* __restrict__ hist) {
  __shared__ int warp_sum[8];
  const VoxSeg sg = segs[blockIdx.x];
  const int d = threadIdx.x, lane = d & 31, wid = d >> 5;
  int* h = hist + (size_t)sg.blk0 * 256 + d;
  int total = 0;
  for (int b = 0; b < sg.nblk; b++) total += h[(size_t)b * 256];
  int incl = total;
#pragma unroll
  for (int s = 1; s < 32; s <<= 1) {
    const int t = __shfl_up_sync(0xffffffffu, incl, s);
    if (lane >= s) incl += t;
  }
  if (lane == 31) warp_sum[wid] = incl;
  __syncthreads();
  int run = sg.pt0 + incl - total;
  for (int w = 0; w < wid; w++) run += warp_sum[w];
  for (int b = 0; b < sg.nblk; b++) {
    const int t = h[(size_t)b * 256];
    h[(size_t)b * 256] = run;
    run += t;
  }
}

// The block's points go to their digit's positions in raster order: round by round, warp by warp, lane by lane.
__global__ void __launch_bounds__(kVoxThreads) k_vox_scatter(const uint32_t* __restrict__ key_in, const uint32_t* __restrict__ idx_in,
                                                             uint32_t* __restrict__ key_out, uint32_t* __restrict__ idx_out, int shift,
                                                             const int2* __restrict__ blocks, const VoxSeg* __restrict__ segs,
                                                             const int* __restrict__ hist) {
  __shared__ int warp_pos[kVoxThreads / 32][256];
  __shared__ int next[256];
  const int2 blk = blocks[blockIdx.x];
  const VoxSeg sg = segs[blk.x];
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  next[threadIdx.x] = hist[blockIdx.x * 256 + threadIdx.x];
#pragma unroll 1
  for (int k = 0; k < kVoxRounds; k++) {
#pragma unroll
    for (int w = 0; w < kVoxThreads / 32; w++) warp_pos[w][threadIdx.x] = 0;
    __syncthreads();
    const int i = blk.y + k * kVoxThreads + threadIdx.x;
    const bool valid = i < sg.npts;
    uint32_t kk = 0, ii = 0;
    if (valid) {
      kk = key_in[sg.pt0 + i];
      ii = idx_in[sg.pt0 + i];
    }
    const int d = (int)((kk >> shift) & 255u);
    const unsigned peers = __match_any_sync(0xffffffffu, valid ? d : 256 + lane);  // the lanes of this warp with the same digit
    if (valid && lane == __ffs(peers) - 1) warp_pos[wid][d] = __popc(peers);
    __syncthreads();
    {
      int acc = next[threadIdx.x];
#pragma unroll
      for (int w = 0; w < kVoxThreads / 32; w++) {
        const int t = warp_pos[w][threadIdx.x];
        warp_pos[w][threadIdx.x] = acc;
        acc += t;
      }
      next[threadIdx.x] = acc;
    }
    __syncthreads();
    if (valid) {
      const int dst = warp_pos[wid][d] + __popc(peers & ((1u << lane) - 1u));
      key_out[dst] = kk;
      idx_out[dst] = ii;
    }
    __syncthreads();
  }
}

// ---- runs ------------------------------------------------------------------------------------------------------------------

// Point i of a node's sorted segment starts a voxel's run.
__device__ __forceinline__ bool vox_is_head(const uint32_t* __restrict__ key, const VoxSeg& sg, int i) {
  const uint32_t k = key[sg.pt0 + i];
  return k != kVoxNoKey && (i == 0 || key[sg.pt0 + i - 1] != k);
}

// LIST false: counts[block] = its run heads.  LIST true: heads[offs[block] + rank] = (position in the chunk, node).
template <bool LIST>
__global__ void __launch_bounds__(kVoxThreads) k_vox_heads(const uint32_t* __restrict__ key, const int2* __restrict__ blocks,
                                                           const VoxSeg* __restrict__ segs, int* __restrict__ counts,
                                                           const long long* __restrict__ offs, int2* __restrict__ heads) {
  __shared__ int warp_cnt[kVoxThreads / 32];
  const int2 blk = blocks[blockIdx.x];
  const VoxSeg sg = segs[blk.x];
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  long long next = LIST ? offs[blockIdx.x] : 0;
#pragma unroll 1
  for (int k = 0; k < kVoxRounds; k++) {
    const int i = blk.y + k * kVoxThreads + threadIdx.x;
    const bool head = i < sg.npts && vox_is_head(key, sg, i);
    const unsigned bal = __ballot_sync(0xffffffffu, head);
    if (lane == 0) warp_cnt[wid] = __popc(bal);
    __syncthreads();
    int before = 0, total = 0;
#pragma unroll
    for (int w = 0; w < kVoxThreads / 32; w++) {
      const int c = warp_cnt[w];
      before += w < wid ? c : 0;
      total += c;
    }
    if (LIST && head) heads[next + before + __popc(bal & ((1u << lane) - 1u))] = make_int2(sg.pt0 + i, blk.x);
    next += total;
    __syncthreads();
  }
  if (!LIST && threadIdx.x == 0) counts[blockIdx.x] = (int)next;
}

// The centroid of one voxel (PCL 1.7 voxel_grid.hpp, downsample_all_data_): x, y, z, r, g, b summed one point after the
// other in float, each sum times 1.0f / n (Eigen 3.2's operator/=(Scalar) multiplies by the reciprocal), the colour means
// truncated to bytes.
__global__ void __launch_bounds__(kVoxThreads) k_vox_centroids(const MapNode* __restrict__ nodes, const VoxSeg* __restrict__ segs,
                                                               const uint32_t* __restrict__ key, const uint32_t* __restrict__ idx,
                                                               const long long* __restrict__ offs, const int2* __restrict__ heads,
                                                               long long nvoxels, float* __restrict__ slab) {
  const long long v = (long long)blockIdx.x * kVoxThreads + threadIdx.x;
  if (v >= nvoxels) return;
  const int2 hd = heads[v];
  const MapNode& nd = nodes[hd.y];
  const VoxSeg sg = segs[hd.y];
  const MapArgs a = vox_args();
  const uint32_t k = key[hd.x];
  const int end = sg.pt0 + sg.npts;
  float sx = 0.f, sy = 0.f, sz = 0.f, sr = 0.f, sgr = 0.f, sb = 0.f;
  int n = 0;
  for (int j = hd.x; j < end && key[j] == k; j++, n++) {
    MapOut o;
    map_point(nd, (int)idx[j], a, o);
    sx = __fadd_rn(sx, o.x);
    sy = __fadd_rn(sy, o.y);
    sz = __fadd_rn(sz, o.z);
    sr = __fadd_rn(sr, (float)((o.rgb >> 16) & 255u));
    sgr = __fadd_rn(sgr, (float)((o.rgb >> 8) & 255u));
    sb = __fadd_rn(sb, (float)(o.rgb & 255u));
  }
  const float rn = __fdiv_rn(1.0f, (float)n);
  const long long first = offs[sg.blk0], count = offs[sg.blk0 + sg.nblk] - first;
  float* out = slab + 4 * first;
  const long long at = v - first;
  out[at] = __fmul_rn(sx, rn);
  out[count + at] = __fmul_rn(sy, rn);
  out[2 * count + at] = __fmul_rn(sz, rn);
  const uint32_t r = (uint32_t)(int)__fmul_rn(sr, rn), gg = (uint32_t)(int)__fmul_rn(sgr, rn), bb = (uint32_t)(int)__fmul_rn(sb, rn);
  reinterpret_cast<uint32_t*>(out)[3 * count + at] = (r << 16) | (gg << 8) | bb;
}

// ---- launchers -------------------------------------------------------------------------------------------------------------

cudaError_t launch_vox_keys(const VoxBufs& b, int nnodes, int nblocks, float inv_leaf, cudaStream_t st, int* n_launches) {
  cudaError_t e = cudaMemsetAsync(b.bmin, 0xff, sizeof(uint32_t) * 3 * (size_t)nnodes, st);
  if (e == cudaSuccess) e = cudaMemsetAsync(b.bmax, 0, sizeof(uint32_t) * 3 * (size_t)nnodes, st);
  if (e != cudaSuccess) return e;
  if (nblocks > 0) {
    k_vox_bounds<<<nblocks, kVoxThreads, 0, st>>>(b.nodes, b.blocks, b.bmin, b.bmax);
    ++*n_launches;
  }
  k_vox_grid<<<(nnodes + 127) / 128, 128, 0, st>>>(nnodes, b.bmin, b.bmax, inv_leaf, b.grid);
  ++*n_launches;
  if (nblocks > 0) {
    k_vox_keys<<<nblocks, kVoxThreads, 0, st>>>(b.nodes, b.blocks, b.segs, b.grid, inv_leaf, b.key[0], b.idx[0]);
    ++*n_launches;
  }
  return cudaGetLastError();
}

cudaError_t launch_vox_sort(const VoxBufs& b, int nnodes, int nblocks, int passes, cudaStream_t st, int* n_launches) {
  if (nblocks > 0) {
    for (int p = 0; p < passes; p++) {
      const int in = p & 1, shift = 8 * p;
      k_vox_hist<<<nblocks, kVoxThreads, 0, st>>>(b.key[in], shift, b.blocks, b.segs, b.hist);
      k_vox_offsets<<<nnodes, 256, 0, st>>>(b.segs, b.hist);
      k_vox_scatter<<<nblocks, kVoxThreads, 0, st>>>(b.key[in], b.idx[in], b.key[in ^ 1], b.idx[in ^ 1], shift, b.blocks, b.segs,
                                                     b.hist);
      *n_launches += 3;
    }
    k_vox_heads<false><<<nblocks, kVoxThreads, 0, st>>>(b.key[passes & 1], b.blocks, b.segs, b.counts, nullptr, nullptr);
    ++*n_launches;
  }
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return e;
  e = launch_map_scan(b.counts, nblocks, b.offs, st);
  ++*n_launches;
  if (e != cudaSuccess || nblocks == 0) return e;
  k_vox_heads<true><<<nblocks, kVoxThreads, 0, st>>>(b.key[passes & 1], b.blocks, b.segs, nullptr, b.offs, b.heads);
  ++*n_launches;
  return cudaGetLastError();
}

cudaError_t launch_vox_centroids(const VoxBufs& b, int passes, long long nvoxels, float* slab, cudaStream_t st) {
  if (nvoxels <= 0) return cudaSuccess;
  k_vox_centroids<<<(unsigned)((nvoxels + kVoxThreads - 1) / kVoxThreads), kVoxThreads, 0, st>>>(
      b.nodes, b.segs, b.key[passes & 1], b.idx[passes & 1], b.offs, b.heads, nvoxels, slab);
  return cudaGetLastError();
}

}  // namespace rb200
