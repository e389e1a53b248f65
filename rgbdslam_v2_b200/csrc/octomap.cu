// octomap.cu -- the colour OctoMap of the nodes' stored clouds (ColorOctomapServer::insertCloudCallback, ColorOcTree::write):
//   k_oct_count / k_oct_emit  per point its ray cells (computeRayKeys), its occupied cell and its colour entry, counted per
//                             point and per 1024-point block, then written at the block's scanned offset in point order
//   k_oct_radix_*             stable 8-bit LSD radix sort of the entries on the key bytes that vary
//   k_oct_flag_keep           per (cell, scan) one free-or-occupied entry, occupied winning: one update per key and scan
//   k_oct_fold                one thread per cell: the scans' log-odds updates and the points' colours in order
//   k_oct_merge               the new leaves into the sorted leaf array
//   k_oct_reduce / _offsets / _records
//                             the writer: inner nodes level by level, pre-order record offsets top down, 8-byte records
//   k_ocf_flags / _scatter    the occupancy filter of the stored clouds: per point its keep flag from three leaf lookups,
//                             then the kept points of the changed nodes into new x / y / z / colour planes, in order
// The float and double chains are written with explicit _rn intrinsics: octomap on x86-64 does not contract.
#include <cfloat>
#include <climits>

#include "map.cuh"
#include "octomap.cuh"

namespace rb200 {

constexpr int kOctThreads = 256;
constexpr int kOctTile = 4096;  // items per CTA of the scan and the radix passes (16 per thread)
constexpr int kOctPer = kOctTile / kOctThreads;

__device__ __forceinline__ uint64_t oct_spread(uint32_t v) {  // bit i of v -> bit 3 i
  uint64_t x = v & 0xffffu;
  x = (x | (x << 32)) & 0x1f00000000ffffull;
  x = (x | (x << 16)) & 0x1f0000ff0000ffull;
  x = (x | (x << 8)) & 0x100f00f00f00f00full;
  x = (x | (x << 4)) & 0x10c30c30c30c30c3ull;
  x = (x | (x << 2)) & 0x1249249249249249ull;
  return x;
}
__device__ __forceinline__ uint64_t oct_morton(const uint32_t k[3]) {
  return oct_spread(k[0]) | (oct_spread(k[1]) << 1) | (oct_spread(k[2]) << 2);
}

// coordToKeyChecked: (int)floor(rf * c) + 32768 inside [0, 65536); x86's (int) of a NaN or out-of-range value fails the test too
__device__ __forceinline__ bool oct_key(double rf, float c, uint32_t& k) {
  const double v = floor(__dmul_rn(rf, (double)c));
  if (!(v >= -32768.0 && v < 32768.0)) return false;
  k = (uint32_t)((int)v + 32768);
  return true;
}
__device__ __forceinline__ bool oct_key3(double rf, float x, float y, float z, uint32_t k[3]) {
  return oct_key(rf, x, k[0]) && oct_key(rf, y, k[1]) && oct_key(rf, z, k[2]);
}

// computeRayKeys(origin, end): f(key) for every cell of the ray in order (none when a key fails or both keys are equal)
template <class F>
__device__ __forceinline__ void oct_ray(const OctArgs& a, const float o[3], const float e[3], F&& f) {
  uint32_t ko[3], ke[3];
  if (!oct_key3(a.rf, o[0], o[1], o[2], ko) || !oct_key3(a.rf, e[0], e[1], e[2], ke)) return;
  if (ko[0] == ke[0] && ko[1] == ke[1] && ko[2] == ke[2]) return;
  f(ko);
  float d[3];
#pragma unroll
  for (int i = 0; i < 3; i++) d[i] = __fsub_rn(e[i], o[i]);
  const float nsq = __fadd_rn(__fadd_rn(__fmul_rn(d[0], d[0]), __fmul_rn(d[1], d[1])), __fmul_rn(d[2], d[2]));
  const float len = __double2float_rn(__dsqrt_rn((double)nsq));
  int step[3];
  double tmax[3], tdelta[3];
#pragma unroll
  for (int i = 0; i < 3; i++) {
    d[i] = __fdiv_rn(d[i], len);
    step[i] = d[i] > 0.f ? 1 : (d[i] < 0.f ? -1 : 0);
    if (step[i] != 0) {
      // keyToCoord(key) + (float)(step * res * 0.5), in double
      const double border = __dadd_rn(__dmul_rn(__dadd_rn((double)((int)ko[i] - 32768), 0.5), a.res),
                                      (double)__double2float_rn(__dmul_rn(__dmul_rn((double)step[i], a.res), 0.5)));
      tmax[i] = __ddiv_rn(__dsub_rn(border, (double)o[i]), (double)d[i]);
      tdelta[i] = __ddiv_rn(a.res, (double)fabsf(d[i]));
    } else {
      tmax[i] = DBL_MAX;
      tdelta[i] = DBL_MAX;
    }
  }
  // the walk indexes nothing by the chosen axis, so that every array stays in registers
  uint32_t cur[3] = {ko[0], ko[1], ko[2]};
  const double dlen = (double)len;
  for (;;) {
    if (tmax[0] < tmax[1] && tmax[0] < tmax[2]) {
      cur[0] = (cur[0] + step[0]) & 0xffffu;
      tmax[0] = __dadd_rn(tmax[0], tdelta[0]);
    } else if (!(tmax[0] < tmax[1]) && tmax[1] < tmax[2]) {
      cur[1] = (cur[1] + step[1]) & 0xffffu;
      tmax[1] = __dadd_rn(tmax[1], tdelta[1]);
    } else {
      cur[2] = (cur[2] + step[2]) & 0xffffu;
      tmax[2] = __dadd_rn(tmax[2], tdelta[2]);
    }
    if (cur[0] == ke[0] && cur[1] == ke[1] && cur[2] == ke[2]) return;
    if (fmin(fmin(tmax[0], tmax[1]), tmax[2]) > dlen) return;
    f(cur);
  }
}

// Point i of node nd as insertCloudCallback sees it: v(key, kind, colour word) for each of its entries.
template <class V>
__device__ __forceinline__ void oct_point(const MapNode& nd, int i, const OctArgs& a, V&& v) {
  const MapArgs ma{0.f, 0, 1, 1, 32};  // every point, transformed, no depth filter
  MapOut p;
  map_point(nd, i, ma, p);
  if (!(isfinite(p.x) && isfinite(p.y) && isfinite(p.z))) return;
  const float o[3] = {nd.m[3], nd.m[7], nd.m[11]};
  const float e[3] = {p.x, p.y, p.z};
  float d[3];
#pragma unroll
  for (int k = 0; k < 3; k++) d[k] = __fsub_rn(e[k], o[k]);
  // Vector3::norm(): the float squared norm, its square root in double
  const double norm = __dsqrt_rn((double)__fadd_rn(__fadd_rn(__fmul_rn(d[0], d[0]), __fmul_rn(d[1], d[1])), __fmul_rn(d[2], d[2])));
  uint32_t k[3];
  if (a.max_range < 0.0 || norm <= a.max_range) {
    oct_ray(a, o, e, [&](const uint32_t* c) { v(c, 0u, 0u); });
    if (oct_key3(a.rf, e[0], e[1], e[2], k)) v(k, 1u, 0u);
  } else {  // origin + normalized(p - origin) * (float)max_range, all free
    const float len = (float)norm, mr = (float)a.max_range;
    float q[3];
#pragma unroll
    for (int c = 0; c < 3; c++) q[c] = __fadd_rn(o[c], __fmul_rn(norm > 0.0 ? __fdiv_rn(d[c], len) : d[c], mr));
    oct_ray(a, o, q, [&](const uint32_t* c) { v(c, 0u, 0u); });
  }
  if (oct_key3(a.rf, e[0], e[1], e[2], k)) v(k, 2u, p.rgb);
}

__device__ __forceinline__ int oct_block_sum(int c, int* warp_sum) {
#pragma unroll
  for (int s = 16; s > 0; s >>= 1) c += __shfl_xor_sync(0xffffffffu, c, s);
  if ((threadIdx.x & 31) == 0) warp_sum[threadIdx.x >> 5] = c;
  __syncthreads();
  int t = 0;
#pragma unroll
  for (int w = 0; w < kOctThreads / 32; w++) t += warp_sum[w];
  __syncthreads();
  return t;
}

// Exclusive block scan of c (thread order); *total receives the block's sum.
__device__ __forceinline__ long long oct_block_excl(long long c, long long* warp_sum, long long* total) {
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  long long incl = c;
#pragma unroll
  for (int s = 1; s < 32; s <<= 1) {
    const long long t = __shfl_up_sync(0xffffffffu, incl, s);
    if (lane >= s) incl += t;
  }
  if (lane == 31) warp_sum[wid] = incl;
  __syncthreads();
  long long before = 0, all = 0;
#pragma unroll
  for (int w = 0; w < kOctThreads / 32; w++) {
    before += w < wid ? warp_sum[w] : 0;
    all += warp_sum[w];
  }
  __syncthreads();
  *total = all;
  return before + incl - c;
}

// Per point its entry count (pcount[block * 1024 + point - first point]) and per block their sum.
__global__ void __launch_bounds__(kOctThreads) k_oct_count(const MapNode* __restrict__ nodes, const int2* __restrict__ blocks, OctArgs a,
                                                           int* __restrict__ counts, int* __restrict__ pcount) {
  __shared__ int warp_sum[kOctThreads / 32];
  const int2 blk = blocks[blockIdx.x];
  const MapNode& nd = nodes[blk.x];
  const int P = nd.cw * nd.ch;
  int c = 0;
#pragma unroll 1
  for (int r = 0; r < kMapBlockPoints / kOctThreads; r++) {
    const int i = blk.y + r * kOctThreads + threadIdx.x;
    int ci = 0;
    if (i < P) oct_point(nd, i, a, [&](const uint32_t*, uint32_t, uint32_t) { ci++; });
    pcount[(size_t)blockIdx.x * kMapBlockPoints + r * kOctThreads + threadIdx.x] = ci;
    c += ci;
  }
  const int t = oct_block_sum(c, warp_sum);
  if (threadIdx.x == 0) counts[blockIdx.x] = t;
}

__global__ void __launch_bounds__(kOctThreads) k_oct_emit(const MapNode* __restrict__ nodes, const int2* __restrict__ blocks, int b0,
                                                          int node0, const long long* __restrict__ offs, const int* __restrict__ pcount,
                                                          OctArgs a, unsigned long long* __restrict__ keys, uint32_t* __restrict__ vals) {
  __shared__ long long warp_sum[kOctThreads / 32];
  const int b = b0 + blockIdx.x;
  const int2 blk = blocks[b];
  const MapNode& nd = nodes[blk.x];
  const unsigned long long scan = (unsigned long long)(blk.x - node0) << 2;
  const int P = nd.cw * nd.ch;
  long long next = offs[blockIdx.x];
#pragma unroll 1
  for (int r = 0; r < kMapBlockPoints / kOctThreads; r++) {
    const int i = blk.y + r * kOctThreads + threadIdx.x;
    const int c = pcount[(size_t)b * kMapBlockPoints + r * kOctThreads + threadIdx.x];
    long long total;
    long long w = next + oct_block_excl(c, warp_sum, &total);
    if (i < P)
      oct_point(nd, i, a, [&](const uint32_t* k, uint32_t kind, uint32_t rgb) {
        keys[w] = (oct_morton(k) << 16) | scan | kind;
        vals[w] = rgb;
        w++;
      });
    next += total;
  }
}

// ---- scan, key bits, radix sort --------------------------------------------------------------------------------------------

__global__ void __launch_bounds__(kOctThreads) k_oct_tile_sums(const uint32_t* __restrict__ in, long long n, int* __restrict__ sums) {
  __shared__ int warp_sum[kOctThreads / 32];
  const long long base = (long long)blockIdx.x * kOctTile + (long long)threadIdx.x * kOctPer;
  int c = 0;
#pragma unroll
  for (int k = 0; k < kOctPer; k++) c += base + k < n ? (int)in[base + k] : 0;
  const int t = oct_block_sum(c, warp_sum);
  if (threadIdx.x == 0) sums[blockIdx.x] = t;
}

__global__ void __launch_bounds__(kOctThreads) k_oct_tile_apply(const uint32_t* __restrict__ in, long long n,
                                                                const long long* __restrict__ tile_offs, uint32_t* __restrict__ out) {
  __shared__ long long warp_sum[kOctThreads / 32];
  const long long base = (long long)blockIdx.x * kOctTile + (long long)threadIdx.x * kOctPer;
  uint32_t v[kOctPer];
  long long c = 0;
#pragma unroll
  for (int k = 0; k < kOctPer; k++) {
    v[k] = base + k < n ? in[base + k] : 0u;
    c += v[k];
  }
  long long total;
  long long run = tile_offs[blockIdx.x] + oct_block_excl(c, warp_sum, &total);
#pragma unroll
  for (int k = 0; k < kOctPer; k++) {
    if (base + k < n) out[base + k] = (uint32_t)run;
    run += v[k];
  }
}

int oct_scan_tiles(long long n) { return (int)std::max<long long>(1, (n + kOctTile - 1) / kOctTile); }

cudaError_t launch_oct_scan(const uint32_t* flags, long long n, uint32_t* offs, int* tile_sums, long long* tile_offs, cudaStream_t st) {
  const int nt = oct_scan_tiles(n);
  k_oct_tile_sums<<<nt, kOctThreads, 0, st>>>(flags, n, tile_sums);
  cudaError_t e = launch_map_scan(tile_sums, nt, tile_offs, st);
  if (e != cudaSuccess) return e;
  k_oct_tile_apply<<<nt, kOctThreads, 0, st>>>(flags, n, tile_offs, offs);
  return cudaGetLastError();
}

__global__ void __launch_bounds__(kOctThreads) k_oct_key_bits(const unsigned long long* __restrict__ keys, long long n,
                                                              unsigned long long* __restrict__ bits) {
  unsigned long long o = 0, an = ~0ull;
  for (long long i = (long long)blockIdx.x * kOctThreads + threadIdx.x; i < n; i += (long long)gridDim.x * kOctThreads) {
    o |= keys[i];
    an &= keys[i];
  }
#pragma unroll
  for (int s = 16; s > 0; s >>= 1) {
    o |= __shfl_xor_sync(0xffffffffu, o, s);
    an &= __shfl_xor_sync(0xffffffffu, an, s);
  }
  if ((threadIdx.x & 31) == 0) {
    atomicOr(&bits[0], o);
    atomicAnd(&bits[1], an);
  }
}

cudaError_t launch_oct_key_bits(const unsigned long long* keys, long long n, unsigned long long* d_bits, cudaStream_t st) {
  const unsigned long long init[2] = {0ull, ~0ull};
  cudaError_t e = cudaMemcpyAsync(d_bits, init, sizeof(init), cudaMemcpyHostToDevice, st);
  if (e != cudaSuccess) return e;
  const long long blocks = std::min<long long>(1024, std::max<long long>(1, (n + kOctThreads - 1) / kOctThreads));
  k_oct_key_bits<<<(int)blocks, kOctThreads, 0, st>>>(keys, n, d_bits);
  return cudaGetLastError();
}

// digit-major histogram: hist[d * ntiles + tile]
__global__ void __launch_bounds__(kOctThreads) k_oct_radix_hist(const unsigned long long* __restrict__ keys, long long n, int shift,
                                                                uint32_t* __restrict__ hist) {
  __shared__ uint32_t h[256];
  h[threadIdx.x] = 0;
  __syncthreads();
  const long long base = (long long)blockIdx.x * kOctTile;
#pragma unroll 4
  for (int k = 0; k < kOctPer; k++) {
    const long long i = base + k * kOctThreads + threadIdx.x;
    if (i < n) atomicAdd(&h[(keys[i] >> shift) & 0xff], 1u);
  }
  __syncthreads();
  hist[(size_t)threadIdx.x * gridDim.x + blockIdx.x] = h[threadIdx.x];
}

// Stable scatter: the tile's items go in index order, 256 per round; inside a round an item's place among equal digits is
// its warp's count of them before it plus its rank among its warp's peers.
__global__ void __launch_bounds__(kOctThreads) k_oct_radix_scatter(const unsigned long long* __restrict__ kin,
                                                                   const uint32_t* __restrict__ vin, long long n, int shift,
                                                                   const uint32_t* __restrict__ hist_offs,
                                                                   unsigned long long* __restrict__ kout, uint32_t* __restrict__ vout) {
  constexpr int W = kOctThreads / 32;
  __shared__ uint32_t base[256];
  __shared__ uint16_t wcnt[W][256];
  base[threadIdx.x] = hist_offs[(size_t)threadIdx.x * gridDim.x + blockIdx.x];
#pragma unroll
  for (int w = 0; w < W; w++) wcnt[w][threadIdx.x] = 0;
  __syncthreads();
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  const long long tile = (long long)blockIdx.x * kOctTile;
#pragma unroll 1
  for (int r = 0; r < kOctPer; r++) {
    const long long i = tile + r * kOctThreads + threadIdx.x;
    const bool ok = i < n;
    const unsigned long long key = ok ? kin[i] : 0ull;
    const uint32_t d = ok ? (uint32_t)((key >> shift) & 0xff) : 256u;
    const unsigned peers = __match_any_sync(0xffffffffu, d);
    const int rank = __popc(peers & ((1u << lane) - 1u));
    if (ok && rank == 0) wcnt[wid][d] = (uint16_t)__popc(peers);
    __syncthreads();
    if (ok) {
      uint32_t pos = base[d] + rank;
      for (int w = 0; w < wid; w++) pos += wcnt[w][d];
      kout[pos] = key;
      vout[pos] = vin[i];
    }
    __syncthreads();
    uint32_t add = 0;
#pragma unroll
    for (int w = 0; w < W; w++) {
      add += wcnt[w][threadIdx.x];
      wcnt[w][threadIdx.x] = 0;
    }
    base[threadIdx.x] += add;
    __syncthreads();
  }
}

cudaError_t launch_oct_radix_pass(const unsigned long long* kin, const uint32_t* vin, long long n, int shift, uint32_t* hist,
                                  uint32_t* hist_offs, int* tile_sums, long long* tile_offs, unsigned long long* kout,
                                  uint32_t* vout, cudaStream_t st) {
  const int nt = oct_scan_tiles(n);
  k_oct_radix_hist<<<nt, kOctThreads, 0, st>>>(kin, n, shift, hist);
  cudaError_t e = launch_oct_scan(hist, 256ll * nt, hist_offs, tile_sums, tile_offs, st);
  if (e != cudaSuccess) return e;
  k_oct_radix_scatter<<<nt, kOctThreads, 0, st>>>(kin, vin, n, shift, hist_offs, kout, vout);
  return cudaGetLastError();
}

// ---- reduction to one update per (cell, scan), the fold, the merge ---------------------------------------------------------

__global__ void k_oct_flag_keep(const unsigned long long* __restrict__ keys, long long n, uint32_t* __restrict__ flags) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const unsigned long long k = keys[i];
  // a free / occupied entry is kept when it is the last one of its (cell, scan): kind 1 then says "some ray ended here"
  flags[i] = (k & 3) == 2 || i + 1 == n || (keys[i + 1] >> 2) != (k >> 2) || (keys[i + 1] & 3) == 2;
}

__global__ void k_oct_compact(const unsigned long long* __restrict__ kin, const uint32_t* __restrict__ vin, const uint32_t* __restrict__ flags,
                              const uint32_t* __restrict__ offs, long long n, unsigned long long* __restrict__ kout,
                              uint32_t* __restrict__ vout) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n || !flags[i]) return;
  kout[offs[i]] = kin[i];
  vout[offs[i]] = vin[i];
}

__global__ void k_oct_flag_heads(const unsigned long long* __restrict__ keys, long long n, int shift, uint32_t* __restrict__ flags) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  flags[i] = i == 0 || (keys[i] >> shift) != (keys[i - 1] >> shift);
}

__global__ void k_oct_index(const uint32_t* __restrict__ flags, const uint32_t* __restrict__ offs, long long n, uint32_t* __restrict__ out) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n && flags[i]) out[offs[i]] = (uint32_t)i;
}

__device__ __forceinline__ long long oct_lower_bound(const unsigned long long* __restrict__ k, long long n, unsigned long long x) {
  long long lo = 0, hi = n;
  while (lo < hi) {
    const long long mid = (lo + hi) >> 1;
    if (k[mid] < x) lo = mid + 1;
    else hi = mid;
  }
  return lo;
}

// averageNodeColor on a leaf colour (r << 16 | g << 8 | b; kOctWhite = unset)
__device__ __forceinline__ uint32_t oct_average(uint32_t prev, uint32_t word) {
  const uint32_t c = word & 0xffffffu;
  if (prev == kOctWhite) return c;
  uint32_t out = 0;
#pragma unroll
  for (int s = 0; s < 24; s += 8) out |= ((((prev >> s) & 0xff) + ((c >> s) & 0xff)) / 2) << s;
  return out;
}

__global__ void k_oct_fold(const unsigned long long* __restrict__ ck, const uint32_t* __restrict__ cv, long long c,
                           const uint32_t* __restrict__ starts, long long m, OctArgs a, const unsigned long long* __restrict__ lk,
                           float* __restrict__ llo, uint32_t* __restrict__ lrgb, long long nleaves, unsigned long long* __restrict__ nk,
                           float* __restrict__ nlo, uint32_t* __restrict__ nrgb, uint32_t* __restrict__ new_flag) {
  const long long j = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= m) return;
  const long long b = starts[j], e = j + 1 < m ? (long long)starts[j + 1] : c;
  const unsigned long long cell = ck[b] >> 16;
  const long long idx = oct_lower_bound(lk, nleaves, cell);
  const bool existed = idx < nleaves && lk[idx] == cell;
  float lo = existed ? llo[idx] : 0.f;
  uint32_t rgb = existed ? lrgb[idx] : kOctWhite;
  bool live = existed;
  for (long long i = b; i < e; i++) {
    const uint32_t kind = (uint32_t)(ck[i] & 3);
    if (kind <= 1) {  // updateNodeLogOdds: add, then clamp
      live = true;
      lo = __fadd_rn(lo, kind ? a.hit : a.miss);
      if (lo < a.cmin) lo = a.cmin;
      if (lo > a.cmax) lo = a.cmax;
    } else if (live) {
      rgb = oct_average(rgb, cv[i]);
    }
  }
  if (existed) {
    llo[idx] = lo;
    lrgb[idx] = rgb;
  }
  nk[j] = cell;
  nlo[j] = lo;
  nrgb[j] = rgb;
  new_flag[j] = !existed && live;
}

__global__ void k_oct_merge_old(const unsigned long long* __restrict__ lk, const float* __restrict__ llo, const uint32_t* __restrict__ lrgb,
                                long long nleaves, const unsigned long long* __restrict__ newk, long long nnew,
                                unsigned long long* __restrict__ ok, float* __restrict__ olo, uint32_t* __restrict__ orgb) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= nleaves) return;
  const long long p = i + oct_lower_bound(newk, nnew, lk[i]);
  ok[p] = lk[i];
  olo[p] = llo[i];
  orgb[p] = lrgb[i];
}

__global__ void k_oct_gather_new(const unsigned long long* __restrict__ nk, const uint32_t* __restrict__ new_flag,
                                 const uint32_t* __restrict__ offs, long long m, unsigned long long* __restrict__ newk) {
  const long long j = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (j < m && new_flag[j]) newk[offs[j]] = nk[j];
}

__global__ void k_oct_merge_new(const unsigned long long* __restrict__ lk, long long nleaves, const unsigned long long* __restrict__ nk,
                                const float* __restrict__ nlo, const uint32_t* __restrict__ nrgb, const uint32_t* __restrict__ new_flag,
                                const uint32_t* __restrict__ offs, long long m, unsigned long long* __restrict__ ok,
                                float* __restrict__ olo, uint32_t* __restrict__ orgb) {
  const long long j = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= m || !new_flag[j]) return;
  const long long p = offs[j] + oct_lower_bound(lk, nleaves, nk[j]);
  ok[p] = nk[j];
  olo[p] = nlo[j];
  orgb[p] = nrgb[j];
}

// ---- the writer ------------------------------------------------------------------------------------------------------------

__global__ void k_oct_leaf_level(OctLevel l) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= l.n) return;
  l.size[i] = 1;
  l.mask[i] = 0;
}

// ColorOcTreeNode::updateOccupancyChildren (maximum child log-odds) and updateColorChildren (int mean of the set colours)
__global__ void k_oct_reduce(OctLevel p, OctLevel c) {
  const long long j = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= p.n) return;
  const long long b = p.first[j], e = j + 1 < p.n ? (long long)p.first[j + 1] : c.n;
  float lo = -FLT_MAX;
  uint32_t mask = 0, sr = 0, sg = 0, sb = 0, cnt = 0;
  unsigned long long size = 1;
  for (long long i = b; i < e; i++) {
    mask |= 1u << (c.key[i] & 7);
    if (c.lo[i] > lo) lo = c.lo[i];
    const uint32_t rgb = c.rgb[i];
    if (rgb != kOctWhite) {
      sr += rgb >> 16;
      sg += (rgb >> 8) & 0xff;
      sb += rgb & 0xff;
      cnt++;
    }
    size += c.size[i];
  }
  p.key[j] = c.key[b] >> 3;
  p.lo[j] = lo;
  p.rgb[j] = cnt ? ((sr / cnt) << 16) | ((sg / cnt) << 8) | (sb / cnt) : kOctWhite;
  p.mask[j] = (uint8_t)mask;
  p.size[j] = size;
}

__global__ void k_oct_offsets(OctLevel p, OctLevel c) {
  const long long j = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= p.n) return;
  const long long b = p.first[j], e = j + 1 < p.n ? (long long)p.first[j + 1] : c.n;
  unsigned long long o = p.off[j] + 1;
  for (long long i = b; i < e; i++) {
    c.off[i] = o;
    o += c.size[i];
  }
}

__global__ void k_oct_records(OctLevel l, uint2* __restrict__ out) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= l.n) return;
  const uint32_t rgb = l.rgb[i];
  // float value, then Color {r, g, b}, then the child bits (ColorOcTreeNode::writeValue)
  out[l.off[i]] = make_uint2(__float_as_uint(l.lo[i]),
                             (rgb >> 16) | (((rgb >> 8) & 0xff) << 8) | ((rgb & 0xff) << 16) | ((uint32_t)l.mask[i] << 24));
}

// ---- the occupancy filter --------------------------------------------------------------------------------------------------

// coordToKey unchecked: (uint16)((int)floor(rf * c) + 32768), (int) as x86-64's cvttsd2si (INT_MIN for NaN, +-inf and out of
// range)
__device__ __forceinline__ uint32_t ocf_key(double rf, float c) {
  const double v = floor(__dmul_rn(rf, (double)c));
  const int k = v >= -2147483648.0 && v < 2147483648.0 ? (int)v : INT_MIN;
  return ((uint32_t)k + 32768u) & 0xffffu;
}

// keyToCoord: (double((int)key - 32768) + 0.5) * res
__device__ __forceinline__ double ocf_coord(double res, uint32_t k) { return __dmul_rn(__dadd_rn((double)((int)k - 32768), 0.5), res); }

// ColorOctomapServer::occupancyFilter for one point p (as stored) under the sensor pose s (qx qy qz qw ox oy oz)
__device__ __forceinline__ bool ocf_keep(const OcfArgs& a, const float* s, float px, float py, float pz) {
  const float qx = s[0], qy = s[1], qz = s[2], qw = s[3];
  // Eigen's _transformVector: uv = q.vec() x p; uv += uv; v = p + w uv + q.vec() x uv; then + t
  float ux = __fsub_rn(__fmul_rn(qy, pz), __fmul_rn(qz, py));
  float uy = __fsub_rn(__fmul_rn(qz, px), __fmul_rn(qx, pz));
  float uz = __fsub_rn(__fmul_rn(qx, py), __fmul_rn(qy, px));
  ux = __fadd_rn(ux, ux);
  uy = __fadd_rn(uy, uy);
  uz = __fadd_rn(uz, uz);
  const float ix = __fadd_rn(__fadd_rn(__fadd_rn(px, __fmul_rn(qw, ux)), __fsub_rn(__fmul_rn(qy, uz), __fmul_rn(qz, uy))), s[4]);
  const float iy = __fadd_rn(__fadd_rn(__fadd_rn(py, __fmul_rn(qw, uy)), __fsub_rn(__fmul_rn(qz, ux), __fmul_rn(qx, uz))), s[5]);
  const float iz = __fadd_rn(__fadd_rn(__fadd_rn(pz, __fmul_rn(qw, uz)), __fsub_rn(__fmul_rn(qx, uy), __fmul_rn(qy, ux))), s[6]);
  if (isnan(iz)) return false;
  // the reference's nested loops never reset y_a / z_a: only (kx - 1, ky - 1, kz - 1 + d), d = 0, 1, 2, are visited
  const uint32_t k[3] = {(ocf_key(a.rf, ix) + 0xffffu) & 0xffffu, (ocf_key(a.rf, iy) + 0xffffu) & 0xffffu,
                         (ocf_key(a.rf, iz) + 0xffffu) & 0xffffu};
  const double dx = __dsub_rn(ocf_coord(a.res, k[0]), (double)ix);
  const double dy = __dsub_rn(ocf_coord(a.res, k[1]), (double)iy);
  const double dxy = __dadd_rn(__dmul_rn(dx, dx), __dmul_rn(dy, dy));
  double so = 0.0, sw = 0.0;
#pragma unroll 1
  for (int d = 0; d < 3; d++) {
    const uint32_t c[3] = {k[0], k[1], (k[2] + d) & 0xffffu};
    const unsigned long long key = oct_morton(c);
    const long long idx = oct_lower_bound(a.lk, a.nleaves, key);
    if (idx < a.nleaves && a.lk[idx] == key) {
      const double dz = __dsub_rn(ocf_coord(a.res, c[2]), (double)iz);
      const double w = __dadd_rn(dxy, __dmul_rn(dz, dz));
      so = __dadd_rn(so, __ddiv_rn(a.occ[idx], w));
      sw = __dadd_rn(sw, w);
    }
  }
  return so < __dmul_rn(a.threshold, sw);
}

__global__ void __launch_bounds__(kOctThreads) k_ocf_flags(const MapNode* __restrict__ nodes, const int2* __restrict__ blocks,
                                                           const float* __restrict__ sensor7, OcfArgs a, uint8_t* __restrict__ flags,
                                                           int* __restrict__ counts, uint8_t* __restrict__ keep0) {
  __shared__ int warp_sum[kOctThreads / 32];
  const int2 blk = blocks[blockIdx.x];
  const MapNode& nd = nodes[blk.x];
  const float* s = sensor7 + 7 * (size_t)blk.x;
  const int P = nd.cw * nd.ch;
  const MapArgs ma{0.f, 0, 1, 0, 32};  // every point, as stored
  int c = 0;
#pragma unroll 1
  for (int r = 0; r < kMapBlockPoints / kOctThreads; r++) {
    const int i = blk.y + r * kOctThreads + threadIdx.x;
    bool keep = false;
    if (i < P) {
      MapOut p;
      map_point(nd, i, ma, p);
      keep = ocf_keep(a, s, p.x, p.y, p.z);
    }
    flags[(size_t)blockIdx.x * kMapBlockPoints + r * kOctThreads + threadIdx.x] = keep;
    if (i == 0) keep0[blk.x] = keep;
    c += keep;
  }
  const int t = oct_block_sum(c, warp_sum);
  if (threadIdx.x == 0) counts[blockIdx.x] = t;
}

__global__ void __launch_bounds__(kOctThreads) k_ocf_scatter(const MapNode* __restrict__ nodes, const int2* __restrict__ blocks,
                                                             const uint8_t* __restrict__ flags, const long long* __restrict__ offs,
                                                             const OcfOut* __restrict__ out, float* __restrict__ slab) {
  __shared__ int warp_cnt[kOctThreads / 32];
  const int2 blk = blocks[blockIdx.x];
  const OcfOut o = out[blk.x];
  if (o.dst < 0) return;  // the whole CTA: the node keeps its cloud
  const MapNode& nd = nodes[blk.x];
  const int P = nd.cw * nd.ch;
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  float* x = slab + 4 * o.dst;
  long long next = offs[blockIdx.x] - o.first;
  const MapArgs ma{0.f, 0, 1, 0, 32};
#pragma unroll 1
  for (int r = 0; r < kMapBlockPoints / kOctThreads; r++) {
    const int i = blk.y + r * kOctThreads + threadIdx.x;
    const bool keep = i < P && flags[(size_t)blockIdx.x * kMapBlockPoints + r * kOctThreads + threadIdx.x];
    const unsigned bal = __ballot_sync(0xffffffffu, keep);
    if (lane == 0) warp_cnt[wid] = __popc(bal);
    __syncthreads();
    int before = 0, total = 0;
#pragma unroll
    for (int w = 0; w < kOctThreads / 32; w++) {
      const int c = warp_cnt[w];
      before += w < wid ? c : 0;
      total += c;
    }
    if (keep) {
      MapOut p;
      map_point(nd, i, ma, p);
      const long long j = next + before + __popc(bal & ((1u << lane) - 1u));
      x[j] = p.x;
      x[o.count + j] = p.y;
      x[2 * o.count + j] = p.z;
      reinterpret_cast<uint32_t*>(x)[3 * o.count + j] = p.rgb;
    }
    next += total;
    __syncthreads();
  }
}

// ---- launchers -------------------------------------------------------------------------------------------------------------

cudaError_t launch_ocf_flags(const MapNode* d_nodes, const int2* d_blocks, int nblocks, const float* d_sensor7, const OcfArgs& a,
                             uint8_t* d_flags, int* d_counts, uint8_t* d_keep0, cudaStream_t st) {
  if (nblocks <= 0) return cudaSuccess;
  k_ocf_flags<<<nblocks, kOctThreads, 0, st>>>(d_nodes, d_blocks, d_sensor7, a, d_flags, d_counts, d_keep0);
  return cudaGetLastError();
}

cudaError_t launch_ocf_scatter(const MapNode* d_nodes, const int2* d_blocks, int nblocks, const uint8_t* d_flags, const long long* d_offs,
                               const OcfOut* d_out, float* slab, cudaStream_t st) {
  if (nblocks <= 0) return cudaSuccess;
  k_ocf_scatter<<<nblocks, kOctThreads, 0, st>>>(d_nodes, d_blocks, d_flags, d_offs, d_out, slab);
  return cudaGetLastError();
}

static inline unsigned grid_of(long long n) { return (unsigned)std::max<long long>(1, (n + kOctThreads - 1) / kOctThreads); }

cudaError_t launch_oct_count(const MapNode* d_nodes, const int2* d_blocks, int nblocks, const OctArgs& a, int* d_counts,
                             int* d_pcount, cudaStream_t st) {
  if (nblocks <= 0) return cudaSuccess;
  k_oct_count<<<nblocks, kOctThreads, 0, st>>>(d_nodes, d_blocks, a, d_counts, d_pcount);
  return cudaGetLastError();
}

cudaError_t launch_oct_emit(const MapNode* d_nodes, const int2* d_blocks, int b0, int b1, int node0, const long long* d_offs,
                            const int* d_pcount, const OctArgs& a, unsigned long long* keys, uint32_t* vals, cudaStream_t st) {
  if (b1 <= b0) return cudaSuccess;
  k_oct_emit<<<b1 - b0, kOctThreads, 0, st>>>(d_nodes, d_blocks, b0, node0, d_offs, d_pcount, a, keys, vals);
  return cudaGetLastError();
}

cudaError_t launch_oct_flag_keep(const unsigned long long* keys, long long n, uint32_t* flags, cudaStream_t st) {
  k_oct_flag_keep<<<grid_of(n), kOctThreads, 0, st>>>(keys, n, flags);
  return cudaGetLastError();
}

cudaError_t launch_oct_compact(const unsigned long long* kin, const uint32_t* vin, const uint32_t* flags, const uint32_t* offs,
                               long long n, unsigned long long* kout, uint32_t* vout, cudaStream_t st) {
  k_oct_compact<<<grid_of(n), kOctThreads, 0, st>>>(kin, vin, flags, offs, n, kout, vout);
  return cudaGetLastError();
}

cudaError_t launch_oct_flag_heads(const unsigned long long* keys, long long n, int shift, uint32_t* flags, cudaStream_t st) {
  k_oct_flag_heads<<<grid_of(n), kOctThreads, 0, st>>>(keys, n, shift, flags);
  return cudaGetLastError();
}

cudaError_t launch_oct_index(const uint32_t* flags, const uint32_t* offs, long long n, uint32_t* out, cudaStream_t st) {
  k_oct_index<<<grid_of(n), kOctThreads, 0, st>>>(flags, offs, n, out);
  return cudaGetLastError();
}

cudaError_t launch_oct_fold(const unsigned long long* ck, const uint32_t* cv, long long c, const uint32_t* starts, long long m,
                            const OctArgs& a, const unsigned long long* lk, float* llo, uint32_t* lrgb, long long nleaves,
                            unsigned long long* nk, float* nlo, uint32_t* nrgb, uint32_t* new_flag, cudaStream_t st) {
  if (m <= 0) return cudaSuccess;
  k_oct_fold<<<grid_of(m), kOctThreads, 0, st>>>(ck, cv, c, starts, m, a, lk, llo, lrgb, nleaves, nk, nlo, nrgb, new_flag);
  return cudaGetLastError();
}

cudaError_t launch_oct_merge(const unsigned long long* lk, const float* llo, const uint32_t* lrgb, long long nleaves,
                             const unsigned long long* nk, const float* nlo, const uint32_t* nrgb, const uint32_t* new_flag,
                             const uint32_t* offs, long long m, unsigned long long* newk, long long nnew, unsigned long long* ok,
                             float* olo, uint32_t* orgb, cudaStream_t st) {
  if (m > 0) k_oct_gather_new<<<grid_of(m), kOctThreads, 0, st>>>(nk, new_flag, offs, m, newk);
  if (nleaves > 0) k_oct_merge_old<<<grid_of(nleaves), kOctThreads, 0, st>>>(lk, llo, lrgb, nleaves, newk, nnew, ok, olo, orgb);
  if (m > 0) k_oct_merge_new<<<grid_of(m), kOctThreads, 0, st>>>(lk, nleaves, nk, nlo, nrgb, new_flag, offs, m, ok, olo, orgb);
  return cudaGetLastError();
}

cudaError_t launch_oct_leaf_level(OctLevel l, cudaStream_t st) {
  k_oct_leaf_level<<<grid_of(l.n), kOctThreads, 0, st>>>(l);
  return cudaGetLastError();
}

cudaError_t launch_oct_reduce(OctLevel p, OctLevel c, cudaStream_t st) {
  k_oct_reduce<<<grid_of(p.n), kOctThreads, 0, st>>>(p, c);
  return cudaGetLastError();
}

cudaError_t launch_oct_offsets(OctLevel p, OctLevel c, cudaStream_t st) {
  k_oct_offsets<<<grid_of(p.n), kOctThreads, 0, st>>>(p, c);
  return cudaGetLastError();
}

cudaError_t launch_oct_records(OctLevel l, uint8_t* out, cudaStream_t st) {
  k_oct_records<<<grid_of(l.n), kOctThreads, 0, st>>>(l, reinterpret_cast<uint2*>(out));
  return cudaGetLastError();
}

}  // namespace rb200
