// api_octomap.cu -- C ABI of the colour OctoMap (include/rgbdslam_b200/octomap.h), host orchestration of octomap.cu:
//   insert: count every node's entries once, then per batch of whole nodes (bounded by kOctBatchEntries) emit -> sort ->
//           one update per (cell, scan) -> fold per cell -> merge the new leaves into the sorted leaf array
//   write / stats: the inner levels from the leaves, bottom up; pre-order offsets top down; the records
//   filter_clouds: the leaves' occupancy from the host's libm (cached until the map changes), then per chunk of whole nodes
//           keep flags -> block scan -> the kept points of the nodes that lose some into one new slab
#include <algorithm>
#include <cmath>
#include <cstdio>
#include <cstring>
#include <string>
#include <unordered_map>
#include <vector>

#include "../../include/rgbdslam_b200/octomap.h"
#include "octomap.cuh"
#include "state.h"

namespace rb200 {

constexpr long long kOctBatchEntries = 1ll << 26;  // sort entries per batch: about 1.6 GB of work buffers (24 bytes each)
constexpr int kOctDepth = 16;
constexpr long long kOcfChunkPoints = 1ll << 25;  // points one filter chunk flags and scatters: 1 byte of flags each

struct OctoMap {
  static constexpr uint32_t kMagic = 0x4f43544du;  // 'OCTM'
  uint32_t magic = kMagic;
  rgbdslam_b200_octomap_params p;
  OctArgs a;
  long long nleaves = 0;
  int cur = 0;
  DevBuf lk[2], llo[2], lrgb[2];  // the leaves, sorted by Morton code: ping-pong for the merge
  DevBuf nodes, blocks, counts, pcount, offs, key[2], val[2], flags, scan, tsum, toffs, bits, starts, nk, nlo, nrgb, newk;
  // the filter: per leaf its occupancy (valid while occ_ok; insert and clear reset it), and the work buffers
  DevBuf occ, sensor, pflags, keep0, outs;
  bool occ_ok = false;
  // the writer's levels 0..15 (level 16 is the leaves): key, lo, rgb, first, mask, size, off
  DevBuf lvl[kOctDepth + 1][7];
  void release() {
    for (int b = 0; b < 2; b++) {
      lk[b].release();
      llo[b].release();
      lrgb[b].release();
      key[b].release();
      val[b].release();
    }
    DevBuf* all[] = {&nodes, &blocks, &counts, &pcount, &offs, &flags, &scan, &tsum, &toffs, &bits, &starts, &nk, &nlo, &nrgb, &newk,
                     &occ, &sensor, &pflags, &keep0, &outs};
    for (DevBuf* b : all) b->release();
    for (auto& l : lvl)
      for (DevBuf& b : l) b.release();
    occ_ok = false;
  }
};

static OctoMap* get_octomap(uint64_t h) {
  OctoMap* m = (OctoMap*)(uintptr_t)h;
  if (!m || m->magic != OctoMap::kMagic) {
    set_error("invalid octomap handle");
    return nullptr;
  }
  return m;
}

static float logodds(double p) { return (float)std::log(p / (1 - p)); }  // octomap::logodds

static bool prob_ok(double p) { return p > 0.0 && p < 1.0; }

// Exclusive scan of n flags into m.scan; returns the total through *total (host).
static int oct_scan(OctoMap& m, const uint32_t* flags, long long n, uint32_t* offs, long long* total, cudaStream_t st) {
  const int nt = oct_scan_tiles(n);
  int rc;
  if ((rc = m.tsum.ensure(4 * (size_t)nt)) || (rc = m.toffs.ensure(8 * ((size_t)nt + 1)))) return rc;
  RB200_CUDA(launch_oct_scan(flags, n, offs, (int*)m.tsum.ptr, (long long*)m.toffs.ptr, st));
  RB200_CUDA(cudaMemcpyAsync(total, (long long*)m.toffs.ptr + nt, 8, cudaMemcpyDeviceToHost, st));
  RB200_CUDA(cudaStreamSynchronize(st));
  g_state.launches += 3;
  return 0;
}

// One batch: nodes [k0, k1) of the table, their blocks [b0, b1), E entries in all.
static int oct_batch(OctoMap& m, int k0, int b0, int b1, long long E) {
  State& s = g_state;
  cudaStream_t st = s.stream;
  int rc;
  const size_t e = (size_t)std::max(E, 1ll);
  const int nt = oct_scan_tiles(E);
  const size_t hist = 256 * (size_t)nt;
  for (int b = 0; b < 2; b++)
    if ((rc = m.key[b].ensure(8 * e)) || (rc = m.val[b].ensure(4 * e))) return rc;
  if ((rc = m.flags.ensure(4 * std::max(e, hist))) || (rc = m.scan.ensure(4 * std::max(e, hist))) ||
      (rc = m.offs.ensure(8 * ((size_t)(b1 - b0) + 1))) || (rc = m.bits.ensure(16)) || (rc = m.starts.ensure(4 * e)) ||
      (rc = m.nk.ensure(8 * e)) || (rc = m.nlo.ensure(4 * e)) || (rc = m.nrgb.ensure(4 * e)))
    return rc;
  unsigned long long* key[2] = {(unsigned long long*)m.key[0].ptr, (unsigned long long*)m.key[1].ptr};
  uint32_t* val[2] = {(uint32_t*)m.val[0].ptr, (uint32_t*)m.val[1].ptr};
  uint32_t* flags = (uint32_t*)m.flags.ptr;
  uint32_t* scan = (uint32_t*)m.scan.ptr;
  RB200_CUDA(launch_map_scan((const int*)m.counts.ptr + b0, b1 - b0, (long long*)m.offs.ptr, st));
  RB200_CUDA(launch_oct_emit((const MapNode*)m.nodes.ptr, (const int2*)m.blocks.ptr, b0, b1, k0, (const long long*)m.offs.ptr,
                             (const int*)m.pcount.ptr, m.a,
                             key[0], val[0], st));
  RB200_CUDA(launch_oct_key_bits(key[0], E, (unsigned long long*)m.bits.ptr, st));
  unsigned long long bits[2];
  RB200_CUDA(cudaMemcpyAsync(bits, m.bits.ptr, 16, cudaMemcpyDeviceToHost, st));
  RB200_CUDA(cudaStreamSynchronize(st));
  s.launches += 3;
  if ((rc = m.tsum.ensure(4 * (size_t)oct_scan_tiles((long long)hist))) ||
      (rc = m.toffs.ensure(8 * ((size_t)oct_scan_tiles((long long)hist) + 1))))
    return rc;
  // the sort: one stable pass per key byte that is not the same in every entry
  int c = 0;
  const unsigned long long vary = bits[0] ^ bits[1];
  for (int shift = 0; shift < 64; shift += 8) {
    if (((vary >> shift) & 0xff) == 0) continue;
    RB200_CUDA(launch_oct_radix_pass(key[c], val[c], E, shift, flags, scan, (int*)m.tsum.ptr, (long long*)m.toffs.ptr, key[1 - c],
                                     val[1 - c], st));
    s.launches += 5;
    c = 1 - c;
  }
  // one free-or-occupied entry per (cell, scan), every colour entry
  long long C = 0, M = 0, K = 0;
  RB200_CUDA(launch_oct_flag_keep(key[c], E, flags, st));
  if ((rc = oct_scan(m, flags, E, scan, &C, st))) return rc;
  RB200_CUDA(launch_oct_compact(key[c], val[c], flags, scan, E, key[1 - c], val[1 - c], st));
  s.launches += 2;
  c = 1 - c;
  // cell segments
  RB200_CUDA(launch_oct_flag_heads(key[c], C, 16, flags, st));
  if ((rc = oct_scan(m, flags, C, scan, &M, st))) return rc;
  RB200_CUDA(launch_oct_index(flags, scan, C, (uint32_t*)m.starts.ptr, st));
  const int L = m.cur;
  RB200_CUDA(launch_oct_fold(key[c], val[c], C, (const uint32_t*)m.starts.ptr, M, m.a, (const unsigned long long*)m.lk[L].ptr,
                             (float*)m.llo[L].ptr, (uint32_t*)m.lrgb[L].ptr, m.nleaves, (unsigned long long*)m.nk.ptr, (float*)m.nlo.ptr,
                             (uint32_t*)m.nrgb.ptr, flags, st));
  s.launches += 3;
  if ((rc = oct_scan(m, flags, M, scan, &K, st))) return rc;
  if (K == 0) return 0;
  const size_t n2 = (size_t)(m.nleaves + K);
  if ((rc = m.lk[1 - L].ensure(8 * n2)) || (rc = m.llo[1 - L].ensure(4 * n2)) || (rc = m.lrgb[1 - L].ensure(4 * n2)) ||
      (rc = m.newk.ensure(8 * (size_t)K)))
    return rc;
  RB200_CUDA(launch_oct_merge((const unsigned long long*)m.lk[L].ptr, (const float*)m.llo[L].ptr, (const uint32_t*)m.lrgb[L].ptr,
                              m.nleaves, (const unsigned long long*)m.nk.ptr, (const float*)m.nlo.ptr, (const uint32_t*)m.nrgb.ptr, flags,
                              scan, M, (unsigned long long*)m.newk.ptr, K, (unsigned long long*)m.lk[1 - L].ptr,
                              (float*)m.llo[1 - L].ptr, (uint32_t*)m.lrgb[1 - L].ptr, st));
  RB200_CUDA(cudaStreamSynchronize(st));
  s.launches += 3;
  m.cur = 1 - L;
  m.nleaves += K;
  return 0;
}

static int oct_insert(OctoMap& m, const std::vector<MapNode>& table) {
  State& s = g_state;
  cudaStream_t st = s.stream;
  const int n = (int)table.size();
  std::vector<int> first_block;
  const std::vector<int2> blocks = map_blocks(table, &first_block);
  const int nb = (int)blocks.size();
  if (nb == 0) return 0;
  int rc;
  if ((rc = m.nodes.ensure(sizeof(MapNode) * n)) || (rc = m.blocks.ensure(sizeof(int2) * nb)) || (rc = m.counts.ensure(4 * (size_t)nb)) ||
      (rc = m.pcount.ensure(4 * (size_t)nb * kMapBlockPoints)))
    return rc;
  RB200_CUDA(cudaMemcpyAsync(m.nodes.ptr, table.data(), sizeof(MapNode) * n, cudaMemcpyHostToDevice, st));
  RB200_CUDA(cudaMemcpyAsync(m.blocks.ptr, blocks.data(), sizeof(int2) * nb, cudaMemcpyHostToDevice, st));
  RB200_CUDA(launch_oct_count((const MapNode*)m.nodes.ptr, (const int2*)m.blocks.ptr, nb, m.a, (int*)m.counts.ptr, (int*)m.pcount.ptr,
                              st));
  std::vector<int> counts(nb);
  RB200_CUDA(cudaMemcpyAsync(counts.data(), m.counts.ptr, 4 * (size_t)nb, cudaMemcpyDeviceToHost, st));
  RB200_CUDA(cudaStreamSynchronize(st));
  s.launches += 1;
  const long long limit = chunk_limit(kOctBatchEntries, "RB200_OCT_BATCH_ENTRIES");
  // batches of whole nodes, at least one, in order
  for (int k0 = 0; k0 < n;) {
    long long E = 0;
    int k1 = k0;
    do {
      for (int b = first_block[k1]; b < first_block[k1 + 1]; b++) E += counts[b];
      k1++;
      long long next = 0;
      if (k1 < n)
        for (int b = first_block[k1]; b < first_block[k1 + 1]; b++) next += counts[b];
      if (k1 >= n || k1 - k0 >= kOctMaxScans || E + next > limit) break;
    } while (true);
    if (E > 0xffffffffll) {
      set_error("octomap_insert: one node has more than 2^32 ray cells");
      return RGBDSLAM_B200_ERR_ARG;
    }
    if (E > 0 && (rc = oct_batch(m, k0, first_block[k0], first_block[k1], E))) return rc;
    k0 = k1;
  }
  return 0;
}

// The occupancy of every leaf, OcTreeNode::getOccupancy = 1 - 1 / (1 + exp(lo)), computed here with the host's libm so that
// the filter's decisions are glibc's (CUDA's double exp is only faithful to within 1 ulp).  Each distinct log-odds value is
// evaluated once: the clamped float sums of a few increments take few values.
static int oct_occupancy(OctoMap& m) {
  if (m.occ_ok || m.nleaves == 0) return 0;
  cudaStream_t st = g_state.stream;
  const size_t n = (size_t)m.nleaves;
  std::vector<uint32_t> lo(n);
  RB200_CUDA(cudaMemcpyAsync(lo.data(), m.llo[m.cur].ptr, 4 * n, cudaMemcpyDeviceToHost, st));
  RB200_CUDA(cudaStreamSynchronize(st));
  std::vector<double> occ(n);
  std::unordered_map<uint32_t, double> seen;
  for (size_t i = 0; i < n; i++) {
    auto it = seen.find(lo[i]);
    if (it == seen.end()) {
      float l;
      std::memcpy(&l, &lo[i], 4);
      it = seen.emplace(lo[i], 1.0 - 1.0 / (1.0 + std::exp((double)l))).first;
    }
    occ[i] = it->second;
  }
  int rc;
  if ((rc = m.occ.ensure(8 * n))) return rc;
  RB200_CUDA(cudaMemcpyAsync(m.occ.ptr, occ.data(), 8 * n, cudaMemcpyHostToDevice, st));
  RB200_CUDA(cudaStreamSynchronize(st));
  m.occ_ok = true;
  return 0;
}

// Filters nodes [k0, k1) of the call into one new slab.  Appends a CloudResult per node that loses
// points and writes n_points[k].
static int ocf_chunk(OctoMap& m, const std::vector<NodeDev*>& nds, const float* sensor7, int k0, int k1, const OcfArgs& a,
                     std::vector<CloudResult>& results, std::vector<NodeSlab*>& slabs, int32_t* n_points) {
  State& s = g_state;
  cudaStream_t st = s.stream;
  const int nn = k1 - k0;
  std::vector<MapNode> nodes(nn);
  for (int k = 0; k < nn; k++) nodes[k] = map_node(nds[k0 + k], nullptr);
  std::vector<int> first_block;
  const std::vector<int2> blocks = map_blocks(nodes, &first_block);
  const int nb = (int)blocks.size();
  int rc;
  if ((rc = m.nodes.ensure(sizeof(MapNode) * nn)) || (rc = m.blocks.ensure(sizeof(int2) * std::max(nb, 1))) ||
      (rc = m.counts.ensure(4 * (size_t)std::max(nb, 1))) || (rc = m.offs.ensure(8 * ((size_t)nb + 1))) ||
      (rc = m.sensor.ensure(28 * (size_t)nn)) || (rc = m.pflags.ensure((size_t)kMapBlockPoints * std::max(nb, 1))) ||
      (rc = m.keep0.ensure((size_t)nn)) || (rc = m.outs.ensure(sizeof(OcfOut) * nn)))
    return rc;
  RB200_CUDA(cudaMemcpyAsync(m.nodes.ptr, nodes.data(), sizeof(MapNode) * nn, cudaMemcpyHostToDevice, st));
  RB200_CUDA(cudaMemcpyAsync(m.sensor.ptr, sensor7 + 7 * (size_t)k0, 28 * (size_t)nn, cudaMemcpyHostToDevice, st));
  if (nb > 0) RB200_CUDA(cudaMemcpyAsync(m.blocks.ptr, blocks.data(), sizeof(int2) * nb, cudaMemcpyHostToDevice, st));
  RB200_CUDA(cudaMemsetAsync(m.keep0.ptr, 0, (size_t)nn, st));
  RB200_CUDA(launch_ocf_flags((const MapNode*)m.nodes.ptr, (const int2*)m.blocks.ptr, nb, (const float*)m.sensor.ptr, a,
                              (uint8_t*)m.pflags.ptr, (int*)m.counts.ptr, (uint8_t*)m.keep0.ptr, st));
  RB200_CUDA(launch_map_scan((const int*)m.counts.ptr, nb, (long long*)m.offs.ptr, st));
  std::vector<long long> offs(nb + 1);
  std::vector<uint8_t> keep0(nn);
  RB200_CUDA(cudaMemcpyAsync(offs.data(), m.offs.ptr, 8 * ((size_t)nb + 1), cudaMemcpyDeviceToHost, st));
  RB200_CUDA(cudaMemcpyAsync(keep0.data(), m.keep0.ptr, (size_t)nn, cudaMemcpyDeviceToHost, st));
  RB200_CUDA(cudaStreamSynchronize(st));
  s.launches += (nb > 0) + 1;
  // the nodes that lose points get their planes in the new slab, back to back; the others keep their clouds
  std::vector<OcfOut> out(nn);
  long long dst = 0;
  for (int k = 0; k < nn; k++) {
    const long long first = offs[first_block[k]], count = offs[first_block[k + 1]] - first;
    const bool changed = count < (long long)nodes[k].cw * nodes[k].ch;
    out[k] = OcfOut{changed ? dst : -1, first, count};
    if (changed) dst += count;
    n_points[k0 + k] = (int32_t)count;
  }
  if (std::none_of(out.begin(), out.end(), [](const OcfOut& o) { return o.dst >= 0; })) return 0;
  NodeSlab* slab = new_slab(dst, "cudaMalloc(occupancy-filtered clouds)", slabs);
  if (!slab) return RGBDSLAM_B200_ERR_CUDA;
  RB200_CUDA(cudaMemcpyAsync(m.outs.ptr, out.data(), sizeof(OcfOut) * nn, cudaMemcpyHostToDevice, st));
  RB200_CUDA(launch_ocf_scatter((const MapNode*)m.nodes.ptr, (const int2*)m.blocks.ptr, nb, (const uint8_t*)m.pflags.ptr,
                                (const long long*)m.offs.ptr, (const OcfOut*)m.outs.ptr, (float*)slab->base, st));
  RB200_CUDA(cudaStreamSynchronize(st));  // the work buffers are the next chunk's
  s.launches += nb > 0;
  for (int k = 0; k < nn; k++) {
    if (out[k].dst < 0) continue;
    NodeDev* nd = nds[k0 + k];
    CloudResult r{nd, slab_cloud(nd->pc, slab, out[k].dst, out[k].count)};
    r.pc.w = (int32_t)out[k].count;
    r.pc.h = 1;
    r.pc.unorganised = true;
    r.pc.point0_one = (nd->pc.step > 0 || nd->pc.point0_one) && keep0[k];  // the kept point 0 stays point 0
    results.push_back(r);
  }
  return 0;
}

// The levels of the tree in m.lvl (level 16: the leaves); returns the node count (0 for an empty map) through *count.
static int oct_levels(OctoMap& m, OctLevel* lv, long long* count) {
  cudaStream_t st = g_state.stream;
  *count = 0;
  if (m.nleaves == 0) return 0;
  int rc;
  auto alloc = [&](int d, long long n, bool leaves) -> int {
    DevBuf* b = m.lvl[d];
    const size_t k = (size_t)std::max(n, 1ll);
    if (!leaves && ((rc = b[0].ensure(8 * k)) || (rc = b[1].ensure(4 * k)) || (rc = b[2].ensure(4 * k)))) return rc;
    if ((rc = b[3].ensure(4 * k)) || (rc = b[4].ensure(k)) || (rc = b[5].ensure(8 * k)) || (rc = b[6].ensure(8 * k))) return rc;
    OctLevel& l = lv[d];
    l.key = leaves ? (unsigned long long*)m.lk[m.cur].ptr : (unsigned long long*)b[0].ptr;
    l.lo = leaves ? (float*)m.llo[m.cur].ptr : (float*)b[1].ptr;
    l.rgb = leaves ? (uint32_t*)m.lrgb[m.cur].ptr : (uint32_t*)b[2].ptr;
    l.first = (uint32_t*)b[3].ptr;
    l.mask = (uint8_t*)b[4].ptr;
    l.size = (unsigned long long*)b[5].ptr;
    l.off = (unsigned long long*)b[6].ptr;
    l.n = n;
    return 0;
  };
  if ((rc = alloc(kOctDepth, m.nleaves, true))) return rc;
  RB200_CUDA(launch_oct_leaf_level(lv[kOctDepth], st));
  const size_t e = (size_t)m.nleaves;
  if ((rc = m.flags.ensure(4 * e)) || (rc = m.scan.ensure(4 * e))) return rc;
  long long total = m.nleaves;
  for (int d = kOctDepth - 1; d >= 0; d--) {
    const OctLevel& c = lv[d + 1];
    long long np = 0;
    RB200_CUDA(launch_oct_flag_heads(c.key, c.n, 3, (uint32_t*)m.flags.ptr, st));
    if ((rc = oct_scan(m, (const uint32_t*)m.flags.ptr, c.n, (uint32_t*)m.scan.ptr, &np, st))) return rc;
    if ((rc = alloc(d, np, false))) return rc;
    RB200_CUDA(launch_oct_index((const uint32_t*)m.flags.ptr, (const uint32_t*)m.scan.ptr, c.n, lv[d].first, st));
    RB200_CUDA(launch_oct_reduce(lv[d], c, st));
    g_state.launches += 3;
    total += np;
  }
  RB200_CUDA(cudaMemsetAsync(lv[0].off, 0, 8, st));
  for (int d = 0; d < kOctDepth; d++) RB200_CUDA(launch_oct_offsets(lv[d], lv[d + 1], st));
  g_state.launches += kOctDepth + 1;
  *count = total;
  return 0;
}

static std::string oct_header(const OctoMap& m, long long nodes) {
  char buf[256];
  std::snprintf(buf, sizeof(buf),
                "# Octomap OcTree file\n# (feel free to add / change comments, but leave the first line as it is!)\n#\n"
                "id ColorOcTree\nsize %lld\nres %g\ndata\n",
                nodes, m.p.resolution);
  return buf;
}

}  // namespace rb200

using namespace rb200;

extern "C" {

void rgbdslam_b200_octomap_default_params(rgbdslam_b200_octomap_params* p) {
  if (!p) return;
  p->resolution = 0.05;
  p->prob_hit = 0.9;
  p->prob_miss = 0.4;
  p->clamping_min = 0.001;
  p->clamping_max = 0.999;
}

int rgbdslam_b200_octomap_create(const rgbdslam_b200_octomap_params* p, uint64_t* map) {
  RB200_ENTER_INITED();
  if (!p || !map || !(p->resolution > 0.0) || !std::isfinite(p->resolution) || !prob_ok(p->prob_hit) || !prob_ok(p->prob_miss) ||
      !prob_ok(p->clamping_min) || !prob_ok(p->clamping_max) || !(p->clamping_min <= p->clamping_max)) {
    set_error("octomap_create: resolution > 0, probabilities in (0, 1) and clamping_min <= clamping_max are needed");
    return RGBDSLAM_B200_ERR_ARG;
  }
  OctoMap* m = new OctoMap();
  m->p = *p;
  m->a.res = p->resolution;
  m->a.rf = 1.0 / p->resolution;
  m->a.max_range = -1.0;
  m->a.hit = logodds(p->prob_hit);
  m->a.miss = logodds(p->prob_miss);
  m->a.cmin = logodds(p->clamping_min);
  m->a.cmax = logodds(p->clamping_max);
  *map = (uint64_t)(uintptr_t)m;
  return 0;
}

int rgbdslam_b200_octomap_insert(uint64_t map, int n, const uint64_t* nodes, const float* transforms12, double max_range) {
  RB200_ENTER_INITED();
  OctoMap* m = get_octomap(map);
  if (!m) return RGBDSLAM_B200_ERR_ARG;
  if (n < 0 || (n > 0 && (!nodes || !transforms12)) || std::isnan(max_range)) {
    set_error("octomap_insert: n >= 0, non-null nodes and transforms and a max_range that is not NaN are needed");
    return RGBDSLAM_B200_ERR_ARG;
  }
  std::vector<NodeDev*> nds;
  int rc;
  if ((rc = check_finite("octomap_insert", "transform", n, 12, transforms12)) ||
      (rc = stored_cloud_nodes("octomap_insert", n, nodes, false, &nds)))
    return rc;
  std::vector<MapNode> table(n);
  for (int k = 0; k < n; k++) table[k] = map_node(nds[k], transforms12 + (size_t)k * 12);
  m->a.max_range = max_range;
  m->occ_ok = false;
  return oct_insert(*m, table);
}

int rgbdslam_b200_octomap_filter_clouds(uint64_t map, int n, const uint64_t* nodes, const float* sensor7, double occupancy_threshold,
                                        int32_t* n_points) {
  RB200_ENTER_INITED();
  OctoMap* m = get_octomap(map);
  if (!m) return RGBDSLAM_B200_ERR_ARG;
  if (n < 0 || (n > 0 && (!nodes || !sensor7)) || std::isnan(occupancy_threshold)) {
    set_error("octomap_filter_clouds: n >= 0, non-null nodes and sensor poses and a threshold that is not NaN are needed");
    return RGBDSLAM_B200_ERR_ARG;
  }
  std::vector<NodeDev*> nds;
  int rc;
  if ((rc = check_finite("octomap_filter_clouds", "sensor pose", n, 7, sensor7)) ||
      (rc = stored_cloud_nodes("octomap_filter_clouds", n, nodes, true, &nds)))
    return rc;
  if (n == 0) return 0;
  if ((rc = oct_occupancy(*m))) return rc;
  const OcfArgs a{m->p.resolution, m->a.rf, occupancy_threshold, (const unsigned long long*)m->lk[m->cur].ptr, (const double*)m->occ.ptr,
                  m->nleaves};
  std::vector<int32_t> counts(n);
  rc = rebuild_clouds(nds, chunk_limit(kOcfChunkPoints, "RB200_OCF_CHUNK_POINTS"),
                      [&](int k0, int k1, long long, auto& results, auto& slabs) {
                        return ocf_chunk(*m, nds, sensor7, k0, k1, a, results, slabs, counts.data());
                      });
  if (rc) return rc;
  if (n_points) std::copy(counts.begin(), counts.end(), n_points);
  return 0;
}

int rgbdslam_b200_octomap_write(uint64_t map, void* out, int64_t capacity, int64_t* n_bytes) {
  RB200_ENTER_INITED();
  OctoMap* m = get_octomap(map);
  if (!m) return RGBDSLAM_B200_ERR_ARG;
  if (!n_bytes || (out && capacity < 0)) {
    set_error("octomap_write: n_bytes must be non-null and capacity >= 0");
    return RGBDSLAM_B200_ERR_ARG;
  }
  OctLevel lv[kOctDepth + 1];
  long long count = 0;
  int rc;
  if ((rc = oct_levels(*m, lv, &count))) return rc;
  const std::string head = oct_header(*m, count);
  const long long total = (long long)head.size() + 8 * count;
  *n_bytes = total;
  if (!out) return 0;
  if (capacity < total) {
    set_error("octomap_write: capacity " + std::to_string(capacity) + " < " + std::to_string(total) + " bytes");
    return RGBDSLAM_B200_ERR_ARG;
  }
  std::memcpy(out, head.data(), head.size());
  if (count == 0) return 0;
  cudaStream_t st = g_state.stream;
  if ((rc = m->key[0].ensure(8 * (size_t)count))) return rc;  // the records, staged in the sort buffer
  for (int d = 0; d <= kOctDepth; d++) RB200_CUDA(launch_oct_records(lv[d], (uint8_t*)m->key[0].ptr, st));
  g_state.launches += kOctDepth + 1;
  RB200_CUDA(cudaMemcpyAsync((uint8_t*)out + head.size(), m->key[0].ptr, 8 * (size_t)count, cudaMemcpyDeviceToHost, st));
  RB200_CUDA(cudaStreamSynchronize(st));
  return 0;
}

int rgbdslam_b200_octomap_stats(uint64_t map, int64_t* nodes, int64_t* leaves) {
  RB200_ENTER_INITED();
  OctoMap* m = get_octomap(map);
  if (!m) return RGBDSLAM_B200_ERR_ARG;
  if (!nodes || !leaves) {
    set_error("octomap_stats: null output");
    return RGBDSLAM_B200_ERR_ARG;
  }
  OctLevel lv[kOctDepth + 1];
  long long count = 0;
  int rc;
  if ((rc = oct_levels(*m, lv, &count))) return rc;
  RB200_CUDA(cudaStreamSynchronize(g_state.stream));
  *nodes = count;
  *leaves = m->nleaves;
  return 0;
}

int rgbdslam_b200_octomap_clear(uint64_t map) {
  RB200_ENTER_INITED();
  OctoMap* m = get_octomap(map);
  if (!m) return RGBDSLAM_B200_ERR_ARG;
  RB200_CUDA(cudaStreamSynchronize(g_state.stream));
  m->release();  // the leaves and every work buffer: the reference resets to free memory (octomap_clear_after_save)
  m->nleaves = 0;
  m->cur = 0;
  return 0;
}

int rgbdslam_b200_node_clear_cloud(uint64_t node_handle) {
  RB200_ENTER_INITED();
  NodeDev* nd = get_node(node_handle);
  if (!nd) return RGBDSLAM_B200_ERR_ARG;
  RB200_CUDA(cudaStreamSynchronize(g_state.stream));
  release_slab(nd->pc.slab);
  nd->pc = NodeCloud();
  return 0;
}

int rgbdslam_b200_octomap_destroy(uint64_t map) {
  std::lock_guard<std::mutex> lk(g_state.mu);
  OctoMap* m = get_octomap(map);
  if (!m) return RGBDSLAM_B200_ERR_ARG;
  if (g_state.inited) {
    cudaSetDevice(g_state.device);
    cudaStreamSynchronize(g_state.stream);
  }
  m->release();
  m->magic = 0;
  delete m;
  return 0;
}

}  // extern "C"
