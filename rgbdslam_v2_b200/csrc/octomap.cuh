// octomap.cuh -- the colour OctoMap kernels (octomap.cu) as the host side (api_octomap.cu) launches them.
#pragma once
#include "kernels.h"

namespace rb200 {

// A sort entry: key = morton(cell) << 16 | scan << 2 | kind, value = the colour word of a kind-2 entry.  Kinds sort in the
// order the reference applies them inside a scan: 0 free cell, 1 occupied cell, 2 colour of a point.  morton interleaves the
// 16-bit keys x, y, z with x lowest, so ascending order is the depth-first pre-order of the tree with children 0..7.
constexpr int kOctMaxScans = 1 << 14;  // scans (nodes) one batch may hold
constexpr uint32_t kOctWhite = 0xffffffu;  // colour (255, 255, 255): "unset"

struct OctArgs {
  double res, rf;        // resolution and 1 / resolution
  double max_range;      // < 0: none
  float hit, miss;       // logodds(prob_hit), logodds(prob_miss)
  float cmin, cmax;      // logodds of the clamping thresholds
};

// Every call below runs on stream st.  Scans count into *d_total (long long, device) where one is given.
// entries per 1024-point block of the table (blocks: (node, first point)) into d_counts, and per point into
// d_pcount[block * 1024 + point - first point]
cudaError_t launch_oct_count(const MapNode* d_nodes, const int2* d_blocks, int nblocks, const OctArgs& a, int* d_counts,
                             int* d_pcount, cudaStream_t st);
// the entries of blocks [b0, b1), whose output offsets (map scan of their counts) are offs[b - b0]; node index - node0 is the scan
cudaError_t launch_oct_emit(const MapNode* d_nodes, const int2* d_blocks, int b0, int b1, int node0, const long long* d_offs,
                            const int* d_pcount, const OctArgs& a, unsigned long long* keys, uint32_t* vals, cudaStream_t st);
// exclusive scan of n flags into offs (uint32) and the total into *d_total; tile_sums / tile_offs: scratch of
// scan_tiles(n) ints / scan_tiles(n) + 1 long longs
int oct_scan_tiles(long long n);
cudaError_t launch_oct_scan(const uint32_t* flags, long long n, uint32_t* offs, int* tile_sums, long long* tile_offs, cudaStream_t st);
// OR and AND of n keys into d_bits[0], d_bits[1] (set to 0 / ~0 first by the call)
cudaError_t launch_oct_key_bits(const unsigned long long* keys, long long n, unsigned long long* d_bits, cudaStream_t st);
// one stable 8-bit LSD pass on the byte at `shift`; hist: 256 * scan_tiles(n) uint32, hist_offs the same
cudaError_t launch_oct_radix_pass(const unsigned long long* kin, const uint32_t* vin, long long n, int shift, uint32_t* hist,
                                  uint32_t* hist_offs, int* tile_sums, long long* tile_offs, unsigned long long* kout,
                                  uint32_t* vout, cudaStream_t st);
// flags: keep the last free / occupied entry of each (cell, scan) and every colour entry
cudaError_t launch_oct_flag_keep(const unsigned long long* keys, long long n, uint32_t* flags, cudaStream_t st);
cudaError_t launch_oct_compact(const unsigned long long* kin, const uint32_t* vin, const uint32_t* flags, const uint32_t* offs,
                               long long n, unsigned long long* kout, uint32_t* vout, cudaStream_t st);
// flags: key >> shift differs from the previous key's
cudaError_t launch_oct_flag_heads(const unsigned long long* keys, long long n, int shift, uint32_t* flags, cudaStream_t st);
// out[offs[i]] = i where flags[i]
cudaError_t launch_oct_index(const uint32_t* flags, const uint32_t* offs, long long n, uint32_t* out, cudaStream_t st);
// one thread per cell segment [starts[j], starts[j + 1]) of the compacted entries (m segments, c entries): the scans' updates
// and colours of that cell in order, onto the leaf (updated in place) or a new leaf (nk / nlo / nrgb, new_flag[j])
cudaError_t launch_oct_fold(const unsigned long long* ck, const uint32_t* cv, long long c, const uint32_t* starts, long long m,
                            const OctArgs& a, const unsigned long long* lk, float* llo, uint32_t* lrgb, long long nleaves,
                            unsigned long long* nk, float* nlo, uint32_t* nrgb, uint32_t* new_flag, cudaStream_t st);
// the leaves (nleaves, sorted) and the new leaves (nnew, sorted, disjoint) merged into the output arrays; the new leaves are
// the entries j of nk / nlo / nrgb with new_flag[j], at position offs[j] among them
cudaError_t launch_oct_merge(const unsigned long long* lk, const float* llo, const uint32_t* lrgb, long long nleaves,
                             const unsigned long long* nk, const float* nlo, const uint32_t* nrgb, const uint32_t* new_flag,
                             const uint32_t* offs, long long m, unsigned long long* newk, long long nnew, unsigned long long* ok,
                             float* olo, uint32_t* orgb, cudaStream_t st);

// One level of the tree for the writer: nodes in pre-order, each with its children's range in the level below.
struct OctLevel {
  unsigned long long* key;  // morton prefix (level d: morton >> 3 (16 - d))
  float* lo;
  uint32_t* rgb;
  uint32_t* first;          // first child in the level below (inner levels)
  uint8_t* mask;            // child-existence bits (0 for leaves)
  unsigned long long* size; // records in the subtree
  unsigned long long* off;  // record index of the node
  long long n;
};
// level p from level c (its children): first[] must already hold the children's starts (launch_oct_index of the heads)
cudaError_t launch_oct_reduce(OctLevel p, OctLevel c, cudaStream_t st);
// offsets of level c's nodes from their parents' (level p)
cudaError_t launch_oct_offsets(OctLevel p, OctLevel c, cudaStream_t st);
// the 8-byte records of one level: float log-odds, r, g, b, child bits
cudaError_t launch_oct_records(OctLevel l, uint8_t* out, cudaStream_t st);
cudaError_t launch_oct_leaf_level(OctLevel l, cudaStream_t st);  // size 1, mask 0

// ---- the occupancy filter (ColorOctomapServer::occupancyFilter, DESIGN.md 4.15) --------------------------------------------
struct OcfArgs {
  double res, rf;      // resolution and 1 / resolution
  double threshold;    // occupancy_filter_threshold
  const unsigned long long* lk;  // the map's leaves (Morton keys, sorted) and their occupancy 1 - 1 / (1 + exp(lo)), libm's
  const double* occ;
  long long nleaves;
};
// Where the kept points of one node of the chunk go: its planes at slab point dst (dst < 0: the node keeps its cloud), the
// first of its offsets (map scan of the block counts) and its kept count.
struct OcfOut {
  long long dst, first;
  long long count;
};
// The keep flag of every point of the blocks (node, first point), flags[block * 1024 + point - first point]; per block the
// kept count; keep0[node] = the flag of the node's point 0.  sensor7: per node qx qy qz qw ox oy oz.
cudaError_t launch_ocf_flags(const MapNode* d_nodes, const int2* d_blocks, int nblocks, const float* d_sensor7, const OcfArgs& a,
                             uint8_t* d_flags, int* d_counts, uint8_t* d_keep0, cudaStream_t st);
// The kept points of the blocks, as stored, into the x / y / z / colour planes of their node at slab + 4 * out[node].dst floats.
cudaError_t launch_ocf_scatter(const MapNode* d_nodes, const int2* d_blocks, int nblocks, const uint8_t* d_flags, const long long* d_offs,
                               const OcfOut* d_out, float* slab, cudaStream_t st);

}  // namespace rb200
