// hamming_tc.cu -- brute-force descriptor matching on the Hopper tensor cores (wgmma, sm_90a).
//
// Two kernels:
//  * tc_hamming_b1_kernel     -- bruteForceSearchORB (features.cpp:168-182) for all query rows of all pairs, exact, as a BINARY
//    GEMM: one wgmma .b1 .and.popc per 64 query rows and 128 train rows gives popcount(a & b) of the raw 256-bit descriptors,
//    and hd = pa + pb - 2 popcount(a & b).  Warp-specialised: a producer warp group claims work items and copies the
//    descriptor rows into shared memory (a ring of train-tile stages on mbarriers), four consumer warp groups issue the MMAs
//    and take the row arg-min independently of each other;
//  * tc_match256_kernel<1|2>  -- the float-descriptor matchers (bf16 RootSIFT scores / SiftGPU's u8 dot products): operand
//    tiles resident in HBM in the layout below, each staged by ONE cp.async.bulk completing on an mbarrier, one producer warp
//    and four consumer warp groups that run independently of each other (one group's epilogue overlaps another's MMAs).
// Both keep the accumulators in registers (64 per thread of an m64n128 MMA) and read their operand tiles in the canonical
// K-major no-swizzle ("interleave") shared-memory layout  tile[row_group][k_chunk][row_in_group 8][16 B]  (8 x 16 B core
// matrices): 16 k-chunks per 256-byte float-descriptor row, 2 per 32-byte ORB row.
#include <type_traits>

#include "kernels.h"

namespace rb200 {

// ---------------------------------------------------------------------------------------------
// PTX helpers
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count));
}
__device__ __forceinline__ void mbar_expect_tx(uint32_t bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint32_t bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity) {
  asm volatile(
      "{\n"
      ".reg .pred p;\n"
      "WAIT_LOOP:\n"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n"
      "@p bra WAIT_DONE;\n"
      "bra WAIT_LOOP;\n"
      "WAIT_DONE:\n"
      "}\n" ::"r"(bar),
      "r"(parity)
      : "memory");
}
__device__ __forceinline__ void bulk_g2s(uint32_t dst_smem, const void* src, uint32_t bytes, uint32_t bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(dst_smem),
               "l"(src), "r"(bytes), "r"(bar)
               : "memory");
}
__device__ __forceinline__ void fence_proxy_async_smem() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }
__device__ __forceinline__ void sts128(uint32_t addr, uint32_t a, uint32_t b, uint32_t c, uint32_t d) {
  asm volatile("st.shared.v4.b32 [%0], {%1, %2, %3, %4};" ::"r"(addr), "r"(a), "r"(b), "r"(c), "r"(d) : "memory");
}

// wgmma shared-memory matrix descriptor, K-major, no swizzle ("interleave"):
//   bits [0,14)  start address >> 4
//   bits [16,30) leading-dimension byte offset >> 4 = distance between the two 8 x 16 B core matrices of one K = 32 B step
//   bits [32,46) stride-dimension byte offset >> 4  = distance between consecutive 8-row groups
//   base offset 0, layout type 0 (interleave)
__device__ __forceinline__ uint64_t make_desc(uint32_t smem_addr, uint32_t lbo_bytes, uint32_t sbo_bytes) {
  return (uint64_t)((smem_addr >> 4) & 0x3FFFu) | ((uint64_t)(lbo_bytes >> 4) << 16) | ((uint64_t)(sbo_bytes >> 4) << 32);
}
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_wait_all() { asm volatile("wgmma.wait_group.sync.aligned 0;" ::: "memory"); }

// The 64 accumulator registers of an m64n128 wgmma.  Element j of thread t of the warp group holds
//   row 16 (t / 32) + (t % 32) / 4 + 8 ((j / 2) % 2),  column 8 (j / 4) + 2 (t % 4) + j % 2.
#define RB_WG_D                                                                                                          \
  "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, " \
  "%25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, "   \
  "%48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}"
#define RB_WG_OPS(C, d)                                                                                                  \
  C(d[0]), C(d[1]), C(d[2]), C(d[3]), C(d[4]), C(d[5]), C(d[6]), C(d[7]), C(d[8]), C(d[9]), C(d[10]), C(d[11]), C(d[12]),  \
      C(d[13]), C(d[14]), C(d[15]), C(d[16]), C(d[17]), C(d[18]), C(d[19]), C(d[20]), C(d[21]), C(d[22]), C(d[23]),     \
      C(d[24]), C(d[25]), C(d[26]), C(d[27]), C(d[28]), C(d[29]), C(d[30]), C(d[31]), C(d[32]), C(d[33]), C(d[34]),     \
      C(d[35]), C(d[36]), C(d[37]), C(d[38]), C(d[39]), C(d[40]), C(d[41]), C(d[42]), C(d[43]), C(d[44]), C(d[45]),     \
      C(d[46]), C(d[47]), C(d[48]), C(d[49]), C(d[50]), C(d[51]), C(d[52]), C(d[53]), C(d[54]), C(d[55]), C(d[56]),     \
      C(d[57]), C(d[58]), C(d[59]), C(d[60]), C(d[61]), C(d[62]), C(d[63])

// D = popcount(A & B^T), b1 x b1 -> s32 (ORB), M64 N128 K256 (one 32-byte descriptor per row)
__device__ __forceinline__ void wgmma_b1(uint32_t (&d)[64], uint64_t da, uint64_t db) {
  asm volatile("wgmma.mma_async.sync.aligned.m64n128k256.s32.b1.b1.and.popc " RB_WG_D ", %64, %65, 0;\n"
               : RB_WG_OPS("+r", d)
               : "l"(da), "l"(db));
}
// u8 x u8 -> s32 (SiftGPU matcher), M64 N128 K32
__device__ __forceinline__ void wgmma_acc(uint32_t (&d)[64], uint64_t da, uint64_t db, uint32_t acc) {
  asm volatile(
      "{\n.reg .pred p;\nsetp.ne.b32 p, %66, 0;\n"
      "wgmma.mma_async.sync.aligned.m64n128k32.s32.u8.u8 " RB_WG_D ", %64, %65, p;\n}\n"
      : RB_WG_OPS("+r", d)
      : "l"(da), "l"(db), "r"(acc));
}
// bf16 x bf16 -> f32 (RootSIFT scores), M64 N128 K16 (32 bytes of K per instruction as well)
__device__ __forceinline__ void wgmma_acc(float (&d)[64], uint64_t da, uint64_t db, uint32_t acc) {
  asm volatile(
      "{\n.reg .pred p;\nsetp.ne.b32 p, %66, 0;\n"
      "wgmma.mma_async.sync.aligned.m64n128k16.f32.bf16.bf16 " RB_WG_D ", %64, %65, p, 1, 1, 0, 0;\n}\n"
      : RB_WG_OPS("+f", d)
      : "l"(da), "l"(db), "r"(acc));
}
#undef RB_WG_OPS
#undef RB_WG_D

constexpr int kNoBest = (int)0x80000000;
constexpr uint32_t kGroupStride = 2048;     // bytes per 8-row group of a 256-byte-row operand tile
constexpr uint32_t kWgRows = 64 * 256;      // 16 KiB: the 64 query rows of one warp group
constexpr uint32_t kA256 = 256 * 256;       // 64 KiB: the 256 query rows of a work item
constexpr uint32_t kB128 = 128 * 256;       // 32 KiB: one train tile

// ---------------------------------------------------------------------------------------------
// Float-descriptor matchers.  Warps 0-15: four consumer warp groups (64 query rows each), warp 16: bulk-copy producer.
// smem: A (the item's 256 query rows, 64 KiB) + a 3-deep ring of 32 KiB train tiles + barriers.
constexpr int kBSt = 3;
constexpr int kTc256ConsumerWarps = 16;
constexpr int kTc256Threads = (kTc256ConsumerWarps + 1) * 32;  // 544
constexpr uint32_t kTc256BarsOff = kA256 + kBSt * kB128;
constexpr uint32_t kTc256SmemBytes = kTc256BarsOff + 128;
static_assert(kTc256SmemBytes <= 232448, "tc_match256: shared memory over the 227 KiB per-CTA limit");
constexpr int kBarAFull = 0, kBarAEmpty = 1, kBarBFull = 2, kBarBEmpty = 2 + kBSt;  // 8 barriers

// top-4 of one query row, ordered by (score descending, column ascending)
struct Top4 {
  float s0 = -3.0e38f, s1 = -3.0e38f, s2 = -3.0e38f, s3 = -3.0e38f;
  int i0 = -1, i1 = -1, i2 = -1, i3 = -1;
  __device__ static bool ahead(float s, int i, float t, int j) { return s > t || (s == t && i < j); }
  __device__ __forceinline__ void insert(float sc, int col) {
    if (!ahead(sc, col, s3, i3)) return;
    if (ahead(sc, col, s2, i2)) {
      s3 = s2; i3 = i2;
      if (ahead(sc, col, s1, i1)) {
        s2 = s1; i2 = i1;
        if (ahead(sc, col, s0, i0)) { s1 = s0; i1 = i0; s0 = sc; i0 = col; }
        else { s1 = sc; i1 = col; }
      } else { s2 = sc; i2 = col; }
    } else { s3 = sc; i3 = col; }
  }
  // merge with the list of the lane `mask` away (the four lanes of a quad share a row)
  __device__ __forceinline__ void merge_xor(int mask) {
    const float t0 = __shfl_xor_sync(0xffffffffu, s0, mask), t1 = __shfl_xor_sync(0xffffffffu, s1, mask),
                t2 = __shfl_xor_sync(0xffffffffu, s2, mask), t3 = __shfl_xor_sync(0xffffffffu, s3, mask);
    const int j0 = __shfl_xor_sync(0xffffffffu, i0, mask), j1 = __shfl_xor_sync(0xffffffffu, i1, mask),
              j2 = __shfl_xor_sync(0xffffffffu, i2, mask), j3 = __shfl_xor_sync(0xffffffffu, i3, mask);
    if (j0 >= 0) insert(t0, j0);
    if (j1 >= 0) insert(t1, j1);
    if (j2 >= 0) insert(t2, j2);
    if (j3 >= 0) insert(t3, j3);
  }
};

// SiftGPU RowMatch / ColMatch bookkeeping of one query row (ProgramCU.cu:1708-1736, 1463-1478, 1771-1777): strict >, only
// positive dots register, the runner-up VALUE counts duplicates of the maximum.  best = (dot << 17) | (0x1FFFF - tie priority),
// -1 = no positive dot yet; next = the largest dot of every other column -- both independent of the visiting order.
struct U8Best {
  long long best = -1;
  int next = 0;
  __device__ __forceinline__ void add_key(long long key) {
    if (key > best) {
      if (best >= 0) next = max(next, (int)(best >> 17));
      best = key;
    } else {
      next = max(next, (int)(key >> 17));
    }
  }
  __device__ __forceinline__ void add(int dv, int col, int tie_rule) {
    // common case first: a dot product below the current best only feeds the runner-up value
    if (dv > 0 && dv >= (best >= 0 ? (int)(best >> 17) : 0)) {
      const int prio = tie_rule ? col : (((col & 31) << 12) | (col >> 5));
      add_key(((long long)dv << 17) | (long long)(0x1FFFF - prio));
    } else {
      next = max(next, dv);
    }
  }
  __device__ __forceinline__ void merge_xor(int mask) {
    const long long pb = __shfl_xor_sync(0xffffffffu, best, mask);
    const int pn = __shfl_xor_sync(0xffffffffu, next, mask);
    if (pb >= 0) add_key(pb);
    next = max(next, pn);
  }
};

template <int MODE>
__global__ void __launch_bounds__(kTc256Threads, 1) tc_match256_kernel(const HamItem* __restrict__ items, int n_items) {
  extern __shared__ __align__(1024) uint8_t smem[];
  const uint32_t sA = smem_u32(smem);
  const uint32_t sB = sA + kA256;
  const uint32_t bars = sA + kTc256BarsOff;
  auto bar = [&](int i) { return bars + 8u * (uint32_t)i; };
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;

  if (threadIdx.x == 0) {
    mbar_init(bar(kBarAFull), 1);
    mbar_init(bar(kBarAEmpty), kTc256ConsumerWarps);
    for (int i = 0; i < kBSt; i++) {
      mbar_init(bar(kBarBFull + i), 1);
      mbar_init(bar(kBarBEmpty + i), kTc256ConsumerWarps);
    }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();

  if (warp == kTc256ConsumerWarps) {
    if (lane == 0) {
      uint32_t na = 0, nb_seq = 0;
      for (int it = blockIdx.x; it < n_items; it += gridDim.x) {
        const HamItem item = items[it];
        mbar_wait(bar(kBarAEmpty), (na & 1u) ^ 1u);
        na++;
        mbar_expect_tx(bar(kBarAFull), kA256);
        bulk_g2s(sA, item.a, kA256, bar(kBarAFull));
        for (int nb = 0; nb < item.n_btiles; nb++, nb_seq++) {
          const uint32_t slot = nb_seq % kBSt;
          mbar_wait(bar(kBarBEmpty + slot), ((nb_seq / kBSt) & 1u) ^ 1u);
          mbar_expect_tx(bar(kBarBFull + slot), kB128);
          bulk_g2s(sB + slot * kB128, item.b + (size_t)nb * kB128, kB128, bar(kBarBFull + slot));
        }
      }
    }
    return;
  }

  const int wg = warp >> 2;                                   // warp group = 64-row block of the query tile
  const int r0 = 16 * (warp & 3) + (lane >> 2);               // this thread's rows: r0 and r0 + 8 of the block
  const int cq = 2 * (lane & 3);                              // and columns cq, cq + 1 of every 8-column block
  const uint64_t da = make_desc(sA + wg * kWgRows, 128, kGroupStride);
  using Acc = typename std::conditional<MODE == 2, uint32_t, float>::type;
  Acc d[64];
  uint32_t na = 0, nb_seq = 0;
  for (int it = blockIdx.x; it < n_items; it += gridDim.x) {
    const HamItem item = items[it];
    Top4 t4[2];
    U8Best u8[2];
    mbar_wait(bar(kBarAFull), na & 1u);
    na++;
    for (int nb = 0; nb < item.n_btiles; nb++, nb_seq++) {
      const uint32_t slot = nb_seq % kBSt;
      mbar_wait(bar(kBarBFull + slot), (nb_seq / kBSt) & 1u);
      const uint64_t db = make_desc(sB + slot * kB128, 128, kGroupStride);
      wgmma_fence();
#pragma unroll
      for (int k = 0; k < (MODE == 2 ? 4 : 8); k++)  // u8 SIFT rows carry 128 B of data: 4 k-steps of 32 B
        wgmma_acc(d, da + (uint64_t)((k * 256) >> 4), db + (uint64_t)((k * 256) >> 4), k > 0 ? 1u : 0u);
      wgmma_commit();
      wgmma_wait_all();
      __syncwarp();
      if (lane == 0) mbar_arrive(bar(kBarBEmpty + slot));
      const int colb = nb * 128 + cq;
      if (MODE == 2) {
        const int nvalid = item.nsearch;  // columns col < nvalid exist; dot products are >= 0 and 0 never registers
#pragma unroll
        for (int j = 0; j < 64; j++) {
          const int col = colb + 8 * (j >> 2) + (j & 1);
          u8[(j >> 1) & 1].add(col < nvalid ? (int)d[j] : 0, col, item.pad_);
        }
      } else {
        // |b|^2 of this thread's two columns of every 8-column block; columns past the last train row get +inf = score -inf
#pragma unroll
        for (int i = 0; i < 16; i++) {
          const int col = colb + 8 * i;
          float2 bn = __ldg(reinterpret_cast<const float2*>(item.bnorm + col));
          if (col >= item.nsearch) bn.x = __int_as_float(0x7f800000);
          if (col + 1 >= item.nsearch) bn.y = __int_as_float(0x7f800000);
          t4[0].insert(fmaf(2.f, (float)d[4 * i], -bn.x), col);
          t4[0].insert(fmaf(2.f, (float)d[4 * i + 1], -bn.y), col + 1);
          t4[1].insert(fmaf(2.f, (float)d[4 * i + 2], -bn.x), col);
          t4[1].insert(fmaf(2.f, (float)d[4 * i + 3], -bn.y), col + 1);
        }
      }
    }
    __syncwarp();
    if (lane == 0) mbar_arrive(bar(kBarAEmpty));
#pragma unroll
    for (int h = 0; h < 2; h++) {
      if (MODE == 2) {
        u8[h].merge_xor(1);
        u8[h].merge_xor(2);
      } else {
        t4[h].merge_xor(1);
        t4[h].merge_xor(2);
      }
      const int row = wg * 64 + r0 + 8 * h;
      if ((lane & 3) == 0 && row < item.nq_valid) {
        if (MODE == 2) {
          int4 o = make_int4(0, -1, u8[h].next, 0);
          if (u8[h].best >= 0) {
            const int prio = 0x1FFFF - (int)(u8[h].best & 0x1FFFF);
            o.x = (int)(u8[h].best >> 17);
            o.y = item.pad_ ? prio : (((prio & 0xFFF) << 5) | (prio >> 12));
          }
          reinterpret_cast<int4*>(item.out)[row] = o;
        } else {
          reinterpret_cast<int4*>(item.out)[row] = make_int4(t4[h].i0, t4[h].i1, t4[h].i2, t4[h].i3);
        }
      }
    }
  }
}

template <int MODE>
static cudaError_t launch_tc256(const HamItem* d_items, int n_items, int sm_count, cudaStream_t stream) {
  if (n_items <= 0) return cudaSuccess;
  static bool attr_set = false;
  if (!attr_set) {
    cudaError_t e = cudaFuncSetAttribute(tc_match256_kernel<MODE>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kTc256SmemBytes);
    if (e != cudaSuccess) return e;
    attr_set = true;
  }
  const int grid = n_items < sm_count ? n_items : sm_count;
  tc_match256_kernel<MODE><<<grid, kTc256Threads, kTc256SmemBytes, stream>>>(d_items, n_items);
  return cudaGetLastError();
}
cudaError_t launch_l2_tc256(const HamItem* d_items, int n_items, int sm_count, cudaStream_t stream) {
  return launch_tc256<1>(d_items, n_items, sm_count, stream);
}
cudaError_t launch_siftgpu_tc256(const HamItem* d_items, int n_items, int sm_count, cudaStream_t stream) {
  return launch_tc256<2>(d_items, n_items, sm_count, stream);
}

// ---------------------------------------------------------------------------------------------
// Hamming match as a binary GEMM (the default ORB path, `set_hamming_path(1)`).
//
// One wgmma.mma_async m64n128k256 .b1 .and.popc per 64 query rows and 128-row train tile takes c = popcount(a & b) over the
// whole 256-bit descriptor pair.  The operands are the raw 32-byte rows, copied into the K-major no-swizzle layout
// [row_group][k_chunk 2][row_in_group 8][16 B] (256 B per 8 rows): nothing is expanded.
//   hd(i, j) = pa_i + pb_j - 2 c(i, j)      (pa, pb: popcounts of the query / train row)
// For a fixed query row pa_i is a constant, so the reference's argmin with the lowest index on ties is the arg-max of
// (2 c - pb_j, -j).  The producer writes, per train tile, one int32 per column  cj = (4095 - col) - 4096 pb_j,  and the
// epilogue forms  key = 8192 c + cj = 4096 (2 c - pb_j) + (4095 - col)  with one IMAD per element before the three-input
// maximum (VIMNMX3).  At the end  m = key >> 12 (arithmetic) = 2 c - pb_j,  hd = pa_i - m,  col = 4095 - (key & 4095).
// Exact in int32: |2 c - pb_j| <= 256, col <= 4095.  Columns past the searched train rows have zero rows (c = 0) and
// cj = INT_MIN, so their key is kNoBest and no column is masked in the epilogue.
//
// Warp-specialised, 640 threads = five warp groups, one CTA per SM, persistent:
//  * warp groups 0-3 (consumers, 64 query rows each): wait for a train stage, issue one MMA, load the tile's cj, release the
//    stage, take the row maxima.  No CTA-wide barrier inside the item loop: the groups drift apart, so one group's epilogue
//    runs under the others' MMAs;
//  * warp group 4 (producer): claims work items from the launch's ticket counter, fetches the next item's 256 query rows
//    (8 KiB) with one cp.async.bulk while the current item runs, prefetches each train tile's rows (one row per thread) into
//    registers one tile ahead, copies them into a ring of kBinStages B stages with their cj, and copies the query rows into
//    the A area with their popcounts (each consumer group's 2 KiB slice is refilled as soon as that group has finished its
//    last tile of the previous item).  Stages are published with fence.proxy.async + an mbarrier arrive.
// The producer's order per item is B0, B1, A, B2, ...: the first two train tiles of the next item are copied while the
// consumers still run the previous one (a ring of >= 2 stages keeps that order deadlock-free: B tile j of an item only waits
// for stages of earlier items, or, for j >= 2, of tiles whose A has been published).
constexpr int kBinConsumerGroups = 4;
constexpr int kBinThreads = (kBinConsumerGroups + 1) * 128;
constexpr int kBinStages = 8;
constexpr uint32_t kBinRowGroup = 256;              // bytes per 8-row group of a 32-byte-row operand tile
constexpr uint32_t kBinWgA = 64 * 32;               // 2 KiB: the 64 query rows of one consumer group
constexpr uint32_t kBinRawA = 256 * 32;             // 8 KiB: the raw query rows of one item
constexpr uint32_t kBinB = 128 * 32;                // 4 KiB: one train tile
// cj of a tile, ordered for the epilogue: lane quad position q = (col & 7) / 2 reads the 32 words [36 q, 36 q + 32) (columns
// 8 i + 2 q + e at 36 q + 2 i + e) with eight LDS.128; the stride of 36 words puts the four quads on distinct banks
constexpr int kBinCjQuadStride = 36;
constexpr uint32_t kBinCj = 4 * kBinCjQuadStride * 4;  // 576 B per stage
constexpr uint32_t kBinBOff = kBinConsumerGroups * kBinWgA;
constexpr uint32_t kBinCjOff = kBinBOff + kBinStages * kBinB;
constexpr uint32_t kBinRawOff = kBinCjOff + kBinStages * kBinCj;
constexpr uint32_t kBinPaOff = kBinRawOff + 2 * kBinRawA;  // pa of the 256 query rows in the A area
constexpr uint32_t kBinBarsOff = kBinPaOff + 256 * 4;
constexpr int kBinBarAFull = 0, kBinBarAEmpty = kBinConsumerGroups, kBinBarBFull = 2 * kBinConsumerGroups,
              kBinBarBEmpty = kBinBarBFull + kBinStages, kBinBarRaw = kBinBarBEmpty + kBinStages, kBinNumBars = kBinBarRaw + 2;
constexpr uint32_t kBinSmemBytes = kBinBarsOff + 8 * kBinNumBars + 4 * (kBinConsumerGroups + 2);
static_assert(kBinSmemBytes <= 232448, "tc_hamming_b1: shared memory over the 227 KiB per-CTA limit");
// Registers: 640 threads start with 65536 / 640 -> 96 each.  The producer gives registers back, the consumers take them:
constexpr int kBinProducerRegs = 64, kBinConsumerRegs = 104;
static_assert(kBinConsumerGroups * 128 * kBinConsumerRegs + 128 * kBinProducerRegs <= kBinThreads * 96,
              "tc_hamming_b1: setmaxnreg budget over the registers the CTA is launched with");

template <uint32_t R>
__device__ __forceinline__ void setmaxnreg_inc() { asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(R)); }
template <uint32_t R>
__device__ __forceinline__ void setmaxnreg_dec() { asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(R)); }
// barrier 1 among the producer warp group's 128 threads (barrier 0 is __syncthreads)
__device__ __forceinline__ void producer_bar_sync() { asm volatile("bar.sync 1, 128;" ::: "memory"); }
__device__ __forceinline__ uint4 lds128(uint32_t addr) {
  uint4 v;
  asm volatile("ld.shared.v4.b32 {%0, %1, %2, %3}, [%4];" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "r"(addr) : "memory");
  return v;
}
__device__ __forceinline__ void sts32(uint32_t addr, int v) { asm volatile("st.shared.b32 [%0], %1;" ::"r"(addr), "r"(v) : "memory"); }
__device__ __forceinline__ int popc4(uint4 v) { return __popc(v.x) + __popc(v.y) + __popc(v.z) + __popc(v.w); }
// byte offset of k-chunk 0 of row r in a [row_group][k_chunk 2][8][16 B] tile (k-chunk 1 is 128 B further)
__device__ __forceinline__ uint32_t row_offset(int r) { return (uint32_t)(r >> 3) * kBinRowGroup + (uint32_t)(r & 7) * 16u; }

// generic-proxy operand stores of this warp -> visible to the tensor core (async proxy) once `bar` completes
__device__ __forceinline__ void publish(uint32_t bar) {
  fence_proxy_async_smem();
  __syncwarp();
  if ((threadIdx.x & 31) == 0) mbar_arrive(bar);
}

// The train rows of one item the producer needs.
struct TrainRows {
  const uint4* b;
  int nsearch, n_btiles;
};
// row `r` of train tile nb (32 B; rows past the searched ones are zeros -- c = 0 in their columns, which cj = INT_MIN masks)
__device__ __forceinline__ void load_train_row(const TrainRows& t, int nb, int r, uint4& v0, uint4& v1) {
  const int row = nb * 128 + r;
  v0 = v1 = make_uint4(0, 0, 0, 0);
  if (row < t.nsearch) {
    v0 = __ldg(t.b + 2 * (size_t)row);
    v1 = __ldg(t.b + 2 * (size_t)row + 1);
  }
}

__device__ __forceinline__ void hamming_producer(const HamItem* __restrict__ items, int n_items, unsigned long long* claim,
                                                 unsigned long long claim_base, uint32_t sA, uint32_t sB, uint32_t sCj,
                                                 uint32_t sRaw, uint32_t sPa, uint32_t bars, volatile int* s_item) {
  setmaxnreg_dec<kBinProducerRegs>();
  const int pt = threadIdx.x - kBinConsumerGroups * 128;  // 0..127
  auto bar = [&](int i) { return bars + 8u * (uint32_t)i; };
  // Claims the CTA's item number k (-1: none left) and starts the bulk copy of its query rows into raw buffer k & 1.  A CTA
  // stops after its first -1, so a launch takes exactly n_items + gridDim.x tickets (the host advances claim_base by that).
  auto claim_item = [&](uint32_t k) -> int {
    if (pt == 0) {
      const unsigned long long t = atomicAdd(claim, 1ull) - claim_base;
      s_item[kBinConsumerGroups + (k & 1)] = t < (unsigned long long)n_items ? (int)t : -1;
    }
    producer_bar_sync();  // publishes the claim; every thread is done copying from raw buffer k & 1 (item k - 2)
    const int it = s_item[kBinConsumerGroups + (k & 1)];
    if (pt == 0 && it >= 0) {
      const uint32_t bytes = 32u * (uint32_t)items[it].nq_valid, rb = bar(kBinBarRaw + (int)(k & 1));
      mbar_expect_tx(rb, bytes);
      bulk_g2s(sRaw + (k & 1) * kBinRawA, items[it].a, bytes, rb);
    }
    return it;
  };
  auto train_rows = [&](int it) {
    TrainRows t{nullptr, 0, 0};
    if (it >= 0) t = TrainRows{reinterpret_cast<const uint4*>(items[it].b), items[it].nsearch, items[it].n_btiles};
    return t;
  };
  // item k's query rows and their popcounts -> each consumer group's A slice as soon as that group has finished item k - 1
  // (it = -1: end marker)
  auto produce_a = [&](uint32_t k, int it) {
    if (it >= 0) mbar_wait(bar(kBinBarRaw + (int)(k & 1)), (k >> 1) & 1u);
    const int r = pt >> 1, hw = pt & 1;  // two threads per query row, one 16-byte k-chunk each
#pragma unroll 1
    for (int g = 0; g < kBinConsumerGroups; g++) {
      mbar_wait(bar(kBinBarAEmpty + g), (k & 1u) ^ 1u);
      if (it >= 0) {
        const uint4 v = lds128(sRaw + (k & 1) * kBinRawA + (uint32_t)(g * 64 + r) * 32u + 16u * hw);
        sts128(sA + (uint32_t)g * kBinWgA + row_offset(r) + 128u * hw, v.x, v.y, v.z, v.w);
        int pa = popc4(v);
        pa += __shfl_xor_sync(0xffffffffu, pa, 1);
        if (hw == 0) sts32(sPa + 4u * (uint32_t)(g * 64 + r), pa);
      }
      if (pt == 0) s_item[g] = it;
      publish(bar(kBinBarAFull + g));
    }
  };

  // this thread's train row pt of every tile goes to cj word 36 q + 2 i + e  (i = pt / 8, q = (pt % 8) / 2, e = pt % 2)
  const uint32_t cj_off = 4u * (uint32_t)(kBinCjQuadStride * ((pt & 7) >> 1) + 2 * (pt >> 3) + (pt & 1));
  uint32_t k = 0, s = 0;  // items claimed by this CTA, B stages produced
  int cur = claim_item(0);
  TrainRows ct = train_rows(cur);
  uint4 p0, p1;  // this thread's row (pt) of the next train tile to copy
  load_train_row(ct, 0, pt, p0, p1);
  for (; cur >= 0; k++) {
    const int nxt = claim_item(k + 1);
    const TrainRows nt = train_rows(nxt);
    if (ct.n_btiles == 0) {  // no train rows (nt <= 1): every query row gets "no match"; the next item's tile 0 comes now
      produce_a(k, cur);
      load_train_row(nt, 0, pt, p0, p1);
    }
#pragma unroll 1
    for (int nb = 0; nb < ct.n_btiles; nb++, s++) {
      const uint4 v0 = p0, v1 = p1;
      if (nb + 1 < ct.n_btiles) load_train_row(ct, nb + 1, pt, p0, p1);
      else load_train_row(nt, 0, pt, p0, p1);
      const int col = nb * 128 + pt;
      const int cj = col < ct.nsearch ? (4095 - col) - 4096 * (popc4(v0) + popc4(v1)) : kNoBest;
      const uint32_t slot = s % kBinStages;
      mbar_wait(bar(kBinBarBEmpty + (int)slot), ((s / kBinStages) & 1u) ^ 1u);
      const uint32_t dst = sB + slot * kBinB + row_offset(pt);
      sts128(dst, v0.x, v0.y, v0.z, v0.w);
      sts128(dst + 128u, v1.x, v1.y, v1.z, v1.w);
      sts32(sCj + slot * kBinCj + cj_off, cj);
      publish(bar(kBinBarBFull + (int)slot));
      if (nb == min(1, ct.n_btiles - 1)) produce_a(k, cur);
    }
    cur = nxt;
    ct = nt;
  }
  produce_a(k, -1);
}

__global__ void __launch_bounds__(kBinThreads, 1)
    tc_hamming_b1_kernel(const HamItem* __restrict__ items, int n_items, unsigned long long* __restrict__ claim,
                         unsigned long long claim_base) {
  extern __shared__ __align__(1024) uint8_t smem[];
  const uint32_t sA = smem_u32(smem);
  const uint32_t sB = sA + kBinBOff, sCj = sA + kBinCjOff, sRaw = sA + kBinRawOff, sPa = sA + kBinPaOff, bars = sA + kBinBarsOff;
  // [0, 4): the item in each consumer group's A slice (-1: no more); [4, 6): the producer's claims
  volatile int* s_item = reinterpret_cast<volatile int*>(smem + kBinBarsOff + 8 * kBinNumBars);
  auto bar = [&](int i) { return bars + 8u * (uint32_t)i; };
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, wg = warp >> 2;

  if (threadIdx.x == 0) {
    for (int g = 0; g < kBinConsumerGroups; g++) {
      mbar_init(bar(kBinBarAFull + g), 4);   // the producer's four warps
      mbar_init(bar(kBinBarAEmpty + g), 4);  // the group's four warps
    }
    for (int i = 0; i < kBinStages; i++) {
      mbar_init(bar(kBinBarBFull + i), 4);
      mbar_init(bar(kBinBarBEmpty + i), 4 * kBinConsumerGroups);
    }
    mbar_init(bar(kBinBarRaw), 1);
    mbar_init(bar(kBinBarRaw + 1), 1);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();

  if (wg == kBinConsumerGroups) {
    hamming_producer(items, n_items, claim, claim_base, sA, sB, sCj, sRaw, sPa, bars, s_item);
    return;
  }

  setmaxnreg_inc<kBinConsumerRegs>();
  const int r0 = 16 * (warp & 3) + (lane >> 2);  // this thread's accumulator rows: r0 and r0 + 8 of the group's 64
  const uint32_t cj_lane = 4u * (uint32_t)(kBinCjQuadStride * (lane & 3));  // cj of columns 8 i + 2 (lane % 4) + e
  const uint64_t da = make_desc(sA + wg * kBinWgA, 128, kBinRowGroup);
  uint32_t d[64];
  uint32_t s = 0;  // B stages consumed
  for (uint32_t k = 0;; k++) {
    mbar_wait(bar(kBinBarAFull + wg), k & 1u);
    const int it = s_item[wg];
    if (it < 0) break;
    const HamItem item = items[it];
    // popcounts of this thread's two query rows, read before the A slice is released
    const int pa0 = reinterpret_cast<volatile int*>(smem + kBinPaOff)[wg * 64 + r0];
    const int pa1 = reinterpret_cast<volatile int*>(smem + kBinPaOff)[wg * 64 + r0 + 8];
    int best[2] = {kNoBest, kNoBest};
#pragma unroll 1
    for (int nb = 0; nb < item.n_btiles; nb++, s++) {
      const uint32_t slot = s % kBinStages;
      mbar_wait(bar(kBinBarBFull + (int)slot), (s / kBinStages) & 1u);
      wgmma_fence();
      wgmma_b1(d, da, make_desc(sB + slot * kBinB, 128, kBinRowGroup));
      wgmma_commit();
      wgmma_wait_all();
      // key of column 8 i + cq + e of the tile in row r0 + 8 h:  8192 c + cj  (cj = INT_MIN past the searched rows, c = 0)
      const uint32_t cjs = sCj + slot * kBinCj + cj_lane;
      int m[2][2] = {{kNoBest, kNoBest}, {kNoBest, kNoBest}};
#pragma unroll
      for (int i2 = 0; i2 < 8; i2++) {  // columns of blocks i = 2 i2, 2 i2 + 1
        const uint4 cj = lds128(cjs + 16u * (uint32_t)i2);
        const int c4[4] = {(int)cj.x, (int)cj.y, (int)cj.z, (int)cj.w};
#pragma unroll
        for (int h = 0; h < 2; h++) {
#pragma unroll
          for (int ii = 0; ii < 2; ii++) {
            const int i = 2 * i2 + ii;
            m[h][ii] = __vimax3_s32(m[h][ii], (int)d[4 * i + 2 * h] * 8192 + c4[2 * ii],
                                    (int)d[4 * i + 2 * h + 1] * 8192 + c4[2 * ii + 1]);
          }
        }
      }
      __syncwarp();
      if (lane == 0) mbar_arrive(bar(kBinBarBEmpty + (int)slot));
      best[0] = __vimax3_s32(best[0], m[0][0], m[0][1]);
      best[1] = __vimax3_s32(best[1], m[1][0], m[1][1]);
    }
    __syncwarp();
    if (lane == 0) mbar_arrive(bar(kBinBarAEmpty + wg));  // every MMA of this item has completed: the A slice may be refilled
#pragma unroll
    for (int h = 0; h < 2; h++) {
      int b = best[h];
      b = max(b, __shfl_xor_sync(0xffffffffu, b, 1));
      b = max(b, __shfl_xor_sync(0xffffffffu, b, 2));
      const int row = wg * 64 + r0 + 8 * h;
      if ((lane & 3) == 0 && row < item.nq_valid) {
        int2 o = make_int2(257, -1);  // features.cpp:172-173
        if (b != kNoBest) {
          o.x = (h ? pa1 : pa0) - (b >> 12);  // pa - (2 c - pb)
          o.y = 4095 - (b & 4095);
        }
        item.out[row] = o;
      }
    }
  }
}

cudaError_t launch_hamming_tc_b1(const HamItem* d_items, int n_items, int sm_count, ClaimCounter& claim, cudaStream_t stream) {
  if (n_items <= 0) return cudaSuccess;
  static bool attr_set = false;
  if (!attr_set) {
    cudaError_t e = cudaFuncSetAttribute(tc_hamming_b1_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kBinSmemBytes);
    if (e != cudaSuccess) return e;
    attr_set = true;
  }
  const int grid = n_items < sm_count ? n_items : sm_count;
  tc_hamming_b1_kernel<<<grid, kBinThreads, kBinSmemBytes, stream>>>(d_items, n_items, claim.ticket, claim.base);
  cudaError_t e = cudaGetLastError();
  if (e == cudaSuccess) claim.base += (unsigned long long)(n_items + grid);
  return e;
}

}  // namespace rb200
