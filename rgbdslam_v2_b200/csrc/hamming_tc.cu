// hamming_tc.cu -- brute-force descriptor matching on the Hopper tensor cores (wgmma, sm_90a).
//
// bruteForceSearchORB (features.cpp:168-182) for all query rows of all pairs, exact:
//   for two 256-bit descriptors a, b read as +-1 vectors:  a . b = 256 - 2 * hamming(a, b)   (exact in int32)
//   => argmin_j hd(q_i, t_j)  ==  argmax_j (Q T^T)_ij, ties -> lowest j  (features.cpp:176 strict <).
// The N x M distance matrix is therefore an int8 GEMM with a row-arg-max epilogue.  A work item is 256 queries of one pair
// against all train rows of the other node, in 128-row train tiles; each of four warp groups owns 64 query rows and issues
// wgmma.mma_async m64n128 (K = 32 bytes per instruction) with the accumulators in registers (64 per thread).  Operand tiles
// use the canonical K-major no-swizzle ("interleave") shared-memory layout:
//   tile[row_group][k_chunk 16][row_in_group 8][16 B]   (8 x 16 B core matrices, 2048 B per 8-row group)
//
// Two kernels:
//  * tc_hamming_expand_kernel -- the ORB path, warp-specialised: a producer warp group claims work items and expands the 32-byte
//    descriptors to +-64 operands straight into shared memory (a ring of train-tile stages on mbarriers), four consumer warp
//    groups issue the MMAs independently of each other, and a ninth k-step carries the column index;
//  * tc_match256_kernel<1|2>  -- the float-descriptor matchers (bf16 RootSIFT scores / SiftGPU's u8 dot products): operand
//    tiles resident in HBM in the layout above, each staged by ONE cp.async.bulk completing on an mbarrier, one producer warp
//    and four consumer warp groups that run independently of each other (one group's epilogue overlaps another's MMAs).
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

// D (+)= A B^T, s8 x s8 -> s32 (ORB), M64 N128 K32
__device__ __forceinline__ void wgmma_s8(uint32_t (&d)[64], uint64_t da, uint64_t db, uint32_t acc) {
  asm volatile(
      "{\n.reg .pred p;\nsetp.ne.b32 p, %66, 0;\n"
      "wgmma.mma_async.sync.aligned.m64n128k32.s32.s8.s8 " RB_WG_D ", %64, %65, p;\n}\n"
      : RB_WG_OPS("+r", d)
      : "l"(da), "l"(db), "r"(acc));
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
// Hamming match with IN-KERNEL operand expansion (the default ORB path, `set_hamming_path(1)`).
//
// The 32-byte descriptors are expanded straight into the operand layout in shared memory (8 x the descriptor bytes: expanding
// in HBM would multiply the stage's DRAM traffic by that).  Two more things ride on it:
//  * operands are +-64 instead of +-1, so the accumulator holds 4096 * dot;
//  * a NINTH k-step multiplies two constant operand blocks, A_idx rows (64, 1, 0 ...) x B_idx row j (hi_j, lo_j, 0 ...) with
//    64 hi_j + lo_j = 127 - j: the accumulator of column j of a train tile becomes  4096 * dot + (127 - j),  i.e. the
//    (dot product, lowest-column-wins) key the arg-max needs is produced BY THE TENSOR CORE, and the epilogue is a plain
//    three-input maximum (VIMNMX3) per two elements.  Against adding the column term on the ALU (one IADD3 per element) in
//    the same warp-specialised structure, the extra MMA is the faster of the two: 0.104-0.106 ms vs 0.108-0.109 ms per C2
//    launch on an H100 80GB HBM3 at 700 W and 1980 MHz (DESIGN.md section 5).  The tensor pipe is not what binds this kernel.
// Exactness: |4096 dot| <= 2^20, 127 - j in [0, 128), global key = acc + (3968 - 128 tile) = 4096 dot + (4095 - col) with
// col <= 4095 -- all exact in int32; dot = key >> 12 (arithmetic), col = 4095 - (key & 4095).
//
// Warp-specialised, 640 threads = five warp groups, one CTA per SM, persistent:
//  * warp groups 0-3 (consumers, 64 query rows each): wait for an operand stage, issue the nine m64n128k32 MMAs of a train
//    tile, release the stage after their wgmma.wait_group, take the row maxima.  No CTA-wide barrier inside the item loop:
//    the groups drift apart, so one group's epilogue runs under the others' MMAs;
//  * warp group 4 (producer): claims work items from the launch's ticket counter, fetches the next item's 256 query rows
//    (8 KiB) with one cp.async.bulk while the current item runs, prefetches each train tile's rows (one row per thread) into
//    registers one tile ahead, and expands them into a ring of kXStages B stages and into the A area (each consumer group's
//    16 KiB slice is refilled as soon as that group has finished its last tile of the previous item).  Stages are published
//    with fence.proxy.async + an mbarrier arrive.
// The producer's order per item is B0, B1, A, B2, ...: the first two train tiles of the next item are expanded while the
// consumers still run the previous one (a ring of >= 2 stages keeps that order deadlock-free: B tile j of an item only waits
// for stages of earlier items, or, for j >= 2, of tiles whose A has been published).
// Shared memory: A 64 KiB + kXStages x 32 KiB + the two 4 KiB index blocks + 2 x 8 KiB raw query staging + barriers.
constexpr int kXConsumerGroups = 4;
constexpr int kXThreads = (kXConsumerGroups + 1) * 128;
constexpr int kXStages = 4;
constexpr uint32_t kXRawA = 256 * 32;  // raw query rows of one item
constexpr uint32_t kXBOff = kA256;
constexpr uint32_t kXIdxOff = kXBOff + kXStages * kB128;
constexpr uint32_t kXRawOff = kXIdxOff + 2 * 4096;
constexpr uint32_t kXBarsOff = kXRawOff + 2 * kXRawA;
constexpr int kXBarAFull = 0, kXBarAEmpty = kXConsumerGroups, kXBarBFull = 2 * kXConsumerGroups,
              kXBarBEmpty = kXBarBFull + kXStages, kXBarRaw = kXBarBEmpty + kXStages, kXNumBars = kXBarRaw + 2;
constexpr uint32_t kXSmemBytes = kXBarsOff + 8 * kXNumBars + 4 * (kXConsumerGroups + 2);
static_assert(kXSmemBytes <= 232448, "tc_hamming_expand: shared memory over the 227 KiB per-CTA limit");
// Registers: 640 threads start with 65536 / 640 -> 96 each.  The producer gives registers back, the consumers take them:
constexpr int kXLaunchRegs = 96, kXProducerRegs = 64, kXConsumerRegs = 104;
static_assert(kXConsumerGroups * 128 * kXConsumerRegs + 128 * kXProducerRegs <= kXThreads * kXLaunchRegs,
              "tc_hamming_expand: setmaxnreg budget over the registers the CTA is launched with");

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

// 4 descriptor bits (bits 0-3 of x, x < 16) -> 4 int8: bit set -> +64, clear -> -64
// (x & 0x80808080) ^ 0xC0C0C0C0 in ONE LOP3 (immLut (a & b) ^ c = (0xF0 & 0xCC) ^ 0xAA = 0x6A): bit 7 of every byte of x selects
// 0x40 (+64, bit set) or 0xC0 (-64, bit clear)
__device__ __forceinline__ uint32_t pm64_from_bit7(uint32_t x) {
  uint32_t r;
  asm("lop3.b32 %0, %1, %2, %3, 0x6A;" : "=r"(r) : "r"(x), "r"(0x80808080u), "r"(0xC0C0C0C0u));
  return r;
}
// Descriptor word wi (0..7) of a row becomes 32 int8 (+-64) in k-chunks 2 wi and 2 wi + 1 of the row at row_addr.
// The order of the 256 k positions inside a row is free as long as both operands use the same one (a dot product is a sum),
// so no bit is ever moved to a "natural" place: output word s of a chunk is the four bits 7-s, 15-s, 23-s, 31-s (shifted by
// 4 for the second chunk), brought to bit 7 of their byte by one left shift and turned into +-64 by one LOP3.
__device__ __forceinline__ void expand_word(uint32_t row_addr, int wi, uint32_t w) {
#pragma unroll
  for (int hf = 0; hf < 2; hf++)
    sts128(row_addr + (uint32_t)(2 * wi + hf) * 128u, pm64_from_bit7(w << (4 * hf)), pm64_from_bit7(w << (4 * hf + 1)),
           pm64_from_bit7(w << (4 * hf + 2)), pm64_from_bit7(w << (4 * hf + 3)));
}
__device__ __forceinline__ uint32_t row_offset(int r) { return (uint32_t)(r >> 3) * kGroupStride + (uint32_t)(r & 7) * 16u; }

// generic-proxy operand stores of this warp -> visible to the tensor core (async proxy) once `bar` completes
__device__ __forceinline__ void publish(uint32_t bar) {
  fence_proxy_async_smem();
  __syncwarp();
  if ((threadIdx.x & 31) == 0) mbar_arrive(bar);
}

// The train rows of one item the producer needs (a whole HamItem would not fit its register budget).
struct TrainRows {
  const uint4* b;
  int nsearch, n_btiles;
};
// row `r` of train tile nb (32 B; rows past the searched ones are zeros -- their columns are masked in the epilogue)
__device__ __forceinline__ void load_train_row(const TrainRows& t, int nb, int r, uint4& v0, uint4& v1) {
  const int row = nb * 128 + r;
  v0 = v1 = make_uint4(0, 0, 0, 0);
  if (row < t.nsearch) {
    v0 = __ldg(t.b + 2 * (size_t)row);
    v1 = __ldg(t.b + 2 * (size_t)row + 1);
  }
}

__device__ __forceinline__ void hamming_producer(const HamItem* __restrict__ items, int n_items, unsigned long long* claim,
                                                 unsigned long long claim_base, uint32_t sA, uint32_t sB, uint32_t sRaw,
                                                 uint32_t bars, volatile int* s_item) {
  setmaxnreg_dec<kXProducerRegs>();
  const int pt = threadIdx.x - kXConsumerGroups * 128;  // 0..127
  auto bar = [&](int i) { return bars + 8u * (uint32_t)i; };
  // Claims the CTA's item number k (-1: none left) and starts the bulk copy of its query rows into raw buffer k & 1.  A CTA
  // stops after its first -1, so a launch takes exactly n_items + gridDim.x tickets (the host advances claim_base by that).
  auto claim_item = [&](uint32_t k) -> int {
    if (pt == 0) {
      const unsigned long long t = atomicAdd(claim, 1ull) - claim_base;
      s_item[kXConsumerGroups + (k & 1)] = t < (unsigned long long)n_items ? (int)t : -1;
    }
    producer_bar_sync();  // publishes the claim; every thread is done expanding from raw buffer k & 1 (item k - 2)
    const int it = s_item[kXConsumerGroups + (k & 1)];
    if (pt == 0 && it >= 0) {
      const uint32_t bytes = 32u * (uint32_t)items[it].nq_valid, rb = bar(kXBarRaw + (int)(k & 1));
      mbar_expect_tx(rb, bytes);
      bulk_g2s(sRaw + (k & 1) * kXRawA, items[it].a, bytes, rb);
    }
    return it;
  };
  auto train_rows = [&](int it) {
    TrainRows t{nullptr, 0, 0};
    if (it >= 0) t = TrainRows{reinterpret_cast<const uint4*>(items[it].b), items[it].nsearch, items[it].n_btiles};
    return t;
  };
  // item k's query rows -> each consumer group's A slice as soon as that group has finished item k - 1 (it = -1: end marker)
  auto produce_a = [&](uint32_t k, int it) {
    if (it >= 0) mbar_wait(bar(kXBarRaw + (int)(k & 1)), (k >> 1) & 1u);
    const int r = pt >> 1, hw = pt & 1;  // two threads per query row, four descriptor words each
#pragma unroll 1
    for (int g = 0; g < kXConsumerGroups; g++) {
      mbar_wait(bar(kXBarAEmpty + g), (k & 1u) ^ 1u);
      if (it >= 0) {
        const uint4 v = lds128(sRaw + (k & 1) * kXRawA + (uint32_t)(g * 64 + r) * 32u + 16u * hw);
        const uint32_t ra = sA + (uint32_t)g * kWgRows + row_offset(r);
        expand_word(ra, 4 * hw, v.x);
        expand_word(ra, 4 * hw + 1, v.y);
        expand_word(ra, 4 * hw + 2, v.z);
        expand_word(ra, 4 * hw + 3, v.w);
      }
      if (pt == 0) s_item[g] = it;
      publish(bar(kXBarAFull + g));
    }
  };

  uint32_t k = 0, s = 0;  // items claimed by this CTA, B stages produced
  int cur = claim_item(0);
  TrainRows ct = train_rows(cur);
  uint4 p0, p1;  // this thread's row (pt) of the next train tile to expand
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
      const uint32_t slot = s % kXStages;
      mbar_wait(bar(kXBarBEmpty + (int)slot), ((s / kXStages) & 1u) ^ 1u);
      const uint32_t dst = sB + slot * kB128 + row_offset(pt);
      expand_word(dst, 0, v0.x);
      expand_word(dst, 1, v0.y);
      expand_word(dst, 2, v0.z);
      expand_word(dst, 3, v0.w);
      expand_word(dst, 4, v1.x);
      expand_word(dst, 5, v1.y);
      expand_word(dst, 6, v1.z);
      expand_word(dst, 7, v1.w);
      publish(bar(kXBarBFull + (int)slot));
      if (nb == min(1, ct.n_btiles - 1)) produce_a(k, cur);
    }
    cur = nxt;
    ct = nt;
  }
  produce_a(k, -1);
}

__global__ void __launch_bounds__(kXThreads, 1)
    tc_hamming_expand_kernel(const HamItem* __restrict__ items, int n_items, unsigned long long* __restrict__ claim,
                             unsigned long long claim_base) {
  extern __shared__ __align__(1024) uint8_t smem[];
  const uint32_t sA = smem_u32(smem);
  const uint32_t sB = sA + kXBOff, sRaw = sA + kXRawOff, bars = sA + kXBarsOff;
  const uint32_t sIdxA = sA + kXIdxOff, sIdxB = sIdxA + 4096;
  // [0, 4): the item in each consumer group's A slice (-1: no more); [4, 6): the producer's claims
  volatile int* s_item = reinterpret_cast<volatile int*>(smem + kXBarsOff + 8 * kXNumBars);
  auto bar = [&](int i) { return bars + 8u * (uint32_t)i; };
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, wg = warp >> 2;

  if (threadIdx.x == 0) {
    for (int g = 0; g < kXConsumerGroups; g++) {
      mbar_init(bar(kXBarAFull + g), 4);   // the producer's four warps
      mbar_init(bar(kXBarAEmpty + g), 4);  // the group's four warps
    }
    for (int i = 0; i < kXStages; i++) {
      mbar_init(bar(kXBarBFull + i), 4);
      mbar_init(bar(kXBarBEmpty + i), 4 * kXConsumerGroups);
    }
    mbar_init(bar(kXBarRaw), 1);
    mbar_init(bar(kXBarRaw + 1), 1);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  if (threadIdx.x < 128) {
    // index blocks, K-major no-swizzle: [row_group 16][k_chunk 2][row 8][16 B]; only bytes 0 and 1 of a row are non-zero
    const int r = threadIdx.x;
    const uint32_t off = (uint32_t)(r >> 3) * 256u + (uint32_t)(r & 7) * 16u;
    sts128(sIdxA + off, 0x00000140u, 0, 0, 0);  // (64, 1, 0, ...)
    sts128(sIdxA + off + 128u, 0, 0, 0, 0);
    const uint32_t rem = 127u - (uint32_t)r;    // 64 * hi + lo
    sts128(sIdxB + off, (rem >> 6) | ((rem & 63u) << 8), 0, 0, 0);
    sts128(sIdxB + off + 128u, 0, 0, 0, 0);
    fence_proxy_async_smem();
  }
  __syncthreads();

  if (wg == kXConsumerGroups) {
    hamming_producer(items, n_items, claim, claim_base, sA, sB, sRaw, bars, s_item);
    return;
  }

  setmaxnreg_inc<kXConsumerRegs>();
  const int r0 = 16 * (warp & 3) + (lane >> 2);  // this thread's accumulator rows: r0 and r0 + 8 of the group's 64
  const int cq = 2 * (lane & 3);                 // and columns cq, cq + 1 of every 8-column block
  const uint64_t da = make_desc(sA + wg * kWgRows, 128, kGroupStride);
  const uint64_t dia = make_desc(sIdxA, 128, 256), dib = make_desc(sIdxB, 128, 256);
  uint32_t d[64];
  uint32_t s = 0;  // B stages consumed
  for (uint32_t k = 0;; k++) {
    mbar_wait(bar(kXBarAFull + wg), k & 1u);
    const int it = s_item[wg];
    if (it < 0) break;
    const HamItem item = items[it];
    int best[2] = {kNoBest, kNoBest};
#pragma unroll 1
    for (int nb = 0; nb < item.n_btiles; nb++, s++) {
      const uint32_t slot = s % kXStages;
      mbar_wait(bar(kXBarBFull + (int)slot), (s / kXStages) & 1u);
      const uint64_t db = make_desc(sB + slot * kB128, 128, kGroupStride);
      wgmma_fence();
#pragma unroll
      for (int ks = 0; ks < 8; ks++) wgmma_s8(d, da + (uint64_t)((ks * 256) >> 4), db + (uint64_t)((ks * 256) >> 4), ks > 0 ? 1u : 0u);
      wgmma_s8(d, dia, dib, 1u);
      wgmma_commit();
      wgmma_wait_all();
      __syncwarp();
      if (lane == 0) mbar_arrive(bar(kXBarBEmpty + (int)slot));
      const int nvalid = item.nsearch - nb * 128;  // train rows of this tile that exist (>= 128: all)
      // key of column 8 i + cq + e of the tile, in this thread's row r0 + 8 h
      auto key = [&](int i, int e, int h) { return (int)d[4 * i + 2 * h + e]; };
#pragma unroll
      for (int h = 0; h < 2; h++) {
        int m = kNoBest;
        if (nvalid >= 128) {
          int m0 = __vimax3_s32(key(0, 0, h), key(0, 1, h), key(1, 0, h));
          int m1 = __vimax3_s32(key(1, 1, h), key(2, 0, h), key(2, 1, h));
#pragma unroll
          for (int i = 3; i < 15; i += 2) {
            m0 = __vimax3_s32(m0, key(i, 0, h), key(i, 1, h));
            m1 = __vimax3_s32(m1, key(i + 1, 0, h), key(i + 1, 1, h));
          }
          m = __vimax3_s32(m0, m1, max(key(15, 0, h), key(15, 1, h)));
        } else {
#pragma unroll
          for (int i = 0; i < 16; i++) {
            if (8 * i + cq < nvalid) m = max(m, key(i, 0, h));
            if (8 * i + cq + 1 < nvalid) m = max(m, key(i, 1, h));
          }
        }
        if (m != kNoBest) best[h] = max(best[h], m + (3968 - 128 * nb));  // 4096 dot + (4095 - col)
      }
    }
    __syncwarp();
    if (lane == 0) mbar_arrive(bar(kXBarAEmpty + wg));  // every MMA of this item has completed: the A slice may be refilled
#pragma unroll
    for (int h = 0; h < 2; h++) {
      int b = best[h];
      b = max(b, __shfl_xor_sync(0xffffffffu, b, 1));
      b = max(b, __shfl_xor_sync(0xffffffffu, b, 2));
      const int row = wg * 64 + r0 + 8 * h;
      if ((lane & 3) == 0 && row < item.nq_valid) {
        int2 o = make_int2(257, -1);  // features.cpp:172-173
        if (b != kNoBest) {
          const int dot = b >> 12;
          o.x = (256 - dot) >> 1;
          o.y = 4095 - (b & 4095);
        }
        item.out[row] = o;
      }
    }
  }
}

cudaError_t launch_hamming_tc_expand(const HamItem* d_items, int n_items, int sm_count, ClaimCounter& claim, cudaStream_t stream) {
  if (n_items <= 0) return cudaSuccess;
  static bool attr_set = false;
  if (!attr_set) {
    cudaError_t e = cudaFuncSetAttribute(tc_hamming_expand_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kXSmemBytes);
    if (e != cudaSuccess) return e;
    attr_set = true;
  }
  const int grid = n_items < sm_count ? n_items : sm_count;
  tc_hamming_expand_kernel<<<grid, kXThreads, kXSmemBytes, stream>>>(d_items, n_items, claim.ticket, claim.base);
  cudaError_t e = cudaGetLastError();
  if (e == cudaSuccess) claim.base += (unsigned long long)(n_items + grid);
  return e;
}

}  // namespace rb200
