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
//  * tc_hamming_expand_kernel -- the ORB path: the threads expand the 32-byte descriptors to +-64 operands straight into shared
//    memory, a ninth k-step carries the column index, and the expansion of train tile n+1 runs while the MMAs of tile n execute;
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
// The threads read the 32-byte descriptors themselves and expand them straight into the operand layout in shared memory
// (8 x the descriptor bytes: expanding in HBM would multiply the stage's DRAM traffic by that).  Two more things ride on it:
//  * operands are +-64 instead of +-1, so the accumulator holds 4096 * dot;
//  * a NINTH k-step multiplies two constant operand blocks, A_idx rows (64, 1, 0 ...) x B_idx row j (hi_j, lo_j, 0 ...) with
//    64 hi_j + lo_j = 127 - j: the accumulator of column j of a train tile becomes  4096 * dot + (127 - j),  i.e. the
//    (dot product, lowest-column-wins) key the arg-max needs is produced BY THE TENSOR CORE, and the epilogue is a plain
//    three-input maximum (VIMNMX3) per two elements.
// Exactness: |4096 dot| <= 2^20, 127 - j in [0, 128), global key = acc + (3968 - 128 tile) = 4096 dot + (4095 - col) with
// col <= 4095 -- all exact in int32; dot = key >> 12 (arithmetic), col = 4095 - (key & 4095).
//
// 512 threads = four warp groups of 64 query rows.  Per item: all threads expand the 256 query rows (two threads per row) and
// train tile 0; then per train tile n: every warp group issues its nine MMAs asynchronously, all threads expand tile n+1 into
// the other half of the double-buffered B area (four threads per row), wait for the MMAs, and take the row maxima.
// Shared memory: A 64 KiB + B 2 x 32 KiB + the two 4 KiB index blocks.
constexpr int kXThreads = 512;
constexpr uint32_t kXBOff = kA256;
constexpr uint32_t kXIdxOff = kXBOff + 2 * kB128;
constexpr uint32_t kXSmemBytes = kXIdxOff + 2 * 4096;
static_assert(kXSmemBytes <= 232448, "tc_hamming_expand: shared memory over the 227 KiB per-CTA limit");

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

// train tile nb of the item -> the B buffer at dst (four threads per row, two descriptor words each; missing rows: zeros)
__device__ __forceinline__ uint2 load_b_words(const HamItem& item, int nb) {
  const int r = threadIdx.x >> 2, row = nb * 128 + r;
  if (row < item.nsearch) return __ldg(reinterpret_cast<const uint2*>(item.b) + 4 * (size_t)row + (threadIdx.x & 3));
  return make_uint2(0, 0);
}
__device__ __forceinline__ void store_b_words(uint32_t dst, uint2 v) {
  const int r = threadIdx.x >> 2, w0 = 2 * (threadIdx.x & 3);
  expand_word(dst + row_offset(r), w0, v.x);
  expand_word(dst + row_offset(r), w0 + 1, v.y);
}

__global__ void __launch_bounds__(kXThreads, 1) tc_hamming_expand_kernel(const HamItem* __restrict__ items, int n_items) {
  extern __shared__ __align__(1024) uint8_t smem[];
  const uint32_t sA = smem_u32(smem);
  const uint32_t sB = sA + kXBOff;
  const uint32_t sIdxA = sA + kXIdxOff, sIdxB = sIdxA + 4096;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;

  if (threadIdx.x < 128) {
    // index blocks, K-major no-swizzle: [row_group 16][k_chunk 2][row 8][16 B]; only bytes 0 and 1 of a row are non-zero
    const int r = threadIdx.x;
    const uint32_t off = (uint32_t)(r >> 3) * 256u + (uint32_t)(r & 7) * 16u;
    sts128(sIdxA + off, 0x00000140u, 0, 0, 0);  // (64, 1, 0, ...)
    sts128(sIdxA + off + 128u, 0, 0, 0, 0);
    const uint32_t rem = 127u - (uint32_t)r;    // 64 * hi + lo
    sts128(sIdxB + off, (rem >> 6) | ((rem & 63u) << 8), 0, 0, 0);
    sts128(sIdxB + off + 128u, 0, 0, 0, 0);
  }
  const int wg = warp >> 2;
  const int r0 = 16 * (warp & 3) + (lane >> 2);  // this thread's accumulator rows: r0 and r0 + 8 of the warp group's 64
  const int cq = 2 * (lane & 3);                 // and columns cq, cq + 1 of every 8-column block
  const uint64_t da = make_desc(sA + wg * kWgRows, 128, kGroupStride);
  const uint64_t dia = make_desc(sIdxA, 128, 256), dib = make_desc(sIdxB, 128, 256);
  uint32_t d[64];

  for (int it = blockIdx.x; it < n_items; it += gridDim.x) {
    const HamItem item = items[it];
    __syncthreads();  // every MMA of the previous item has completed: A and both B buffers may be rewritten
    {
      const int r = threadIdx.x >> 1, hw = threadIdx.x & 1;  // two threads per query row, four descriptor words each
      uint4 v = make_uint4(0, 0, 0, 0);
      if (r < item.nq_valid) v = __ldg(reinterpret_cast<const uint4*>(item.a) + 2 * (size_t)r + hw);
      const uint2 b0 = item.n_btiles > 0 ? load_b_words(item, 0) : make_uint2(0, 0);
      const uint32_t ra = sA + row_offset(r);
      expand_word(ra, 4 * hw, v.x);
      expand_word(ra, 4 * hw + 1, v.y);
      expand_word(ra, 4 * hw + 2, v.z);
      expand_word(ra, 4 * hw + 3, v.w);
      if (item.n_btiles > 0) store_b_words(sB, b0);
    }
    fence_proxy_async_smem();  // generic-proxy operand writes -> visible to the tensor core's (async proxy) reads
    __syncthreads();
    int best[2] = {kNoBest, kNoBest};
    for (int nb = 0; nb < item.n_btiles; nb++) {
      const uint64_t db = make_desc(sB + (uint32_t)(nb & 1) * kB128, 128, kGroupStride);
      wgmma_fence();
#pragma unroll
      for (int ks = 0; ks < 8; ks++) wgmma_s8(d, da + (uint64_t)((ks * 256) >> 4), db + (uint64_t)((ks * 256) >> 4), ks > 0 ? 1u : 0u);
      wgmma_s8(d, dia, dib, 1u);
      wgmma_commit();
      if (nb + 1 < item.n_btiles) store_b_words(sB + (uint32_t)((nb + 1) & 1) * kB128, load_b_words(item, nb + 1));
      wgmma_wait_all();
      const int nvalid = item.nsearch - nb * 128;  // train rows of this tile that exist (>= 128: all)
#pragma unroll
      for (int h = 0; h < 2; h++) {
        int m = kNoBest;
        if (nvalid >= 128) {
          int m0 = __vimax3_s32((int)d[2 * h], (int)d[2 * h + 1], (int)d[4 + 2 * h]);
          int m1 = __vimax3_s32((int)d[4 + 2 * h + 1], (int)d[8 + 2 * h], (int)d[8 + 2 * h + 1]);
#pragma unroll
          for (int i = 3; i < 15; i += 2) {
            m0 = __vimax3_s32(m0, (int)d[4 * i + 2 * h], (int)d[4 * i + 2 * h + 1]);
            m1 = __vimax3_s32(m1, (int)d[4 * i + 4 + 2 * h], (int)d[4 * i + 4 + 2 * h + 1]);
          }
          m = __vimax3_s32(m0, m1, max((int)d[60 + 2 * h], (int)d[60 + 2 * h + 1]));
        } else {
#pragma unroll
          for (int i = 0; i < 16; i++) {
            if (8 * i + cq < nvalid) m = max(m, (int)d[4 * i + 2 * h]);
            if (8 * i + cq + 1 < nvalid) m = max(m, (int)d[4 * i + 2 * h + 1]);
          }
        }
        if (m != kNoBest) best[h] = max(best[h], m + (3968 - 128 * nb));  // 4096 dot + (4095 - col)
      }
      fence_proxy_async_smem();
      __syncthreads();  // tile nb+1 is complete, and every warp group is done with tile nb's buffer
    }
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

cudaError_t launch_hamming_tc_expand(const HamItem* d_items, int n_items, int sm_count, cudaStream_t stream) {
  if (n_items <= 0) return cudaSuccess;
  static bool attr_set = false;
  if (!attr_set) {
    cudaError_t e = cudaFuncSetAttribute(tc_hamming_expand_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kXSmemBytes);
    if (e != cudaSuccess) return e;
    attr_set = true;
  }
  const int grid = n_items < sm_count ? n_items : sm_count;
  tc_hamming_expand_kernel<<<grid, kXThreads, kXSmemBytes, stream>>>(d_items, n_items);
  return cudaGetLastError();
}

}  // namespace rb200
