// posegraph.cu -- pose-graph Levenberg-Marquardt on the GPU (float64), the optimiser behind
// GraphManager::optimizeGraph (src/graph_manager.cpp:900-1066) as configured by createOptimizer
// (src/graph_manager.cpp:107-201): OptimizationAlgorithmLevenberg / BlockSolver<6,3> / LinearSolverPCG,
// EdgeSE3 edges with RobustKernelHuber(delta), vertex fixation (graph_manager.cpp:911-937).
// The reference never marginalises (no Schur step anywhere, SURVEY 8a-a20): H is the 6x6-block sparse Hpp.
//
// Kernels (all deterministic: fixed-order reductions, no atomics):
//   pg_linearize_kernel : per edge  e, Ji, Jj, Huber weight -> blocks A=Ji'WJi, B=Jj'WJj, C=Ji'WJj, gi, gj
//   pg_assemble_kernel  : per vertex (CSR of incident edges) H_vv = sum A|B, b_v = -sum g ; max diag
//   pg_pcg_kernel       : whole block-Jacobi PCG in ONE cooperative launch, two grid barriers per iteration;
//                         matrix-free SpMV: y_v = (H_vv + lambda I) s_v + sum_inc (C s_j | C' s_i)
//   pg_update_kernel    : X <- X * fromVectorMQT(delta)      (VertexSE3::oplusImpl)
//   pg_chi2_kernel      : sum rho(e'We) and sum e'We          (activeRobustChi2 / chi2)
// Host: the pose-edge module (PoseEdges, also the camera-camera term of landmark_ba.cu), the solver's steps for lm_optimize
// (posegraph.h: OptimizationAlgorithmLevenberg) and the optimizeGraphImpl stop rule (graph_manager.cpp:998-1014).
#include <cooperative_groups.h>
#include <cuda_runtime.h>

#include <algorithm>
#include <cfloat>
#include <cmath>
#include <cstdlib>
#include <cstring>
#include <vector>

#include "posegraph.h"
#include "se3_graph.cuh"
#include "state.h"

namespace cg = cooperative_groups;

namespace rb200 {

// EdgeSE3::computeError: e = toVectorMQT(Z^-1 Xi^-1 Xj); optionally the exact Jacobians w.r.t. the
// right-multiplicative increments of VertexSE3::oplusImpl:
//   Ji = [ -Ra , 2 Ra [tb]x ; 0 , -(we I + [ve]x) Rb' ]   Jj = [ Re , 0 ; 0 , we I + [ve]x ]
// with Ra = Rz', Rb = Ri' Rj, tb = Ri'(tj - ti), Re = Ra Rb, qe = (ve, we) the error quaternion (we >= 0).
__device__ void edge_error(const double* xi, const double* xj, const double* z, double* e, double* Ji, double* Jj) {
  double Ri[9], Rj[9], Rz[9];
  quat_to_R(xi + 3, Ri);
  quat_to_R(xj + 3, Rj);
  quat_to_R(z + 3, Rz);
  const double d0 = xj[0] - xi[0], d1 = xj[1] - xi[1], d2 = xj[2] - xi[2];
  double tb[3], Rb[9];
#pragma unroll
  for (int r = 0; r < 3; r++) tb[r] = Ri[r] * d0 + Ri[3 + r] * d1 + Ri[6 + r] * d2;
#pragma unroll
  for (int r = 0; r < 3; r++)
#pragma unroll
    for (int c = 0; c < 3; c++) Rb[3 * r + c] = Ri[r] * Rj[c] + Ri[3 + r] * Rj[3 + c] + Ri[6 + r] * Rj[6 + c];
  const double dd0 = tb[0] - z[0], dd1 = tb[1] - z[1], dd2 = tb[2] - z[2];
#pragma unroll
  for (int r = 0; r < 3; r++) e[r] = Rz[r] * dd0 + Rz[3 + r] * dd1 + Rz[6 + r] * dd2;
  double qi[4] = {-xi[3], -xi[4], -xi[5], xi[6]}, qj[4] = {xj[3], xj[4], xj[5], xj[6]}, qz[4] = {-z[3], -z[4], -z[5], z[6]};
  quat_norm(qi); quat_norm(qj); quat_norm(qz);
  double tmp[4], qe[4];
  quat_mul(qz, qi, tmp);
  quat_mul(tmp, qj, qe);
  quat_norm(qe);
  if (qe[3] < 0) { qe[0] = -qe[0]; qe[1] = -qe[1]; qe[2] = -qe[2]; qe[3] = -qe[3]; }
  e[3] = qe[0]; e[4] = qe[1]; e[5] = qe[2];
  if (!Ji) return;
  const double we = qe[3], vx = qe[0], vy = qe[1], vz = qe[2];
  const double Q[9] = {we, -vz, vy, vz, we, -vx, -vy, vx, we};
  const double Tx[9] = {0, -tb[2], tb[1], tb[2], 0, -tb[0], -tb[1], tb[0], 0};
#pragma unroll
  for (int i = 0; i < 36; i++) { Ji[i] = 0; Jj[i] = 0; }
#pragma unroll
  for (int r = 0; r < 3; r++)
#pragma unroll
    for (int c = 0; c < 3; c++) {
      const double ra0 = Rz[r], ra1 = Rz[3 + r], ra2 = Rz[6 + r];  // row r of Ra = column r of Rz
      Ji[6 * r + c] = -Rz[3 * c + r];
      Ji[6 * r + 3 + c] = 2.0 * (ra0 * Tx[c] + ra1 * Tx[3 + c] + ra2 * Tx[6 + c]);
      Ji[6 * (3 + r) + 3 + c] = -(Q[3 * r] * Rb[3 * c] + Q[3 * r + 1] * Rb[3 * c + 1] + Q[3 * r + 2] * Rb[3 * c + 2]);
      Jj[6 * r + c] = ra0 * Rb[c] + ra1 * Rb[3 + c] + ra2 * Rb[6 + c];
      Jj[6 * (3 + r) + 3 + c] = Q[3 * r + c];
    }
}

// out = s * A' (W B), all 6x6 row-major
__device__ void AtWB(const double* A, const double* W, const double* B, double s, double* out) {
  double WB[36];
  for (int r = 0; r < 6; r++)
    for (int c = 0; c < 6; c++) {
      double a = 0;
#pragma unroll
      for (int k = 0; k < 6; k++) a += W[6 * r + k] * B[6 * k + c];
      WB[6 * r + c] = a;
    }
  for (int r = 0; r < 6; r++)
    for (int c = 0; c < 6; c++) {
      double a = 0;
#pragma unroll
      for (int k = 0; k < 6; k++) a += A[6 * k + r] * WB[6 * k + c];
      out[6 * r + c] = s * a;
    }
}

__global__ void __launch_bounds__(128) pg_linearize_kernel(int ne, const double* __restrict__ x, const int2* __restrict__ ij,
                                                           const double* __restrict__ meas, const double* __restrict__ info,
                                                           double delta, double* __restrict__ blk) {
  const int k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= ne) return;
  const int2 v = ij[k];
  double e[6], Ji[36], Jj[36], W[36];
  edge_error(x + 7 * (size_t)v.x, x + 7 * (size_t)v.y, meas + 7 * (size_t)k, e, Ji, Jj);
  for (int i = 0; i < 36; i++) W[i] = info[36 * (size_t)k + i];
  double We[6], e2 = 0;
  for (int a = 0; a < 6; a++) {
    double s = 0;
    for (int c = 0; c < 6; c++) s += W[6 * a + c] * e[c];
    We[a] = s;
    e2 += e[a] * s;
  }
  const double w = (e2 <= delta * delta) ? 1.0 : delta / sqrt(e2);  // RobustKernelHuber rho'
  double* o = blk + (size_t)k * kEdgeBlk;
  double t[36];
  AtWB(Ji, W, Ji, w, t);
  for (int i = 0; i < 36; i++) o[kEdgeA + i] = t[i];
  AtWB(Jj, W, Jj, w, t);
  for (int i = 0; i < 36; i++) o[kEdgeB + i] = t[i];
  AtWB(Ji, W, Jj, w, t);
  for (int i = 0; i < 36; i++) o[kEdgeC + i] = t[i];
  for (int c = 0; c < 6; c++) {
    double si = 0, sj = 0;
    for (int a = 0; a < 6; a++) {
      si += Ji[6 * a + c] * We[a];
      sj += Jj[6 * a + c] * We[a];
    }
    o[kEdgeGi + c] = w * si;
    o[kEdgeGj + c] = w * sj;
  }
}

// CSR adjacency: inc[off[v] .. off[v+1]) = (edge << 1 | role), role 0: v is vertex i of the edge, 1: vertex j.
__global__ void __launch_bounds__(128) pg_assemble_kernel(int nv, const int* __restrict__ off, const int* __restrict__ inc,
                                                          const uint8_t* __restrict__ fixed, const double* __restrict__ blk,
                                                          double* __restrict__ Hd, double* __restrict__ b,
                                                          double* __restrict__ maxdiag_part) {
  // one thread per (vertex, entry): 42 entries = 36 of H_vv + 6 of b_v; blockDim = 128 -> 3 vertices x 42 (+2 idle)
  const int lv = threadIdx.x / 42, ent = threadIdx.x % 42;
  const int v = blockIdx.x * 3 + lv;
  double val = 0.0;
  const bool act = (lv < 3) && (v < nv);
  if (act) {
    for (int p = off[v]; p < off[v + 1]; p++) {
      const int code = inc[p];
      const double* o = edge_blocks(blk, code >> 1);
      if (ent < 36) val += o[edge_diag(code & 1) + ent];
      else val -= o[edge_grad(code & 1) + (ent - 36)];
    }
    if (ent < 36) Hd[(size_t)v * 36 + ent] = val;
    else b[(size_t)v * 6 + (ent - 36)] = fixed[v] ? 0.0 : val;
  }
  // max |diag| over free vertices (computeLambdaInit): block partial, fixed order
  __shared__ double sm[128];
  double d = 0.0;
  if (act && ent < 36 && (ent % 7) == 0 && !fixed[v]) d = fabs(val);
  sm[threadIdx.x] = d;
  __syncthreads();
  for (int s = 64; s > 0; s >>= 1) {
    if (threadIdx.x < s) sm[threadIdx.x] = fmax(sm[threadIdx.x], sm[threadIdx.x + s]);
    __syncthreads();
  }
  if (threadIdx.x == 0) maxdiag_part[blockIdx.x] = sm[0];
}

struct PcgArgs {
  int nv, ne;
  const int* off;
  const int* inc;
  const int* oth;      // per incidence: the vertex at the other end of the edge
  const int2* ij;
  const uint8_t* fixed;
  const double* blk;   // per-edge blocks (se3_graph.cuh)
  const double* Hd;    // nv x 36
  const double* b;     // nv x 6 (0 for fixed)
  double* Minv;        // nv x 36
  double* x;           // out: nv x 6
  double* r;
  double* s;           // M^-1 r
  double* d;
  double* q;
  double* part;        // grid partial sums (2 x gridDim)
  double* result;      // [0] iterations, [1] final dn, [2] scale = x'(lambda x + b), [3] breakdown flag
  double lambda;
  double tol;
  int maxit;
};

// ---- block-Jacobi PCG with TWO grid barriers per iteration -----------------------------------------------------------
// The textbook iteration needs a barrier after each of: the SpMV q = A d (every vertex reads its neighbours' d), the dot d.q,
// the dot r.s, the update of d -- at 5000 vertices each of them is pure latency (37 us per iteration measured).  Written with
//     q_{k+1} = A d_{k+1} = A s_{k+1} + beta_k q_k        (d_{k+1} = s_{k+1} + beta_k d_k,  s = M^-1 r)
// the SpMV runs on s, which is complete as soon as the dot r.s is, so one iteration is two phases, each ending in one barrier
// that also carries that phase's dot product:
//   phase 1 (vertex-local)   x += alpha d ; r -= alpha q ; s = M^-1 r ; partial r.s              -> barrier -> beta
//   phase 2 (SpMV on s)      q = A s + beta q ; d = s + beta d ; partial d.q                     -> barrier -> alpha
// Same recurrences as g2o's LinearSolverPCG in exact arithmetic (carried residual, absolute tolerance on r'M^-1 r), different
// rounding of q only.  Deterministic: vertex v is always handled by the same warp, dot products are reduced in a fixed order.
__device__ __forceinline__ double block_partial(double v, double* sm) {  // fixed-order CTA sum, result in every thread
  v = warp_sum_d(v);
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  __syncthreads();  // sm may still be read by the previous reduction
  if (lane == 0) sm[warp] = v;
  __syncthreads();
  double s = 0;
  for (int w = 0; w < (int)(blockDim.x >> 5); w++) s += sm[w];
  return s;
}
// every CTA's partial is in part[0 .. gridDim.x): every warp adds them in the same fixed order (strided by lane, then a butterfly)
__device__ __forceinline__ double grid_total(const double* part) {
  const int lane = threadIdx.x & 31;
  double t = 0;
  for (int i = lane; i < (int)gridDim.x; i += 32) t += __ldcg(part + i);
  return warp_sum_d(t);
}

// off-diagonal part of row block v applied to `vec` (lanes split the incident edges), summed over the warp
__device__ __forceinline__ void spmv_offdiag(const PcgArgs& a, int v, int lane, const double* __restrict__ vec, double (&acc)[6]) {
#pragma unroll
  for (int r = 0; r < 6; r++) acc[r] = 0;
  for (int p = a.off[v] + lane; p < a.off[v + 1]; p += 32) {
    const int code = a.inc[p];
    const int other = a.oth[p];
    if (other == v) continue;  // self edge: no off-diagonal block
    const double* C = edge_blocks(a.blk, code >> 1) + kEdgeC;
    const double* o = vec + 6 * (size_t)other;
    double ov[6];
#pragma unroll
    for (int c = 0; c < 6; c++) ov[c] = __ldcg(o + c);
    if ((code & 1) == 0) {  // v == i: C * d_j
#pragma unroll
      for (int r = 0; r < 6; r++)
#pragma unroll
        for (int c = 0; c < 6; c++) acc[r] += C[6 * r + c] * ov[c];
    } else {  // v == j: C' * d_i
#pragma unroll
      for (int r = 0; r < 6; r++)
#pragma unroll
        for (int c = 0; c < 6; c++) acc[c] += C[6 * r + c] * ov[r];
    }
  }
#pragma unroll
  for (int r = 0; r < 6; r++) acc[r] = warp_sum_d(acc[r]);
}

// block-Jacobi preconditioner: M^-1 = (H_vv + lambda I)^-1 per free vertex (own kernel: the Gauss-Jordan working set would
// otherwise set the register budget of the PCG loop)
__global__ void __launch_bounds__(128) pg_precond_kernel(int nv, const double* __restrict__ Hd, const uint8_t* __restrict__ fixed,
                                                         double lambda, double* __restrict__ Minv) {
  const int v = blockIdx.x * blockDim.x + threadIdx.x;
  if (v >= nv) return;
  double A[36], Ai[36];
  for (int i = 0; i < 36; i++) A[i] = Hd[36 * (size_t)v + i];
  for (int k = 0; k < 6; k++) A[7 * k] += lambda;
  const bool ok = !fixed[v] && inv6(A, Ai);
  for (int i = 0; i < 36; i++) Minv[36 * (size_t)v + i] = ok ? Ai[i] : 0.0;
}

__global__ void __launch_bounds__(512, 1) pg_pcg_kernel(PcgArgs a) {
  cg::grid_group grid = cg::this_grid();
  __shared__ double sm[16];
  const int tid = blockIdx.x * blockDim.x + threadIdx.x;
  const int nthreads = gridDim.x * blockDim.x;
  const int lane = threadIdx.x & 31;
  const int gwarp = tid >> 5, nwarps = nthreads >> 5;
  double* part_a = a.part;               // partials of r.s
  double* part_b = a.part + gridDim.x;   // partials of d.q (two arrays: a CTA may already write the next phase's partial
                                         // while another one still reads this phase's)

  // (the preconditioner M^-1 = (H_vv + lambda I)^-1 was written by pg_precond_kernel, launched just before on the same stream)
  // x = 0, r = b, s = M^-1 r (kept in a.d until phase 2 turns it into d), dn = r.s
  double loc = 0;
  for (int v = gwarp; v < a.nv; v += nwarps) {
    double rr = 0, sv = 0;
    if (lane < 6) rr = a.b[6 * (size_t)v + lane];
    double rv[6];
#pragma unroll
    for (int c = 0; c < 6; c++) rv[c] = __shfl_sync(0xffffffffu, rr, c);
    if (lane < 6) {
#pragma unroll
      for (int c = 0; c < 6; c++) sv += a.Minv[36 * (size_t)v + 6 * lane + c] * rv[c];
      a.x[6 * (size_t)v + lane] = 0.0;
      a.r[6 * (size_t)v + lane] = rr;
      a.s[6 * (size_t)v + lane] = sv;
      a.d[6 * (size_t)v + lane] = 0.0;
      a.q[6 * (size_t)v + lane] = 0.0;
      loc += rr * sv;
    }
  }
  {
    const double p = block_partial(loc, sm);
    if (threadIdx.x == 0) part_a[blockIdx.x] = p;
  }
  grid.sync();
  double dn = grid_total(part_a);
  double beta = 0.0;  // first phase 2: d = s, q = A s
  int it = 0;
  bool breakdown = false;
  for (;;) {
    // ---- phase 2: q = A s + beta q ; d = s + beta d ; partial d.q
    loc = 0;
    for (int v = gwarp; v < a.nv; v += nwarps) {
      const bool fx = a.fixed[v] != 0;
      double acc[6];
      if (!fx) spmv_offdiag(a, v, lane, a.s, acc);
      if (lane < 6) {
        double qn = 0, dnw = 0;
        if (!fx) {
          const double* H = a.Hd + 36 * (size_t)v + 6 * lane;
          const double* sv = a.s + 6 * (size_t)v;
          double t = 0;
#pragma unroll
          for (int c = 0; c < 6; c++) t += H[c] * sv[c];
          t += a.lambda * sv[lane];
          double o = 0;
#pragma unroll
          for (int r = 0; r < 6; r++) o = (r == lane) ? acc[r] : o;
          t += o;
          qn = t + beta * a.q[6 * (size_t)v + lane];
          dnw = sv[lane] + beta * a.d[6 * (size_t)v + lane];
        }
        a.q[6 * (size_t)v + lane] = qn;
        a.d[6 * (size_t)v + lane] = dnw;
        loc += dnw * qn;
      }
    }
    {
      const double p = block_partial(loc, sm);
      if (threadIdx.x == 0) part_b[blockIdx.x] = p;
    }
    grid.sync();
    if (it >= a.maxit || dn <= a.tol) break;  // (the extra SpMV of the last round is the price of the two-barrier form)
    const double dq = grid_total(part_b);
    if (!(dq > 0)) { breakdown = true; break; }
    const double alpha = dn / dq;
    // ---- phase 1: x += alpha d ; r -= alpha q (recursive residual: g2o never resets it) ; s = M^-1 r ; partial r.s
    loc = 0;
    for (int v = gwarp; v < a.nv; v += nwarps) {
      double rr = 0;
      if (lane < 6) {
        const size_t i = 6 * (size_t)v + lane;
        a.x[i] += alpha * a.d[i];
        rr = a.r[i] - alpha * a.q[i];
        a.r[i] = rr;
      }
      double rv[6];
#pragma unroll
      for (int c = 0; c < 6; c++) rv[c] = __shfl_sync(0xffffffffu, rr, c);
      if (lane < 6) {
        double sv = 0;
#pragma unroll
        for (int c = 0; c < 6; c++) sv += a.Minv[36 * (size_t)v + 6 * lane + c] * rv[c];
        a.s[6 * (size_t)v + lane] = sv;
        loc += rr * sv;
      }
    }
    {
      const double p = block_partial(loc, sm);
      if (threadIdx.x == 0) part_a[blockIdx.x] = p;
    }
    grid.sync();
    const double dn_new = grid_total(part_a);
    beta = dn_new / dn;
    dn = dn_new;
    it++;
  }
  // computeScale(): sum x_j (lambda x_j + b_j)
  loc = 0;
  const int n = 6 * a.nv;
  for (int i = tid; i < n; i += nthreads) loc += a.x[i] * (a.lambda * a.x[i] + a.b[i]);
  {
    const double p = block_partial(loc, sm);
    if (threadIdx.x == 0) part_a[blockIdx.x] = p;
  }
  grid.sync();
  const double scale = grid_total(part_a);
  if (tid == 0) {
    a.result[0] = (double)it;
    a.result[1] = dn;
    a.result[2] = scale;
    a.result[3] = breakdown ? 1.0 : 0.0;
  }
}

// ---- the same iteration for graphs that fit the chip: everything a vertex owns stays ON the SM ------------------------------
// Up to 80 vertices per CTA (16 warps x 5 groups of 6 lanes: lane = one of the 6 rows of one vertex).  A lane keeps its row of
// x, r, d, q, s, b, M^-1 and H_vv + lambda I in REGISTERS for the whole solve; the CTA stages the off-diagonal 6x6 blocks of
// its vertices' incident edges (already oriented for the owner: C or C', written once per linearisation by pg_orient_kernel,
// contiguous per CTA because the CSR is vertex-major) and the neighbour indices in SHARED memory.  The only global traffic of
// an iteration is the publication of s (48 B per vertex) and the gather of the neighbours' s; the SpMV of a row is a
// sequential sum over its incidences in one lane -- no warp reduction, no atomics, fixed order.  Two grid barriers per
// iteration as in pg_pcg_kernel, but a barrier that carries the dot product itself (pg_tree_barrier).
// C5 (5000 V / 30 000 E, 7814 PCG iterations): 25.5 -> 10.9 us per iteration, 0.20 -> 0.085 s for the whole solve.  Where the
// remaining time goes (clock64 profile): the two barriers 2 x 3.4 us (three fences and two global
// store -> poll hops each), gather + SpMV 2.4 us, block sums 0.9 us.
// Incidences beyond the shared-memory capacity of a CTA (hub vertices) are read from the global copy.
constexpr int kPgResGroups = 5, kPgResWarps = 16, kPgResSlots = kPgResGroups * kPgResWarps;

__global__ void __launch_bounds__(128) pg_orient_kernel(int nv, const int* __restrict__ off, const int* __restrict__ inc,
                                                        const int* __restrict__ oth, const double* __restrict__ blk,
                                                        double* __restrict__ incblk) {
  const int v = blockIdx.x * 4 + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (v >= nv) return;
  for (int p = off[v]; p < off[v + 1]; p++) {
    const int code = inc[p];
    const bool self = oth[p] == v;  // self edge: no off-diagonal block
    const double* C = edge_blocks(blk, code >> 1) + kEdgeC;
    for (int e = lane; e < 36; e += 32) {
      const int r = e / 6, c = e - 6 * r;
      incblk[36 * (size_t)p + e] = self ? 0.0 : ((code & 1) == 0 ? C[6 * r + c] : C[6 * c + r]);
    }
  }
}

// Grid barrier that CARRIES the dot product (resident solver), two levels so that no cache line is polled by more than one
// warp per CTA and no CTA reads more than one line per level:
//   level 1: a CTA publishes its partial sum in slot[bid]; the first CTA of every group of kPgGroup consecutive CTAs polls
//            the group's slots (one 128-byte line), adds them in slot order and publishes the group sum in gslot[group];
//   level 2: every CTA polls the <= 32 group sums (one or two lines) and adds them in order.
// A published double carries the parity of the barrier's use count in its lowest mantissa bit (st.relaxed after a
// __threadfence; polled with relaxed loads, one __threadfence after the last poll): value and flag travel in one word, one
// global round trip per level.  The flag bit is part of the value every reader sees, so the sum is identical in every CTA and
// from run to run.  Two slot sets used alternately (a CTA can only reach the next use of a set after every CTA has consumed
// the previous one: the barrier in between needs all of them).  Measured: 3.4 us per barrier; cooperative-groups grid.sync()
// followed by every warp loading the 148 partials cost the same iteration 4.5 us, a one-level version in which every CTA
// polls all 148 slots 5 us (148 warps hammering the same ten cache lines).  Needs all CTAs co-resident (cooperative launch);
// the host presets all slots to all-ones (parity 1; the first use expects 0).
constexpr int kPgGroup = 12;  // 12 x 8 B = 96 B: the slots of a group share one 128-byte line (slots are 128-byte aligned per group)
__device__ __forceinline__ unsigned long long pg_flagged(double v, unsigned parity) {
  return ((unsigned long long)__double_as_longlong(v) & ~1ull) | (unsigned long long)parity;
}
__device__ __forceinline__ void pg_st_relaxed(double* p, unsigned long long u) {
  asm volatile("st.relaxed.gpu.global.u64 [%0], %1;" ::"l"(p), "l"(u) : "memory");
}
__device__ __forceinline__ unsigned long long pg_ld_relaxed(const double* p) {
  unsigned long long u;
  asm volatile("ld.relaxed.gpu.global.u64 %0, [%1];" : "=l"(u) : "l"(p) : "memory");
  return u;
}
// slots: [group][16] doubles (12 used), gslots: [32] doubles, both per set.  Returns the grid total in every thread.
// fence.acq_rel is all the barrier needs (release before a publication, acquire after the last poll); __threadfence() is the
// sequentially consistent fence
__device__ __forceinline__ void pg_fence() { asm volatile("fence.acq_rel.gpu;" ::: "memory"); }
__device__ __forceinline__ double pg_tree_barrier(double block_sum, double* slots, double* gslots, unsigned parity, double* sm) {
  const int bid = blockIdx.x, grp = bid / kPgGroup, idx = bid - grp * kPgGroup;
  const int n_groups = ((int)gridDim.x + kPgGroup - 1) / kPgGroup;
  if (threadIdx.x < 32) {
    const int lane = threadIdx.x;
    if (lane == 0) {
      pg_fence();  // the CTA's s rows (ordered before this thread by the __syncthreads of block_partial) become visible first
      pg_st_relaxed(slots + 16 * grp + idx, pg_flagged(block_sum, parity));
    }
    if (idx == 0) {  // group leader
      const int members = min(kPgGroup, (int)gridDim.x - grp * kPgGroup);
      unsigned long long u;
      bool ok;
      do {
        u = lane < members ? pg_ld_relaxed(slots + 16 * grp + lane) : (unsigned long long)parity;
        ok = __all_sync(0xffffffffu, (u & 1ull) == (unsigned long long)parity);
      } while (!ok);
      const double t = warp_sum_d(lane < members ? __longlong_as_double((long long)u) : 0.0);
      if (lane == 0) {
        pg_fence();
        pg_st_relaxed(gslots + grp, pg_flagged(t, parity));
      }
    }
    unsigned long long u;
    bool ok;
    do {
      u = lane < n_groups ? pg_ld_relaxed(gslots + lane) : (unsigned long long)parity;
      ok = __all_sync(0xffffffffu, (u & 1ull) == (unsigned long long)parity);
    } while (!ok);
    const double t = warp_sum_d(lane < n_groups ? __longlong_as_double((long long)u) : 0.0);
    pg_fence();
    if (lane == 0) sm[0] = t;
  }
  __syncthreads();
  const double r = sm[0];
  return r;  // (the next block_partial starts with a __syncthreads before it reuses sm)
}
constexpr int kPgBarrierDoubles = 2 * (16 * 32 + 32);  // two sets of (<= 32 groups x 16 slots) + 32 group sums: grids up to 384 CTAs

__global__ void __launch_bounds__(kPgResWarps * 32, 1) pg_pcg_resident_kernel(PcgArgs a, const double* __restrict__ incblk, int vpc, int cap) {
  extern __shared__ __align__(16) unsigned char pg_dsm[];
  double* sm = reinterpret_cast<double*>(pg_dsm);  // 16 doubles of block_partial
  double* blk_s = sm + 16;                         // cap x 36
  double* sg_s = blk_s + 36 * (size_t)cap;         // cap x 6: the neighbours' s rows of the current iteration
  int* src_s = reinterpret_cast<int*>(sg_s + 6 * (size_t)cap);  // cap x 6: where element i of sg_s comes from (index into s)
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int g = lane / 6, row = lane - 6 * g;
  const int v0 = blockIdx.x * vpc, v1 = min(a.nv, v0 + vpc);
  const int p0 = v0 < a.nv ? a.off[v0] : 0, p1 = v0 < a.nv ? a.off[v1] : 0;
  const int n_s = min(p1 - p0, cap);
  for (int i = threadIdx.x; i < 36 * n_s; i += blockDim.x) blk_s[i] = incblk[36 * (size_t)p0 + i];
  for (int i = threadIdx.x; i < 6 * n_s; i += blockDim.x) {
    const int li = i / 6;
    src_s[i] = 6 * a.oth[p0 + li] + (i - 6 * li);
  }
  const int slot = warp * kPgResGroups + g;
  const int v = v0 + slot;
  const bool act = g < kPgResGroups && slot < vpc && v < v1;
  const int gbase = 6 * g;
  double* slots_a = a.part;                 // set A (r.s and the final scale), set B (d.q)
  double* gslots_a = a.part + 16 * 32;
  double* slots_b = a.part + 16 * 32 + 32;
  double* gslots_b = slots_b + 16 * 32;

  double Mrow[6], Hrow[6], xb = 0, rr = 0, dd = 0, qq = 0, sv = 0, bb = 0;
  bool fx = true;
  int pb = 0, pe = 0;
#pragma unroll
  for (int c = 0; c < 6; c++) { Mrow[c] = 0; Hrow[c] = 0; }
  if (act) {
    fx = a.fixed[v] != 0;
#pragma unroll
    for (int c = 0; c < 6; c++) {
      Mrow[c] = a.Minv[36 * (size_t)v + 6 * row + c];
      Hrow[c] = a.Hd[36 * (size_t)v + 6 * row + c] + (c == row ? a.lambda : 0.0);
    }
    bb = a.b[6 * (size_t)v + row];
    pb = a.off[v];
    pe = a.off[v + 1];
  }
  __syncthreads();
  // x = 0, r = b, s = M^-1 r, dn = r.s
  rr = bb;
  {
    double t = 0;
#pragma unroll
    for (int c = 0; c < 6; c++) t += Mrow[c] * __shfl_sync(0xffffffffu, rr, (gbase + c) & 31);
    sv = t;
  }
  if (act) a.s[6 * (size_t)v + row] = sv;
  unsigned ea = 0, eb = 0;  // use counts of the two slot sets
  double bsum;
  {
    bsum = block_partial(act ? rr * sv : 0.0, sm);
  }
  double dn = pg_tree_barrier(bsum, slots_a, gslots_a, ea & 1u, sm);
  ea++;
  double beta = 0.0;
  int it = 0;
  bool breakdown = false;
  for (;;) {
    // ---- phase 2: q = A s + beta q ; d = s + beta d ; partial d.q
    // the s rows of all neighbours of this CTA's vertices, fetched by the whole CTA in ONE round trip (one double per thread
    // and step, all independent) into shared memory; a lane then sums its row over its incidences out of shared memory only --
    // the time of the phase no longer depends on the largest vertex degree in the grid
    for (int base = 0; base < 6 * n_s; base += 8 * (int)blockDim.x) {
      double tmp[8];
#pragma unroll
      for (int u = 0; u < 8; u++) {  // eight independent loads in flight per thread
        const int i = base + u * (int)blockDim.x + (int)threadIdx.x;
        tmp[u] = i < 6 * n_s ? __ldcg(a.s + src_s[i]) : 0.0;
      }
#pragma unroll
      for (int u = 0; u < 8; u++) {
        const int i = base + u * (int)blockDim.x + (int)threadIdx.x;
        if (i < 6 * n_s) sg_s[i] = tmp[u];
      }
    }
    __syncthreads();
    double acc = 0;
    if (act && !fx) {
      // six independent accumulators (one per column) and two incidences per step: a single running sum would serialise
      // degree x 6 dependent FP64 FMAs (their latency, not their number, was the cost of the phase)
      double ac0[6] = {0, 0, 0, 0, 0, 0}, ac1[6] = {0, 0, 0, 0, 0, 0};
      const int pe_s = min(pe, p0 + n_s);
      int p = pb;
      for (; p + 1 < pe_s; p += 2) {
        const int li = p - p0;
        const double* C0 = blk_s + 36 * li + 6 * row;
        const double* o0 = sg_s + 6 * li;
#pragma unroll
        for (int c = 0; c < 6; c++) {
          ac0[c] += C0[c] * o0[c];
          ac1[c] += C0[36 + c] * o0[6 + c];
        }
      }
      if (p < pe_s) {
        const int li = p - p0;
        const double* C0 = blk_s + 36 * li + 6 * row;
        const double* o0 = sg_s + 6 * li;
#pragma unroll
        for (int c = 0; c < 6; c++) ac0[c] += C0[c] * o0[c];
        p++;
      }
      for (; p < pe; p++) {  // beyond the shared-memory capacity of the CTA (hub vertices): straight from global memory
        const double* C = incblk + 36 * (size_t)p + 6 * row;
        const double* o = a.s + 6 * (size_t)a.oth[p];
#pragma unroll
        for (int c = 0; c < 6; c++) ac1[c] += C[c] * __ldcg(o + c);
      }
      acc = ((ac0[0] + ac1[0]) + (ac0[1] + ac1[1])) + ((ac0[2] + ac1[2]) + (ac0[3] + ac1[3])) + ((ac0[4] + ac1[4]) + (ac0[5] + ac1[5]));
    }
    double qn = 0, dnw = 0;
    {
      double t = 0;
#pragma unroll
      for (int c = 0; c < 6; c++) t += Hrow[c] * __shfl_sync(0xffffffffu, sv, (gbase + c) & 31);
      if (act && !fx) {
        qn = t + acc + beta * qq;
        dnw = sv + beta * dd;
      }
    }
    qq = qn;
    dd = dnw;
    {
      bsum = block_partial(act ? dnw * qn : 0.0, sm);
    }
    const double dq = pg_tree_barrier(bsum, slots_b, gslots_b, eb & 1u, sm);
    eb++;
    if (it >= a.maxit || dn <= a.tol) break;
    if (!(dq > 0)) { breakdown = true; break; }
    const double alpha = dn / dq;
    // ---- phase 1: x += alpha d ; r -= alpha q ; s = M^-1 r ; partial r.s
    xb += alpha * dd;
    rr -= alpha * qq;
    {
      double t = 0;
#pragma unroll
      for (int c = 0; c < 6; c++) t += Mrow[c] * __shfl_sync(0xffffffffu, rr, (gbase + c) & 31);
      sv = t;
    }
    if (act) a.s[6 * (size_t)v + row] = sv;
    {
      bsum = block_partial(act ? rr * sv : 0.0, sm);
    }
    const double dn_new = pg_tree_barrier(bsum, slots_a, gslots_a, ea & 1u, sm);
    ea++;
    beta = dn_new / dn;
    dn = dn_new;
    it++;
  }
  if (act) a.x[6 * (size_t)v + row] = xb;
  {
    bsum = block_partial(act ? xb * (a.lambda * xb + bb) : 0.0, sm);
  }
  const double scale = pg_tree_barrier(bsum, slots_a, gslots_a, ea & 1u, sm);
  if (blockIdx.x == 0 && threadIdx.x == 0) {
    a.result[0] = (double)it;
    a.result[1] = dn;
    a.result[2] = scale;
    a.result[3] = breakdown ? 1.0 : 0.0;
  }
}

__global__ void __launch_bounds__(128) pg_update_kernel(int nv, const double* __restrict__ xin, const double* __restrict__ dlt,
                                                        const uint8_t* __restrict__ fixed, double* __restrict__ xout) {
  const int v = blockIdx.x * blockDim.x + threadIdx.x;
  if (v >= nv) return;
  double x[7];
  for (int i = 0; i < 7; i++) x[i] = xin[7 * (size_t)v + i];
  if (!fixed[v]) {
    const double* d = dlt + 6 * (size_t)v;
    double R[9];
    quat_to_R(x + 3, R);
    for (int r = 0; r < 3; r++) x[r] += R[3 * r] * d[0] + R[3 * r + 1] * d[1] + R[3 * r + 2] * d[2];
    const double w = 1.0 - (d[3] * d[3] + d[4] * d[4] + d[5] * d[5]);
    if (w >= 0) {  // fromCompactQuaternion: w < 0 -> identity rotation
      double dq[4] = {d[3], d[4], d[5], sqrt(w)}, q[4] = {x[3], x[4], x[5], x[6]}, o[4];
      quat_mul(q, dq, o);
      quat_norm(o);
      x[3] = o[0]; x[4] = o[1]; x[5] = o[2]; x[6] = o[3];
    }
  }
  for (int i = 0; i < 7; i++) xout[7 * (size_t)v + i] = x[i];
}

// per-edge chi2 -> block partials of (robust, plain); optional per-edge output
__global__ void __launch_bounds__(256) pg_chi2_kernel(int ne, const double* __restrict__ x, const int2* __restrict__ ij,
                                                      const double* __restrict__ meas, const double* __restrict__ info,
                                                      double delta, double* __restrict__ part, double* __restrict__ per_edge) {
  const int k = blockIdx.x * blockDim.x + threadIdx.x;
  double rob = 0, pl = 0;
  if (k < ne) {
    const int2 v = ij[k];
    double e[6];
    edge_error(x + 7 * (size_t)v.x, x + 7 * (size_t)v.y, meas + 7 * (size_t)k, e, nullptr, nullptr);
    const double* W = info + 36 * (size_t)k;
    double e2 = 0;
    for (int a = 0; a < 6; a++)
      for (int c = 0; c < 6; c++) e2 += e[a] * W[6 * a + c] * e[c];
    pl = e2;
    rob = (e2 <= delta * delta) ? e2 : 2 * sqrt(e2) * delta - delta * delta;
    if (per_edge) per_edge[k] = e2;
  }
  __shared__ double s0[256], s1[256];
  s0[threadIdx.x] = rob;
  s1[threadIdx.x] = pl;
  __syncthreads();
  for (int s = 128; s > 0; s >>= 1) {
    if (threadIdx.x < s) {
      s0[threadIdx.x] += s0[threadIdx.x + s];
      s1[threadIdx.x] += s1[threadIdx.x + s];
    }
    __syncthreads();
  }
  if (threadIdx.x == 0) {
    part[2 * blockIdx.x] = s0[0];
    part[2 * blockIdx.x + 1] = s1[0];
  }
}

// ================================================================================================
// Host side

// ---- the pose-edge module (posegraph.h)
int PoseEdges::ensure(int nv, int n_edges) {
  const size_t nv_ = (size_t)(nv > 0 ? nv : 1), ne_ = (size_t)(n_edges > 0 ? n_edges : 1);
  int rc;
  if ((rc = ij.ensure(8 * ne_)) || (rc = meas.ensure(56 * ne_)) || (rc = info.ensure(288 * ne_)) || (rc = off.ensure(4 * (nv_ + 1))) ||
      (rc = inc.ensure(8 * ne_)) || (rc = oth.ensure(8 * ne_)) || (rc = blk.ensure(8 * kEdgeBlk * ne_)))
    return rc;
  return 0;
}

int PoseEdges::upload(int nv, int n_edges, const int32_t* h_ij, const double* h_meas, const double* h_info, double huber_delta,
                      bool incidence, cudaStream_t st) {
  for (size_t k = 0; k < 2 * (size_t)n_edges; k++)
    if (h_ij[k] < 0 || h_ij[k] >= nv) {
      set_error("pose edges: vertex index out of range");
      return RGBDSLAM_B200_ERR_ARG;
    }
  if (int rc = ensure(nv, n_edges)) return rc;
  ne = n_edges;
  delta = huber_delta;
  if (ne > 0) {
    RB200_CUDA(cudaMemcpyAsync(meas.ptr, h_meas, 56 * (size_t)ne, cudaMemcpyHostToDevice, st));
    RB200_CUDA(cudaMemcpyAsync(info.ptr, h_info, 288 * (size_t)ne, cudaMemcpyHostToDevice, st));
    RB200_CUDA(cudaMemcpyAsync(ij.ptr, h_ij, 8 * (size_t)ne, cudaMemcpyHostToDevice, st));
  }
  if (!incidence) return 0;
  // edge order within a vertex's incidences => deterministic sums
  h_off.assign(nv + 1, 0);
  h_inc.resize(2 * (size_t)ne);
  h_oth.resize(2 * (size_t)ne);
  for (size_t k = 0; k < 2 * (size_t)ne; k++) h_off[h_ij[k] + 1]++;
  for (int v = 0; v < nv; v++) h_off[v + 1] += h_off[v];
  std::vector<int> cur(h_off.begin(), h_off.end() - 1);
  for (int k = 0; k < ne; k++) {
    const int i = h_ij[2 * k], j = h_ij[2 * k + 1];
    h_oth[cur[i]] = j;
    h_inc[cur[i]++] = k << 1;
    h_oth[cur[j]] = i;
    h_inc[cur[j]++] = k << 1 | 1;
  }
  RB200_CUDA(cudaMemcpyAsync(off.ptr, h_off.data(), 4 * (size_t)(nv + 1), cudaMemcpyHostToDevice, st));
  if (ne > 0) {
    RB200_CUDA(cudaMemcpyAsync(inc.ptr, h_inc.data(), 8 * (size_t)ne, cudaMemcpyHostToDevice, st));
    RB200_CUDA(cudaMemcpyAsync(oth.ptr, h_oth.data(), 8 * (size_t)ne, cudaMemcpyHostToDevice, st));
  }
  return 0;
}

int PoseEdges::linearize(const double* x, cudaStream_t st, int64_t& launches) {
  if (ne == 0) return 0;
  pg_linearize_kernel<<<(ne + 127) / 128, 128, 0, st>>>(ne, x, (const int2*)ij.ptr, (const double*)meas.ptr, (const double*)info.ptr,
                                                        delta, (double*)blk.ptr);
  RB200_CUDA(cudaGetLastError());
  launches++;
  return 0;
}

int PoseEdges::chi2(const double* x, double* part, double* per_edge, cudaStream_t st, int64_t& launches) const {
  if (ne == 0) return 0;
  pg_chi2_kernel<<<chi2_blocks(), 256, 0, st>>>(ne, x, (const int2*)ij.ptr, (const double*)meas.ptr, (const double*)info.ptr, delta,
                                                part, per_edge);
  RB200_CUDA(cudaGetLastError());
  launches++;
  return 0;
}

cudaError_t pg_launch_update(int nv, const double* xin, const double* dlt, const uint8_t* fixed, double* xout, cudaStream_t st) {
  pg_update_kernel<<<(nv + 127) / 128, 128, 0, st>>>(nv, xin, dlt, fixed, xout);
  return cudaGetLastError();
}

// ---- the pose-graph solver
struct PgDevice {
  PoseEdges edges;
  DevBuf x, xtrial, fixed, Hd, b, Minv, dx, r, sv, d, q, part, result, chipart, maxpart, per_edge, incblk;
  ~PgDevice() {
    DevBuf* all[] = {&x, &xtrial, &fixed, &Hd, &b, &Minv, &dx, &r, &sv, &d, &q, &part, &result, &chipart, &maxpart, &per_edge, &incblk};
    for (DevBuf* bb : all) bb->release();
  }
};

// The solver's device buffers live for the lifetime of the library (grow-only): a cudaMalloc / cudaFree pair per buffer and call
// costs far more than the solve itself once the process holds gigabytes of pinned memory (measured: ~200 ms of cudaFree per call
// in the 2000-frame sequence run against 30 ms inside the PCG kernels).  Guarded by the state mutex like every entry point.
static PgDevice* g_pg_dev = nullptr;
void posegraph_release() {
  delete g_pg_dev;
  g_pg_dev = nullptr;
}

struct PgCtx {
  PgDevice& dev;
  explicit PgCtx(PgDevice& d) : dev(d) {}
  int nv = 0;
  cudaStream_t st = nullptr;
  int pcg_grid = 0;
  int64_t launches = 0;
  int cg_iters = 0;
  double pcg_residual = -1.0;  // LinearSolverPCG::_residual
  // resident solver (pg_pcg_resident_kernel): vertices per CTA, shared-memory capacity in incidences, dynamic bytes; vpc == 0: off
  int res_vpc = 0, res_cap = 0, res_smem = 0;
};

static int pg_errors(PgCtx& c, const double* dx_poses, double* robust, double* plain, double* per_edge) {
  const PoseEdges& E = c.dev.edges;
  const int nb = E.chi2_blocks();
  if (E.ne == 0) {
    *robust = *plain = 0;
    return 0;
  }
  if (int rc = E.chi2(dx_poses, (double*)c.dev.chipart.ptr, per_edge, c.st, c.launches)) return rc;
  std::vector<double> part(2 * (size_t)nb);
  RB200_CUDA(cudaMemcpyAsync(part.data(), c.dev.chipart.ptr, sizeof(double) * 2 * nb, cudaMemcpyDeviceToHost, c.st));
  RB200_CUDA(cudaStreamSynchronize(c.st));
  double r = 0, p = 0;
  for (int i = 0; i < nb; i++) {
    r += part[2 * i];
    p += part[2 * i + 1];
  }
  *robust = r;
  *plain = p;
  return 0;
}

static int pg_build(PgCtx& c, double* maxdiag) {
  const PoseEdges& E = c.dev.edges;
  if (int rc = c.dev.edges.linearize((const double*)c.dev.x.ptr, c.st, c.launches)) return rc;
  const int nb = (c.nv + 2) / 3;
  pg_assemble_kernel<<<nb, 128, 0, c.st>>>(c.nv, (const int*)E.off.ptr, (const int*)E.inc.ptr, (const uint8_t*)c.dev.fixed.ptr,
                                           (const double*)E.blk.ptr, (double*)c.dev.Hd.ptr, (double*)c.dev.b.ptr,
                                           (double*)c.dev.maxpart.ptr);
  RB200_CUDA(cudaGetLastError());
  c.launches++;
  if (c.res_vpc > 0 && E.ne > 0) {
    pg_orient_kernel<<<(c.nv + 3) / 4, 128, 0, c.st>>>(c.nv, (const int*)E.off.ptr, (const int*)E.inc.ptr, (const int*)E.oth.ptr,
                                                       (const double*)E.blk.ptr, (double*)c.dev.incblk.ptr);
    RB200_CUDA(cudaGetLastError());
    c.launches++;
  }
  if (maxdiag) {
    std::vector<double> part(nb);
    RB200_CUDA(cudaMemcpyAsync(part.data(), c.dev.maxpart.ptr, sizeof(double) * nb, cudaMemcpyDeviceToHost, c.st));
    RB200_CUDA(cudaStreamSynchronize(c.st));
    double m = 0;
    for (double v : part) m = v > m ? v : m;
    *maxdiag = m;
  }
  return 0;
}

static int pg_pcg(PgCtx& c, double lambda, double* scale, bool* ok) {
  PcgArgs a;
  const PoseEdges& E = c.dev.edges;
  a.nv = c.nv;
  a.ne = E.ne;
  a.off = (const int*)E.off.ptr;
  a.inc = (const int*)E.inc.ptr;
  a.oth = (const int*)E.oth.ptr;
  a.ij = (const int2*)E.ij.ptr;
  a.fixed = (const uint8_t*)c.dev.fixed.ptr;
  a.blk = (const double*)E.blk.ptr;
  a.Hd = (const double*)c.dev.Hd.ptr;
  a.b = (const double*)c.dev.b.ptr;
  a.Minv = (double*)c.dev.Minv.ptr;
  a.x = (double*)c.dev.dx.ptr;
  a.r = (double*)c.dev.r.ptr;
  a.d = (double*)c.dev.d.ptr;
  a.q = (double*)c.dev.q.ptr;
  a.s = (double*)c.dev.sv.ptr;
  a.part = (double*)c.dev.part.ptr;
  a.result = (double*)c.dev.result.ptr;
  a.lambda = lambda;
  a.tol = (c.pcg_residual > 0.0 && c.pcg_residual > 1e-6) ? c.pcg_residual : 1e-6;
  a.maxit = 6 * c.nv;
  void* args[] = {&a};
  pg_precond_kernel<<<(c.nv + 127) / 128, 128, 0, c.st>>>(c.nv, a.Hd, a.fixed, lambda, a.Minv);
  RB200_CUDA(cudaGetLastError());
  c.launches++;
  if (c.res_vpc > 0) {
    RB200_CUDA(cudaMemsetAsync(c.dev.part.ptr, 0xFF, 8 * (size_t)kPgBarrierDoubles, c.st));  // barrier slots: parity 1
    const double* incblk = (const double*)c.dev.incblk.ptr;
    void* rargs[] = {&a, &incblk, &c.res_vpc, &c.res_cap};
    RB200_CUDA(cudaLaunchCooperativeKernel((void*)pg_pcg_resident_kernel, dim3(c.pcg_grid), dim3(kPgResWarps * 32), rargs,
                                        (size_t)c.res_smem, c.st));
  } else {
    RB200_CUDA(cudaLaunchCooperativeKernel((void*)pg_pcg_kernel, dim3(c.pcg_grid), dim3(512), args, 0, c.st));
  }
  c.launches++;
  double res[4];
  RB200_CUDA(cudaMemcpyAsync(res, c.dev.result.ptr, sizeof(res), cudaMemcpyDeviceToHost, c.st));
  RB200_CUDA(cudaStreamSynchronize(c.st));
  c.cg_iters += (int)res[0];
  c.pcg_residual = 0.5 * res[1];
  *scale = res[2];
  *ok = res[3] == 0.0;
  return 0;
}

// SparseOptimizer::optimize(iterations); every iteration starts by re-evaluating the chi2 (computeActiveErrors)
static int pg_optimize(PgCtx& c, int iterations, int* done) {
  PgDevice& d = c.dev;
  double chi2 = 0, plain;
  auto linearize = [&](double& cur, double* maxdiag) {
    const int rc = pg_errors(c, (const double*)d.x.ptr, &cur, &plain, nullptr);
    return rc ? rc : pg_build(c, maxdiag);
  };
  auto trial = [&](double lambda, double& temp, double& scale, bool& ok) {
    if (int rc = pg_pcg(c, lambda, &scale, &ok)) return rc;
    RB200_CUDA(pg_launch_update(c.nv, (const double*)d.x.ptr, (const double*)d.dx.ptr, (const uint8_t*)d.fixed.ptr,
                                (double*)d.xtrial.ptr, c.st));
    c.launches++;
    return pg_errors(c, (const double*)d.xtrial.ptr, &temp, &plain, nullptr);
  };
  return lm_optimize(iterations, chi2, done, linearize, trial, [&] { std::swap(d.x, d.xtrial); });
}

// grow-only device buffers of a solve with nv vertices and ne edges (rgbdslam_b200_posegraph_reserve: a caller that knows how
// large its graph will get takes the allocations out of its first solve)
static int pg_ensure(PgDevice& d, int nv, int ne) {
  int rc;
  const size_t nv_ = (size_t)(nv > 0 ? nv : 1), ne_ = (size_t)(ne > 0 ? ne : 1);
  const int chi_blocks = (ne + 255) / 256 + 1, max_blocks = (nv + 2) / 3 + 1;
  if ((rc = d.edges.ensure(nv, ne)) || (rc = d.x.ensure(56 * nv_)) || (rc = d.xtrial.ensure(56 * nv_)) || (rc = d.fixed.ensure(nv_)) ||
      (rc = d.Hd.ensure(288 * nv_)) || (rc = d.b.ensure(48 * nv_)) || (rc = d.Minv.ensure(288 * nv_)) || (rc = d.dx.ensure(48 * nv_)) ||
      (rc = d.r.ensure(48 * nv_)) || (rc = d.d.ensure(48 * nv_)) || (rc = d.q.ensure(48 * nv_)) || (rc = d.sv.ensure(48 * nv_)) ||
      (rc = d.result.ensure(128)) || (rc = d.chipart.ensure(16 * (size_t)chi_blocks)) ||
      (rc = d.maxpart.ensure(8 * (size_t)max_blocks)) || (rc = d.per_edge.ensure(8 * ne_)) || (rc = d.incblk.ensure(288 * 2 * ne_)))
    return rc;
  return 0;
}
int posegraph_reserve(int nv, int ne) {
  if (!g_pg_dev) g_pg_dev = new PgDevice();
  return pg_ensure(*g_pg_dev, nv, ne);
}

int posegraph_optimize(int nv, double* poses, const uint8_t* fixed, int ne, const int32_t* ij, const double* meas,
                       const double* info, double stop, double huber_delta, double* chi2_out, int* iters_out, int* cg_iters_out) {
  State& s = g_state;
  if (!g_pg_dev) g_pg_dev = new PgDevice();
  PgDevice& d = *g_pg_dev;
  PgCtx c(d);
  c.nv = nv;
  c.st = s.stream;
  int rc;
  if ((rc = d.edges.upload(nv, ne, ij, meas, info, huber_delta, true, c.st))) return rc;
  if ((rc = pg_ensure(d, nv, ne))) return rc;
  // cooperative grid: all co-resident blocks of the PCG kernel
  int per_sm = 0;
  RB200_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, pg_pcg_kernel, 512, 0));
  if (per_sm < 1) {
    set_error("posegraph: PCG kernel cannot be made resident");
    return RGBDSLAM_B200_ERR_CUDA;
  }
  c.pcg_grid = s.sm_count;  // one 512-thread CTA per SM: the barrier cost grows with the CTA count, the work per iteration is tiny
  if ((rc = d.part.ensure(16 * (size_t)c.pcg_grid + 8 * (size_t)kPgBarrierDoubles))) return rc;
  {
    // resident solver when every vertex gets its own 6-lane group (RB200_PG_RESIDENT=0 forces the general kernel)
    const char* env = std::getenv("RB200_PG_RESIDENT");
    const int vpc = (nv + c.pcg_grid - 1) / c.pcg_grid;
    if (!(env && env[0] == '0') && nv > 0 && vpc <= kPgResSlots && c.pcg_grid <= 32 * kPgGroup) {
      const std::vector<int>& off = d.edges.h_off;
      int max_inc = 0;
      for (int v0 = 0; v0 < nv; v0 += vpc) {
        const int v1 = v0 + vpc < nv ? v0 + vpc : nv;
        max_inc = std::max(max_inc, off[v1] - off[v0]);
      }
      const int cap_max = (200 * 1024 - 128) / 360;  // 36 + 6 doubles + 6 source indices per incidence
      c.res_cap = max_inc < cap_max ? max_inc : cap_max;
      c.res_smem = 128 + 360 * c.res_cap;
      c.res_smem = (c.res_smem + 15) & ~15;
      static int attr_bytes = 0;
      if (c.res_smem > attr_bytes) {
        RB200_CUDA(cudaFuncSetAttribute(pg_pcg_resident_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024 + 16));
        attr_bytes = 200 * 1024 + 16;
      }
      int per_sm_res = 0;
      RB200_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm_res, pg_pcg_resident_kernel, kPgResWarps * 32, (size_t)c.res_smem));
      if (per_sm_res >= 1) {
        c.res_vpc = vpc;
      }
    }
  }
  cudaStream_t st = c.st;
  RB200_CUDA(cudaMemcpyAsync(d.x.ptr, poses, 56 * (size_t)nv, cudaMemcpyHostToDevice, st));
  RB200_CUDA(cudaMemcpyAsync(d.fixed.ptr, fixed, (size_t)nv, cudaMemcpyHostToDevice, st));
  RB200_CUDA(cudaStreamSynchronize(st));

  // graph_manager.cpp:998-1014
  int it = 0;
  double chi2 = DBL_MAX, robust = 0;
  if (stop >= 1.0) {
    const int step = (int)std::ceil(stop / 10);
    do {
      int done = 0;
      if ((rc = pg_optimize(c, step, &done))) return rc;
      it += done;
    } while (it < stop && it > 0);
    if ((rc = pg_errors(c, (const double*)d.x.ptr, &robust, &chi2, nullptr))) return rc;
  } else {
    double prev;
    do {
      prev = chi2;
      int done = 0;
      if ((rc = pg_optimize(c, 5, &done))) return rc;
      it += done;
      if ((rc = pg_errors(c, (const double*)d.x.ptr, &robust, &chi2, nullptr))) return rc;
    } while (chi2 / prev < (1.0 - stop));
  }
  RB200_CUDA(cudaMemcpyAsync(poses, d.x.ptr, 56 * (size_t)nv, cudaMemcpyDeviceToHost, st));
  RB200_CUDA(cudaStreamSynchronize(st));
  if (chi2_out) *chi2_out = chi2;
  if (iters_out) *iters_out = it;
  if (cg_iters_out) *cg_iters_out = c.cg_iters;
  s.launches += c.launches;
  return 0;
}

int posegraph_chi2(int nv, const double* poses, int ne, const int32_t* ij, const double* meas, const double* info,
                   double huber_delta, double* chi2_out, double* per_edge_chi2) {
  State& s = g_state;
  if (!g_pg_dev) g_pg_dev = new PgDevice();
  PgDevice& d = *g_pg_dev;
  PgCtx c(d);
  c.nv = nv;
  c.st = s.stream;
  int rc;
  if ((rc = d.edges.upload(nv, ne, ij, meas, info, huber_delta, false, c.st))) return rc;
  if ((rc = pg_ensure(d, nv, ne))) return rc;
  RB200_CUDA(cudaMemcpyAsync(d.x.ptr, poses, 56 * (size_t)nv, cudaMemcpyHostToDevice, c.st));
  double robust, chi2;
  if ((rc = pg_errors(c, (const double*)d.x.ptr, &robust, &chi2, per_edge_chi2 ? (double*)d.per_edge.ptr : nullptr))) return rc;
  if (per_edge_chi2 && ne > 0)
    RB200_CUDA(cudaMemcpyAsync(per_edge_chi2, d.per_edge.ptr, 8 * (size_t)ne, cudaMemcpyDeviceToHost, c.st));
  RB200_CUDA(cudaStreamSynchronize(c.st));
  if (chi2_out) *chi2_out = chi2;
  s.launches += c.launches;
  return 0;
}

}  // namespace rb200
