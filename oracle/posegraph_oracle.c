/*
 * posegraph_oracle.c -- CPU ORACLE (test infrastructure, NOT product code) for the pose-graph solve:
 * GraphManager::optimizeGraph / optimizeGraphImpl (src/graph_manager.cpp:900-1066) with the optimizer
 * built by createOptimizer (src/graph_manager.cpp:107-201): g2o::OptimizationAlgorithmLevenberg over
 * BlockSolver<6,3> with LinearSolverPCG (backend_solver "pcg", parameter_server.cpp:123), EdgeSE3 edges
 * with a shared RobustKernelHuber(delta = 1) (graph_manager.cpp:867-876, graph_manager.h:382), vertex
 * fixation per fixationOfVertices (graph_manager.cpp:911-937).
 *
 * PARITY STATUS: "parity unpinned".  g2o is an un-vendored dependency (fork felixendres/g2o, branch c++03,
 * no commit pinned -- install.sh:42) and is absent here; there are no golden vectors.  The published g2o
 * algorithms are restated (SURVEY.md appendix D):
 *   EdgeSE3::computeError      e = toVectorMQT(Z^-1 * Xi^-1 * Xj)  (t, then qx,qy,qz with w >= 0)
 *   VertexSE3::oplusImpl       X <- X * fromVectorMQT(delta)
 *   RobustKernelHuber          rho(e2) = e2 | 2*sqrt(e2)*d - d^2 ; weight = 1 | d/sqrt(e2)
 *   OptimizationAlgorithmLevenberg::solve  (lambda_init = 1e-5 * max diag H, nu doubling, <=10 trials,
 *                              rho = (chi_old - chi_new) / (x^T(lambda x + b) + 1e-3), lambda *= clamp(1-(2rho-1)^3, 1/3, 2/3))
 *   LinearSolverPCG            CG with block-Jacobi preconditioner, stop when r^T M^-1 r <= d0 with
 *                              d0 = max(1e-6, 0.5 * final r^T M^-1 r of the previous solve) (absolute tolerance
 *                              mode, _residual carried between solves), max iterations = matrix dimension,
 *                              residual updated recursively (the periodic reset is a TODO in g2o)
 * The Jacobians are the exact derivatives of that error under that oplus (g2o uses the same, analytically);
 * tests/test_posegraph_oracle.py checks them against finite differences and the converged solution against an
 * independent scipy sparse Gauss-Newton.
 *
 * Pose / measurement format: 7 doubles (tx,ty,tz,qx,qy,qz,qw), the g2o VERTEX_SE3:QUAT / TUM trajectory order
 * (src/misc.cpp:90-93 logTransform).
 */
#include <math.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>
#include <float.h>

typedef struct {
  double R[9]; /* row-major */
  double t[3];
} iso_t;

static void quat_to_R(const double* q /* x y z w */, double* R) {
  double x = q[0], y = q[1], z = q[2], w = q[3];
  double n = sqrt(x * x + y * y + z * z + w * w);
  x /= n; y /= n; z /= n; w /= n;
  R[0] = 1 - 2 * (y * y + z * z); R[1] = 2 * (x * y - z * w);     R[2] = 2 * (x * z + y * w);
  R[3] = 2 * (x * y + z * w);     R[4] = 1 - 2 * (x * x + z * z); R[5] = 2 * (y * z - x * w);
  R[6] = 2 * (x * z - y * w);     R[7] = 2 * (y * z + x * w);     R[8] = 1 - 2 * (x * x + y * y);
}

static void quat_mul(const double* a, const double* b, double* o) { /* (x y z w) Hamilton product a*b */
  double ax = a[0], ay = a[1], az = a[2], aw = a[3], bx = b[0], by = b[1], bz = b[2], bw = b[3];
  o[0] = aw * bx + ax * bw + ay * bz - az * by;
  o[1] = aw * by - ax * bz + ay * bw + az * bx;
  o[2] = aw * bz + ax * by - ay * bx + az * bw;
  o[3] = aw * bw - ax * bx - ay * by - az * bz;
}
static void quat_conj(const double* a, double* o) { o[0] = -a[0]; o[1] = -a[1]; o[2] = -a[2]; o[3] = a[3]; }
static void quat_normalize(double* q) {
  double n = sqrt(q[0] * q[0] + q[1] * q[1] + q[2] * q[2] + q[3] * q[3]);
  for (int i = 0; i < 4; i++) q[i] /= n;
}

/* EdgeSE3::computeError + exact Jacobians.  xi, xj, z: 7-vectors (t, q).  e[6], Ji[36], Jj[36] row-major. */
void oracle_edge_se3(const double* xi, const double* xj, const double* z, double* e, double* Ji, double* Jj) {
  double Ri[9], Rz[9], Rj[9];
  quat_to_R(xi + 3, Ri);
  quat_to_R(xj + 3, Rj);
  quat_to_R(z + 3, Rz);
  /* tb = Ri^T (tj - ti);  Rb = Ri^T Rj */
  double d[3] = {xj[0] - xi[0], xj[1] - xi[1], xj[2] - xi[2]};
  double tb[3], Rb[9];
  for (int r = 0; r < 3; r++) tb[r] = Ri[0 + r] * d[0] + Ri[3 + r] * d[1] + Ri[6 + r] * d[2];
  for (int r = 0; r < 3; r++)
    for (int c = 0; c < 3; c++) Rb[3 * r + c] = Ri[0 + r] * Rj[0 + c] + Ri[3 + r] * Rj[3 + c] + Ri[6 + r] * Rj[6 + c];
  /* te = Rz^T (tb - tz) ; Ra = Rz^T */
  double dd[3] = {tb[0] - z[0], tb[1] - z[1], tb[2] - z[2]};
  for (int r = 0; r < 3; r++) e[r] = Rz[0 + r] * dd[0] + Rz[3 + r] * dd[1] + Rz[6 + r] * dd[2];
  /* qe = qz^* qi^* qj */
  double qi[4] = {xi[3], xi[4], xi[5], xi[6]}, qj[4] = {xj[3], xj[4], xj[5], xj[6]}, qz[4] = {z[3], z[4], z[5], z[6]};
  quat_normalize(qi); quat_normalize(qj); quat_normalize(qz);
  double qic[4], qzc[4], tmp[4], qe[4];
  quat_conj(qi, qic); quat_conj(qz, qzc);
  quat_mul(qzc, qic, tmp);
  quat_mul(tmp, qj, qe);
  quat_normalize(qe);
  if (qe[3] < 0) for (int k = 0; k < 4; k++) qe[k] = -qe[k];
  e[3] = qe[0]; e[4] = qe[1]; e[5] = qe[2];
  if (!Ji) return;
  const double we = qe[3], vx = qe[0], vy = qe[1], vz = qe[2];
  /* Q = we I + [ve]x */
  double Q[9] = {we, -vz, vy, vz, we, -vx, -vy, vx, we};
  double Ra[9];
  for (int r = 0; r < 3; r++) for (int c = 0; c < 3; c++) Ra[3 * r + c] = Rz[3 * c + r];
  double Re[9];
  for (int r = 0; r < 3; r++) for (int c = 0; c < 3; c++) Re[3 * r + c] = Ra[3 * r] * Rb[c] + Ra[3 * r + 1] * Rb[3 + c] + Ra[3 * r + 2] * Rb[6 + c];
  memset(Ji, 0, 36 * sizeof(double));
  memset(Jj, 0, 36 * sizeof(double));
  double Tx[9] = {0, -tb[2], tb[1], tb[2], 0, -tb[0], -tb[1], tb[0], 0};
  for (int r = 0; r < 3; r++)
    for (int c = 0; c < 3; c++) {
      Ji[6 * r + c] = -Ra[3 * r + c];                                                                      /* d te / d ti */
      Ji[6 * r + 3 + c] = 2.0 * (Ra[3 * r] * Tx[c] + Ra[3 * r + 1] * Tx[3 + c] + Ra[3 * r + 2] * Tx[6 + c]); /* d te / d qi */
      Ji[6 * (3 + r) + 3 + c] = -(Q[3 * r] * Rb[3 * c] + Q[3 * r + 1] * Rb[3 * c + 1] + Q[3 * r + 2] * Rb[3 * c + 2]); /* -Q Rb^T */
      Jj[6 * r + c] = Re[3 * r + c];                                                                       /* d te / d tj */
      Jj[6 * (3 + r) + 3 + c] = Q[3 * r + c];                                                              /* d qe / d qj */
    }
}

/* VertexSE3::oplusImpl: X <- X * fromVectorMQT(delta) */
void oracle_vertex_oplus(double* x, const double* dlt) {
  double R[9];
  quat_to_R(x + 3, R);
  for (int r = 0; r < 3; r++) x[r] += R[3 * r] * dlt[0] + R[3 * r + 1] * dlt[1] + R[3 * r + 2] * dlt[2];
  double w = 1.0 - (dlt[3] * dlt[3] + dlt[4] * dlt[4] + dlt[5] * dlt[5]);
  if (w < 0) return; /* fromCompactQuaternion: identity rotation */
  double dq[4] = {dlt[3], dlt[4], dlt[5], sqrt(w)}, q[4] = {x[3], x[4], x[5], x[6]}, o[4];
  quat_mul(q, dq, o);
  quat_normalize(o);
  memcpy(x + 3, o, sizeof(o));
}

typedef struct {
  int nv, ne;
  const uint8_t* fixed;
  const int32_t* ij;
  const double* meas;
  const double* info;
  double delta;
  /* linear system */
  double* Hd;  /* nv x 36 */
  double* Ho;  /* ne x 36: Ji^T W Jj */
  double* b;   /* nv x 6 */
  double* Minv; /* nv x 36 block-Jacobi */
  double pcg_residual; /* LinearSolverPCG::_residual (-1 initially) */
  /* trace of one LM iteration (oracle_posegraph_lm_trace; NULL elsewhere), per trial t: tr_trial[8 t ..] = lambda, PCG
   * tolerance, PCG iterations, computeScale, trial chi2 (robust), rho, accepted, PCG ok; tr_dx[6 nv t ..] the PCG step;
   * tr_dn[(6 nv + 1) t + k] = r^T M^-1 r before PCG iteration k (k = 0 .. iterations) */
  double *tr_trial, *tr_dx, *tr_dn;
  int tr_n;
  double* babs; /* nv x 6: sum of |terms| of b (oracle_posegraph_system; NULL elsewhere) */
} pg_t;

static void mat6_AtWB(const double* A, const double* W, const double* B, double s, double* out /* += s*A^T W B */) {
  double WB[36];
  for (int r = 0; r < 6; r++)
    for (int c = 0; c < 6; c++) {
      double a = 0;
      for (int k = 0; k < 6; k++) a += W[6 * r + k] * B[6 * k + c];
      WB[6 * r + c] = a;
    }
  for (int r = 0; r < 6; r++)
    for (int c = 0; c < 6; c++) {
      double a = 0;
      for (int k = 0; k < 6; k++) a += A[6 * k + r] * WB[6 * k + c];
      out[6 * r + c] += s * a;
    }
}

/* returns robust chi2 (sum rho0) and plain chi2 (sum e^T W e) */
static void pg_errors(const pg_t* g, const double* x, double* robust, double* plain) {
  double r = 0, p = 0;
  for (int k = 0; k < g->ne; k++) {
    int i = g->ij[2 * k], j = g->ij[2 * k + 1];
    double e[6];
    oracle_edge_se3(x + 7 * i, x + 7 * j, g->meas + 7 * k, e, NULL, NULL);
    const double* W = g->info + 36 * k;
    double e2 = 0;
    for (int a = 0; a < 6; a++) for (int c = 0; c < 6; c++) e2 += e[a] * W[6 * a + c] * e[c];
    p += e2;
    double d2 = g->delta * g->delta;
    r += (e2 <= d2) ? e2 : 2 * sqrt(e2) * g->delta - d2;
  }
  *robust = r;
  *plain = p;
}

static void pg_build(pg_t* g, const double* x) {
  memset(g->Hd, 0, sizeof(double) * 36 * g->nv);
  memset(g->b, 0, sizeof(double) * 6 * g->nv);
  for (int k = 0; k < g->ne; k++) {
    int i = g->ij[2 * k], j = g->ij[2 * k + 1];
    double e[6], Ji[36], Jj[36];
    oracle_edge_se3(x + 7 * i, x + 7 * j, g->meas + 7 * k, e, Ji, Jj);
    const double* W = g->info + 36 * k;
    double We[6], e2 = 0;
    for (int a = 0; a < 6; a++) {
      We[a] = 0;
      for (int c = 0; c < 6; c++) We[a] += W[6 * a + c] * e[c];
      e2 += e[a] * We[a];
    }
    double w = (e2 <= g->delta * g->delta) ? 1.0 : g->delta / sqrt(e2);
    mat6_AtWB(Ji, W, Ji, w, g->Hd + 36 * i);
    mat6_AtWB(Jj, W, Jj, w, g->Hd + 36 * j);
    memset(g->Ho + 36 * k, 0, 36 * sizeof(double));
    mat6_AtWB(Ji, W, Jj, w, g->Ho + 36 * k);
    for (int c = 0; c < 6; c++) {
      double si = 0, sj = 0;
      for (int a = 0; a < 6; a++) { si += Ji[6 * a + c] * We[a]; sj += Jj[6 * a + c] * We[a]; }
      g->b[6 * i + c] -= w * si;
      g->b[6 * j + c] -= w * sj;
      if (g->babs) {
        g->babs[6 * i + c] += fabs(w * si);
        g->babs[6 * j + c] += fabs(w * sj);
      }
    }
  }
}

static void pg_spmv(const pg_t* g, double lambda, const double* v, double* out) {
  for (int i = 0; i < g->nv; i++)
    for (int r = 0; r < 6; r++) {
      double a = 0;
      if (!g->fixed[i]) {
        for (int c = 0; c < 6; c++) a += g->Hd[36 * i + 6 * r + c] * v[6 * i + c];
        a += lambda * v[6 * i + r];
      }
      out[6 * i + r] = a;
    }
  for (int k = 0; k < g->ne; k++) {
    int i = g->ij[2 * k], j = g->ij[2 * k + 1];
    if (g->fixed[i] || g->fixed[j] || i == j) continue;
    const double* C = g->Ho + 36 * k;
    for (int r = 0; r < 6; r++)
      for (int c = 0; c < 6; c++) {
        out[6 * i + r] += C[6 * r + c] * v[6 * j + c];
        out[6 * j + c] += C[6 * r + c] * v[6 * i + r];
      }
  }
}

static int inv6(const double* A, double* Ai) { /* Gauss-Jordan with partial pivoting */
  double M[6][12];
  for (int r = 0; r < 6; r++) for (int c = 0; c < 6; c++) { M[r][c] = A[6 * r + c]; M[r][6 + c] = (r == c); }
  for (int c = 0; c < 6; c++) {
    int p = c;
    for (int r = c + 1; r < 6; r++) if (fabs(M[r][c]) > fabs(M[p][c])) p = r;
    if (fabs(M[p][c]) < 1e-300) return 0;
    if (p != c) for (int k = 0; k < 12; k++) { double t = M[c][k]; M[c][k] = M[p][k]; M[p][k] = t; }
    double d = M[c][c];
    for (int k = 0; k < 12; k++) M[c][k] /= d;
    for (int r = 0; r < 6; r++) if (r != c) { double f = M[r][c]; if (f != 0) for (int k = 0; k < 12; k++) M[r][k] -= f * M[c][k]; }
  }
  for (int r = 0; r < 6; r++) for (int c = 0; c < 6; c++) Ai[6 * r + c] = M[r][6 + c];
  return 1;
}

/* LinearSolverPCG: solve (H + lambda I) x = b on the free vertices.  Returns iterations (<0 on breakdown). */
static int pg_pcg(pg_t* g, double lambda, double* x, int* iters_out) {
  const int n = 6 * g->nv;
  double* r = (double*)malloc(sizeof(double) * n * 4);
  double *d = r + n, *q = d + n, *s = q + n;
  for (int i = 0; i < g->nv; i++) {
    double A[36];
    memcpy(A, g->Hd + 36 * i, sizeof(A));
    for (int k = 0; k < 6; k++) A[7 * k] += lambda;
    if (g->fixed[i] || !inv6(A, g->Minv + 36 * i)) memset(g->Minv + 36 * i, 0, 36 * sizeof(double));
  }
  memset(x, 0, sizeof(double) * n);
  for (int i = 0; i < n; i++) r[i] = g->fixed[i / 6] ? 0.0 : g->b[i];
  double dn = 0;
  for (int i = 0; i < g->nv; i++)
    for (int a = 0; a < 6; a++) {
      double v = 0;
      for (int c = 0; c < 6; c++) v += g->Minv[36 * i + 6 * a + c] * r[6 * i + c];
      d[6 * i + a] = v;
      dn += r[6 * i + a] * v;
    }
  const double tol = (g->pcg_residual > 0.0 && g->pcg_residual > 1e-6) ? g->pcg_residual : 1e-6;
  int it = 0, maxit = n;
  int ok = 1;
  double* trace = g->tr_dn ? g->tr_dn + (size_t)g->tr_n * (n + 1) : NULL;
  if (g->tr_trial) g->tr_trial[8 * g->tr_n + 1] = tol;
  for (; it < maxit; it++) {
    if (trace) trace[it] = dn;
    if (dn <= tol) break;
    pg_spmv(g, lambda, d, q);
    double dq = 0;
    for (int i = 0; i < n; i++) dq += d[i] * q[i];
    if (!(dq > 0)) { ok = 0; break; }
    double alpha = dn / dq;
    for (int i = 0; i < n; i++) x[i] += alpha * d[i];
    for (int i = 0; i < n; i++) r[i] -= alpha * q[i]; /* g2o: "TODO: reset residual here every 50 iterations" (not done) */
    double dold = dn;
    dn = 0;
    for (int i = 0; i < g->nv; i++)
      for (int a = 0; a < 6; a++) {
        double v = 0;
        for (int c = 0; c < 6; c++) v += g->Minv[36 * i + 6 * a + c] * r[6 * i + c];
        s[6 * i + a] = v;
        dn += r[6 * i + a] * v;
      }
    double beta = dn / dold;
    for (int i = 0; i < n; i++) d[i] = s[i] + beta * d[i];
  }
  if (trace && it == maxit) trace[it] = dn;
  free(r);
  g->pcg_residual = 0.5 * dn;
  if (iters_out) *iters_out += it;
  return ok;
}

typedef struct {
  double lambda, ni;
} lm_state_t;

/* OptimizationAlgorithmLevenberg::solve(iteration).  Returns 1 = OK, 0 = Terminate. */
static int pg_lm_solve(pg_t* g, double* x, int iteration, lm_state_t* st, int* cg_iters) {
  const int n = 6 * g->nv;
  double cur, plain;
  pg_errors(g, x, &cur, &plain);
  double temp = cur;
  pg_build(g, x);
  if (iteration == 0) {
    double mx = 0;
    for (int i = 0; i < g->nv; i++)
      if (!g->fixed[i]) for (int k = 0; k < 6; k++) mx = fmax(mx, fabs(g->Hd[36 * i + 7 * k]));
    st->lambda = 1e-5 * mx;
    st->ni = 2;
  }
  double* dx = (double*)malloc(sizeof(double) * n);
  double* backup = (double*)malloc(sizeof(double) * 7 * g->nv);
  double rho = 0;
  int qmax = 0;
  do {
    memcpy(backup, x, sizeof(double) * 7 * g->nv);
    const double lambda = st->lambda;
    const int cg0 = *cg_iters;
    int ok2 = pg_pcg(g, st->lambda, dx, cg_iters);
    for (int i = 0; i < g->nv; i++) if (!g->fixed[i]) oracle_vertex_oplus(x + 7 * i, dx + 6 * i);
    pg_errors(g, x, &temp, &plain);
    if (!ok2) temp = DBL_MAX;
    rho = cur - temp;
    double scale = 0;
    for (int i = 0; i < n; i++) if (!g->fixed[i / 6]) scale += dx[i] * (st->lambda * dx[i] + g->b[i]);
    if (g->tr_trial) {
      double* t = g->tr_trial + 8 * g->tr_n;
      t[0] = lambda; t[2] = *cg_iters - cg0; t[3] = scale; t[4] = temp; t[5] = rho / (scale + 1e-3);
      t[6] = rho / (scale + 1e-3) > 0 && isfinite(temp); t[7] = ok2;
      memcpy(g->tr_dx + (size_t)n * g->tr_n, dx, sizeof(double) * n);
      g->tr_n++;
    }
    scale += 1e-3;
    rho /= scale;
    if (rho > 0 && isfinite(temp)) {
      double alpha = 1. - pow(2 * rho - 1, 3);
      alpha = fmin(alpha, 2. / 3.);
      double sf = fmax(1. / 3., alpha);
      st->lambda *= sf;
      st->ni = 2;
      cur = temp;
    } else {
      st->lambda *= st->ni;
      st->ni *= 2;
      memcpy(x, backup, sizeof(double) * 7 * g->nv);
      if (!isfinite(st->lambda)) break;
    }
    qmax++;
  } while (rho < 0 && qmax < 10);
  free(dx);
  free(backup);
  if (qmax == 10 || rho == 0) return 0;
  return 1;
}

static int pg_optimize(pg_t* g, double* x, int iterations, int* cg_iters) { /* SparseOptimizer::optimize */
  lm_state_t st = {0, 2};
  int cj = 0;
  for (int i = 0; i < iterations; i++) {
    int ok = pg_lm_solve(g, x, i, &st, cg_iters);
    cj++;
    if (!ok) break;
  }
  return cj;
}

static void pg_init(pg_t* g, int nv, const uint8_t* fixed, int ne, const int32_t* ij, const double* meas, const double* info,
                    double huber_delta) {
  memset(g, 0, sizeof(*g));
  g->nv = nv; g->ne = ne; g->fixed = fixed; g->ij = ij; g->meas = meas; g->info = info; g->delta = huber_delta;
  g->Hd = (double*)malloc(sizeof(double) * 36 * (nv > 0 ? nv : 1));
  g->Ho = (double*)malloc(sizeof(double) * 36 * (ne > 0 ? ne : 1));
  g->b = (double*)malloc(sizeof(double) * 6 * (nv > 0 ? nv : 1));
  g->Minv = (double*)malloc(sizeof(double) * 36 * (nv > 0 ? nv : 1));
  g->pcg_residual = -1.0;
}
static void pg_free(pg_t* g) { free(g->Hd); free(g->Ho); free(g->b); free(g->Minv); }

/* GraphManager::optimizeGraphImpl stop rule (graph_manager.cpp:998-1014).
 * poses: nv x 7 in/out.  stop >= 1: iteration budget; 0 < stop < 1: relative chi2 convergence in chunks of 5.
 * Returns chi2 (sum e^T Omega e, optimizer_->chi2()). */
double oracle_posegraph_optimize(int nv, double* poses, const uint8_t* fixed, int ne, const int32_t* ij, const double* meas,
                                 const double* info, double stop, double huber_delta, int* iters_out, int* cg_iters_out) {
  pg_t g;
  pg_init(&g, nv, fixed, ne, ij, meas, info, huber_delta);
  int it = 0, cg = 0;
  double chi2 = DBL_MAX, robust;
  if (stop >= 1.0) {
    int step = (int)ceil(stop / 10);
    do { it += pg_optimize(&g, poses, step, &cg); } while (it < stop && it > 0);
    pg_errors(&g, poses, &robust, &chi2);
  } else {
    double prev;
    do {
      prev = chi2;
      it += pg_optimize(&g, poses, 5, &cg);
      pg_errors(&g, poses, &robust, &chi2);
    } while (chi2 / prev < (1.0 - stop));
  }
  pg_free(&g);
  if (iters_out) *iters_out = it;
  if (cg_iters_out) *cg_iters_out = cg;
  return chi2;
}

/* One LM iteration exactly as oracle_posegraph_optimize(stop = 1) runs it (ceil(1 / 10) = 1: one pg_optimize(1)), with every
 * trial traced (pg_t.tr_*): trials[10 x 8], dx[10 x 6 nv], dn[10 x (6 nv + 1)] (layouts at pg_t).  poses: nv x 7 in/out.
 * Returns the number of trials; *chi2_out = chi2 of the returned poses, *cg_iters_out = PCG iterations of all trials. */
int oracle_posegraph_lm_trace(int nv, double* poses, const uint8_t* fixed, int ne, const int32_t* ij, const double* meas,
                              const double* info, double huber_delta, double* trials, double* dx, double* dn, double* chi2_out,
                              int* cg_iters_out) {
  pg_t g;
  pg_init(&g, nv, fixed, ne, ij, meas, info, huber_delta);
  g.tr_trial = trials; g.tr_dx = dx; g.tr_dn = dn;
  int cg = 0;
  double robust;
  pg_optimize(&g, poses, 1, &cg);
  pg_errors(&g, poses, &robust, chi2_out);
  pg_free(&g);
  *cg_iters_out = cg;
  return g.tr_n;
}

/* The damped system one PCG solves at the poses: Hd[nv x 36] = H_vv + lambda I for a free vertex (H_vv for a fixed one),
 * Ho[ne x 36] = Ji^T W Jj (Huber-weighted) of every edge, b[nv x 6] = -sum J^T W e and babs[nv x 6] = sum |J^T W e| (both 0 for
 * a fixed vertex).  The PCG's operator is the free rows and columns of that matrix, without the off-diagonal block of a self
 * edge (pg_spmv). */
void oracle_posegraph_system(int nv, const double* poses, const uint8_t* fixed, int ne, const int32_t* ij, const double* meas,
                             const double* info, double huber_delta, double lambda, double* Hd, double* Ho, double* b, double* babs) {
  pg_t g;
  memset(&g, 0, sizeof(g));
  g.nv = nv; g.ne = ne; g.fixed = fixed; g.ij = ij; g.meas = meas; g.info = info; g.delta = huber_delta;
  g.Hd = Hd; g.Ho = Ho; g.b = b; g.babs = babs;
  memset(babs, 0, sizeof(double) * 6 * nv);
  pg_build(&g, poses);
  for (int i = 0; i < nv; i++) {
    if (fixed[i]) { memset(b + 6 * i, 0, 6 * sizeof(double)); memset(babs + 6 * i, 0, 6 * sizeof(double)); continue; }
    for (int k = 0; k < 6; k++) Hd[36 * i + 7 * k] += lambda;
  }
}

/* chi2 only (optimizer_->computeActiveErrors(); chi2()) */
double oracle_posegraph_chi2(int nv, const double* poses, int ne, const int32_t* ij, const double* meas, const double* info,
                             double huber_delta, double* robust_out) {
  pg_t g;
  memset(&g, 0, sizeof(g));
  g.nv = nv; g.ne = ne; g.ij = ij; g.meas = meas; g.info = info; g.delta = huber_delta;
  double r, p;
  pg_errors(&g, poses, &r, &p);
  if (robust_out) *robust_out = r;
  return p;
}
