// Pose graph: ceres' Levenberg-Marquardt on the reference's PoseGraph3dErrorTerm (ceres_pose_graph_3d.hpp:198-352), one CTA, one launch per
// solve.  The host uploads the inputs and the elimination plan (pg_plan.h) once and reads the poses and the summary back once.
//
// Per LM iteration: one thread per edge evaluates its residual and its two 6 x 6 Jacobian blocks (analytic, in the tangent space of each
// endpoint); per free node the diagonal block and the gradient are summed over its edges in ascending edge order; the cost is a fixed-order
// reduction.  The step solve is exact: the odometry segments by block cyclic reduction (pg_block.cuh, every segment and every position of a
// level in parallel), the Schur complement on the border by a dense Cholesky factorization, then back substitution.  Every sum has a fixed
// order, so the same input gives the same bits.  Built -fmad=false, like the oracle (-ffp-contract=off).
#include <cfloat>
#include <cmath>
#include "kernels.cuh"
#include "pg_block.cuh"
#include "pg_plan.h"

#define PG_THREADS 256

struct PgOut { double initial_cost, final_cost, cost; int iterations, evaluations, termination, xi, valid; long long cyc[4]; };

struct PgArgs {
  int N, M, F, nb, n_pos, n_levels, max_iterations, mode; double radius_in;
  const int *ea, *eb, *free_of_node, *free_node, *inc_ptr, *inc, *free_pos, *free_border, *pos_free, *pos_border, *cpl_ptr, *cpl;
  const int *elim_ptr, *elim, *upd_ptr, *upd, *border, *bd_ptr, *bd, *bb_ptr, *bb;
  const double *meas, *sqi;
  double* x[2];
  double *r[2], *ja[2], *jb[2], *ec[2];
  double *eoff, *emod, *H, *g, *scaling, *diag, *Adiag, *rhs, *delta, *D, *C, *b, *Lf, *Wl, *Wr, *y, *xs, *Bm, *Bv, *out_step;
  PgOut* out;
};

// The arena: inputs first (uploaded in one copy from a host image with the same layout), then the work arrays.
struct PgSizes { int N, M, F, n_pos, n_elim, n_upd, n_levels, nb, n_bd, n_bb; };
template <typename Args> static size_t pg_layout(Carve& c, const PgSizes& s, Args& a, size_t* in_bytes) {
  const size_t N = s.N, M = s.M, F = s.F, P = s.n_pos, nb = s.nb;
  a.ea = c.take<int>(M); a.eb = c.take<int>(M); a.free_of_node = c.take<int>(N); a.free_node = c.take<int>(F); a.inc_ptr = c.take<int>(F + 1);
  a.inc = c.take<int>(2 * M); a.free_pos = c.take<int>(F); a.free_border = c.take<int>(F); a.pos_free = c.take<int>(P); a.pos_border = c.take<int>(P);
  a.cpl_ptr = c.take<int>(P + 1); a.cpl = c.take<int>(M); a.elim_ptr = c.take<int>(s.n_levels + 1); a.elim = c.take<int>(3 * (size_t)s.n_elim);
  a.upd_ptr = c.take<int>(s.n_levels + 1); a.upd = c.take<int>(3 * (size_t)s.n_upd); a.border = c.take<int>(nb); a.bd_ptr = c.take<int>(nb * nb + 1);
  a.bd = c.take<int>(3 * (size_t)s.n_bd); a.bb_ptr = c.take<int>(nb + 1); a.bb = c.take<int>(2 * (size_t)s.n_bb);
  a.meas = c.take<double>(7 * M); a.sqi = c.take<double>(36 * M); a.x[0] = c.take<double>(7 * N);
  *in_bytes = c.bytes;
  a.x[1] = c.take<double>(7 * N);
  for (int k = 0; k < 2; k++) { a.r[k] = c.take<double>(6 * M); a.ja[k] = c.take<double>(36 * M); a.jb[k] = c.take<double>(36 * M); a.ec[k] = c.take<double>(M); }
  a.eoff = c.take<double>(36 * M); a.emod = c.take<double>(M);
  a.H = c.take<double>(36 * F); a.g = c.take<double>(6 * F); a.scaling = c.take<double>(6 * F); a.diag = c.take<double>(6 * F); a.Adiag = c.take<double>(36 * F);
  a.rhs = c.take<double>(6 * F); a.delta = c.take<double>(6 * F); a.out_step = c.take<double>(6 * F);
  a.D = c.take<double>(36 * P); a.C = c.take<double>(36 * P); a.b = c.take<double>(6 * P); a.Lf = c.take<double>(36 * P); a.Wl = c.take<double>(36 * P);
  a.Wr = c.take<double>(36 * P); a.y = c.take<double>(6 * P); a.xs = c.take<double>(6 * P);
  a.Bm = c.take<double>(36 * nb * nb); a.Bv = c.take<double>(6 * nb);
  a.out = c.take<PgOut>(1);
  return c.bytes;
}
// Host-side image of the input region: the same layout with writable pointers.
struct PgHostArgs {
  int *ea, *eb, *free_of_node, *free_node, *inc_ptr, *inc, *free_pos, *free_border, *pos_free, *pos_border, *cpl_ptr, *cpl;
  int *elim_ptr, *elim, *upd_ptr, *upd, *border, *bd_ptr, *bd, *bb_ptr, *bb;
  double *meas, *sqi; double* x[2];
  double *r[2], *ja[2], *jb[2], *ec[2];
  double *eoff, *emod, *H, *g, *scaling, *diag, *Adiag, *rhs, *delta, *D, *C, *b, *Lf, *Wl, *Wr, *y, *xs, *Bm, *Bv, *out_step;
  PgOut* out;
};

struct ll_pose_graph {
  ll_ctx* ctx = nullptr;
  DevBuf arena;
  std::vector<char> host;
  PgPlan plan;
};

// ------------------------------------------------------------------------------------------------ device
__device__ __forceinline__ void pg_cross(const double* a, const double* b, double* o) {
  o[0] = a[1] * b[2] - a[2] * b[1]; o[1] = a[2] * b[0] - a[0] * b[2]; o[2] = a[0] * b[1] - a[1] * b[0];
}
// derivative of d_qrot(q, v) (Eigen's _transformVector) in q along dq
__device__ __forceinline__ void pg_drot(const double* q, const double* dq, const double* v, double* o) {
  double c[3], dc[3], t1[3], t2[3];
  pg_cross(q + 1, v, c); pg_cross(dq + 1, v, dc);
  for (int k = 0; k < 3; k++) { c[k] += c[k]; dc[k] += dc[k]; }
  pg_cross(dq + 1, c, t1); pg_cross(q + 1, dc, t2);
  for (int k = 0; k < 3; k++) o[k] = dq[0] * c[k] + q[0] * dc[k] + t1[k] + t2[k];
}
// 2 vec(qm (qa qb)^*)
__device__ __forceinline__ void pg_eq(const double* qm, const double* qa, const double* qb, double* o) {
  double t[4], tc[4], d[4];
  d_qmul(qa, qb, t); tc[0] = t[0]; tc[1] = -t[1]; tc[2] = -t[2]; tc[3] = -t[3];
  d_qmul(qm, tc, d);
  o[0] = 2.0 * d[1]; o[1] = 2.0 * d[2]; o[2] = 2.0 * d[3];
}
// Residual, Jacobian blocks (rows e_p, e_q; columns position, rotation tangent) and cost of edge e at the poses X.
__device__ void pg_eval_edge(const PgArgs& A, int e, const double* X, double* r, double* Ja, double* Jb, double* cost) {
  const int a = A.ea[e], bn = A.eb[e];
  const double *qa = X + 7 * a, *pa = X + 7 * a + 4, *qb = X + 7 * bn, *pb = X + 7 * bn + 4, *qm = A.meas + 7 * e, *pm = A.meas + 7 * e + 4;
  const double qac[4] = {qa[0], -qa[1], -qa[2], -qa[3]};
  const double dp[3] = {pb[0] - pa[0], pb[1] - pa[1], pb[2] - pa[2]};
  double ev[6];
  d_qrot(qac, dp, ev); for (int k = 0; k < 3; k++) ev[k] -= pm[k];
  pg_eq(qm, qac, qb, ev + 3);
  double JA[36], JB[36];
  for (int i = 0; i < 36; i++) { JA[i] = 0.0; JB[i] = 0.0; }
  for (int k = 0; k < 3; k++) {
    const double ek[3] = {k == 0 ? 1.0 : 0.0, k == 1 ? 1.0 : 0.0, k == 2 ? 1.0 : 0.0};
    const double pk[4] = {0.0, ek[0], ek[1], ek[2]};
    double col[3];
    d_qrot(qac, ek, col);
    for (int i = 0; i < 3; i++) { JB[i * 6 + k] = col[i]; JA[i * 6 + k] = -col[i]; }
    double dqb[4], dqa[4], dqac[4], o[3];
    d_qmul(pk, qb, dqb); pg_eq(qm, qac, dqb, o);
    for (int i = 0; i < 3; i++) JB[(3 + i) * 6 + 3 + k] = o[i];
    d_qmul(pk, qa, dqa); dqac[0] = dqa[0]; dqac[1] = -dqa[1]; dqac[2] = -dqa[2]; dqac[3] = -dqa[3];
    pg_drot(qac, dqac, dp, o);
    for (int i = 0; i < 3; i++) JA[i * 6 + 3 + k] = o[i];
    pg_eq(qm, dqac, qb, o);
    for (int i = 0; i < 3; i++) JA[(3 + i) * 6 + 3 + k] = o[i];
  }
  const double* L = A.sqi + 36 * e;
  double c = 0.0;
  for (int i = 0; i < 6; i++) {
    double s = 0.0; for (int k = 0; k <= i; k++) s += L[i * 6 + k] * ev[k];
    r[i] = s; c += s * s;
    for (int j = 0; j < 6; j++) {
      double sa = 0.0, sb = 0.0; for (int k = 0; k <= i; k++) { sa += L[i * 6 + k] * JA[k * 6 + j]; sb += L[i * 6 + k] * JB[k * 6 + j]; }
      Ja[i * 6 + j] = sa; Jb[i * 6 + j] = sb;
    }
  }
  *cost = 0.5 * c;
}
// EigenQuaternionParameterization::Plus on q (w,x,y,z) and the Euclidean plus on t, for one pose
__device__ __forceinline__ void pg_plus(const double* x, const double* d /* position, rotation */, double* o) {
  const double nd = sqrt(d[3] * d[3] + d[4] * d[4] + d[5] * d[5]);
  if (nd > 0.0) {
    const double sbd = sin(nd) / nd, dq[4] = {cos(nd), sbd * d[3], sbd * d[4], sbd * d[5]};
    d_qmul(dq, x, o);
  } else { o[0] = x[0]; o[1] = x[1]; o[2] = x[2]; o[3] = x[3]; }
  for (int k = 0; k < 3; k++) o[4 + k] = x[4 + k] + d[k];
}

__device__ double pg_sum(double v, double* sh) {   // fixed-order CTA sum
  sh[threadIdx.x] = v; __syncthreads();
  for (int s = PG_THREADS / 2; s > 0; s >>= 1) { if ((int)threadIdx.x < s) sh[threadIdx.x] += sh[threadIdx.x + s]; __syncthreads(); }
  const double r = sh[0]; __syncthreads(); return r;
}
__device__ double pg_max(double v, double* sh) {
  sh[threadIdx.x] = v; __syncthreads();
  for (int s = PG_THREADS / 2; s > 0; s >>= 1) { if ((int)threadIdx.x < s) sh[threadIdx.x] = fmax(sh[threadIdx.x], sh[threadIdx.x + s]); __syncthreads(); }
  const double r = sh[0]; __syncthreads(); return r;
}
// all edges at X into buffer k; returns the cost (any non-finite value: +inf)
__device__ double pg_evaluate(const PgArgs& A, const double* X, int k, double* sh) {
  double c = 0.0;
  for (int e = threadIdx.x; e < A.M; e += PG_THREADS) { pg_eval_edge(A, e, X, A.r[k] + 6 * e, A.ja[k] + 36 * e, A.jb[k] + 36 * e, A.ec[k] + e); c += A.ec[k][e]; }
  const double s = pg_sum(c, sh);
  return isfinite(s) ? s : INFINITY;
}
// normal-equation blocks at buffer k: per free node H and g (incident edges ascending), per free-free edge J_a^T J_b
__device__ void pg_assemble(const PgArgs& A, int k) {
  for (int f = threadIdx.x; f < A.F; f += PG_THREADS) {
    double H[36], g[6];
    for (int i = 0; i < 36; i++) H[i] = 0.0; for (int i = 0; i < 6; i++) g[i] = 0.0;
    for (int q = A.inc_ptr[f]; q < A.inc_ptr[f + 1]; q++) {
      const int e = A.inc[q] >> 1; const double* J = (A.inc[q] & 1) ? A.jb[k] + 36 * e : A.ja[k] + 36 * e; const double* r = A.r[k] + 6 * e;
      for (int i = 0; i < 6; i++) {
        double s = 0.0; for (int t = 0; t < 6; t++) s += J[t * 6 + i] * r[t]; g[i] += s;
        for (int j = 0; j < 6; j++) { double h = 0.0; for (int t = 0; t < 6; t++) h += J[t * 6 + i] * J[t * 6 + j]; H[i * 6 + j] += h; }
      }
    }
    for (int i = 0; i < 36; i++) A.H[36 * f + i] = H[i]; for (int i = 0; i < 6; i++) A.g[6 * f + i] = g[i];
  }
  for (int e = threadIdx.x; e < A.M; e += PG_THREADS) {
    if (A.free_of_node[A.ea[e]] < 0 || A.free_of_node[A.eb[e]] < 0) continue;
    const double *Ja = A.ja[k] + 36 * e, *Jb = A.jb[k] + 36 * e;
    for (int i = 0; i < 6; i++) for (int j = 0; j < 6; j++) { double h = 0.0; for (int t = 0; t < 6; t++) h += Ja[t * 6 + i] * Jb[t * 6 + j]; A.eoff[36 * e + i * 6 + j] = h; }
  }
  __syncthreads();
}
// the scaled coupling of edge e stored as row = lower node (transposed: a is the higher node)
__device__ __forceinline__ void pg_edge_coupling(const PgArgs& A, int e, int tr, double* acc) {
  const int lo = A.free_of_node[tr ? A.eb[e] : A.ea[e]], hi = A.free_of_node[tr ? A.ea[e] : A.eb[e]];
  pg_add_scaled(acc, A.eoff + 36 * e, tr != 0, A.scaling + 6 * lo, A.scaling + 6 * hi);
}
// The LM step: (S H S + D / radius) step = -S g, delta = S step.  Returns false when a pivot is not positive or the step is not finite.
__device__ bool pg_linear(const PgArgs& A, double radius, bool reuse_diag, int* sh_flag, double* shd, long long* cyc) {
  long long t0 = clock64();
  if (threadIdx.x == 0) *sh_flag = 1;
  for (int f = threadIdx.x; f < A.F; f += PG_THREADS) {
    const double* s = A.scaling + 6 * f; const double* H = A.H + 36 * f; double* Ad = A.Adiag + 36 * f;
    for (int i = 0; i < 6; i++) {
      if (!reuse_diag) A.diag[6 * f + i] = fmin(fmax(H[i * 6 + i] * s[i] * s[i], 1e-6), 1e32);
      for (int j = 0; j < 6; j++) Ad[i * 6 + j] = s[i] * H[i * 6 + j] * s[j];
      A.rhs[6 * f + i] = s[i] * A.g[6 * f + i];
    }
    for (int i = 0; i < 6; i++) { const double d = sqrt(A.diag[6 * f + i] / radius); Ad[i * 6 + i] += d * d; }
  }
  __syncthreads();
  for (int p = threadIdx.x; p < A.n_pos; p += PG_THREADS) {
    const int f = A.pos_free[p];
    double* D = A.D + 36 * p; double* C = A.C + 36 * p; double* b = A.b + 6 * p;
    for (int i = 0; i < 36; i++) { D[i] = f >= 0 ? A.Adiag[36 * f + i] : 0.0; C[i] = 0.0; }
    for (int i = 0; i < 6; i++) b[i] = f >= 0 ? A.rhs[6 * f + i] : 0.0;
    for (int q = A.cpl_ptr[p]; q < A.cpl_ptr[p + 1]; q++) pg_edge_coupling(A, A.cpl[q] >> 1, A.cpl[q] & 1, C);
  }
  __syncthreads();
  for (int lv = 0; lv < A.n_levels; lv++) {
    for (int q = A.elim_ptr[lv] + threadIdx.x; q < A.elim_ptr[lv + 1]; q += PG_THREADS) {
      const int pl = A.elim[3 * q], p = A.elim[3 * q + 1];
      if (!pg_elim(A.D + 36 * p, A.C + 36 * pl, A.C + 36 * p, A.b + 6 * p, A.Lf + 36 * p, A.Wl + 36 * p, A.Wr + 36 * p, A.y + 6 * p)) *sh_flag = 0;
    }
    __syncthreads();
    for (int q = A.upd_ptr[lv] + threadIdx.x; q < A.upd_ptr[lv + 1]; q += PG_THREADS) {
      const int s = A.upd[3 * q], l = A.upd[3 * q + 1], r = A.upd[3 * q + 2];
      pg_update(A.D + 36 * s, A.b + 6 * s, A.C + 36 * s, l >= 0 ? A.Wr + 36 * l : nullptr, l >= 0 ? A.y + 6 * l : nullptr, r >= 0 ? A.Wl + 36 * r : nullptr,
                r >= 0 ? A.Wr + 36 * r : nullptr, r >= 0 ? A.y + 6 * r : nullptr);
    }
    __syncthreads();
  }
  long long t1 = clock64();
  // the border system (lower triangle of Bm) and its dense Cholesky factorization
  const int n = 6 * A.nb;
  if (n > 0) {
    for (int w = threadIdx.x; w < A.nb * A.nb * 36; w += PG_THREADS) {
      const int pair = w / 36, ent = w % 36, i = pair / A.nb, j = pair % A.nb, rr = ent / 6, cc = ent % 6;
      if (j < i) continue;
      double v = 0.0;
      for (int q = A.bd_ptr[pair]; q < A.bd_ptr[pair + 1]; q++) {
        const int kind = A.bd[3 * q], idx = A.bd[3 * q + 1], tr = A.bd[3 * q + 2];
        if (kind == 0) v += A.Adiag[36 * idx + ent];
        else if (kind == 1) { double acc[36]; for (int t = 0; t < 36; t++) acc[t] = 0.0; pg_edge_coupling(A, idx, tr, acc); v += acc[ent]; }
        else if (kind == 2) v += A.D[36 * idx + ent];
        else v += A.C[36 * idx + ent];
      }
      A.Bm[(size_t)(6 * j + cc) * n + 6 * i + rr] = v;
    }
    for (int w = threadIdx.x; w < n; w += PG_THREADS) {
      const int i = w / 6, rr = w % 6; double v = 0.0;
      for (int q = A.bb_ptr[i]; q < A.bb_ptr[i + 1]; q++) v += A.bb[2 * q] == 0 ? A.rhs[6 * A.bb[2 * q + 1] + rr] : A.b[6 * A.bb[2 * q + 1] + rr];
      A.Bv[w] = v;
    }
    __syncthreads();
    for (int k = 0; k < n; k++) {
      if (threadIdx.x == 0) { const double d = A.Bm[(size_t)k * n + k]; if (!(d > 0.0)) *sh_flag = 0; A.Bm[(size_t)k * n + k] = sqrt(d); }
      __syncthreads();
      if (!*sh_flag) break;
      const double piv = A.Bm[(size_t)k * n + k];
      for (int i = k + 1 + threadIdx.x; i < n; i += PG_THREADS) A.Bm[(size_t)i * n + k] /= piv;
      __syncthreads();
      const int m = n - k - 1;
      for (int w = threadIdx.x; w < m * m; w += PG_THREADS) {
        const int i = k + 1 + w / m, j = k + 1 + w % m;
        if (j <= i) A.Bm[(size_t)i * n + j] -= A.Bm[(size_t)i * n + k] * A.Bm[(size_t)j * n + k];
      }
      __syncthreads();
    }
    if (*sh_flag) {
      for (int k = 0; k < n; k++) {   // L y = v
        if (threadIdx.x == 0) A.Bv[k] /= A.Bm[(size_t)k * n + k];
        __syncthreads();
        for (int i = k + 1 + threadIdx.x; i < n; i += PG_THREADS) A.Bv[i] -= A.Bm[(size_t)i * n + k] * A.Bv[k];
        __syncthreads();
      }
      for (int k = n - 1; k >= 0; k--) {   // L^T x = y
        if (threadIdx.x == 0) A.Bv[k] /= A.Bm[(size_t)k * n + k];
        __syncthreads();
        for (int i = threadIdx.x; i < k; i += PG_THREADS) A.Bv[i] -= A.Bm[(size_t)k * n + i] * A.Bv[k];
        __syncthreads();
      }
    }
  }
  __syncthreads();
  long long t2 = clock64();
  const bool ok = *sh_flag != 0;
  if (ok) {
    for (int p = threadIdx.x; p < A.n_pos; p += PG_THREADS) {
      if (A.pos_free[p] >= 0) continue;
      const int sb = A.pos_border[p];
      for (int i = 0; i < 6; i++) A.xs[6 * p + i] = sb >= 0 ? A.Bv[6 * sb + i] : 0.0;
    }
    __syncthreads();
    for (int lv = A.n_levels - 1; lv >= 0; lv--) {
      for (int q = A.elim_ptr[lv] + threadIdx.x; q < A.elim_ptr[lv + 1]; q += PG_THREADS) {
        const int pl = A.elim[3 * q], p = A.elim[3 * q + 1], pr = A.elim[3 * q + 2];
        pg_backsub(A.Lf + 36 * p, A.Wl + 36 * p, A.Wr + 36 * p, A.y + 6 * p, A.xs + 6 * pl, A.xs + 6 * pr, A.xs + 6 * p);
      }
      __syncthreads();
    }
    int bad = 0;
    for (int f = threadIdx.x; f < A.F; f += PG_THREADS) {
      const int sb = A.free_border[f]; const double* x = sb >= 0 ? A.Bv + 6 * sb : A.xs + 6 * A.free_pos[f];
      for (int i = 0; i < 6; i++) {
        const double st = -x[i]; if (!isfinite(st)) bad = 1;
        A.out_step[6 * f + i] = st; A.delta[6 * f + i] = st * A.scaling[6 * f + i];
      }
    }
    if (bad) *sh_flag = 0;
  }
  __syncthreads();
  const bool ok2 = *sh_flag != 0;
  __syncthreads();
  long long t3 = clock64();
  cyc[1] += (t1 - t0) + (t3 - t2); cyc[2] += t2 - t1;
  (void)shd;
  return ok2;
}

__global__ void __launch_bounds__(PG_THREADS) pg_solve_kernel(PgArgs A) {
  __shared__ double sh[PG_THREADS];
  __shared__ int flag, done, accept;
  __shared__ double x_cost, cand_cost, radius, dfac, mcc, x_norm, gmax, min_iter_cost, rel;
  __shared__ int iteration, num_invalid, reuse_diag, last_succ, termination, evals, xi, ei;
  long long cyc[4] = {0, 0, 0, 0};
  const long long t_start = clock64();
  const int tid = threadIdx.x;
  // per free node: sum of squares of the pose (x_norm), and the gradient test |x - Plus(x, -g)|_inf
  auto norms = [&](int k) {
    double s = 0.0, m = 0.0;
    for (int f = tid; f < A.F; f += PG_THREADS) {
      const double* x = A.x[k] + 7 * A.free_node[f]; double ng[6], pg[7];
      for (int i = 0; i < 7; i++) s += x[i] * x[i];
      for (int i = 0; i < 6; i++) ng[i] = -A.g[6 * f + i];
      pg_plus(x, ng, pg);
      for (int i = 0; i < 7; i++) m = fmax(m, fabs(x[i] - pg[i]));
    }
    const double ss = pg_sum(s, sh), mm = pg_max(m, sh);
    if (tid == 0) { x_norm = sqrt(ss); gmax = mm; }
  };
  if (tid == 0) { xi = 0; ei = 0; evals = 1; iteration = 0; num_invalid = 0; reuse_diag = 0; last_succ = 1; radius = 1e4; dfac = 2.0; done = 0; termination = 0; }
  for (int i = tid; i < 7 * A.N; i += PG_THREADS) A.x[1][i] = A.x[0][i];
  __syncthreads();
  long long te = clock64();
  const double c0 = pg_evaluate(A, A.x[0], 0, sh);
  if (tid == 0) { x_cost = c0; min_iter_cost = c0; }
  pg_assemble(A, 0);
  for (int f = tid; f < A.F; f += PG_THREADS) for (int i = 0; i < 6; i++) A.scaling[6 * f + i] = 1.0 / (1.0 + sqrt(A.H[36 * f + i * 7]));
  __syncthreads();
  norms(0);
  cyc[0] += clock64() - te;
  if (A.mode == 1) {   // ll_pose_graph_step
    const bool ok = pg_linear(A, A.radius_in, false, &flag, sh, cyc);
    if (tid == 0) { A.out->cost = x_cost; A.out->valid = ok ? 1 : 0; }
    return;
  }
  if (tid == 0 && !isfinite(c0)) { done = 1; termination = 4; }
  __syncthreads();
  while (!done) {
    if (tid == 0) {
      if (iteration >= A.max_iterations) { done = 1; termination = 0; }
      else if (last_succ && gmax <= LM_GTOL) { done = 1; termination = 1; }
      else if (radius <= 1e-32) { done = 1; termination = 5; }
      else iteration++;
    }
    __syncthreads();
    if (done) break;
    bool ok = pg_linear(A, radius, reuse_diag != 0, &flag, sh, cyc);
    te = clock64();
    if (tid == 0) reuse_diag = 1;
    if (ok) {   // model cost change: -sum (J delta) . (r + J delta / 2)
      double s = 0.0;
      for (int e = tid; e < A.M; e += PG_THREADS) {
        const int fa = A.free_of_node[A.ea[e]], fb = A.free_of_node[A.eb[e]];
        const double *Ja = A.ja[ei] + 36 * e, *Jb = A.jb[ei] + 36 * e, *r = A.r[ei] + 6 * e;
        double t = 0.0;
        for (int i = 0; i < 6; i++) {
          double m = 0.0;
          for (int j = 0; j < 6; j++) { if (fa >= 0) m += Ja[i * 6 + j] * A.delta[6 * fa + j]; if (fb >= 0) m += Jb[i * 6 + j] * A.delta[6 * fb + j]; }
          t += m * (r[i] + m / 2.0);
        }
        s += t;
      }
      const double mc = -pg_sum(s, sh);
      if (tid == 0) mcc = mc;
      ok = mc > 0.0;
    }
    if (!ok) {   // HandleInvalidStep
      if (tid == 0) {
        if (++num_invalid >= 5) { done = 1; termination = 4; }
        else { radius = radius / dfac; dfac *= 2.0; last_succ = 0; }
      }
      __syncthreads();
      cyc[0] += clock64() - te;
      continue;
    }
    // the candidate and its cost
    const int xc = 1 - xi, ec = 1 - ei;
    double sn = 0.0;
    for (int f = tid; f < A.F; f += PG_THREADS) {
      const int nd = A.free_node[f]; const double* x = A.x[xi] + 7 * nd; double* o = A.x[xc] + 7 * nd;
      pg_plus(x, A.delta + 6 * f, o);
      for (int i = 0; i < 7; i++) sn += (x[i] - o[i]) * (x[i] - o[i]);
    }
    const double step_norm = sqrt(pg_sum(sn, sh));
    double cc = pg_evaluate(A, A.x[xc], ec, sh);
    if (!isfinite(cc)) cc = DBL_MAX;
    if (tid == 0) {
      num_invalid = 0; evals++; cand_cost = cc; accept = 0;
      if (step_norm <= LM_PTOL * (x_norm + LM_PTOL)) { done = 1; termination = 2; }
      else if (fabs(x_cost - cc) <= LM_FTOL * x_cost) { done = 1; termination = 3; }
      else { rel = (x_cost - cc) / mcc; accept = rel > 1e-3 ? 1 : 0; }
    }
    __syncthreads();
    if (done) { cyc[0] += clock64() - te; break; }
    if (accept) {   // HandleSuccessfulStep
      pg_assemble(A, ec);
      norms(xc);
      if (tid == 0) {
        xi = xc; ei = ec; x_cost = cand_cost; radius = radius_after_success(radius, rel); dfac = 2.0; reuse_diag = 0; last_succ = 1;
        min_iter_cost = fmin(min_iter_cost, x_cost);
      }
    } else if (tid == 0) {   // HandleUnsuccessfulStep
      radius = radius / dfac; dfac *= 2.0; reuse_diag = 1; last_succ = 0; min_iter_cost = fmin(min_iter_cost, cand_cost);
    }
    __syncthreads();
    cyc[0] += clock64() - te;
  }
  if (tid == 0) {
    PgOut* o = A.out;
    o->initial_cost = c0; o->final_cost = fmin(c0, min_iter_cost); o->cost = x_cost; o->iterations = iteration; o->evaluations = evals;
    o->termination = termination; o->xi = xi; o->valid = 1;
    cyc[3] = clock64() - t_start;
    for (int k = 0; k < 4; k++) o->cyc[k] = cyc[k];
  }
}

// ------------------------------------------------------------------------------------------------ host
static bool pg_host_llt(const double* W, double* L) {   // Eigen's LLT<Lower>: W = L L^T; false unless W is symmetric positive definite
  for (int i = 0; i < 6; i++) for (int j = 0; j < 6; j++) if (!(W[i * 6 + j] == W[j * 6 + i])) return false;
  for (int i = 0; i < 36; i++) L[i] = 0.0;
  for (int k = 0; k < 6; k++) {
    double x = W[k * 6 + k]; for (int j = 0; j < k; j++) x -= L[k * 6 + j] * L[k * 6 + j];
    if (!(x > 0.0)) return false;
    x = std::sqrt(x); L[k * 6 + k] = x;
    for (int i = k + 1; i < 6; i++) { double s = W[i * 6 + k]; for (int j = 0; j < k; j++) s -= L[i * 6 + j] * L[k * 6 + j]; L[i * 6 + k] = s / x; }
  }
  return true;
}
static int pg_check(ll_pose_graph* pg, const ll_pose* poses, int n, const ll_pg_edge* edges, int m) {
  ll_ctx* ctx = pg->ctx;
  if (n < 0 || m < 0 || (n > 0 && !poses) || (m > 0 && !edges)) { ctx->set_error("pose graph: null poses / edges or a negative count"); return LL_ERR_INVALID; }
  for (int i = 0; i < n; i++) {
    for (int k = 0; k < 4; k++) if (!std::isfinite(poses[i].q_wxyz[k])) { ctx->set_error("pose " + std::to_string(i) + " is not finite"); return LL_ERR_INVALID; }
    for (int k = 0; k < 3; k++) if (!std::isfinite(poses[i].t[k])) { ctx->set_error("pose " + std::to_string(i) + " is not finite"); return LL_ERR_INVALID; }
  }
  for (int e = 0; e < m; e++) {
    const ll_pg_edge& E = edges[e];
    if (E.id_begin < 0 || E.id_begin >= n || E.id_end < 0 || E.id_end >= n) { ctx->set_error("edge " + std::to_string(e) + ": id outside 0 .. n-1"); return LL_ERR_INVALID; }
    if (E.id_begin == E.id_end) { ctx->set_error("edge " + std::to_string(e) + ": id_begin == id_end"); return LL_ERR_INVALID; }
    bool fin = true;
    for (int k = 0; k < 4; k++) fin = fin && std::isfinite(E.q_wxyz[k]);
    for (int k = 0; k < 3; k++) fin = fin && std::isfinite(E.t[k]);
    for (int k = 0; k < 36; k++) fin = fin && std::isfinite(E.information[k]);
    if (!fin) { ctx->set_error("edge " + std::to_string(e) + " is not finite"); return LL_ERR_INVALID; }
    double L[36];
    if (!pg_host_llt(E.information, L)) { ctx->set_error("edge " + std::to_string(e) + ": information is not symmetric positive definite"); return LL_ERR_INVALID; }
  }
  return LL_OK;
}
static PgSizes pg_sizes(const PgPlan& P) {
  return {P.N, P.M, P.F, P.n_pos, P.elim_ptr.back(), P.upd_ptr.back(), P.n_levels, P.nb, (int)P.bd.size() / 3, (int)P.bb.size() / 2};
}
// Validates, plans, uploads and launches; on success the kernel is enqueued and the arena's pointers are in *A.
static int pg_launch(ll_pose_graph* pg, const ll_pose* poses, int n, const ll_pg_edge* edges, int m, int mode, int max_iterations, double radius, PgArgs* A) {
  ll_ctx* ctx = pg->ctx;
  LL_TRY(pg_check(pg, poses, n, edges, m));
  std::vector<int> ea(m), eb(m);
  for (int e = 0; e < m; e++) { ea[e] = edges[e].id_begin; eb[e] = edges[e].id_end; }
  PgPlan& P = pg->plan;
  if (pg_build_plan(n, m, ea.data(), eb.data(), P) > LL_PG_MAX_BORDER) {
    ctx->set_error("pose graph: " + std::to_string(P.nb) + " border nodes (free endpoints of loop edges), at most " + std::to_string(LL_PG_MAX_BORDER));
    return LL_ERR_CAPACITY;
  }
  const PgSizes S = pg_sizes(P);
  size_t in_bytes = 0;
  PgArgs a{};
  cudaSetDevice(ctx->device);
  LL_CUDA(ctx, pg->arena.carve([&](Carve& c) { pg_layout(c, S, a, &in_bytes); }));
  PgHostArgs h{};
  { Carve c0; size_t ib; pg_layout(c0, S, h, &ib); }
  pg->host.resize(in_bytes);
  { Carve c(pg->host.data()); size_t ib; pg_layout(c, S, h, &ib); }
  auto put = [](int* d, const std::vector<int>& v) { if (!v.empty()) memcpy(d, v.data(), v.size() * sizeof(int)); };
  put(h.ea, ea); put(h.eb, eb); put(h.free_of_node, P.free_of_node); put(h.free_node, P.free_node); put(h.inc_ptr, P.inc_ptr); put(h.inc, P.inc);
  put(h.free_pos, P.free_pos); put(h.free_border, P.free_border); put(h.pos_free, P.pos_free); put(h.pos_border, P.pos_border);
  put(h.cpl_ptr, P.cpl_ptr); put(h.cpl, P.cpl); put(h.elim_ptr, P.elim_ptr); put(h.elim, P.elim); put(h.upd_ptr, P.upd_ptr); put(h.upd, P.upd);
  put(h.border, P.border); put(h.bd_ptr, P.bd_ptr); put(h.bd, P.bd); put(h.bb_ptr, P.bb_ptr); put(h.bb, P.bb);
  for (int e = 0; e < m; e++) {
    memcpy(h.meas + 7 * e, edges[e].q_wxyz, 4 * sizeof(double)); memcpy(h.meas + 7 * e + 4, edges[e].t, 3 * sizeof(double));
    pg_host_llt(edges[e].information, h.sqi + 36 * e);
  }
  static_assert(sizeof(ll_pose) == 7 * sizeof(double), "ll_pose is 7 packed doubles");
  if (n) memcpy(h.x[0], poses, (size_t)n * sizeof(ll_pose));
  a.N = n; a.M = m; a.F = P.F; a.nb = P.nb; a.n_pos = P.n_pos; a.n_levels = P.n_levels; a.max_iterations = max_iterations; a.mode = mode; a.radius_in = radius;
  LL_CUDA(ctx, cudaMemcpyAsync(pg->arena.p, pg->host.data(), in_bytes, cudaMemcpyHostToDevice, ctx->stream));
  pg_solve_kernel<<<1, PG_THREADS, 0, ctx->stream>>>(a);
  ctx->launches++;
  LL_CUDA(ctx, cudaGetLastError());
  *A = a;
  return LL_OK;
}

// Re-posed keyframe clouds (Mapping_refine::refine_pts): after the segmented VoxelGrid, point i of segment k becomes R_aff[k] p + T_aff[k] in
// float, the row sums left to right as Eigen's fixed-size product has them; the intensity is 0, as eigen_to_pcl_pt leaves it.
__global__ void repose_kernel(const float4* __restrict__ in, const int* __restrict__ out_end, int n_seg, const float* __restrict__ aff, float4* __restrict__ out) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= out_end[n_seg - 1]) return;
  int lo = 0, hi = n_seg - 1;   // the first segment whose end is past i
  while (lo < hi) { const int m = (lo + hi) >> 1; if (out_end[m] > i) hi = m; else lo = m + 1; }
  const float* A = aff + 12 * lo; const float4 p = in[i];
  float o[3];
  for (int r = 0; r < 3; r++) o[r] = ((A[3 * r] * p.x + A[3 * r + 1] * p.y) + A[3 * r + 2] * p.z) + A[9 + r];
  out[i] = make_float4(o[0], o[1], o[2], 0.f);
}
static void pg_rotation(const double* q, double* R) {   // Eigen's QuaternionBase::toRotationMatrix, q as w, x, y, z
  const double w = q[0], x = q[1], y = q[2], z = q[3];
  const double tx = 2 * x, ty = 2 * y, tz = 2 * z, twx = tx * w, twy = ty * w, twz = tz * w, txx = tx * x, txy = ty * x, txz = tz * x, tyy = ty * y, tyz = tz * y,
               tzz = tz * z;
  R[0] = 1 - (tyy + tzz); R[1] = txy - twz; R[2] = txz + twy;
  R[3] = txy + twz; R[4] = 1 - (txx + tzz); R[5] = tyz - twx;
  R[6] = txz - twy; R[7] = tyz + twx; R[8] = 1 - (txx + tyy);
}

// ll_keyframes_repose on device input: keyframe k is d_in[seg_end[k - 1] .. seg_end[k]) of n points (host ends, n_kf 1 ... 256), down-sampled into d_mid
// and moved into d_out (each as large as the input); d_end, d_oend (n_kf ints) and d_aff (12 n_kf floats) are the caller's device scratch.
// out_end[k] = the end of keyframe k's output, read back after the work on the context's stream has completed.
int keyframes_repose_dev(ll_ctx* ctx, const float4* d_in, int n, const int* seg_end, int n_kf, const ll_pose* poses_ori, const ll_pose* poses_opt, float leaf,
                         float4* d_mid, float4* d_out, int* d_end, int* d_oend, float* d_aff, int* out_end) {
  cudaStream_t s = ctx->stream;
  std::vector<int> h(seg_end, seg_end + n_kf); std::vector<float> aff(12 * (size_t)n_kf);
  for (int k = 0; k < n_kf; k++) ll_keyframe_affine(&poses_ori[k], &poses_opt[k], &aff[12 * k], &aff[12 * k + 9]);
  LL_CUDA(ctx, cudaMemcpyAsync(d_end, h.data(), n_kf * sizeof(int), cudaMemcpyHostToDevice, s));
  LL_CUDA(ctx, cudaMemcpyAsync(d_aff, aff.data(), aff.size() * sizeof(float), cudaMemcpyHostToDevice, s));
  LL_TRY(launch_voxel_grid_segments(ctx, s, ctx->scratch, d_in, n, d_end, n_kf, leaf, d_mid, d_oend));
  if (n) { repose_kernel<<<ll_div_up(n, 256), 256, 0, s>>>(d_mid, d_oend, n_kf, d_aff, d_out); ctx->launches++; LL_CUDA(ctx, cudaGetLastError()); }
  LL_CUDA(ctx, cudaMemcpyAsync(h.data(), d_oend, n_kf * sizeof(int), cudaMemcpyDeviceToHost, s));
  LL_CUDA(ctx, cudaStreamSynchronize(s));
  std::copy(h.begin(), h.end(), out_end);
  return LL_OK;
}

extern "C" {

void ll_keyframe_affine(const ll_pose* ori, const ll_pose* opt, float R_aff[9], float T_aff[3]) {
  double Ro[9], Rp[9];
  pg_rotation(ori->q_wxyz, Ro); pg_rotation(opt->q_wxyz, Rp);
  for (int i = 0; i < 3; i++) for (int j = 0; j < 3; j++) {   // (R_opm * R_ori^T).cast<float>()
    const double v = (Rp[3 * i] * Ro[3 * j] + Rp[3 * i + 1] * Ro[3 * j + 1]) + Rp[3 * i + 2] * Ro[3 * j + 2];
    R_aff[3 * i + j] = (float)v;
  }
  for (int i = 0; i < 3; i++) {   // (R_aff.cast<double>() * (-t_ori) + t_opm).cast<float>()
    const double v = ((double)R_aff[3 * i] * -ori->t[0] + (double)R_aff[3 * i + 1] * -ori->t[1]) + (double)R_aff[3 * i + 2] * -ori->t[2];
    T_aff[i] = (float)(v + opt->t[i]);
  }
}

int ll_keyframes_repose(ll_ctx* ctx, const ll_point* clouds, size_t n, const size_t* seg_end, int n_kf, const ll_pose* poses_ori, const ll_pose* poses_opt,
                        float leaf, ll_point* out, size_t* n_out_per_seg) {
  if (!ctx || !seg_end || !n_out_per_seg || !poses_ori || !poses_opt || (!clouds && n) || n_kf < 1 || n_kf > 256 || !(leaf > 0.f) || n >= (size_t)1 << 31)
    return LL_ERR_INVALID;
  for (int k = 0; k < n_kf; k++) if (seg_end[k] > n || (k && seg_end[k] < seg_end[k - 1])) { ctx->set_error("segment ends must ascend and stay within n"); return LL_ERR_INVALID; }
  cudaSetDevice(ctx->device);
  cudaStream_t s = ctx->stream;
  float4 *d_in, *d_mid, *d_out; int *d_end, *d_oend; float* d_aff;
  LL_CUDA(ctx, ctx->feat_buf.carve([&](Carve& c) {
    d_in = c.take<float4>(n); d_mid = c.take<float4>(n); d_out = c.take<float4>(n); d_end = c.take<int>(n_kf); d_oend = c.take<int>(n_kf); d_aff = c.take<float>(12 * (size_t)n_kf);
  }));
  std::vector<int> h(n_kf);
  for (int k = 0; k < n_kf; k++) h[k] = (int)seg_end[k];
  LL_TRY(upload_cloud(ctx, s, clouds, n, LL_FMT_XYZI16, LL_HOST, d_in));
  LL_TRY(keyframes_repose_dev(ctx, d_in, (int)n, h.data(), n_kf, poses_ori, poses_opt, leaf, d_mid, d_out, d_end, d_oend, d_aff, h.data()));
  for (int k = 0; k < n_kf; k++) n_out_per_seg[k] = (size_t)(h[k] - (k ? h[k - 1] : 0));
  if (out && h[n_kf - 1] > 0) { LL_CUDA(ctx, cudaMemcpyAsync(out, d_out, (size_t)h[n_kf - 1] * 16, cudaMemcpyDeviceToHost, s)); LL_CUDA(ctx, cudaStreamSynchronize(s)); }
  return LL_OK;
}

int ll_pose_graph_create(ll_ctx* ctx, int reserve_nodes, int reserve_edges, ll_pose_graph** out) {
  if (!ctx || !out || reserve_nodes < 0 || reserve_edges < 0) return LL_ERR_INVALID;
  *out = nullptr;
  ll_pose_graph* pg = new ll_pose_graph();
  pg->ctx = ctx;
  // the largest plan of this size: every node free and in a segment of its own (3 positions each), the border full
  const int N = reserve_nodes, M = reserve_edges, nb = LL_PG_MAX_BORDER;
  const PgSizes S = {N, M, N, 3 * N, N, 2 * N, 32, nb, nb + M + 3 * N, nb + 2 * N};
  PgArgs a{}; size_t ib;
  cudaSetDevice(ctx->device);
  const size_t bytes = layout_bytes([&](Carve& c) { pg_layout(c, S, a, &ib); });
  const cudaError_t e = pg->arena.reserve_floor(bytes);
  if (e != cudaSuccess) { ctx->set_error(std::string("pose graph arena: ") + cudaGetErrorString(e)); delete pg; return LL_ERR_CUDA; }
  pg->host.reserve(ib);
  *out = pg;
  return LL_OK;
}

void ll_pose_graph_release(ll_pose_graph* pg) {
  if (!pg) return;
  cudaSetDevice(pg->ctx->device);
  cudaStreamSynchronize(pg->ctx->stream);
  pg->arena.release();
  delete pg;
}

int ll_pose_graph_optimize(ll_pose_graph* pg, ll_pose* poses, int n, const ll_pg_edge* edges, int m, int max_iterations, ll_pg_summary* summary) {
  if (!pg || !summary) return LL_ERR_INVALID;
  ll_ctx* ctx = pg->ctx;
  memset(summary, 0, sizeof(*summary));
  if (m == 0) { LL_TRY(pg_check(pg, poses, n, edges, m)); return LL_OK; }   // the reference returns before building a problem
  PgArgs a;
  LL_TRY(pg_launch(pg, poses, n, edges, m, 0, max_iterations > 0 ? max_iterations : 200, 0.0, &a));
  PgOut o;
  std::vector<ll_pose> x(n);
  LL_CUDA(ctx, cudaMemcpyAsync(&o, a.out, sizeof(o), cudaMemcpyDeviceToHost, ctx->stream));
  LL_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  LL_CUDA(ctx, cudaMemcpyAsync(x.data(), a.x[o.xi], (size_t)n * sizeof(ll_pose), cudaMemcpyDeviceToHost, ctx->stream));
  LL_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  const PgPlan& P = pg->plan;
  for (int f = 0; f < P.F; f++) poses[P.free_node[f]] = x[P.free_node[f]];
  summary->initial_cost = o.initial_cost; summary->final_cost = o.final_cost; summary->iterations = o.iterations; summary->evaluations = o.evaluations;
  summary->termination = o.termination; summary->border_nodes = P.nb; summary->segments = P.n_seg; summary->levels = P.n_levels; summary->free_nodes = P.F;
  summary->cycles_eval = o.cyc[0]; summary->cycles_elim = o.cyc[1]; summary->cycles_border = o.cyc[2]; summary->cycles_total = o.cyc[3];
  return LL_OK;
}

int ll_pose_graph_step(ll_pose_graph* pg, const ll_pose* poses, int n, const ll_pg_edge* edges, int m, double radius, double* cost, double* gradient,
                       double* scaling, double* step, int* valid) {
  if (!pg || !cost || !gradient || !scaling || !step || !valid) return LL_ERR_INVALID;
  ll_ctx* ctx = pg->ctx;
  if (!(radius > 0.0) || !std::isfinite(radius)) { ctx->set_error("pose graph step: the radius must be positive and finite"); return LL_ERR_INVALID; }
  if (m == 0) { ctx->set_error("pose graph step: no edges"); return LL_ERR_INVALID; }
  PgArgs a;
  LL_TRY(pg_launch(pg, poses, n, edges, m, 1, 0, radius, &a));
  const PgPlan& P = pg->plan;
  PgOut o;
  std::vector<double> g(6 * (size_t)P.F), s(6 * (size_t)P.F), st(6 * (size_t)P.F);
  LL_CUDA(ctx, cudaMemcpyAsync(&o, a.out, sizeof(o), cudaMemcpyDeviceToHost, ctx->stream));
  LL_CUDA(ctx, cudaMemcpyAsync(g.data(), a.g, g.size() * sizeof(double), cudaMemcpyDeviceToHost, ctx->stream));
  LL_CUDA(ctx, cudaMemcpyAsync(s.data(), a.scaling, s.size() * sizeof(double), cudaMemcpyDeviceToHost, ctx->stream));
  LL_CUDA(ctx, cudaMemcpyAsync(st.data(), a.out_step, st.size() * sizeof(double), cudaMemcpyDeviceToHost, ctx->stream));
  LL_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  memset(gradient, 0, 6 * (size_t)n * sizeof(double)); memset(scaling, 0, 6 * (size_t)n * sizeof(double)); memset(step, 0, 6 * (size_t)n * sizeof(double));
  for (int f = 0; f < P.F; f++) {
    const size_t d = 6 * (size_t)P.free_node[f];
    memcpy(gradient + d, &g[6 * f], 48); memcpy(scaling + d, &s[6 * f], 48); memcpy(step + d, &st[6 * f], 48);
  }
  *cost = o.cost; *valid = o.valid;
  return LL_OK;
}

// Eigen::Quaterniond::inverse(): the conjugate divided by the squared norm (an SSE2 build sums it as (x^2 + z^2) + (y^2 + w^2))
static void pg_qinv(const double* q, double* o) {
  const double n2 = (q[1] * q[1] + q[3] * q[3]) + (q[2] * q[2] + q[0] * q[0]);
  if (n2 > 0.0) { o[0] = q[0] / n2; o[1] = -q[1] / n2; o[2] = -q[2] / n2; o[3] = -q[3] / n2; } else { o[0] = o[1] = o[2] = o[3] = 0.0; }
}
static void pg_hmul(const double* a, const double* b, double* o) {
  o[0] = a[0] * b[0] - a[1] * b[1] - a[2] * b[2] - a[3] * b[3];
  o[1] = a[0] * b[1] + a[1] * b[0] + a[2] * b[3] - a[3] * b[2];
  o[2] = a[0] * b[2] + a[2] * b[0] + a[3] * b[1] - a[1] * b[3];
  o[3] = a[0] * b[3] + a[3] * b[0] + a[1] * b[2] - a[2] * b[1];
}
static void pg_hrot(const double* q, const double* v, double* o) {   // Eigen's _transformVector
  double c[3] = {q[2] * v[2] - q[3] * v[1], q[3] * v[0] - q[1] * v[2], q[1] * v[1] - q[2] * v[0]};
  c[0] += c[0]; c[1] += c[1]; c[2] += c[2];
  o[0] = v[0] + q[0] * c[0] + (q[2] * c[2] - q[3] * c[1]); o[1] = v[1] + q[0] * c[1] + (q[3] * c[0] - q[1] * c[2]); o[2] = v[2] + q[0] * c[2] + (q[1] * c[1] - q[2] * c[0]);
}

// The odometry edge of service_loop_detection (laser_mapping.hpp:952-958): q = q_prev^-1 q_cur, t = q_prev^-1 (t_cur - t_prev), information = I.
void pg_odometry_edge(const ll_pose* prev, int id_prev, const ll_pose* cur, int id_cur, ll_pg_edge* out) {
  double qi[4], d[3];
  memset(out, 0, sizeof(*out));
  pg_qinv(prev->q_wxyz, qi);
  for (int k = 0; k < 3; k++) d[k] = cur->t[k] - prev->t[k];
  pg_hrot(qi, d, out->t);
  pg_hmul(qi, cur->q_wxyz, out->q_wxyz);
  out->id_begin = id_prev; out->id_end = id_cur;
  for (int k = 0; k < 6; k++) out->information[7 * k] = 1.0;
}

void ll_pose_graph_loop_edge(const double icp_q_wxyz[4], const double icp_t[3], const ll_pose* pose_a, int id_a, const ll_pose* pose_b, int id_b, ll_pg_edge* out) {
  memset(out, 0, sizeof(*out));
  double iq[4], it[3], nt[3] = {-icp_t[0], -icp_t[1], -icp_t[2]};
  pg_qinv(icp_q_wxyz, iq); pg_hrot(iq, nt, it);   // laser_mapping.hpp:1065-1066: ICP_t = ICP_q^-1 (-ICP_t); ICP_q = ICP_q^-1
  double qbi[4], iqi[4], t1[4];
  pg_qinv(pose_b->q_wxyz, qbi); pg_qinv(iq, iqi);
  pg_hmul(qbi, iqi, t1); pg_hmul(t1, pose_a->q_wxyz, out->q_wxyz);
  const double d[3] = {pose_a->t[0] - it[0], pose_a->t[1] - it[1], pose_a->t[2] - it[2]};
  double r[3]; pg_hrot(iqi, d, r);
  const double u[3] = {r[0] - pose_b->t[0], r[1] - pose_b->t[1], r[2] - pose_b->t[2]};
  pg_hrot(qbi, u, out->t);
  out->id_begin = id_b; out->id_end = id_a;
  for (int k = 0; k < 6; k++) out->information[k * 7] = 1.0;
}

}  // extern "C"
