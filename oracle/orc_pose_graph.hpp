// ORACLE — CPU restatement of Ceres_pose_graph_3d::pose_graph_optimization (ceres_pose_graph_3d.hpp:198-352) and of
// Scene_alignment::add_constrain_of_loop (scene_alignment.hpp:97-127).  Test infrastructure only (tests/cpp/pg_oracle.cpp wraps it).
// The residual is differentiated with Jets in its 14 ambient parameters (p_a, q_a as x,y,z,w, p_b, q_b), as AutoDiffCostFunction does, and
// multiplied by EigenQuaternionParameterization's 4 x 3 local Jacobian.  The minimizer is orc_solver.hpp's TrustRegionMinimizer restatement
// without bounds (so without line search), over all free poses; its exact linear solve is an envelope (skyline) LL^T in pose order.
#pragma once
#include <algorithm>
#include <cmath>
#include <limits>
#include <vector>
#include "orc_cloud.hpp"
#include "orc_math.hpp"

namespace orc_pg {
using orc::Jet;

struct Pose { double q[4]; double t[3]; };   // q as w, x, y, z
struct Edge { int a, b; double q[4]; double t[3]; double W[36]; };
struct Summary { double initial_cost = 0, final_cost = 0; int iterations = 0, evaluations = 0, termination = 0; };

template <typename T> inline void qmul(const T* a, const T* b, T* o) {   // (w, x, y, z), Eigen's operation order
  o[0] = a[0] * b[0] - a[1] * b[1] - a[2] * b[2] - a[3] * b[3];
  o[1] = a[0] * b[1] + a[1] * b[0] + a[2] * b[3] - a[3] * b[2];
  o[2] = a[0] * b[2] + a[2] * b[0] + a[3] * b[1] - a[1] * b[3];
  o[3] = a[0] * b[3] + a[3] * b[0] + a[1] * b[2] - a[2] * b[1];
}
template <typename T> inline void qrot(const T* q, const T* v, T* o) {   // Eigen's _transformVector
  T c[3] = {q[2] * v[2] - q[3] * v[1], q[3] * v[0] - q[1] * v[2], q[1] * v[1] - q[2] * v[0]};
  for (int k = 0; k < 3; k++) c[k] = c[k] + c[k];
  o[0] = v[0] + q[0] * c[0] + (q[2] * c[2] - q[3] * c[1]);
  o[1] = v[1] + q[0] * c[1] + (q[3] * c[0] - q[1] * c[2]);
  o[2] = v[2] + q[0] * c[2] + (q[1] * c[1] - q[2] * c[0]);
}
// PoseGraph3dErrorTerm::operator() before the sqrt-information product; q_a, q_b as (w, x, y, z)
template <typename T> inline void error6(const T* pa, const T* qa, const T* pb, const T* qb, const Edge& E, T* e) {
  const T qac[4] = {qa[0], -qa[1], -qa[2], -qa[3]};
  const T dp[3] = {pb[0] - pa[0], pb[1] - pa[1], pb[2] - pa[2]};
  T r[3]; qrot(qac, dp, r);
  for (int k = 0; k < 3; k++) e[k] = r[k] - T(E.t[k]);
  T qab[4], qabc[4], d[4]; qmul(qac, qb, qab);
  qabc[0] = qab[0]; qabc[1] = -qab[1]; qabc[2] = -qab[2]; qabc[3] = -qab[3];
  const T qm[4] = {T(E.q[0]), T(E.q[1]), T(E.q[2]), T(E.q[3])};
  qmul(qm, qabc, d);
  for (int k = 0; k < 3; k++) e[3 + k] = T(2.0) * d[1 + k];
}
inline bool llt6(const double* W, double* L) {   // information.llt().matrixL()
  for (int i = 0; i < 36; i++) L[i] = 0.0;
  for (int k = 0; k < 6; k++) {
    double x = W[k * 6 + k]; for (int j = 0; j < k; j++) x -= L[k * 6 + j] * L[k * 6 + j];
    if (!(x > 0.0)) return false;
    x = std::sqrt(x); L[k * 6 + k] = x;
    for (int i = k + 1; i < 6; i++) { double s = W[i * 6 + k]; for (int j = 0; j < k; j++) s -= L[i * 6 + j] * L[k * 6 + j]; L[i * 6 + k] = s / x; }
  }
  return true;
}
// Residual r (6) and tangent Jacobians Ja, Jb (6 x 6 row-major, columns position then rotation) of edge E.
inline void residual(const Pose& A, const Pose& B, const Edge& E, double* r, double* Ja, double* Jb) {
  typedef Jet<14> J;
  J pa[3], qa[4], pb[3], qb[4];
  // ambient order of the parameter blocks: p_a, q_a (x, y, z, w), p_b, q_b (x, y, z, w)
  for (int k = 0; k < 3; k++) { pa[k] = J(A.t[k], k); pb[k] = J(B.t[k], 7 + k); }
  for (int k = 0; k < 3; k++) { qa[1 + k] = J(A.q[1 + k], 3 + k); qb[1 + k] = J(B.q[1 + k], 10 + k); }
  qa[0] = J(A.q[0], 6); qb[0] = J(B.q[0], 13);
  J e[6]; error6(pa, qa, pb, qb, E, e);
  double L[36]; llt6(E.W, L);
  J res[6];
  for (int i = 0; i < 6; i++) { J s(0.0); for (int k = 0; k <= i; k++) s = s + J(L[i * 6 + k]) * e[k]; res[i] = s; }
  auto local = [](const double* q /* w, x, y, z */, double* M /* 4 x 3, rows x, y, z, w */) {
    const double x = q[1], y = q[2], z = q[3], w = q[0];
    const double m[12] = {w, z, -y, -z, w, x, y, -x, w, -x, -y, -z};
    for (int i = 0; i < 12; i++) M[i] = m[i];
  };
  double Ma[12], Mb[12]; local(A.q, Ma); local(B.q, Mb);
  for (int i = 0; i < 6; i++) {
    r[i] = res[i].a;
    for (int k = 0; k < 3; k++) { Ja[i * 6 + k] = res[i].v[k]; Jb[i * 6 + k] = res[i].v[7 + k]; }
    for (int c = 0; c < 3; c++) {
      double sa = 0.0, sb = 0.0;
      for (int k = 0; k < 4; k++) { sa += res[i].v[3 + k] * Ma[k * 3 + c]; sb += res[i].v[10 + k] * Mb[k * 3 + c]; }
      Ja[i * 6 + 3 + c] = sa; Jb[i * 6 + 3 + c] = sb;
    }
  }
}
inline void plus(const Pose& x, const double* d, Pose& o) {   // EigenQuaternionParameterization::Plus and the Euclidean plus
  const double nd = std::sqrt(d[3] * d[3] + d[4] * d[4] + d[5] * d[5]);
  if (nd > 0.0) { const double s = std::sin(nd) / nd, dq[4] = {std::cos(nd), s * d[3], s * d[4], s * d[5]}; qmul(dq, x.q, o.q); }
  else for (int k = 0; k < 4; k++) o.q[k] = x.q[k];
  for (int k = 0; k < 3; k++) o.t[k] = x.t[k] + d[k];
}

// Envelope (skyline) LL^T of an SPD matrix: row r stores columns first[r] .. r.
struct Skyline {
  int n = 0; std::vector<int> first; std::vector<size_t> off; std::vector<double> v;
  void shape(const std::vector<int>& f) {
    n = (int)f.size(); first = f; off.assign(n + 1, 0);
    for (int r = 0; r < n; r++) off[r + 1] = off[r] + (size_t)(r - first[r] + 1);
    v.assign(off[n], 0.0);
  }
  double& at(int r, int c) { return v[off[r] + (c - first[r])]; }   // c in first[r] .. r
  bool factor() {
    for (int r = 0; r < n; r++)
      for (int c = first[r]; c <= r; c++) {
        double s = at(r, c);
        for (int k = std::max(first[r], first[c]); k < c; k++) s -= at(r, k) * at(c, k);
        if (c == r) { if (!(s > 0.0)) return false; at(r, r) = std::sqrt(s); } else at(r, c) = s / at(c, c);
      }
    return true;
  }
  void solve(std::vector<double>& x) {
    for (int r = 0; r < n; r++) { double s = x[r]; for (int k = first[r]; k < r; k++) s -= at(r, k) * x[k]; x[r] = s / at(r, r); }
    for (int r = n - 1; r >= 0; r--) { x[r] /= at(r, r); const double xr = x[r]; for (int k = first[r]; k < r; k++) x[k] -= at(r, k) * xr; }
  }
};

struct Problem {
  int N = 0; std::vector<Edge> E; std::vector<int> fidx, fnode;
  std::vector<double> r, Ja, Jb;
  // cost and (optionally) residuals / Jacobians of every edge at X; false if not finite
  bool evaluate(const std::vector<Pose>& X, double* cost, bool jac) {
    double c = 0.0; double rr[6], a[36], b[36];
    for (size_t e = 0; e < E.size(); e++) {
      residual(X[E[e].a], X[E[e].b], E[e], rr, a, b);
      double s = 0.0; for (int i = 0; i < 6; i++) s += rr[i] * rr[i];
      c += 0.5 * s;
      if (jac) { std::copy(rr, rr + 6, &r[6 * e]); std::copy(a, a + 36, &Ja[36 * e]); std::copy(b, b + 36, &Jb[36 * e]); }
    }
    *cost = c; return std::isfinite(c);
  }
};

// Minimizes in place.  Pose 0 and poses no edge touches do not move.
// function_tolerance, parameter_tolerance: ceres' 1e-6 and 1e-8 by default (a test can tighten them to reach the optimum itself).
inline void optimize(std::vector<Pose>& X, const std::vector<Edge>& edges, int max_iterations, Summary* S, double function_tolerance = 1e-6, double parameter_tolerance = 1e-8) {
  *S = Summary();
  if (edges.empty()) return;
  Problem P; P.N = (int)X.size(); P.E = edges; P.fidx.assign(P.N, -1);
  std::vector<char> touched(P.N, 0); for (auto& e : edges) { touched[e.a] = 1; touched[e.b] = 1; }
  for (int n = 1; n < P.N; n++) if (touched[n]) { P.fidx[n] = (int)P.fnode.size(); P.fnode.push_back(n); }
  const int F = (int)P.fnode.size(), n = 6 * F; const size_t M = edges.size();
  P.r.resize(6 * M); P.Ja.resize(36 * M); P.Jb.resize(36 * M);
  std::vector<int> first(n);
  { std::vector<int> lo(F); for (int f = 0; f < F; f++) lo[f] = f;
    for (auto& e : edges) { const int fa = P.fidx[e.a], fb = P.fidx[e.b]; if (fa >= 0 && fb >= 0) { lo[fa] = std::min(lo[fa], fb); lo[fb] = std::min(lo[fb], fa); } }
    for (int f = 0; f < F; f++) for (int i = 0; i < 6; i++) first[6 * f + i] = 6 * lo[f]; }
  Skyline K;
  auto norm_x = [&](const std::vector<Pose>& Y) { double s = 0; for (int f = 0; f < F; f++) { const Pose& p = Y[P.fnode[f]]; for (int k = 0; k < 4; k++) s += p.q[k] * p.q[k]; for (int k = 0; k < 3; k++) s += p.t[k] * p.t[k]; } return std::sqrt(s); };
  std::vector<double> g(n), scaling(n), diagonal(n), colsq(n), step(n), delta(n);
  double x_cost = 0;
  auto eval_grad_jac = [&](const std::vector<Pose>& Y, bool first_eval) -> bool {
    S->evaluations++;
    if (!P.evaluate(Y, &x_cost, true)) return false;
    std::fill(g.begin(), g.end(), 0.0); std::fill(colsq.begin(), colsq.end(), 0.0);
    for (size_t e = 0; e < M; e++) for (int s = 0; s < 2; s++) {
      const int f = P.fidx[s ? edges[e].b : edges[e].a]; if (f < 0) continue;
      const double* J = s ? &P.Jb[36 * e] : &P.Ja[36 * e];
      for (int c = 0; c < 6; c++) for (int i = 0; i < 6; i++) { g[6 * f + c] += J[i * 6 + c] * P.r[6 * e + i]; colsq[6 * f + c] += J[i * 6 + c] * J[i * 6 + c]; }
    }
    if (first_eval) for (int c = 0; c < n; c++) scaling[c] = 1.0 / (1.0 + std::sqrt(colsq[c]));
    return true;
  };
  auto gmax = [&](const std::vector<Pose>& Y) {
    double m = 0; for (int f = 0; f < F; f++) { double ng[6]; for (int c = 0; c < 6; c++) ng[c] = -g[6 * f + c]; Pose o; const Pose& p = Y[P.fnode[f]]; plus(p, ng, o);
      for (int k = 0; k < 4; k++) m = std::max(m, std::fabs(p.q[k] - o.q[k])); for (int k = 0; k < 3; k++) m = std::max(m, std::fabs(p.t[k] - o.t[k])); }
    return m;
  };
  if (!eval_grad_jac(X, true)) { S->initial_cost = S->final_cost = x_cost; S->termination = 4; return; }
  S->initial_cost = x_cost; double min_iter_cost = x_cost;
  double x_norm = norm_x(X);
  double radius = 1e4, decrease_factor = 2.0; bool reuse_diagonal = false; int num_invalid = 0, iteration = 0; bool last_successful = true; double last_gmax = gmax(X);
  std::vector<Pose> cand = X;
  for (;;) {
    if (iteration >= max_iterations) { S->termination = 0; break; }
    if (last_successful && last_gmax <= 1e-10) { S->termination = 1; break; }
    if (radius <= 1e-32) { S->termination = 5; break; }
    iteration++; S->iterations = iteration;
    if (!reuse_diagonal) for (int c = 0; c < n; c++) diagonal[c] = std::min(std::max(colsq[c] * scaling[c] * scaling[c], 1e-6), 1e32);
    K.shape(first);
    for (size_t e = 0; e < M; e++) {   // (J S)^T (J S), block by block
      const int f[2] = {P.fidx[edges[e].a], P.fidx[edges[e].b]}; const double* Jp[2] = {&P.Ja[36 * e], &P.Jb[36 * e]};
      for (int u = 0; u < 2; u++) for (int v = 0; v < 2; v++) {
        if (f[u] < 0 || f[v] < 0 || f[u] < f[v]) continue;
        for (int i = 0; i < 6; i++) for (int j = 0; j < 6; j++) {
          const int R = 6 * f[u] + i, Cc = 6 * f[v] + j; if (Cc > R) continue;
          double s = 0; for (int k = 0; k < 6; k++) s += (Jp[u][k * 6 + i] * scaling[R]) * (Jp[v][k * 6 + j] * scaling[Cc]);
          K.at(R, Cc) += s;
        }
      }
    }
    for (int c = 0; c < n; c++) { const double d = std::sqrt(diagonal[c] / radius); K.at(c, c) += d * d; }
    for (int c = 0; c < n; c++) step[c] = g[c] * scaling[c];
    bool solved = K.factor();
    if (solved) { K.solve(step); for (int c = 0; c < n; c++) { step[c] = -step[c]; if (!std::isfinite(step[c])) solved = false; } }
    reuse_diagonal = true;
    double mcc = 0; bool valid = false;
    if (solved) {
      for (int c = 0; c < n; c++) delta[c] = step[c] * scaling[c];
      double mc = 0;
      for (size_t e = 0; e < M; e++) {
        const int fa = P.fidx[edges[e].a], fb = P.fidx[edges[e].b];
        for (int i = 0; i < 6; i++) {
          double m = 0; for (int j = 0; j < 6; j++) { if (fa >= 0) m += P.Ja[36 * e + i * 6 + j] * delta[6 * fa + j]; if (fb >= 0) m += P.Jb[36 * e + i * 6 + j] * delta[6 * fb + j]; }
          mc += m * (P.r[6 * e + i] + m / 2.0);
        }
      }
      mcc = -mc; valid = mcc > 0.0;
    }
    if (!valid) {
      if (++num_invalid >= 5) { S->termination = 4; break; }
      radius = radius / decrease_factor; decrease_factor *= 2.0; last_successful = false; continue;
    }
    num_invalid = 0;
    cand = X;
    for (int f = 0; f < F; f++) plus(X[P.fnode[f]], &delta[6 * f], cand[P.fnode[f]]);
    double cand_cost; S->evaluations++;
    if (!P.evaluate(cand, &cand_cost, false)) cand_cost = std::numeric_limits<double>::max();
    double sn = 0; for (int f = 0; f < F; f++) { const Pose &a = X[P.fnode[f]], &b = cand[P.fnode[f]];
      for (int k = 0; k < 4; k++) sn += (a.q[k] - b.q[k]) * (a.q[k] - b.q[k]); for (int k = 0; k < 3; k++) sn += (a.t[k] - b.t[k]) * (a.t[k] - b.t[k]); }
    if (std::sqrt(sn) <= parameter_tolerance * (x_norm + parameter_tolerance)) { S->termination = 2; break; }
    if (std::fabs(x_cost - cand_cost) <= function_tolerance * x_cost) { S->termination = 3; break; }
    const double rel = (x_cost - cand_cost) / mcc;
    if (rel > 1e-3) {
      X = cand; x_norm = norm_x(X);
      S->evaluations--;   // the candidate's evaluation is the new point's
      eval_grad_jac(X, false); last_gmax = gmax(X); last_successful = true;
      radius = std::min(1e16, radius / std::max(1.0 / 3.0, 1.0 - std::pow(2.0 * rel - 1.0, 3))); decrease_factor = 2.0; reuse_diagonal = false;
      min_iter_cost = std::min(min_iter_cost, x_cost);
    } else {
      radius = radius / decrease_factor; decrease_factor *= 2.0; last_successful = false; min_iter_cost = std::min(min_iter_cost, cand_cost);
    }
  }
  S->final_cost = std::min(S->initial_cost, min_iter_cost);
}

// add_constrain_of_loop after laser_mapping.hpp:1065-1066's inversion of the ICP pose.  Eigen's inverse(): conjugate / squared norm.
inline void qinv(const double* q, double* o) {
  const double n2 = (q[1] * q[1] + q[3] * q[3]) + (q[2] * q[2] + q[0] * q[0]);
  if (n2 > 0.0) { o[0] = q[0] / n2; for (int k = 1; k < 4; k++) o[k] = -q[k] / n2; } else for (int k = 0; k < 4; k++) o[k] = 0.0;
}
inline Edge loop_edge(const double* icp_q, const double* icp_t, const Pose& A, int id_a, const Pose& B, int id_b) {
  Edge E{}; double iq[4], it[3], nt[3] = {-icp_t[0], -icp_t[1], -icp_t[2]};
  qinv(icp_q, iq); qrot(iq, nt, it);
  double qbi[4], iqi[4], t1[4]; qinv(B.q, qbi); qinv(iq, iqi);
  qmul(qbi, iqi, t1); qmul(t1, A.q, E.q);
  const double d[3] = {A.t[0] - it[0], A.t[1] - it[1], A.t[2] - it[2]}; double r[3]; qrot(iqi, d, r);
  const double u[3] = {r[0] - B.t[0], r[1] - B.t[1], r[2] - B.t[2]}; qrot(qbi, u, E.t);
  E.a = id_b; E.b = id_a; for (int k = 0; k < 6; k++) E.W[k * 7] = 1.0;
  return E;
}

// Mapping_refine::refine_pts (ceres_pose_graph_3d.hpp:437-451) after the if_save == 0 VoxelGrid of refine_pointcloud (:475-479).
inline void rotation(const double* q, double* R) {   // Eigen's toRotationMatrix, q as w, x, y, z
  const double w = q[0], x = q[1], y = q[2], z = q[3];
  const double tx = 2 * x, ty = 2 * y, tz = 2 * z, twx = tx * w, twy = ty * w, twz = tz * w, txx = tx * x, txy = ty * x, txz = tz * x, tyy = ty * y,
               tyz = tz * y, tzz = tz * z;
  const double m[9] = {1 - (tyy + tzz), txy - twz, txz + twy, txy + twz, 1 - (txx + tzz), tyz - twx, txz - twy, tyz + twx, 1 - (txx + tyy)};
  for (int i = 0; i < 9; i++) R[i] = m[i];
}
// in / out: n points of 4 floats (x, y, z, intensity); returns the count kept.  The output intensity is 0 (eigen_to_pcl_pt sets x, y, z only).
inline int repose(const float* in, int n, float leaf, const Pose& ori, const Pose& opt, float* out) {
  std::vector<float> ds(4 * (size_t)std::max(n, 1));
  const int m = orc::voxel_grid(in, n, leaf, ds.data());
  double Ro[9], Rp[9]; rotation(ori.q, Ro); rotation(opt.q, Rp);
  float Ra[9], Ta[3];
  for (int i = 0; i < 3; i++) for (int j = 0; j < 3; j++) { double v = 0; for (int k = 0; k < 3; k++) v += Rp[3 * i + k] * Ro[3 * j + k]; Ra[3 * i + j] = (float)v; }
  for (int i = 0; i < 3; i++) { double v = 0; for (int k = 0; k < 3; k++) v += (double)Ra[3 * i + k] * (-ori.t[k]); Ta[i] = (float)(v + opt.t[i]); }
  for (int p = 0; p < m; p++) {
    for (int i = 0; i < 3; i++) { float v = 0.f; for (int k = 0; k < 3; k++) v += Ra[3 * i + k] * ds[4 * p + k]; out[4 * p + i] = v + Ta[i]; }
    out[4 * p + 3] = 0.f;
  }
  return m;
}

}  // namespace orc_pg
