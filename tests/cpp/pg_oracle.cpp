// C entry points of the pose-graph oracle (oracle/orc_pose_graph.hpp) for the tests: poses as rows (qw, qx, qy, qz, tx, ty, tz), edges as
// ids (begin, end), measurements as rows of 7 in the same layout and information matrices as 36 doubles, row-major.
#include "../../oracle/orc_pose_graph.hpp"

static orc_pg::Pose pgo_pose(const double* p) { orc_pg::Pose o; for (int k = 0; k < 4; k++) o.q[k] = p[k]; for (int k = 0; k < 3; k++) o.t[k] = p[4 + k]; return o; }
static orc_pg::Edge pgo_edge(int a, int b, const double* meas, const double* W) {
  orc_pg::Edge e; e.a = a; e.b = b;
  for (int k = 0; k < 4; k++) e.q[k] = meas[k];
  for (int k = 0; k < 3; k++) e.t[k] = meas[4 + k];
  for (int k = 0; k < 36; k++) e.W[k] = W[k];
  return e;
}

extern "C" {

// dsum: initial cost, final cost; isum: iterations, evaluations, termination
// ftol, ptol: the function and parameter tolerances (ceres' 1e-6, 1e-8)
void pgo_optimize(double* poses, int n, const int* ids, const double* meas, const double* W, int m, int max_iterations, double ftol, double ptol, double* dsum, int* isum) {
  std::vector<orc_pg::Pose> X(n); for (int i = 0; i < n; i++) X[i] = pgo_pose(poses + 7 * i);
  std::vector<orc_pg::Edge> E(m); for (int e = 0; e < m; e++) E[e] = pgo_edge(ids[2 * e], ids[2 * e + 1], meas + 7 * e, W + 36 * e);
  orc_pg::Summary S; orc_pg::optimize(X, E, max_iterations, &S, ftol, ptol);
  for (int i = 0; i < n; i++) { for (int k = 0; k < 4; k++) poses[7 * i + k] = X[i].q[k]; for (int k = 0; k < 3; k++) poses[7 * i + 4 + k] = X[i].t[k]; }
  dsum[0] = S.initial_cost; dsum[1] = S.final_cost; isum[0] = S.iterations; isum[1] = S.evaluations; isum[2] = S.termination;
}

void pgo_residual(const double* pa, const double* pb, const double* meas, const double* W, double* r, double* Ja, double* Jb) {
  orc_pg::residual(pgo_pose(pa), pgo_pose(pb), pgo_edge(0, 1, meas, W), r, Ja, Jb);
}

// Solves the SPD system A x = b (n x n, row-major, dense input) with the skyline factorization, envelope from the first nonzero per row.
int pgo_skyline_solve(const double* A, const double* b, int n, double* x) {
  std::vector<int> first(n);
  for (int r = 0; r < n; r++) { int c = 0; while (c < r && A[(size_t)r * n + c] == 0.0) c++; first[r] = c; }
  orc_pg::Skyline K; K.shape(first);
  for (int r = 0; r < n; r++) for (int c = first[r]; c <= r; c++) K.at(r, c) = A[(size_t)r * n + c];
  if (!K.factor()) return 0;
  std::vector<double> v(b, b + n); K.solve(v);
  for (int r = 0; r < n; r++) x[r] = v[r];
  return 1;
}

// clouds: n points of 4 floats; keyframe k = [seg_end[k - 1], seg_end[k]); poses as rows of 7.  Returns the total kept.
int pgo_repose(const float* clouds, const long long* seg_end, int n_kf, const double* ori, const double* opt, float leaf, float* out, long long* n_out) {
  int w = 0;
  for (int k = 0; k < n_kf; k++) {
    const long long b = k ? seg_end[k - 1] : 0;
    const int m = orc_pg::repose(clouds + 4 * b, (int)(seg_end[k] - b), leaf, pgo_pose(ori + 7 * k), pgo_pose(opt + 7 * k), out + 4 * (size_t)w);
    n_out[k] = m; w += m;
  }
  return w;
}

void pgo_loop_edge(const double* icp_q, const double* icp_t, const double* pa, int id_a, const double* pb, int id_b, int* ids, double* meas) {
  const orc_pg::Edge e = orc_pg::loop_edge(icp_q, icp_t, pgo_pose(pa), id_a, pgo_pose(pb), id_b);
  ids[0] = e.a; ids[1] = e.b;
  for (int k = 0; k < 4; k++) meas[k] = e.q[k];
  for (int k = 0; k < 3; k++) meas[4 + k] = e.t[k];
}

}
