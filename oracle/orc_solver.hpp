// ORACLE — TEST INFRASTRUCTURE ONLY (see orc_math.hpp header). PARITY UNPINNED.
// CPU restatement of what the reference delegates to Ceres Solver (third-party, not vendored, not
// version-pinned: loam_livox/CMakeLists.txt:23; API use implies 1.10 <= version < 2.2; the 1.14 behaviour
// is restated) for the 7-parameter (q_incre[4] on the Eigen-quaternion manifold + t_incre[3], box-bounded)
// robust least-squares problem built at loam_livox/source/point_cloud_registration.hpp:220-228,323,422
// and solved at :460-474,:501-508.
//
//   residual functors  loam_livox/source/ceres_icp.hpp:238-301 (point2line), :306-380 (point2plane),
//                      :81-148 / :152-233 (motion-deblur variants), evaluated with forward-mode Jets exactly
//                      like ceres::AutoDiffCostFunction<F,3,4,3>
//   loss               ceres::HuberLoss(0.1) shared by every block (:220), Corrector with rho'' <= 0
//   manifold           ceres::EigenQuaternionParameterization (:221)
//   minimizer          ceres TrustRegionMinimizer + LevenbergMarquardtStrategy, library defaults,
//                      is_constrained = true (bounds on t, :143-151) => projected Armijo line search per step
//   linear solver      DENSE_SCHUR (:43) == exact solve of the damped 6x6 normal equations
#pragma once
#include <algorithm>
#include <cmath>
#include <complex>
#include <cstdio>
#include <limits>
#include <vector>
#include "orc_math.hpp"

namespace orc {

struct ResidualBlock {
  int type;        // 0 = point2line, 1 = point2plane
  int motion_blur; // 1 = *_mb functor
  double p[3];     // m_current_pt (scan frame)
  double a[3];     // m_target_line_a
  double v[3];     // m_unit_vec_ab (line) or m_unit_vec_n = u_ab x u_ac, NOT re-normalised (plane)
  double s;        // m_motion_blur_s
  int src;         // 0 corner / 1 surface, index of the generating feature (for tests)
  int src_index;
};

// ceres_icp.hpp:246-260
inline void make_point2line(ResidualBlock& b, const double p[3], const double ta[3], const double tb[3]) {
  b.type = 0; b.motion_blur = 0; b.s = 1.0;
  double u[3] = {tb[0] - ta[0], tb[1] - ta[1], tb[2] - ta[2]};
  double n = std::sqrt(u[0] * u[0] + u[1] * u[1] + u[2] * u[2]);
  for (int k = 0; k < 3; k++) { b.p[k] = p[k]; b.a[k] = ta[k]; b.v[k] = u[k] / n; }
}
// ceres_icp.hpp:314-336
inline void make_point2plane(ResidualBlock& b, const double p[3], const double ta[3], const double tb[3], const double tc[3]) {
  b.type = 1; b.motion_blur = 0; b.s = 1.0;
  double ab[3] = {tb[0] - ta[0], tb[1] - ta[1], tb[2] - ta[2]};
  double nab = std::sqrt(ab[0] * ab[0] + ab[1] * ab[1] + ab[2] * ab[2]);
  for (int k = 0; k < 3; k++) ab[k] = ab[k] / nab;
  double ac[3] = {tc[0] - ta[0], tc[1] - ta[1], tc[2] - ta[2]};
  double nac = std::sqrt(ac[0] * ac[0] + ac[1] * ac[1] + ac[2] * ac[2]);
  for (int k = 0; k < 3; k++) ac[k] = ac[k] / nac;
  b.v[0] = ab[1] * ac[2] - ab[2] * ac[1]; b.v[1] = ab[2] * ac[0] - ab[0] * ac[2]; b.v[2] = ab[0] * ac[1] - ab[1] * ac[0];
  for (int k = 0; k < 3; k++) { b.p[k] = p[k]; b.a[k] = ta[k]; }
}

// operator() of the four functors (ceres_icp.hpp:262-288, :338-366, :106-134, :187-218). _q is Eigen storage order x,y,z,w.
template <typename T>
inline void eval_functor(const ResidualBlock& b, const Qd& q_last_d, const V3d& t_last_d, const T* _q, const T* _t, T* residual) {
  Quat<T> q_last{T(q_last_d.w), T(q_last_d.x), T(q_last_d.y), T(q_last_d.z)};
  Vec3<T> t_last{T(t_last_d.x), T(t_last_d.y), T(t_last_d.z)};
  Quat<T> q_incre{_q[3], _q[0], _q[1], _q[2]};
  Vec3<T> t_incre{_t[0], _t[1], _t[2]};
  Vec3<T> pt{T(b.p[0]), T(b.p[1]), T(b.p[2])};
  Vec3<T> pt_tr;
  if (b.motion_blur) {
    Quat<T> q_id{T(1.0), T(0.0), T(0.0), T(0.0)};
    Quat<T> q_interp = qslerp(q_id, T(b.s), q_incre);
    Vec3<T> t_interp = t_incre * T(b.s);
    pt_tr = qrot(q_last, qrot(q_interp, pt) + t_interp) + t_last;
  } else {
    pt_tr = qrot(q_last, qrot(q_incre, pt) + t_incre) + t_last;
  }
  Vec3<T> a{T(b.a[0]), T(b.a[1]), T(b.a[2])};
  Vec3<T> v{T(b.v[0]), T(b.v[1]), T(b.v[2])};
  Vec3<T> d = pt_tr - a;
  Vec3<T> r;
  if (b.type == 0) r = d - dot(d, v) * v;  // vec_ac - project_on_unit_vector(vec_ac, unit_ab)
  else r = dot(d, v) * v;                  // project_on_unit_vector(vec_ad, n) ; m_weigh == 1
  residual[0] = r.x; residual[1] = r.y; residual[2] = r.z;
}

// ceres::HuberLoss::Evaluate
inline void huber(double a, double s, double rho[3]) {
  const double b = a * a;
  if (s > b) { const double r = std::sqrt(s); rho[0] = 2.0 * a * r - b; rho[1] = std::max(std::numeric_limits<double>::min(), a / r); rho[2] = -rho[1] / (2.0 * s); }
  else { rho[0] = s; rho[1] = 1.0; rho[2] = 0.0; }
}

struct Problem {
  std::vector<ResidualBlock> blocks;
  Qd q_last{1, 0, 0, 0}; V3d t_last{0, 0, 0};
  double huber_a = 0.1;
  double t_bound = 2.0;   // |t_incre[j]| <= m_para_max_speed
  int num_threads = 1;    // CPU-baseline knob only (ceres default is 1)

  // ceres::EigenQuaternionParameterization::Plus + box projection of ParameterBlock::Plus.
  void plus(const double x[7], const double delta[6], double out[7]) const {
    const double nd = std::sqrt(delta[0] * delta[0] + delta[1] * delta[1] + delta[2] * delta[2]);
    if (nd > 0.0) {
      const double sbd = std::sin(nd) / nd;
      Qd dq{std::cos(nd), sbd * delta[0], sbd * delta[1], sbd * delta[2]};
      Qd q{x[3], x[0], x[1], x[2]};
      Qd r = qmul(dq, q);
      out[0] = r.x; out[1] = r.y; out[2] = r.z; out[3] = r.w;
    } else { out[0] = x[0]; out[1] = x[1]; out[2] = x[2]; out[3] = x[3]; }
    for (int k = 0; k < 3; k++) {
      double v = x[4 + k] + delta[3 + k];
      out[4 + k] = std::min(std::max(v, -t_bound), t_bound);
    }
  }

  // ProgramEvaluator::Evaluate: cost = sum 0.5*rho(|r|^2); residuals/jacobian loss-corrected (Corrector, alpha = 0);
  // jacobian in the 6-dim tangent space (3 rows per block, row-major 6 cols), gradient = J^T r.
  bool evaluate(const double x[7], double* cost, std::vector<double>* residuals, double* gradient, std::vector<double>* jac) const {
    const size_t M = blocks.size();
    if (residuals) residuals->assign(3 * M, 0.0);
    if (jac) jac->assign(18 * M, 0.0);
    const bool need_j = (gradient != nullptr) || (jac != nullptr);
    // EigenQuaternionParameterization::ComputeJacobian (4x3, rows x,y,z,w)
    const double PJ[4][3] = {{x[3], x[2], -x[1]}, {-x[2], x[3], x[0]}, {x[1], -x[0], x[3]}, {-x[0], -x[1], -x[2]}};
    double total = 0; double g[6] = {0, 0, 0, 0, 0, 0};
#pragma omp parallel for num_threads(num_threads) reduction(+ : total, g[:6]) schedule(static) if (num_threads > 1)
    for (size_t i = 0; i < M; i++) {
      const ResidualBlock& b = blocks[i];
      double r[3]; double J[3][6];
      if (need_j) {
        typedef Jet<7> J7;
        J7 q[4], t[3], res[3];
        for (int k = 0; k < 4; k++) q[k] = J7(x[k], k);
        for (int k = 0; k < 3; k++) t[k] = J7(x[4 + k], 4 + k);
        eval_functor<J7>(b, q_last, t_last, q, t, res);
        for (int rr = 0; rr < 3; rr++) {
          r[rr] = res[rr].a;
          for (int c = 0; c < 3; c++) J[rr][c] = res[rr].v[0] * PJ[0][c] + res[rr].v[1] * PJ[1][c] + res[rr].v[2] * PJ[2][c] + res[rr].v[3] * PJ[3][c];
          for (int c = 0; c < 3; c++) J[rr][3 + c] = res[rr].v[4 + c];
        }
      } else {
        eval_functor<double>(b, q_last, t_last, x, x + 4, r);
      }
      const double sq = r[0] * r[0] + r[1] * r[1] + r[2] * r[2];
      double rho[3]; huber(huber_a, sq, rho);
      total += 0.5 * rho[0];
      const double sc = std::sqrt(rho[1]);  // Corrector: rho[2] <= 0 => residual_scaling = sqrt(rho'), alpha = 0
      if (need_j) for (int rr = 0; rr < 3; rr++) for (int c = 0; c < 6; c++) J[rr][c] *= sc;
      for (int rr = 0; rr < 3; rr++) r[rr] *= sc;
      if (residuals) for (int rr = 0; rr < 3; rr++) (*residuals)[3 * i + rr] = r[rr];
      if (jac) for (int rr = 0; rr < 3; rr++) for (int c = 0; c < 6; c++) (*jac)[18 * i + 6 * rr + c] = J[rr][c];
      if (gradient) for (int c = 0; c < 6; c++) g[c] += J[0][c] * r[0] + J[1][c] * r[1] + J[2][c] * r[2];
    }
    *cost = total;
    if (gradient) for (int c = 0; c < 6; c++) gradient[c] = g[c];
    return std::isfinite(total);
  }
};

// ---------------------------------------------------------------------------------- polynomial helpers
// ceres/internal/polynomial.cc: FindInterpolatingPolynomial / MinimizePolynomial. Highest degree first.
struct FunctionSample { double x = 0, value = 0, gradient = 0; bool value_is_valid = false, gradient_is_valid = false; };

inline double eval_poly(const std::vector<double>& p, double x) { double v = 0; for (double c : p) v = v * x + c; return v; }

inline bool solve_dense(std::vector<std::vector<double>>& A, std::vector<double>& b) {  // Gaussian elimination, full pivoting
  const int n = (int)b.size(); std::vector<int> perm(n); for (int i = 0; i < n; i++) perm[i] = i;
  for (int c = 0; c < n; c++) {
    int pr = c, pc = c; double best = 0;
    for (int i = c; i < n; i++) for (int j = c; j < n; j++) if (std::fabs(A[i][j]) > best) { best = std::fabs(A[i][j]); pr = i; pc = j; }
    if (best == 0) return false;
    std::swap(A[c], A[pr]); std::swap(b[c], b[pr]);
    for (int i = 0; i < n; i++) std::swap(A[i][c], A[i][pc]);
    std::swap(perm[c], perm[pc]);
    for (int i = c + 1; i < n; i++) { double f = A[i][c] / A[c][c]; for (int j = c; j < n; j++) A[i][j] -= f * A[c][j]; b[i] -= f * b[c]; }
  }
  std::vector<double> y(n);
  for (int i = n - 1; i >= 0; i--) { double s = b[i]; for (int j = i + 1; j < n; j++) s -= A[i][j] * y[j]; y[i] = s / A[i][i]; }
  std::vector<double> xx(n); for (int i = 0; i < n; i++) xx[perm[i]] = y[i];
  b = xx; return true;
}

inline std::vector<double> find_interpolating_polynomial(const std::vector<FunctionSample>& samples) {
  int num_constraints = 0;
  for (auto& s : samples) { if (s.value_is_valid) num_constraints++; if (s.gradient_is_valid) num_constraints++; }
  const int degree = num_constraints - 1;
  std::vector<std::vector<double>> A(num_constraints, std::vector<double>(num_constraints, 0.0)); std::vector<double> rhs(num_constraints, 0.0);
  int row = 0;
  for (auto& s : samples) {
    if (s.value_is_valid) { for (int j = 0; j <= degree; j++) A[row][j] = std::pow(s.x, degree - j); rhs[row] = s.value; row++; }
    if (s.gradient_is_valid) { for (int j = 0; j < degree; j++) A[row][j] = (degree - j) * std::pow(s.x, degree - j - 1); rhs[row] = s.gradient; row++; }
  }
  solve_dense(A, rhs);
  return rhs;
}

// Real parts of all roots (ceres MinimizePolynomial tests the real part of every root, complex ones included).
inline std::vector<double> poly_root_real_parts(std::vector<double> p) {
  while (!p.empty() && p[0] == 0.0) p.erase(p.begin());
  std::vector<double> out; const int deg = (int)p.size() - 1;
  if (deg < 1) return out;
  if (deg == 1) { out.push_back(-p[1] / p[0]); return out; }
  if (deg == 2) {  // FindQuadraticPolynomialRoots
    const double a = p[0], b = p[1], c = p[2], D = b * b - 4 * a * c, sqrt_D = std::sqrt(std::fabs(D));
    if (D >= 0) {
      if (b >= 0) { out.push_back((-b - sqrt_D) / (2.0 * a)); out.push_back((2.0 * c) / (-b - sqrt_D)); }
      else { out.push_back((2.0 * c) / (-b + sqrt_D)); out.push_back((-b + sqrt_D) / (2.0 * a)); }
    } else { out.push_back(-b / (2.0 * a)); out.push_back(-b / (2.0 * a)); }
    return out;
  }
  // general degree: Durand–Kerner on the monic polynomial (ceres uses companion-matrix eigenvalues)
  std::vector<std::complex<double>> z(deg), c(deg + 1);
  for (int i = 0; i <= deg; i++) c[i] = p[i] / p[0];
  double rad = 0; for (int i = 1; i <= deg; i++) rad = std::max(rad, std::abs(c[i]));
  rad = 1.0 + rad;
  for (int i = 0; i < deg; i++) z[i] = std::polar(rad * 0.5, 2.0 * M_PI * i / deg + 0.4);
  for (int it = 0; it < 500; it++) {
    double change = 0;
    for (int i = 0; i < deg; i++) {
      std::complex<double> num = 0; for (int k = 0; k <= deg; k++) num = num * z[i] + c[k];
      std::complex<double> den = 1; for (int j = 0; j < deg; j++) if (j != i) den *= (z[i] - z[j]);
      if (std::abs(den) == 0) den = 1e-300;
      std::complex<double> dz = num / den; z[i] -= dz; change = std::max(change, std::abs(dz));
    }
    if (change < 1e-15 * rad) break;
  }
  for (auto& r : z) out.push_back(r.real());
  return out;
}

inline void minimize_polynomial(const std::vector<double>& poly, double x_min, double x_max, double* optimal_x, double* optimal_value) {
  *optimal_x = (x_min + x_max) / 2.0; *optimal_value = eval_poly(poly, *optimal_x);
  const double vmin = eval_poly(poly, x_min); if (vmin < *optimal_value) { *optimal_value = vmin; *optimal_x = x_min; }
  const double vmax = eval_poly(poly, x_max); if (vmax < *optimal_value) { *optimal_value = vmax; *optimal_x = x_max; }
  if (poly.size() <= 2) return;
  const int deg = (int)poly.size() - 1; std::vector<double> der(deg);
  for (int i = 0; i < deg; i++) der[i] = (deg - i) * poly[i];
  for (double root : poly_root_real_parts(der)) {
    if (!(root >= x_min && root <= x_max)) continue;
    const double v = eval_poly(poly, root); if (v < *optimal_value) { *optimal_value = v; *optimal_x = root; }
  }
}

// ---------------------------------------------------------------------------------- trust-region minimizer
struct SolveOptions {
  int max_num_iterations = 50;
  double initial_trust_region_radius = 1e4, max_trust_region_radius = 1e16, min_trust_region_radius = 1e-32;
  double min_relative_decrease = 1e-3, min_lm_diagonal = 1e-6, max_lm_diagonal = 1e32;
  double function_tolerance = 1e-6, gradient_tolerance = 1e-10, parameter_tolerance = 1e-8;
  int max_num_consecutive_invalid_steps = 5;
  // Armijo line search (projected, because the problem is bounds-constrained)
  double ls_sufficient_decrease = 1e-4, ls_max_step_contraction = 1e-3, ls_min_step_contraction = 0.6, ls_min_step_size = 1e-9;
  int ls_max_num_iterations = 20;
};
struct SolveSummary {
  double initial_cost = 0, final_cost = 0; int num_residual_blocks = 0;
  int iterations = 0, num_successful_steps = 0, num_unsuccessful_steps = 0, num_line_search_steps = 0;
  int num_cost_evals = 0, num_jac_evals = 0;
  int termination = 0;  // 0 no_convergence(max iter) 1 gradient tol 2 parameter tol 3 function tol 4 failure 5 radius
};

inline bool cholesky_solve6(const double A[6][6], const double b[6], double x[6]) {
  double L[6][6] = {};
  for (int i = 0; i < 6; i++)
    for (int j = 0; j <= i; j++) {
      double s = A[i][j]; for (int k = 0; k < j; k++) s -= L[i][k] * L[j][k];
      if (i == j) { if (!(s > 0.0)) return false; L[i][i] = std::sqrt(s); } else L[i][j] = s / L[j][j];
    }
  double y[6];
  for (int i = 0; i < 6; i++) { double s = b[i]; for (int k = 0; k < i; k++) s -= L[i][k] * y[k]; y[i] = s / L[i][i]; }
  for (int i = 5; i >= 0; i--) { double s = y[i]; for (int k = i + 1; k < 6; k++) s -= L[k][i] * x[k]; x[i] = s / L[i][i]; }
  for (int i = 0; i < 6; i++) if (!std::isfinite(x[i])) return false;
  return true;
}

// ceres::Solve on `x` (7 doubles, q in Eigen order x,y,z,w then t). Restates TrustRegionMinimizer::Minimize (1.14).
inline void solve(const Problem& prob, const SolveOptions& opt, double x_io[7], SolveSummary* sum) {
  *sum = SolveSummary(); sum->num_residual_blocks = (int)prob.blocks.size();
  const size_t M = prob.blocks.size();
  if (M == 0) { sum->termination = 3; return; }  // ceres: nothing to optimise, costs stay 0
  double x[7], cand[7]; for (int k = 0; k < 7; k++) x[k] = x_io[k];
  std::vector<double> residuals, jac, model_res(3 * M);
  double gradient[6], scaling[6], x_cost = 0, cand_cost = 0;
  // --- IterationZero: project onto the bounds (Plus with zero delta), evaluate
  { const double z[6] = {0, 0, 0, 0, 0, 0}; prob.plus(x, z, cand); for (int k = 0; k < 7; k++) x[k] = cand[k]; }
  double x_norm = 0; for (int k = 0; k < 7; k++) x_norm += x[k] * x[k]; x_norm = std::sqrt(x_norm);
  auto eval_grad_jac = [&](int iteration) -> bool {
    sum->num_cost_evals++; sum->num_jac_evals++;
    if (!prob.evaluate(x, &x_cost, &residuals, gradient, &jac)) return false;
    if (iteration == 0) {  // jacobi scaling from the initial jacobian only
      double cn[6] = {0, 0, 0, 0, 0, 0};
      for (size_t r = 0; r < 3 * M; r++) for (int c = 0; c < 6; c++) cn[c] += jac[6 * r + c] * jac[6 * r + c];
      for (int c = 0; c < 6; c++) scaling[c] = 1.0 / (1.0 + std::sqrt(cn[c]));
    }
    for (size_t r = 0; r < 3 * M; r++) for (int c = 0; c < 6; c++) jac[6 * r + c] *= scaling[c];
    return true;
  };
  auto gradient_max_norm = [&]() -> double {  // |x - Plus(x, -g)|_inf in the ambient space
    double ng[6], pg[7]; for (int c = 0; c < 6; c++) ng[c] = -gradient[c];
    prob.plus(x, ng, pg); double m = 0; for (int k = 0; k < 7; k++) m = std::max(m, std::fabs(x[k] - pg[k])); return m;
  };
  if (!eval_grad_jac(0)) { sum->termination = 4; return; }
  sum->initial_cost = x_cost; double min_iter_cost = x_cost; double minimum_cost = x_cost;
  for (int k = 0; k < 7; k++) x_io[k] = x[k];  // iteration 0 counts as successful: the projected point is written back
  double radius = opt.initial_trust_region_radius, decrease_factor = 2.0; bool reuse_diagonal = false; double diagonal[6] = {0, 0, 0, 0, 0, 0};
  int num_consecutive_invalid = 0; int iteration = 0; bool last_successful = true; double last_gmax = gradient_max_norm();
  double current_cost_eval = x_cost;  // TrustRegionStepEvaluator (monotonic mode): reference == current
  for (;;) {
    // FinalizeIterationAndCheckIfMinimizerCanContinue
    if (iteration >= opt.max_num_iterations) { sum->termination = 0; break; }
    if (last_successful && last_gmax <= opt.gradient_tolerance) { sum->termination = 1; break; }
    if (radius <= opt.min_trust_region_radius) { sum->termination = 5; break; }
    iteration++; sum->iterations = iteration;
    // --- ComputeTrustRegionStep (LevenbergMarquardtStrategy::ComputeStep)
    if (!reuse_diagonal) {
      for (int c = 0; c < 6; c++) diagonal[c] = 0;
      for (size_t r = 0; r < 3 * M; r++) for (int c = 0; c < 6; c++) diagonal[c] += jac[6 * r + c] * jac[6 * r + c];
      for (int c = 0; c < 6; c++) diagonal[c] = std::min(std::max(diagonal[c], opt.min_lm_diagonal), opt.max_lm_diagonal);
    }
    double A[6][6] = {}, rhs[6] = {0, 0, 0, 0, 0, 0};
    for (size_t r = 0; r < 3 * M; r++) {
      const double* jr = &jac[6 * r];
      for (int i = 0; i < 6; i++) { rhs[i] += jr[i] * residuals[r]; for (int j = 0; j <= i; j++) A[i][j] += jr[i] * jr[j]; }
    }
    for (int i = 0; i < 6; i++) for (int j = i + 1; j < 6; j++) A[i][j] = A[j][i];
    for (int c = 0; c < 6; c++) { const double d = std::sqrt(diagonal[c] / radius); A[c][c] += d * d; }
    double step[6]; bool solved = cholesky_solve6(A, rhs, step);
    for (int c = 0; c < 6; c++) step[c] = -step[c];
    reuse_diagonal = true;
    bool step_is_valid = false; double model_cost_change = 0; double delta[6];
    if (solved) {
      for (size_t r = 0; r < 3 * M; r++) { double s = 0; for (int c = 0; c < 6; c++) s += jac[6 * r + c] * step[c]; model_res[r] = s; }
      double mc = 0; for (size_t r = 0; r < 3 * M; r++) mc += model_res[r] * (residuals[r] + model_res[r] / 2.0);
      model_cost_change = -mc; step_is_valid = model_cost_change > 0.0;
      if (step_is_valid) { for (int c = 0; c < 6; c++) delta[c] = step[c] * scaling[c]; num_consecutive_invalid = 0; }
    }
    if (!step_is_valid) {  // HandleInvalidStep
      if (++num_consecutive_invalid >= opt.max_num_consecutive_invalid_steps) { sum->termination = 4; break; }
      radius = radius / decrease_factor; decrease_factor *= 2.0; reuse_diagonal = true; last_successful = false; continue;
    }
    // --- DoLineSearch (is_constrained): projected Armijo, cubic interpolation
    {
      double gd = 0; for (int c = 0; c < 6; c++) gd += gradient[c] * delta[c];
      double dmax = 0; for (int c = 0; c < 6; c++) dmax = std::max(dmax, std::fabs(delta[c]));
      auto ls_eval = [&](double a, FunctionSample* out) {
        double sd[6], px[7], g2[6], c2 = 0; for (int c = 0; c < 6; c++) sd[c] = a * delta[c];
        prob.plus(x, sd, px); sum->num_cost_evals++; sum->num_jac_evals++;
        out->x = a; out->value_is_valid = prob.evaluate(px, &c2, nullptr, g2, nullptr); out->value = c2;
        double gg = 0; for (int c = 0; c < 6; c++) gg += g2[c] * delta[c]; out->gradient = gg; out->gradient_is_valid = out->value_is_valid && std::isfinite(gg);
      };
      FunctionSample initial; initial.x = 0; initial.value = x_cost; initial.gradient = gd; initial.value_is_valid = initial.gradient_is_valid = true;
      FunctionSample previous, current; int ls_iters = 0; bool success = false;
      ls_eval(1.0, &current);
      for (;;) {
        if (current.value_is_valid && !(current.value > x_cost + opt.ls_sufficient_decrease * gd * current.x)) { success = true; break; }
        if (++ls_iters >= opt.ls_max_num_iterations) break;
        double step_size;
        const double mn = opt.ls_max_step_contraction * current.x, mxs = opt.ls_min_step_contraction * current.x;
        if (!current.value_is_valid) step_size = std::min(std::max(current.x * 0.5, mn), mxs);
        else {
          std::vector<FunctionSample> samples; samples.push_back(initial); samples.push_back(current); if (previous.value_is_valid) samples.push_back(previous);
          double unused; minimize_polynomial(find_interpolating_polynomial(samples), mn, mxs, &step_size, &unused);
        }
        if (step_size * dmax < opt.ls_min_step_size) break;
        previous = current; ls_eval(step_size, &current);
      }
      sum->num_line_search_steps += ls_iters;
      if (success) for (int c = 0; c < 6; c++) delta[c] *= current.x;
    }
    // --- ComputeCandidatePointAndEvaluateCost
    prob.plus(x, delta, cand); sum->num_cost_evals++;
    if (!prob.evaluate(cand, &cand_cost, nullptr, nullptr, nullptr)) cand_cost = std::numeric_limits<double>::max();
    // --- ParameterToleranceReached / FunctionToleranceReached (candidate is NOT taken on convergence)
    double step_norm = 0; for (int k = 0; k < 7; k++) step_norm += (x[k] - cand[k]) * (x[k] - cand[k]); step_norm = std::sqrt(step_norm);
    if (step_norm <= opt.parameter_tolerance * (x_norm + opt.parameter_tolerance)) { sum->termination = 2; break; }
    const double cost_change = x_cost - cand_cost;
    if (std::fabs(cost_change) <= opt.function_tolerance * x_cost) { sum->termination = 3; break; }
    // --- IsStepSuccessful
    const double relative_decrease = (current_cost_eval - cand_cost) / model_cost_change;
    if (relative_decrease > opt.min_relative_decrease) {  // HandleSuccessfulStep
      for (int k = 0; k < 7; k++) x[k] = cand[k];
      x_norm = 0; for (int k = 0; k < 7; k++) x_norm += x[k] * x[k]; x_norm = std::sqrt(x_norm);
      if (!eval_grad_jac(iteration)) { sum->termination = 4; break; }
      last_gmax = gradient_max_norm(); last_successful = true; sum->num_successful_steps++;
      radius = radius / std::max(1.0 / 3.0, 1.0 - std::pow(2.0 * relative_decrease - 1.0, 3));
      radius = std::min(opt.max_trust_region_radius, radius); decrease_factor = 2.0; reuse_diagonal = false;
      current_cost_eval = cand_cost; min_iter_cost = std::min(min_iter_cost, x_cost);
      if (x_cost < minimum_cost) { minimum_cost = x_cost; for (int k = 0; k < 7; k++) x_io[k] = x[k]; }
    } else {  // HandleUnsuccessfulStep
      radius = radius / decrease_factor; decrease_factor *= 2.0; reuse_diagonal = true; last_successful = false; sum->num_unsuccessful_steps++;
      min_iter_cost = std::min(min_iter_cost, cand_cost);  // iteration_summary.cost = candidate_cost
    }
  }
  sum->final_cost = std::min(sum->initial_cost, min_iter_cost);  // SetSummaryFinalCost: min over iteration costs
}

}  // namespace orc
