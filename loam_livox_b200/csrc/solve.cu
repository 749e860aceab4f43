// Robust 6-DoF Levenberg-Marquardt solve of one ICP iteration as ONE persistent kernel (K8 + K9 + K10 front end).
//
// Replaces, on the reference side (Ceres is third-party, restated from its published behaviour, see oracle/orc_solver.hpp):
//   ceres::Problem / AddResidualBlock / Solve x2   loam_livox/source/point_cloud_registration.hpp:220-228,323,422,460-474,501-508
//   residual models (autodiff)                     loam_livox/source/ceres_icp.hpp:262-288 (point2line), :338-366 (point2plane)
//   HuberLoss(0.1), EigenQuaternionParameterization, bounds on t   :220-221, :143-151
//   problem.Evaluate + compute_inlier_residual_threshold   :476-499, :153-161 (K10)
//   pose composition + ICP termination test        :514-531
//
// Design (DESIGN.md §3.2): every residual block is staged once into SHARED MEMORY (SoA) of one of the persistent CTAs (one per SM, 132 on an
// H100) and stays on-chip for the whole solve.  One evaluation = every thread evaluates its blocks' r, J, Huber weight and normal-equation
// terms, a CTA reduce, then a master-less exchange: every CTA publishes its 29 sums in a tagged row, reads all rows and reduces them in fixed
// order, so every CTA holds bit-identical sums and advances its own copy of the trust-region state.  SOLVE_FUSED runs a whole ICP iteration
// in one launch: solve #1, the L1 norms, K10's inlier threshold over the grid (hash-set de-duplication + radix select), the outlier drop,
// solve #2 and the pose.  No host round trip inside a launch.
#include <cfloat>
#include <cstdlib>
#include "common.cuh"
#include "kernels.cuh"
#include "exact_math.cuh"

#define FULL 0xffffffffu
#define NSUM 29          // 21 JtJ (upper, row-major) + 6 Jtr + cost + valid-block count
#define SOLVE_THREADS 256

__device__ __forceinline__ unsigned ld_acquire_u32(const unsigned* p) { unsigned v; asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory"); return v; }
__device__ __forceinline__ void st_release_u32(unsigned* p, unsigned v) { asm volatile("st.release.gpu.global.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory"); }
__device__ __forceinline__ unsigned ld_acquire_sys_u32(const unsigned* p) { unsigned v; asm volatile("ld.acquire.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory"); return v; }
__device__ __forceinline__ void st_release_sys_u32(unsigned* p, unsigned v) { asm volatile("st.release.sys.global.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory"); }

#include "lm_core.cuh"

// ------------------------------------------------------------------------------------------------ per-block evaluation
struct Slot { double px, py, pz, ax, ay, az, vx, vy, vz; double s; int type; };   // s: m_motion_blur_s (deblur only)

struct EvalConst {   // uniform per evaluation, in shared memory
  double x[7];       // trial point: q (x,y,z,w), t
  double PJ[4][3];   // EigenQuaternionParameterization::ComputeJacobian
  double Rl[3][3];   // rotation by q_last (columns = q_last * e_k)
  double tl[3];
  double huber_a, huber_b;
  // Eigen slerp(Identity -> q_incre) pieces that do not depend on the block (deblur only): theta = acos|w|, d(theta)/dw
  double sl_theta, sl_sin, sl_cos, sl_dth_dw; int sl_lerp;
};

__device__ __forceinline__ void cross3(double ax, double ay, double az, double bx, double by, double bz, double& ox, double& oy, double& oz) {
  ox = ay * bz - az * by; oy = az * bx - ax * bz; oz = ax * by - ay * bx;
}
// residual (3), optional Jacobian (3 x 6, tangent space), returns rho' (Huber weight) and adds 0.5*rho to *cost
// MB = the *_mb functors (ceres_icp.hpp:106-134, :187-218): q_incre -> Identity.slerp(s, q_incre) (Eigen: scale0 * I + scale1 * q_incre, scales
// from theta = acos|w|, plain lerp when |w| >= 1 - eps; the result is NOT re-normalised and goes through _transformVector as is) and
// t_incre -> s * t_incre.  The derivative below is the derivative of exactly that expression, which is what the reference's Jets compute.
template <bool MB>
__device__ __forceinline__ void eval_block(const Slot& s, const EvalConst& E, double r[3], double J[6][3], bool want_j) {
  double ux = E.x[0], uy = E.x[1], uz = E.x[2], w = E.x[3];
  double sc1 = 1.0, dsc0 = 0.0, dsc1 = 0.0, ts = 1.0;   // scale1, d(scale0)/dw, d(scale1)/dw, translation scale
  if (MB) {
    const double sb = s.s; double sc0;
    if (E.sl_lerp) { sc0 = 1.0 - sb; sc1 = sb; }
    else {
      double s0, c0, s1, c1; sincos((1.0 - sb) * E.sl_theta, &s0, &c0); sincos(sb * E.sl_theta, &s1, &c1);
      const double inv = 1.0 / E.sl_sin;
      sc0 = s0 * inv; sc1 = s1 * inv;
      dsc0 = ((1.0 - sb) * c0 * E.sl_sin - s0 * E.sl_cos) * inv * inv * E.sl_dth_dw;
      dsc1 = (sb * c1 * E.sl_sin - s1 * E.sl_cos) * inv * inv * E.sl_dth_dw;
    }
    if (E.x[3] < 0.0) { sc1 = -sc1; dsc1 = -dsc1; }
    ux *= sc1; uy *= sc1; uz *= sc1; w = sc0 + sc1 * E.x[3]; ts = sb;
  }
  double cx, cy, cz; cross3(ux, uy, uz, s.px, s.py, s.pz, cx, cy, cz); cx += cx; cy += cy; cz += cz;   // 2 (u x p)
  double ex, ey, ez; cross3(ux, uy, uz, cx, cy, cz, ex, ey, ez);
  const double yx = s.px + w * cx + ex + ts * E.x[4], yy = s.py + w * cy + ey + ts * E.x[5], yz = s.pz + w * cz + ez + ts * E.x[6];
  const double dx = E.Rl[0][0] * yx + E.Rl[0][1] * yy + E.Rl[0][2] * yz + E.tl[0] - s.ax;
  const double dy = E.Rl[1][0] * yx + E.Rl[1][1] * yy + E.Rl[1][2] * yz + E.tl[1] - s.ay;
  const double dz = E.Rl[2][0] * yx + E.Rl[2][1] * yy + E.Rl[2][2] * yz + E.tl[2] - s.az;
  const double dv = dx * s.vx + dy * s.vy + dz * s.vz;
  const bool line = s.type == 1;
  if (line) { r[0] = dx - dv * s.vx; r[1] = dy - dv * s.vy; r[2] = dz - dv * s.vz; }
  else { r[0] = dv * s.vx; r[1] = dv * s.vy; r[2] = dv * s.vz; }
  if (!want_j) return;
#pragma unroll
  for (int c = 0; c < 6; c++) {
    double gx, gy, gz;   // derivative of y = q_incre * p + t_incre along tangent direction c
    if (c < 3) {
      double dux = E.PJ[0][c], duy = E.PJ[1][c], duz = E.PJ[2][c], dw = E.PJ[3][c];
      if (MB) {   // direction of (scale1 u, scale0 + scale1 w) along the ambient direction (du, dw)
        const double k1 = dsc1 * dw;
        dux = k1 * E.x[0] + sc1 * dux; duy = k1 * E.x[1] + sc1 * duy; duz = k1 * E.x[2] + sc1 * duz;
        dw = dsc0 * dw + k1 * E.x[3] + sc1 * dw;
      }
      double ax, ay, az; cross3(dux, duy, duz, s.px, s.py, s.pz, ax, ay, az); ax += ax; ay += ay; az += az;  // 2 (du x p)
      double bx, by, bz; cross3(dux, duy, duz, cx, cy, cz, bx, by, bz);                                       // du x 2(u x p)
      double fx, fy, fz; cross3(ux, uy, uz, ax, ay, az, fx, fy, fz);                                          // u x 2(du x p)
      gx = dw * cx + w * ax + bx + fx; gy = dw * cy + w * ay + by + fy; gz = dw * cz + w * az + bz + fz;
    } else { gx = c == 3 ? ts : 0.0; gy = c == 4 ? ts : 0.0; gz = c == 5 ? ts : 0.0; }
    const double e0 = E.Rl[0][0] * gx + E.Rl[0][1] * gy + E.Rl[0][2] * gz;
    const double e1 = E.Rl[1][0] * gx + E.Rl[1][1] * gy + E.Rl[1][2] * gz;
    const double e2 = E.Rl[2][0] * gx + E.Rl[2][1] * gy + E.Rl[2][2] * gz;
    const double ev = e0 * s.vx + e1 * s.vy + e2 * s.vz;
    if (line) { J[c][0] = e0 - ev * s.vx; J[c][1] = e1 - ev * s.vy; J[c][2] = e2 - ev * s.vz; }
    else { J[c][0] = ev * s.vx; J[c][1] = ev * s.vy; J[c][2] = ev * s.vz; }
  }
}
__device__ __forceinline__ double huber_weight(double sq, double a, double b, double& rho0) {
  if (sq > b) { double r = sqrt(sq); rho0 = 2.0 * a * r - b; return fmax(DBL_MIN, a / r); }
  rho0 = sq; return 1.0;
}

// Per solve: everything that depends on the last pose and the loss only.
__device__ void setup_static(EvalConst& E, const RegDevState* st) {
  const double* ql = st->pose_last;
  for (int k = 0; k < 3; k++) { double e[3] = {k == 0 ? 1.0 : 0.0, k == 1 ? 1.0 : 0.0, k == 2 ? 1.0 : 0.0}, o[3]; d_qrot(ql, e, o); E.Rl[0][k] = o[0]; E.Rl[1][k] = o[1]; E.Rl[2][k] = o[2]; }
  E.tl[0] = st->pose_last[4]; E.tl[1] = st->pose_last[5]; E.tl[2] = st->pose_last[6];
  E.huber_a = st->huber_a; E.huber_b = st->huber_a * st->huber_a;
}
// Per evaluation (on every CTA's critical path): the trial point, the parameterisation Jacobian and, for the *_mb functors only, the slerp terms.
template <bool MB>
__device__ __forceinline__ void setup_trial(EvalConst& E, const double* x) {
  for (int k = 0; k < 7; k++) E.x[k] = x[k];
  E.PJ[0][0] = x[3];  E.PJ[0][1] = x[2];  E.PJ[0][2] = -x[1];
  E.PJ[1][0] = -x[2]; E.PJ[1][1] = x[3];  E.PJ[1][2] = x[0];
  E.PJ[2][0] = x[1];  E.PJ[2][1] = -x[0]; E.PJ[2][2] = x[3];
  E.PJ[3][0] = -x[0]; E.PJ[3][1] = -x[1]; E.PJ[3][2] = -x[2];
  if (MB) { const double d = x[3], ad = fabs(d);
    if (ad >= 1.0 - 2.220446049250313e-16) { E.sl_lerp = 1; E.sl_theta = 0; E.sl_sin = 1; E.sl_cos = 1; E.sl_dth_dw = 0; }
    else { E.sl_lerp = 0; E.sl_theta = acos(ad); E.sl_sin = sin(E.sl_theta); E.sl_cos = cos(E.sl_theta); E.sl_dth_dw = -(d < 0.0 ? -1.0 : 1.0) / sqrt(1.0 - ad * ad); } }
}

// ------------------------------------------------------------------------------------------------ the persistent kernel
// Residual blocks are staged ONCE into shared memory (SoA: 52 B per block) and stay there for the whole solve.
// CTA b owns the 512-slot tiles b, b + grid, b + 2 grid, ...  (coalesced staging, balanced over the SMs).
// ---- fast path (no motion deblur): the same r, J^T J, J^T r in closed form.
// With y = q_incre p, d' = y + t_incre - a' (a' = R_last^T (a - t_last)), w' = R_last^T v, alpha = d'.w':
//   line : r = R_last (d' - alpha w'),  J = R_last (I - w' w'^T) G        plane: r = R_last alpha w',  J = R_last w' w'^T G
//   G = d(y + t)/d(tangent, t) = [ -2 [y]x | I ]   (EigenQuaternionParameterization::Plus is q <- exp(delta) q: dy = 2 delta x y)
// so J^T J and J^T r need only beta = G^T w', G^T G (closed form in y) and G^T r': ~150 fp64 flops per block instead of ~1200.
struct FastSlot { double px, py, pz, ax, ay, az, wx, wy, wz; int type; };
__device__ __forceinline__ void fast_residual(const FastSlot& s, const EvalConst& E, double y[3], double r[3], double& alpha) {
  const double ux = E.x[0], uy = E.x[1], uz = E.x[2], w = E.x[3];
  double cx, cy, cz; cross3(ux, uy, uz, s.px, s.py, s.pz, cx, cy, cz); cx += cx; cy += cy; cz += cz;
  double ex, ey, ez; cross3(ux, uy, uz, cx, cy, cz, ex, ey, ez);
  y[0] = s.px + w * cx + ex; y[1] = s.py + w * cy + ey; y[2] = s.pz + w * cz + ez;
  const double dx = y[0] + E.x[4] - s.ax, dy = y[1] + E.x[5] - s.ay, dz = y[2] + E.x[6] - s.az;
  alpha = dx * s.wx + dy * s.wy + dz * s.wz;
  if (s.type == 1) { r[0] = dx - alpha * s.wx; r[1] = dy - alpha * s.wy; r[2] = dz - alpha * s.wz; }
  else { r[0] = alpha * s.wx; r[1] = alpha * s.wy; r[2] = alpha * s.wz; }
}
__device__ __forceinline__ void fast_accumulate(const FastSlot& s, const EvalConst& E, double acc[NSUM]) {
  double y[3], r[3], alpha; fast_residual(s, E, y, r, alpha);
  double rho0; const double wgt = huber_weight(r[0] * r[0] + r[1] * r[1] + r[2] * r[2], E.huber_a, E.huber_b, rho0);
  acc[27] += 0.5 * rho0; acc[28] += 1.0;
  const bool line = s.type == 1;
  const double wn2 = s.wx * s.wx + s.wy * s.wy + s.wz * s.wz;
  // beta = G^T w' = (2 y x w', w')
  double b[6]; cross3(y[0], y[1], y[2], s.wx, s.wy, s.wz, b[0], b[1], b[2]); b[0] += b[0]; b[1] += b[1]; b[2] += b[2]; b[3] = s.wx; b[4] = s.wy; b[5] = s.wz;
  // gradient: line J^T r = G^T (r - w'(w'.r)); plane J^T r = |w'|^2 G^T r
  double rr[3], cg;
  if (line) { const double wr = s.wx * r[0] + s.wy * r[1] + s.wz * r[2]; rr[0] = r[0] - wr * s.wx; rr[1] = r[1] - wr * s.wy; rr[2] = r[2] - wr * s.wz; cg = wgt; }
  else { rr[0] = r[0]; rr[1] = r[1]; rr[2] = r[2]; cg = wgt * wn2; }
  double g0, g1, g2; cross3(y[0], y[1], y[2], rr[0], rr[1], rr[2], g0, g1, g2);
  acc[21] += cg * (g0 + g0); acc[22] += cg * (g1 + g1); acc[23] += cg * (g2 + g2); acc[24] += cg * rr[0]; acc[25] += cg * rr[1]; acc[26] += cg * rr[2];
  // Hessian: line G^T G - (2 - |w'|^2) beta beta^T ; plane |w'|^2 beta beta^T
  const double cb = line ? -wgt * (2.0 - wn2) : wgt * wn2;
  int h = 0;
#pragma unroll
  for (int i = 0; i < 6; i++) {
#pragma unroll
    for (int j = i; j < 6; j++) { acc[h] += cb * b[i] * b[j]; h++; }
  }
  if (line) {
    const double yy = y[0] * y[0] + y[1] * y[1] + y[2] * y[2], w4 = 4.0 * wgt, w2 = 2.0 * wgt;
    // rows 0..2 of G^T G: [4 (|y|^2 I - y y^T) | 2 [e_i x y]_k], rows 3..5: [ . | I ]
    acc[0] += w4 * (yy - y[0] * y[0]); acc[1] -= w4 * y[0] * y[1]; acc[2] -= w4 * y[0] * y[2];
    acc[4] -= w2 * y[2]; acc[5] += w2 * y[1];                                  // (0,3) = 0, (0,4) = -2 y_z, (0,5) = 2 y_y
    acc[6] += w4 * (yy - y[1] * y[1]); acc[7] -= w4 * y[1] * y[2];
    acc[8] += w2 * y[2]; acc[10] -= w2 * y[0];                                 // (1,3) = 2 y_z, (1,4) = 0, (1,5) = -2 y_x
    acc[11] += w4 * (yy - y[2] * y[2]);
    acc[12] -= w2 * y[1]; acc[13] += w2 * y[0];                                // (2,3) = -2 y_y, (2,4) = 2 y_x, (2,5) = 0
    acc[15] += wgt; acc[18] += wgt; acc[20] += wgt;                            // (3,3), (4,4), (5,5)
  }
}

// One level of the CTA reduce's transposing butterfly: lanes that differ in bit OFF swap halves of w[0 .. 2 OFF) and add, so that w[0 .. OFF) holds
// pairwise sums (after the five levels, lane L holds the warp's total of sum L).
template <int OFF>
__device__ __forceinline__ void butterfly_level(double (&w)[32], int lane) {
  const bool upper = (lane & OFF) != 0;
#pragma unroll
  for (int i = 0; i < OFF; i++) {
    const double send = upper ? w[i] : w[i + OFF];          // the half this lane gives away
    const double keep = upper ? w[i + OFF] : w[i];
    w[i] = keep + __shfl_xor_sync(FULL, send, OFF);
  }
}

struct SmemSlots { float* p[3]; float* a[3]; double* v[3]; double* ap[3]; int* type; float* s; };
// MB (general path): v = line direction / plane normal (world), a = anchor (world, fp32-exact), s = blur factor      -> 56 B / slot
// !MB (fast path):   v = R_last^T v, ap = R_last^T (a - t_last): the evaluation never touches the last pose again   -> 64 B / slot
__device__ __forceinline__ SmemSlots carve(unsigned char* base, int cap, bool mb) {
  SmemSlots s; double* d = (double*)base;
  s.v[0] = d; s.v[1] = d + cap; s.v[2] = d + 2 * cap; d += 3 * (size_t)cap;
  if (!mb) { s.ap[0] = d; s.ap[1] = d + cap; s.ap[2] = d + 2 * cap; d += 3 * (size_t)cap; } else { s.ap[0] = s.ap[1] = s.ap[2] = nullptr; }
  float* f = (float*)d;
  s.p[0] = f; s.p[1] = f + cap; s.p[2] = f + 2 * cap; f += 3 * (size_t)cap;
  if (mb) { s.a[0] = f; s.a[1] = f + cap; s.a[2] = f + 2 * cap; f += 3 * (size_t)cap; s.s = f; f += cap; } else { s.a[0] = s.a[1] = s.a[2] = nullptr; s.s = nullptr; }
  s.type = (int*)f;
  return s;
}
#define SLOT_BYTES 64
#define SLOT_BYTES_MB 56

// ------------------------------------------------------------------------------------------------ grid-wide exchange without a master
// Every CTA owns one 256-byte row per parity in SolveSync: 29 sums + a generation tag.  An exchange = every CTA writes its row and tags it with
// the generation (release), every CTA waits until all rows carry that tag (thread t polls row t: one L2 round trip, no atomics, nobody is special)
// and reduces the rows itself in fixed order -- bit-identical sums everywhere, so every CTA advances its own copy of the solver state and there is
// no publish step.  Rows are double-buffered by generation parity: a CTA can be at most one exchange ahead of the slowest one.  Generations grow
// monotonically over the life of the context (SolveSync::gen is never reset), so a stale tag can never match.
__device__ __forceinline__ double* sync_row(SolveSync* Y, unsigned gen, int cta) { return Y->rows[gen & 1u][cta]; }
// Called by one thread after a warp or CTA barrier that follows the writes it publishes (the CTA's row, K10's histogram atomics).  The release is
// cumulative: it orders every write the barrier made this thread observe, so no separate fence is needed (a __threadfence here is a sequentially
// consistent fence on the path of every exchange).
__device__ __forceinline__ void sync_arrive(SolveSync* Y, unsigned gen) {
  st_release_u32((unsigned*)(sync_row(Y, gen, blockIdx.x) + 31), gen);
}
__device__ __forceinline__ void sync_wait_all(SolveSync* Y, unsigned gen) {   // CTA-collective
  if (threadIdx.x < gridDim.x) { const unsigned* f = (const unsigned*)(sync_row(Y, gen, threadIdx.x) + 31); while (ld_acquire_u32(f) != gen) {} }
  __syncthreads();
}
// plain barrier (no payload)
__device__ __forceinline__ void grid_sync(SolveSync* Y, unsigned& gen) {
  gen++;
  __syncthreads();
  if (threadIdx.x == 0) sync_arrive(Y, gen);
  sync_wait_all(Y, gen);
}

// K10 (compute_inlier_residual_threshold, :153-161) spread over the grid: de-duplicate the per-block L1 norms (std::set<double>), take element
// floor(ratio * size).  Used by the fused section of lm_solve_kernel and by k10_select_kernel (the sharded mode's select between solve #1 and
// solve #2, and the parity hook ll_inlier_select), so that all of them run the same code.
#define K10_PASSES 6
#define L1_EMPTY 0xffffffffffffffffull

// Bit pattern of a non-negative double as an order-preserving key (-0.0 == 0.0 in a std::set).
__device__ __forceinline__ unsigned long long l1_key(double v) { return (unsigned long long)__double_as_longlong(v == 0.0 ? 0.0 : v); }
// Insert into the global hash set: true when this call created the entry, i.e. the caller is the (only) representative of a distinct value.
__device__ __forceinline__ bool l1_set_insert_flag(unsigned long long* __restrict__ table, unsigned table_mask, double v, bool valid) {
  if (!(valid && v < INFINITY)) return false;   // +inf = invalid slot, NaN never compares
  const unsigned long long key = l1_key(v);
  unsigned h = (unsigned)((key * 0x9E3779B97F4A7C15ull) >> 40) & table_mask;
  for (;;) {
    const unsigned long long prev = atomicCAS(&table[h], L1_EMPTY, key);
    if (prev == L1_EMPTY) return true;
    if (prev == key) return false;
    h = (h + 1) & table_mask;
  }
}
// The inlier threshold of solve #2 (:484-485): max(inliner_dis, the K10 order statistic), which counts as 0 when there is no distinct value.
__device__ __forceinline__ double k10_threshold(double inliner_dis, double value, int n_distinct) { return fmax(inliner_dis, n_distinct > 0 ? value : 0.0); }
struct K10Smem { unsigned hist[2048]; unsigned warp_sum[SOLVE_THREADS / 32 + 1]; unsigned long long prefix, mask; int k, cnt_bin, n_distinct, done; int scratch[40]; double result; };

// Clear the hash set of the L1 norms and the K10 histograms / candidate counter; a grid exchange must follow before any insert.
__device__ __forceinline__ void k10_clear(unsigned long long* table, unsigned table_mask, SolveSync* Y) {
  for (unsigned idx = blockIdx.x * SOLVE_THREADS + threadIdx.x; idx <= table_mask; idx += gridDim.x * SOLVE_THREADS) table[idx] = L1_EMPTY;
  for (unsigned idx = blockIdx.x * SOLVE_THREADS + threadIdx.x; idx < K10_PASSES * 2048u + 64u; idx += gridDim.x * SOLVE_THREADS) ((unsigned*)Y->hist)[idx] = 0u;   // hist + list_cnt + pad
}

// The element of rank min(floor(ratio * n), n - 1) among the n DISTINCT values l1[i] of the slots whose flag (bit 8 of type[li], shared memory)
// says this thread represents the value.  Radix select on the bit patterns (non-negative doubles order like their bits), 11-bit digits from the
// exponent down: per pass every CTA histograms the distinct values it represents (shared memory), adds its non-empty bins to the global
// histogram, one exchange, and every CTA finds the bin of the wanted rank in the same histogram.  When that bin holds <= 64 values they are
// collected and ranked directly.  Grid-collective; ends with s_k10.n_distinct and s_k10.result (valid when n_distinct > 0) on every CTA.
__device__ __forceinline__ void k10_select(K10Smem& s_k10, SolveSync* Y, unsigned& gen, const int* type, const double* l1, int M, int tiles_per_cta, int tile, const double* ratio) {
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  if (tid == 0) { s_k10.prefix = 0ull; s_k10.mask = 0ull; s_k10.k = -1; s_k10.done = 0; s_k10.result = 0.0; }
  __syncthreads();
  for (int pass = 0; pass < K10_PASSES && !s_k10.done; pass++) {
    const int shift = pass < 5 ? 52 - 11 * pass : 0; const unsigned dmask = pass < 5 ? 2047u : 255u;   // bits 62..52, 51..41, 40..30, 29..19, 18..8, 7..0
    for (int b = tid; b < 2048; b += SOLVE_THREADS) s_k10.hist[b] = 0u;
    __syncthreads();
    const unsigned long long prefix = s_k10.prefix, himask = s_k10.mask;
    for (int k = 0; k < tiles_per_cta; k++) {
      const int i = (blockIdx.x + gridDim.x * k) * tile + tid, li = k * SOLVE_THREADS + tid;
      if (i < M && tid < tile && (type[li] & 0x100)) {
        const unsigned long long key = l1_key(l1[i]);
        if ((key & himask) == prefix) atomicAdd(&s_k10.hist[(unsigned)(key >> shift) & dmask], 1u);
      }
    }
    __syncthreads();
    unsigned* gh = Y->hist[pass];
    for (int b = tid; b < 2048; b += SOLVE_THREADS) { const unsigned c = s_k10.hist[b]; if (c) atomicAdd(&gh[b], c); }
    grid_sync(Y, gen);
    // every CTA: exclusive scan of the global histogram, find the bin that holds rank k
    constexpr int BPT = 2048 / SOLVE_THREADS;
    unsigned h[BPT], run = 0;
#pragma unroll
    for (int b = 0; b < BPT; b++) { h[b] = __ldcg(&gh[tid * BPT + b]); run += h[b]; }
    unsigned incl = run;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) { const unsigned v = __shfl_up_sync(FULL, incl, o); if (lane >= o) incl += v; }
    if (lane == 31) s_k10.warp_sum[warp] = incl;
    __syncthreads();
    if (tid == 0) { unsigned t = 0; for (int w = 0; w < SOLVE_THREADS / 32; w++) { const unsigned c = s_k10.warp_sum[w]; s_k10.warp_sum[w] = t; t += c; } s_k10.warp_sum[SOLVE_THREADS / 32] = t; }
    __syncthreads();
    if (pass == 0 && tid == 0) {
      const int n = (int)s_k10.warp_sum[SOLVE_THREADS / 32]; s_k10.n_distinct = n;
      int k = (int)(*ratio * (double)n); if (k > n - 1) k = n - 1; s_k10.k = k;
      if (n == 0) s_k10.done = 1;   // no block at all: the solve reported termination -1 already
    }
    __syncthreads();
    if (!s_k10.done) {
      const unsigned excl = s_k10.warp_sum[warp] + incl - run; const unsigned k = (unsigned)s_k10.k;
      __syncthreads();
      if (k >= excl && k < excl + run) {   // exactly one thread
        unsigned below = excl; int j = 0;
#pragma unroll
        for (int b = 0; b < BPT; b++) { if (k >= below + h[b] && j == b) { below += h[b]; j = b + 1; } }
        const int jj = j < BPT ? j : BPT - 1;
        s_k10.k = (int)(k - below); s_k10.cnt_bin = (int)h[jj];
        s_k10.prefix = prefix | ((unsigned long long)(tid * BPT + jj) << shift);
        s_k10.mask = himask | ((unsigned long long)dmask << shift);
      }
      __syncthreads();
      if (s_k10.cnt_bin <= 64 || pass == K10_PASSES - 1) {
        // collect the members of the bin (<= 64 distinct values, or all equal in their 63 bits: then any of them is the answer) and rank them
        const unsigned long long pf = s_k10.prefix, hm = s_k10.mask;
        for (int kk = 0; kk < tiles_per_cta; kk++) {
          const int i = (blockIdx.x + gridDim.x * kk) * tile + tid, li = kk * SOLVE_THREADS + tid;
          if (i < M && tid < tile && (type[li] & 0x100)) {
            const double v = l1[i];
            if ((l1_key(v) & hm) == pf) { const unsigned slot = atomicAdd(&Y->list_cnt, 1u); if (slot < 64u) Y->list[slot] = v; }
          }
        }
        grid_sync(Y, gen);
        {   // rank the <= 64 collected values: one value per thread out of shared memory (distinct values: exactly one has the wanted rank)
          double* cand = (double*)s_k10.hist;
          const int m = min((int)*((volatile unsigned*)&Y->list_cnt), 64);
          if (tid < m) cand[tid] = __ldcg(&Y->list[tid]);
          __syncthreads();
          if (tid < m) { const double mine = cand[tid]; int rank = 0; for (int q = 0; q < m; q++) rank += (cand[q] < mine) ? 1 : 0; if (rank == s_k10.k) s_k10.result = mine; }
          if (tid == 0) s_k10.done = 1;
        }
        __syncthreads();
      }
    }
  }
}

template <bool MB>
__global__ void __launch_bounds__(SOLVE_THREADS, 2) lm_solve_kernel(SolveArgs a, int tiles_per_cta, int tile) {
  extern __shared__ __align__(16) unsigned char s_dyn[];
  __shared__ EvalConst E;
  __shared__ double s_red[SOLVE_THREADS / 32][NSUM + 1];
  __shared__ double s_sum[32];
  __shared__ LmState s_lm;     // EVERY CTA keeps its own copy of the solver state and advances it identically
  __shared__ double s_gmax;
  __shared__ StepOut s_pre[2]; // the next iteration's ComputeStep under both outcomes of the accept test, evaluated by warp 1 while warp 0 decides
  __shared__ K10Smem s_k10;    // SOLVE_FUSED only
  __shared__ long long s_prof[16];   // the master CTA's cycle counters, added to RegDevState::prof once at the end: a global read-modify-write per
                                     // evaluation would put an L2 round trip on the master's path, and every other CTA waits for the master's row
  RegDevState* st = a.st;
  SolveSync* Y = a.sync;
  if ((a.mode == SOLVE_FUSED || a.mode <= SOLVE_SECOND) && *((volatile int*)&st->icp_done)) return;   // ICP work (fused, solve #1 or #2) launched after the ICP loop ended (uniform over the grid)
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int cap = tiles_per_cta * SOLVE_THREADS;
  const SmemSlots S = carve(s_dyn, cap, MB);
  const bool master = blockIdx.x == 0;   // the CTA that writes results back to RegDevState and talks to the peers (nothing waits for it otherwise)
  unsigned gen = *((volatile unsigned*)&Y->gen);   // uniform over the grid: written by the previous launch's CTA 0 at its very end
  if (tid < 16) s_prof[tid] = 0;

  const long long t_k0 = clock64();
  // SOLVE_FUSED = one whole ICP iteration's solver work in ONE launch: solve #1 (prerun iterations) -> L1 norms -> std::set de-duplication + order
  // statistic (K10) -> drop outliers from the staged blocks -> solve #2 -> pose.  The hash set and the histograms are cleared here; the first
  // exchange orders the clear before any insert.
  const bool fused = a.mode == SOLVE_FUSED;
  SolveMode cur_mode = fused ? SOLVE_FIRST : a.mode;
  if (fused) k10_clear(a.table, a.table_mask, Y);
  // ---- stage this CTA's residual blocks
  double thr = 0;
  if (a.mode == SOLVE_SECOND) {   // K10 tail: the threshold from the order statistic and distinct count launch_k10_select left on the device
    thr = k10_threshold(st->inliner_dis, *a.k10_value, *a.k10_n_distinct);
    if (master && tid == 0) st->inlier_threshold = thr;
  }
  // Residual-block cap, drop rule (:434-458): with M blocks and M > cap, block i leaves the problem when rand_i > (float)cap / (float)M.
  float cap_keep = 2.0f; int cap_iter = 0, cap_seed = 0;
  if (a.cap_check) {
    const int nb = a.world > 1 ? st->n_blocks_all : st->n_blocks;
    if (nb > st->cap) cap_keep = (float)st->cap / (float)nb;
    cap_iter = st->icp_iter; cap_seed = st->rng_seed;
  }
  for (int k = 0; k < tiles_per_cta; k++) {
    const int i = (blockIdx.x + gridDim.x * k) * tile + tid, li = k * SOLVE_THREADS + tid;   // tile <= SOLVE_THREADS slots per CTA and pass: threads >= tile idle
    int type = 0;
    if (i < a.M && tid < tile) {
      const float4 ba = a.blk_a[i]; type = __float_as_int(ba.w);
      if (type != 0 && cap_keep <= 1.0f && ll_cap_uniform_f(cap_seed, cap_iter, 2, i) > cap_keep) type = 0;
      if (type != 0 && a.mode == SOLVE_SECOND && (a.l1[i] > thr)) type = 0;
      if (type != 0) {
        const float4 f = a.feat[i];
        S.p[0][li] = f.x; S.p[1][li] = f.y; S.p[2][li] = f.z;
        const double v0 = a.blk_v[(size_t)i * 3], v1 = a.blk_v[(size_t)i * 3 + 1], v2 = a.blk_v[(size_t)i * 3 + 2];
        if (MB) {
          S.a[0][li] = ba.x; S.a[1][li] = ba.y; S.a[2][li] = ba.z; S.v[0][li] = v0; S.v[1][li] = v1; S.v[2][li] = v2;
          S.s[li] = refine_blur_f(f.w, (float)st->min_ts, (float)st->max_ts);   // refine_blur(pointOri.intensity, ...) * 1.0 (:309, :407)
        } else {   // into the frame of the last pose: w' = R_last^T v, a' = R_last^T (a - t_last)
          const double qc[4] = {st->pose_last[0], -st->pose_last[1], -st->pose_last[2], -st->pose_last[3]};
          double vin[3] = {v0, v1, v2}, o[3]; d_qrot(qc, vin, o); S.v[0][li] = o[0]; S.v[1][li] = o[1]; S.v[2][li] = o[2];
          double ain[3] = {(double)ba.x - st->pose_last[4], (double)ba.y - st->pose_last[5], (double)ba.z - st->pose_last[6]}; d_qrot(qc, ain, o);
          S.ap[0][li] = o[0]; S.ap[1][li] = o[1]; S.ap[2][li] = o[2];
        }
      }
    }
    S.type[li] = type;
  }
  const double bound = st->bound;
  double x_start[7]; for (int k = 0; k < 7; k++) x_start[k] = st->x[k];   // read before anybody can write it (CTA 0 does, at the end of a solve)
  for (int ph = 0; ph < (fused ? 2 : 1); ph++) {
  // ---- iteration zero trial point: Plus(x, 0), the projection of the start point onto the bounds (TrustRegionMinimizer::IterationZero).
  if (tid == 0) {
    double z[6] = {0, 0, 0, 0, 0, 0}, tr[7];
    if (ph == 1) for (int k = 0; k < 7; k++) x_start[k] = s_lm.x_best[k];   // phase 2 of the fused mode starts from solve #1's result
    d_plus(x_start, z, bound, tr);
    if (ph == 0) setup_static(E, st);
    setup_trial<MB>(E, tr);
    LmState& L = s_lm;
    L.phase = 0; L.iteration = 0; L.max_iterations = (fused && ph == 0) ? a.prerun_iterations : a.max_iterations; L.num_invalid = 0; L.done = 0; L.termination = 0; L.last_successful = 1; L.reuse_diagonal = 0;
    L.ls_iters = 0; L.n_valid = 0; L.total_iterations = 0; L.total_evaluations = 0; L.pending = -1;
    for (int k = 0; k < 7; k++) { L.trial[k] = tr[k]; L.x_best[k] = tr[k]; }
  }
  __syncthreads();

  if (master && tid == 0 && ph == 0) s_prof[6] += clock64() - t_k0;
  for (;;) {
    const long long t_e0 = clock64();
    // ---- evaluate: r, J, Huber, 29 partial sums per thread
    double acc[NSUM];
#pragma unroll
    for (int i = 0; i < NSUM; i++) acc[i] = 0.0;
    for (int k = 0; k < tiles_per_cta; k++) {
      const int li = k * SOLVE_THREADS + tid;
      const int type = S.type[li];
      if (!MB) {
        if (type != 0) {
          FastSlot fs; fs.type = type; fs.px = S.p[0][li]; fs.py = S.p[1][li]; fs.pz = S.p[2][li]; fs.ax = S.ap[0][li]; fs.ay = S.ap[1][li]; fs.az = S.ap[2][li];
          fs.wx = S.v[0][li]; fs.wy = S.v[1][li]; fs.wz = S.v[2][li];
          fast_accumulate(fs, E, acc);
        }
        continue;
      }
      Slot s; s.type = type;
      if (s.type != 0) {
        s.px = S.p[0][li]; s.py = S.p[1][li]; s.pz = S.p[2][li]; s.ax = S.a[0][li]; s.ay = S.a[1][li]; s.az = S.a[2][li];
        s.vx = S.v[0][li]; s.vy = S.v[1][li]; s.vz = S.v[2][li];
        s.s = (double)S.s[li];
        double r[3], J[6][3]; eval_block<true>(s, E, r, J, true);
        double rho0; const double wgt = huber_weight(r[0] * r[0] + r[1] * r[1] + r[2] * r[2], E.huber_a, E.huber_b, rho0);
        acc[27] += 0.5 * rho0; acc[28] += 1.0;
        int h = 0;
#pragma unroll
        for (int i = 0; i < 6; i++) {
          acc[21 + i] += wgt * (J[i][0] * r[0] + J[i][1] * r[1] + J[i][2] * r[2]);
#pragma unroll
          for (int j = i; j < 6; j++) { acc[h] += wgt * (J[i][0] * J[j][0] + J[i][1] * J[j][1] + J[i][2] * J[j][2]); h++; }
        }
      }
    }
    // ---- CTA reduce: a transposing butterfly over the warp (lane L ends up with the warp's total of sum L: 31 shuffle-adds instead of 29 x 5),
    // then shared memory, fixed order (warps that own no valid block contribute exact zeros)
    if (__any_sync(FULL, acc[28] != 0.0)) {
      double w[32];
#pragma unroll
      for (int i = 0; i < 32; i++) w[i] = i < NSUM ? acc[i] : 0.0;
      // one call per level with a constant width, so that every index is a constant and w stays in registers (a loop over the widths left
      // w in local memory: a dependent local load and store per shuffle)
      butterfly_level<16>(w, lane); butterfly_level<8>(w, lane); butterfly_level<4>(w, lane); butterfly_level<2>(w, lane); butterfly_level<1>(w, lane);
      if (lane < NSUM) s_red[warp][lane] = w[0];
    } else if (lane < NSUM) s_red[warp][lane] = 0.0;
    __syncthreads();
    // ---- exchange: this CTA's 29 sums into its row, tag, wait for every row, reduce all rows in fixed order (every CTA does, identically)
    gen++;
    if (warp == 0) {
      if (lane < NSUM) { double v = 0; for (int wq = 0; wq < SOLVE_THREADS / 32; wq++) v += s_red[wq][lane]; sync_row(Y, gen, blockIdx.x)[lane] = v; }
      __syncwarp();
      if (lane == 0) sync_arrive(Y, gen);
    }
    const long long t_e1 = clock64();
    sync_wait_all(Y, gen);
    const long long t_e2 = clock64();
    {
      // Thread (grp, val) sums value `val` of rows grp, grp + G, grp + 2G, ...: every row load is issued before the first add (one L2 round trip,
      // not one per four rows).  The sum is the fixed-order one every CTA computes: four chains over rows j = 0, 1, 2, 3 (mod 4) while a whole
      // group of four is left, the remaining rows into the first chain, (v0 + v1) + (v2 + v3), then the G group sums in order.
      // (Each thread acquiring the tags of its own rows instead of the poll + barrier above was measured slower: back-to-back acquires do not
      // overlap, each waits for the one before.)
      constexpr int G = SOLVE_THREADS / 32, RMAX = (LL_SYNC_ROWS + G - 1) / G;
      static_assert(RMAX % 4 == 0, "the row loop below runs whole groups of four");
      const int val = tid & 31, grp = tid >> 5, nb = (int)gridDim.x;
      const int n = grp < nb ? (nb - grp + G - 1) / G : 0;   // rows of this group
      if (val < NSUM) {
        double r[RMAX];
#pragma unroll
        for (int j = 0; j < RMAX; j++) r[j] = j < n ? __ldcg(&sync_row(Y, gen, grp + j * G)[val]) : 0.0;
        double v0 = 0, v1 = 0, v2 = 0, v3 = 0;
        const int whole = n & ~3;
#pragma unroll
        for (int j = 0; j < RMAX; j += 4) if (j < whole) { v0 += r[j]; v1 += r[j + 1]; v2 += r[j + 2]; v3 += r[j + 3]; }
#pragma unroll
        for (int j = 0; j < RMAX; j++) if (j >= whole && j < n) v0 += r[j];
        s_red[grp][val] = (v0 + v1) + (v2 + v3);
      }
      __syncthreads();
      if (tid < NSUM) { double t = 0; for (int g = 0; g < G; g++) t += s_red[g][tid]; s_sum[tid] = t; }
      __syncthreads();
    }
    if (a.world > 1) {
      // fused all-reduce over NVLink peer memory (CTA 0 of every rank): every rank writes its 29 sums into slot [rank] of every peer's staging
      // buffer (double-buffered by generation parity), then sums the slots in rank order -> bit-identical on all ranks; the result goes to the
      // other CTAs of this rank through one more tagged row.
      if (master && warp == 0) {
        unsigned* cgen = (unsigned*)((char*)a.comm_local + LL_COMM_CTRL_OFF);   // monotonic over the life of the context
        const unsigned g1 = *cgen + 1; const int par = g1 & 1;
        for (int p = 0; p < a.world; p++) {
          double* dst = a.comm_peer[p] + ((size_t)par * 8 + a.rank) * 64;
          if (lane < NSUM) dst[lane] = s_sum[lane];
        }
        __threadfence_system();
        __syncwarp();
        if (lane < a.world) st_release_sys_u32((unsigned*)(a.comm_peer[lane] + ((size_t)par * 8 + a.rank) * 64 + 32), g1);
        if (lane < a.world) { const unsigned* f = (const unsigned*)(a.comm_local + ((size_t)par * 8 + lane) * 64 + 32); while (ld_acquire_sys_u32(f) != g1) {} }
        __syncwarp();
        double t = 0;
        if (lane < NSUM) for (int p = 0; p < a.world; p++) t += *((volatile double*)(a.comm_local + ((size_t)par * 8 + p) * 64 + lane));
        if (lane < NSUM) Y->bcast[gen & 1u][lane] = t;
        if (lane == 0) *cgen = g1;
        __syncwarp();
        if (lane == 0) { __threadfence(); st_release_u32((unsigned*)&Y->bcast[gen & 1u][31], gen); }
      }
      if (tid == 0) { const unsigned* f = (const unsigned*)&Y->bcast[gen & 1u][31]; while (ld_acquire_u32(f) != gen) {} }
      __syncthreads();
      if (tid < NSUM) s_sum[tid] = __ldcg(&Y->bcast[gen & 1u][tid]);
      __syncthreads();
    }
    const long long t_e3 = clock64();
    // ---- advance the solver: warp 1 evaluates the next iteration's ComputeStep under both outcomes while warp 0 digests the evaluation
    if (cur_mode == SOLVE_EVALUATE) {
      if (tid == 0) { LmState& L = s_lm; for (int i = 0; i < 21; i++) L.H[i] = s_sum[i]; for (int i = 0; i < 6; i++) L.g[i] = s_sum[21 + i]; L.x_cost = s_sum[27]; L.n_valid = (int)(s_sum[28] + 0.5); L.done = 1; }
    } else {
      StepIn in; double gx[7], gg[6];
      if (warp == 1 && lane < 2) lm_hypothesis(s_lm, s_sum, lane, in);   // a private copy of the state BEFORE warp 0 touches it
      if (tid == 64) { for (int k = 0; k < 7; k++) gx[k] = s_lm.trial[k]; for (int c = 0; c < 6; c++) gg[c] = -s_sum[21 + c]; }
      __syncthreads();
      const long long t_h0 = clock64();
      if (warp == 1 && lane < 2) { compute_step(in, bound, s_pre[lane]); if (master && lane == 0) s_prof[13] += clock64() - t_h0; }   // Cholesky + model cost + Plus: the long pole of an LM step ...
      else if (tid == 0) { lm_step(s_lm, s_sum, bound, true); if (master) s_prof[14] += clock64() - t_h0; }   // ... next to the accept test and the bookkeeping ...
      else if (tid == 64) {   // ... and the gradient test of the accepted point (max |x - Plus(x, -g)|), which only the NEXT iteration's entry check reads
        double pg[7]; d_plus(gx, gg, bound, pg); double mx = 0; for (int k = 0; k < 7; k++) mx = fmax(mx, fabs(gx[k] - pg[k])); s_gmax = mx;
      }
      __syncthreads();
      if (tid == 0 && s_lm.pending == 0) s_lm.last_gmax = s_gmax;   // pending == 0 <=> the point just evaluated became x
      if (master && tid == 0) s_prof[15] += clock64() - t_h0;
      if (tid == 0 && s_lm.pending >= 0) lm_next_iteration(s_lm, bound, &s_pre[s_lm.pending]);
    }
    // (volatile: the plain test was if-converted into a load of `done` by EVERY thread, which racecheck reports against thread 0's write in lm_finish --
    // harmless, only thread 0 ever used the value, but there is no reason to keep a flagged access)
    if (tid == 0) { if (!*(volatile int*)&s_lm.done) setup_trial<MB>(E, s_lm.trial); }
    __syncthreads();
    if (master && tid == 0) { const long long t_e4 = clock64(); s_prof[0] += t_e1 - t_e0; s_prof[1] += t_e2 - t_e1; s_prof[2] += t_e3 - t_e2; s_prof[3] += t_e4 - t_e3; s_prof[5] += 1; }
    if (s_lm.done) break;
  }
  // ---- the solve has ended (on every CTA, with the same state)
  if (tid == 0) {
    LmState& L = s_lm;
    setup_trial<MB>(E, L.x_best);   // the epilogue (L1 norms) evaluates at the solution
    if (master) {
      st->lm = L;   // whole solver state (parity hooks / host diagnostics read it)
      if (cur_mode != SOLVE_EVALUATE) {
        for (int k = 0; k < 7; k++) st->x[k] = L.x_best[k];
        st->total_lm_iterations += L.iteration; st->total_evaluations += L.total_evaluations;
      }
      if (cur_mode == SOLVE_SECOND) {   // :514-531 pose composition + ICP termination test
        double qi[4] = {L.x_best[3], L.x_best[0], L.x_best[1], L.x_best[2]}, ti[3] = {L.x_best[4], L.x_best[5], L.x_best[6]};
        const double* ql = st->pose_last; double tcur[3], qcur[4];
        d_qrot(ql, ti, tcur); for (int k = 0; k < 3; k++) tcur[k] += st->pose_last[4 + k];
        d_qmul(ql, qi, qcur);
        for (int k = 0; k < 4; k++) st->pose_curr[k] = qcur[k]; for (int k = 0; k < 3; k++) st->pose_curr[4 + k] = tcur[k];
        st->angular_diff = (double)((float)d_angdist(qcur, ql)) * 57.3;
        double td = 0; for (int k = 0; k < 3; k++) td += (tcur[k] - st->pose_last[4 + k]) * (tcur[k] - st->pose_last[4 + k]); st->t_diff = sqrt(td);
        if (MB) {   // compute_interpolatation_rodrigue (:607-620): Eigen::AngleAxisd(q_incre), used by the next iteration's pointAssociateToMap
          double n = sqrt(qi[1] * qi[1] + qi[2] * qi[2] + qi[3] * qi[3]), ax[3], ang;
          if (n != 0.0) { ang = 2.0 * atan2(n, fabs(qi[0])); if (qi[0] < 0) n = -n; ax[0] = qi[1] / n; ax[1] = qi[2] / n; ax[2] = qi[3] / n; }
          else { ang = 0; ax[0] = 1; ax[1] = 0; ax[2] = 0; }
          const double an = sqrt(ax[0] * ax[0] + ax[1] * ax[1] + ax[2] * ax[2]); for (int k = 0; k < 3; k++) ax[k] /= an;
          double* H = st->interp_hat; for (int k = 0; k < 9; k++) H[k] = 0;
          H[1] = -ax[2]; H[3] = ax[2]; H[2] = ax[1]; H[6] = -ax[1]; H[5] = -ax[0]; H[7] = ax[0];
          for (int i = 0; i < 3; i++) for (int j = 0; j < 3; j++) { double t = 0; for (int k = 0; k < 3; k++) t += H[i * 3 + k] * H[k * 3 + j]; st->interp_hat_sq[i * 3 + j] = t; }
          st->interp_theta = ang;
        }
        if (L.termination == -1) st->icp_done = 1;   // no residual block: the host reports the error; iterations launched ahead must not run
        st->final_cost = L.final_cost; st->initial_cost = L.initial_cost; st->num_residual_blocks = L.n_valid;
        double dt = 0; for (int k = 0; k < 3; k++) dt += (st->t_last_opt[k] - ti[k]) * (st->t_last_opt[k] - ti[k]);
        if (d_angdist(st->q_last_opt, qi) < 57.3 * st->min_icp_R && sqrt(dt) < st->min_icp_T) st->icp_done = 1;
        else { for (int k = 0; k < 4; k++) st->q_last_opt[k] = qi[k]; for (int k = 0; k < 3; k++) st->t_last_opt[k] = ti[k]; }
        st->icp_iter++;
      }
    }
  }
  __syncthreads();
  // ---- epilogue of solve #1: loss-corrected L1 norm of every block at the solution (problem.Evaluate, :476-481)
  const long long t_p0 = clock64();
  if (cur_mode == SOLVE_FIRST) {
    for (int k = 0; k < tiles_per_cta; k++) {
      const int i = (blockIdx.x + gridDim.x * k) * tile + tid, li = k * SOLVE_THREADS + tid;
      double my_l1 = INFINITY;
      if (i < a.M && tid < tile) {
        double l1 = INFINITY;
        Slot s; s.type = S.type[li] & 0xff;
        if (s.type != 0) {
          double r[3];
          if (MB) {
            s.px = S.p[0][li]; s.py = S.p[1][li]; s.pz = S.p[2][li]; s.ax = S.a[0][li]; s.ay = S.a[1][li]; s.az = S.a[2][li];
            s.vx = S.v[0][li]; s.vy = S.v[1][li]; s.vz = S.v[2][li];
            s.s = (double)S.s[li];
            double J[6][3]; eval_block<true>(s, E, r, J, false);
          } else {   // the L1 norm is taken in the world frame: r = R_last r'
            FastSlot fs; fs.type = s.type; fs.px = S.p[0][li]; fs.py = S.p[1][li]; fs.pz = S.p[2][li]; fs.ax = S.ap[0][li]; fs.ay = S.ap[1][li]; fs.az = S.ap[2][li];
            fs.wx = S.v[0][li]; fs.wy = S.v[1][li]; fs.wz = S.v[2][li];
            double y[3], rp[3], alpha; fast_residual(fs, E, y, rp, alpha);
            r[0] = E.Rl[0][0] * rp[0] + E.Rl[0][1] * rp[1] + E.Rl[0][2] * rp[2];
            r[1] = E.Rl[1][0] * rp[0] + E.Rl[1][1] * rp[1] + E.Rl[1][2] * rp[2];
            r[2] = E.Rl[2][0] * rp[0] + E.Rl[2][1] * rp[1] + E.Rl[2][2] * rp[2];
          }
          double rho0; const double wgt = huber_weight(r[0] * r[0] + r[1] * r[1] + r[2] * r[2], E.huber_a, E.huber_b, rho0);
          const double sc = sqrt(wgt);
          l1 = fabs(sc * r[0]) + fabs(sc * r[1]) + fabs(sc * r[2]);
        }
        a.l1[i] = l1;
        my_l1 = l1;
      }
      // std::set de-duplication: the thread whose insert created the entry represents the value from here on (bit 8 of its slot's type)
      if (fused && l1_set_insert_flag(a.table, a.table_mask, my_l1, my_l1 < INFINITY)) S.type[li] |= 0x100;
    }
  }
  if (fused && ph == 0) {
    // ---- K10 over the whole grid (:153-161): the element of rank floor(ratio * n) among the DISTINCT L1 norms (k10_select)
    const long long q0 = clock64();
    k10_select(s_k10, Y, gen, S.type, a.l1, a.M, tiles_per_cta, tile, &st->inlier_ratio);
    const double thr2 = k10_threshold(st->inliner_dis, s_k10.result, s_k10.n_distinct);
    if (master && tid == 0) { st->inlier_threshold = thr2; st->n_unique = s_k10.n_distinct; }
    const long long q3 = clock64();
    for (int k = 0; k < tiles_per_cta; k++) {                // :487-499: blocks above the threshold leave the problem
      const int i = (blockIdx.x + gridDim.x * k) * tile + tid, li = k * SOLVE_THREADS + tid;
      if (i < a.M && tid < tile) { const int t = S.type[li] & 0xff; S.type[li] = (t != 0 && a.l1[i] > thr2) ? 0 : t; }
    }
    cur_mode = SOLVE_SECOND;
    __syncthreads();
    if (master && tid == 0) { const long long q4 = clock64(); s_prof[8] += q0 - t_p0; s_prof[10] += q3 - q0; s_prof[12] += q4 - q3; }
  }
  if (master && tid == 0) s_prof[7] += clock64() - t_p0;
  }   // phase
  // hand the generation base to the next launch (stream-ordered): every CTA ended with the same `gen`
  if (master && tid == 0) {
    *((volatile unsigned*)&Y->gen) = gen;
    for (int k = 0; k < 16; k++) st->prof[k] += s_prof[k];
  }
}

#define SOLVE_MAX_SMEM (200 * 1024)   // up to ~405k slots on 132 SMs; a typical scan (<= 113 KB of slots per CTA) leaves room for a second CTA per SM (another context's solver)

int solve_prepare(ll_ctx* ctx) {
  LL_CUDA(ctx, cudaFuncSetAttribute((void*)lm_solve_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, SOLVE_MAX_SMEM));
  LL_CUDA(ctx, cudaFuncSetAttribute((void*)lm_solve_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, SOLVE_MAX_SMEM));
  if (!ctx->d_sync) {
    void* p = nullptr; LL_CUDA(ctx, cudaMalloc(&p, sizeof(SolveSync))); LL_CUDA(ctx, cudaMemset(p, 0, sizeof(SolveSync))); ctx->d_sync = (SolveSync*)p;
  }
  return LL_OK;
}
// How M slots are spread over the persistent CTAs: CTA b owns the tiles b, b + grid, b + 2 grid, ... of `tile` slots each.
struct SolveGrid { int tile, tiles_per_cta, grid; };
static SolveGrid solve_grid(const ll_ctx* ctx, int M) {
  // The evaluation is fp64-throughput bound (64 DFMA/clk/SM): spread the slots over ALL SMs, even when that leaves CTAs partly empty.
  // tile = slots per CTA and pass (a multiple of 32, <= SOLVE_THREADS); partly empty CTAs on every SM evaluate faster than fewer full ones.
  const int M1 = M > 0 ? M : 1;
  SolveGrid g;
  g.tile = ((ll_div_up(M1, ctx->num_sms) + 31) / 32) * 32; if (g.tile > SOLVE_THREADS) g.tile = SOLVE_THREADS;
  const int tiles = ll_div_up(M1, g.tile);
  g.grid = tiles < ctx->num_sms ? tiles : ctx->num_sms; if (g.grid > LL_SYNC_ROWS) g.grid = LL_SYNC_ROWS;
  g.tiles_per_cta = ll_div_up(tiles, g.grid);
  return g;
}
// Dynamic shared memory of one solver CTA: whole tiles of SOLVE_THREADS slots, SLOT_BYTES (fast path) or SLOT_BYTES_MB (*_mb functors) each.
static size_t solve_smem_bytes(const SolveGrid& sg, int deblur) { return (size_t)sg.tiles_per_cta * SOLVE_THREADS * (deblur ? SLOT_BYTES_MB : SLOT_BYTES); }
int solve_capacity(ll_ctx* ctx, int M, int deblur) {
  if (solve_smem_bytes(solve_grid(ctx, M), deblur) > SOLVE_MAX_SMEM) { ctx->set_error("too many residual-block slots for the shared-memory-resident solver"); return LL_ERR_CAPACITY; }
  return LL_OK;
}
int launch_solve(ll_ctx* ctx, const SolveArgs& a) {
  const SolveGrid sg = solve_grid(ctx, a.M);
  int tile = sg.tile, tiles_per_cta = sg.tiles_per_cta; const int grid = sg.grid;
  const int mb = a.deblur ? 1 : 0;
  LL_TRY(solve_capacity(ctx, a.M, mb));
  const size_t smem = solve_smem_bytes(sg, mb);
  void* fn = mb ? (void*)lm_solve_kernel<true> : (void*)lm_solve_kernel<false>;
  SolveArgs args = a; args.sync = ctx->d_sync; void* kargs[] = {&args, &tiles_per_cta, &tile};
  LL_CUDA(ctx, cudaLaunchCooperativeKernel(fn, dim3(grid), dim3(SOLVE_THREADS), kargs, smem, ctx->stream));   // co-residency of the whole grid is what the exchanges rely on
  ctx->launches++;
  return LL_OK;
}

// The fused kernel's K10 over n given values (the sharded mode's exchanged L1 norms, or the values of ll_inlier_select), spread over the CTAs as
// lm_solve_kernel spreads M = n slots.  Same generation protocol as the solver: `gen` is read at entry and handed to the next launch at the end.
__global__ void __launch_bounds__(SOLVE_THREADS) k10_select_kernel(SolveSync* Y, const double* l1, int n, const double* ratio, unsigned long long* table, unsigned table_mask,
                                                                   int tiles_per_cta, int tile, double* value, int* n_distinct) {
  extern __shared__ int s_flag[];   // [tiles_per_cta * SOLVE_THREADS]: bit 8 = this thread represents its slot's value (lm_solve_kernel: S.type)
  __shared__ K10Smem s_k10;
  const int tid = threadIdx.x;
  unsigned gen = *((volatile unsigned*)&Y->gen);
  k10_clear(table, table_mask, Y);
  grid_sync(Y, gen);   // the clear before any insert
  for (int k = 0; k < tiles_per_cta; k++) {   // as the epilogue of solve #1: +inf / NaN (and slots past n) are not residuals
    const int i = (blockIdx.x + gridDim.x * k) * tile + tid, li = k * SOLVE_THREADS + tid;
    const double v = (i < n && tid < tile) ? l1[i] : INFINITY;
    s_flag[li] = l1_set_insert_flag(table, table_mask, v, v < INFINITY) ? 0x100 : 0;
  }
  k10_select(s_k10, Y, gen, s_flag, l1, n, tiles_per_cta, tile, ratio);
  if (blockIdx.x == 0 && tid == 0) {
    *value = s_k10.n_distinct > 0 ? s_k10.result : 0.0; *n_distinct = s_k10.n_distinct;
    *((volatile unsigned*)&Y->gen) = gen;
  }
}
int launch_k10_select(ll_ctx* ctx, const double* d_l1, int n, const double* d_ratio, unsigned long long* table, unsigned table_mask, double* d_value, int* d_n_distinct) {
  const SolveGrid sg = solve_grid(ctx, n);
  int tile = sg.tile, tiles_per_cta = sg.tiles_per_cta;
  SolveSync* Y = ctx->d_sync;
  const size_t smem = (size_t)tiles_per_cta * SOLVE_THREADS * sizeof(int);   // 4 B per slot: 48 KB up to ~1.6M values on 132 SMs
  if (smem > 48 * 1024) LL_CUDA(ctx, cudaFuncSetAttribute((void*)k10_select_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  void* kargs[] = {&Y, &d_l1, &n, &d_ratio, &table, &table_mask, &tiles_per_cta, &tile, &d_value, &d_n_distinct};
  LL_CUDA(ctx, cudaLaunchCooperativeKernel((void*)k10_select_kernel, dim3(sg.grid), dim3(SOLVE_THREADS), kargs, smem, ctx->stream));
  ctx->launches++;
  return LL_OK;
}


// ---------------------------------------------------------------------------------------------- sharded mode: K10 exchange over peer memory
// The X buffer is single (not double-buffered): rank A may only start overwriting slot i for ICP iteration k+1 after every rank has finished reading X for
// iteration k.  That holds because (1) the select that reads X runs on every rank BEFORE that rank's solve #2 launch (stream order), (2) solve #2's first
// all-reduce cannot complete on any rank before every rank has entered it, and (3) A's next exchange launch follows A's solve #2 in stream order.  The host
// clears X (NaN) at the start of an iteration; the clear of iteration k+1 is ordered after A's solve #2 of iteration k in the same way.
struct L1ExchangeArgs { const double* l1; int M; int rank, world; char* comm_local; char* comm_peer[8]; };
__global__ void __launch_bounds__(256) l1_exchange_kernel(L1ExchangeArgs a) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < a.M) {
    const double v = a.l1[i];
    if (v < INFINITY) for (int p = 0; p < a.world; p++) ((double*)(a.comm_peer[p] + LL_COMM_X_OFF))[i] = v;   // one owner per slot: no write conflicts
  }
  __threadfence_system();
  __syncthreads();
  if (threadIdx.x != 0) return;
  unsigned* ctrl = (unsigned*)(a.comm_local + LL_COMM_CTRL_OFF);
  if (atomicAdd(&ctrl[2], 1u) != gridDim.x - 1) return;
  // last CTA of this rank: all of this rank's pushes are issued and fenced; tell every peer, then wait for every peer
  ctrl[2] = 0u;
  const unsigned g = ctrl[1] + 1u; ctrl[1] = g;
  __threadfence_system();
  for (int p = 0; p < a.world; p++) st_release_sys_u32((unsigned*)(a.comm_peer[p] + LL_COMM_CTRL_OFF) + 16 + a.rank, g);
  for (int p = 0; p < a.world; p++) { const unsigned* f = ctrl + 16 + p; while (ld_acquire_sys_u32(f) != g) {} }
}
// Residual-block cap in sharded mode: the drop probability depends on the number of blocks of ALL ranks.  One warp: push this rank's count into
// every peer's slot (double-buffered by generation parity), flag, wait for every peer's flag, sum in rank order.
struct CountExchangeArgs { RegDevState* st; int rank, world; char* comm_local; char* comm_peer[8]; };
__global__ void count_exchange_kernel(CountExchangeArgs a) {
  const int lane = threadIdx.x;
  unsigned* ctrl = (unsigned*)(a.comm_local + LL_COMM_CTRL_OFF);
  const unsigned g = ctrl[3] + 1u; const int par = g & 1u;
  if (lane < a.world) {
    unsigned* pc = (unsigned*)(a.comm_peer[lane] + LL_COMM_CTRL_OFF);
    pc[64 + par * 8 + a.rank] = (unsigned)a.st->n_blocks;
    __threadfence_system();
    st_release_sys_u32(pc + 80 + a.rank, g);
    while (ld_acquire_sys_u32(ctrl + 80 + lane) != g) {}
  }
  __syncwarp();
  if (lane == 0) {
    int tot = 0; for (int p = 0; p < a.world; p++) tot += (int)*((volatile unsigned*)(ctrl + 64 + par * 8 + p));
    a.st->n_blocks_all = tot; ctrl[3] = g;
  }
}
int launch_count_exchange(ll_ctx* ctx) {
  if (ctx->world <= 1) return LL_OK;
  CountExchangeArgs a; a.st = ctx->d_reg; a.rank = ctx->rank; a.world = ctx->world; a.comm_local = (char*)ctx->comm_local;
  for (int i = 0; i < 8; i++) a.comm_peer[i] = (char*)ctx->comm_peers[i];
  count_exchange_kernel<<<1, 32, 0, ctx->stream>>>(a); ctx->launches++;
  LL_CUDA(ctx, cudaGetLastError());
  return LL_OK;
}
int launch_l1_exchange(ll_ctx* ctx, const double* d_l1, int M) {
  if (ctx->world <= 1 || M == 0) return LL_OK;
  L1ExchangeArgs a; a.l1 = d_l1; a.M = M; a.rank = ctx->rank; a.world = ctx->world; a.comm_local = (char*)ctx->comm_local;
  for (int i = 0; i < 8; i++) a.comm_peer[i] = (char*)ctx->comm_peers[i];
  l1_exchange_kernel<<<ll_div_up(M, 256), 256, 0, ctx->stream>>>(a); ctx->launches++;
  LL_CUDA(ctx, cudaGetLastError());
  return LL_OK;
}
