// Pose graph (posegraph.cu): the 6 x 6 block operations of the exact LM step solve, as plain C++ like lm_core.cuh, so that tests/cpp/pg_host.cpp
// runs the same code on the host.  Blocks are row-major double[36]; a position's blocks are D (diagonal), C (coupling to the next position of the
// current list, row = this position) and b (right-hand side).  Eliminating position p between pl and pr (block rows of an SPD matrix):
//   D_p = L L^T,  Wl = L^-1 C_pl^T,  Wr = L^-1 C_p,  y = L^-1 b_p
// and the survivors take the Schur complement: D_pl -= Wl^T Wl, b_pl -= Wl^T y, D_pr -= Wr^T Wr, b_pr -= Wr^T y, C_pl = -Wl^T Wr.
// Back substitution: x_p = L^-T (y - Wl x_pl - Wr x_pr).
#pragma once
#include <cfloat>
#include <cmath>
#include "lm_state.h"
namespace {   // internal linkage: solve.cu links the same non-inline helpers of lm_core.cuh
#include "lm_core.cuh"
}

LL_HD LL_INLINE bool pg_chol6(const double* A, double* L) {   // A = L L^T, L lower; false if a pivot is not positive
  for (int i = 0; i < 6; i++)
    for (int j = 0; j < 6; j++) {
      if (j > i) { L[i * 6 + j] = 0.0; continue; }
      double s = A[i * 6 + j];
      for (int k = 0; k < j; k++) s -= L[i * 6 + k] * L[j * 6 + k];
      if (i == j) { if (!(s > 0.0)) return false; L[i * 6 + i] = sqrt(s); } else L[i * 6 + j] = s / L[j * 6 + j];
    }
  return true;
}
LL_HD LL_INLINE void pg_fwd(const double* L, double* v) {   // v <- L^-1 v
  for (int i = 0; i < 6; i++) { double s = v[i]; for (int k = 0; k < i; k++) s -= L[i * 6 + k] * v[k]; v[i] = s / L[i * 6 + i]; }
}
LL_HD LL_INLINE void pg_bwd(const double* L, double* v) {   // v <- L^-T v
  for (int i = 5; i >= 0; i--) { double s = v[i]; for (int k = i + 1; k < 6; k++) s -= L[k * 6 + i] * v[k]; v[i] = s / L[i * 6 + i]; }
}
LL_HD LL_INLINE void pg_fwd_block(const double* L, const double* B, bool transposed, double* W) {   // W = L^-1 B (or L^-1 B^T)
  for (int c = 0; c < 6; c++) {
    double v[6]; for (int r = 0; r < 6; r++) v[r] = transposed ? B[c * 6 + r] : B[r * 6 + c];
    pg_fwd(L, v); for (int r = 0; r < 6; r++) W[r * 6 + c] = v[r];
  }
}
LL_HD LL_INLINE void pg_sub_tt(double* D, const double* W1, const double* W2) {   // D -= W1^T W2
  for (int i = 0; i < 6; i++) for (int j = 0; j < 6; j++) { double s = 0.0; for (int k = 0; k < 6; k++) s += W1[k * 6 + i] * W2[k * 6 + j]; D[i * 6 + j] -= s; }
}
LL_HD LL_INLINE void pg_sub_tv(double* b, const double* W, const double* y) {    // b -= W^T y
  for (int i = 0; i < 6; i++) { double s = 0.0; for (int k = 0; k < 6; k++) s += W[k * 6 + i] * y[k]; b[i] -= s; }
}
// One elimination (false: the pivot block is not positive definite).
LL_HD LL_INLINE bool pg_elim(const double* D, const double* C_left, const double* C_self, const double* b, double* Lf, double* Wl, double* Wr, double* y) {
  if (!pg_chol6(D, Lf)) return false;
  pg_fwd_block(Lf, C_left, true, Wl); pg_fwd_block(Lf, C_self, false, Wr);
  for (int i = 0; i < 6; i++) y[i] = b[i];
  pg_fwd(Lf, y);
  return true;
}
// A survivor's update from the eliminated position on its left (its Wr couples to the survivor) and / or on its right (its Wl does), in
// that order; C is the survivor's new coupling to the next survivor (set when there is a right neighbour).
LL_HD LL_INLINE void pg_update(double* D, double* b, double* C, const double* Wr_left, const double* y_left, const double* Wl_right, const double* Wr_right,
                               const double* y_right) {
  if (Wr_left) { pg_sub_tt(D, Wr_left, Wr_left); pg_sub_tv(b, Wr_left, y_left); }
  if (Wl_right) {
    pg_sub_tt(D, Wl_right, Wl_right); pg_sub_tv(b, Wl_right, y_right);
    for (int i = 0; i < 36; i++) C[i] = 0.0;
    pg_sub_tt(C, Wl_right, Wr_right);
  }
}
LL_HD LL_INLINE void pg_backsub(const double* Lf, const double* Wl, const double* Wr, const double* y, const double* x_left, const double* x_right, double* x) {
  double v[6];
  for (int i = 0; i < 6; i++) { double s = y[i]; for (int k = 0; k < 6; k++) s -= Wl[i * 6 + k] * x_left[k] + Wr[i * 6 + k] * x_right[k]; v[i] = s; }
  pg_bwd(Lf, v);
  for (int i = 0; i < 6; i++) x[i] = v[i];
}
// acc += s_row (.) B (.) s_col (B or B^T), the scaled coupling of one edge
LL_HD LL_INLINE void pg_add_scaled(double* acc, const double* B, bool transposed, const double* s_row, const double* s_col) {
  for (int i = 0; i < 6; i++) for (int j = 0; j < 6; j++) acc[i * 6 + j] += s_row[i] * (transposed ? B[j * 6 + i] : B[i * 6 + j]) * s_col[j];
}
