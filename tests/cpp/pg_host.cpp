// The pose-graph step solve's elimination (loam_livox_b200/csrc/pg_plan.h and pg_block.cuh) compiled for the host: the same plan and the same
// 6 x 6 block operations the kernel runs, driven level by level in the kernel's order, with a plain dense Cholesky for the border.
// tests/test_pose_graph_host.py compares the solution with numpy.linalg.solve.
#include <vector>
#include "../../loam_livox_b200/csrc/pg_block.cuh"
#include "../../loam_livox_b200/csrc/pg_plan.h"

extern "C" {

// Solves A x = b, A given as the diagonal block of every free node (node_blocks [N x 36]; rows of nodes that are not free are ignored) and
// the coupling J_a^T J_b of every edge (edge_blocks [M x 36], row = id_begin), b per node [N x 6].  Returns the border size, or -1 when a
// pivot fails.  stats: free nodes, segments, levels.
int pgh_solve(int N, int M, const int* ea, const int* eb, const double* node_blocks, const double* edge_blocks, const double* b_nodes, double* x, int* stats) {
  PgPlan P; pg_build_plan(N, M, ea, eb, P);
  stats[0] = P.F; stats[1] = P.n_seg; stats[2] = P.n_levels;
  const double ones[6] = {1, 1, 1, 1, 1, 1};
  std::vector<double> D(36 * (size_t)P.n_pos), C(36 * (size_t)P.n_pos), b(6 * (size_t)P.n_pos), Lf(D.size()), Wl(D.size()), Wr(D.size()), y(b.size()), xs(b.size());
  auto coupling = [&](int e, int tr, double* acc) { pg_add_scaled(acc, edge_blocks + 36 * e, tr != 0, ones, ones); };
  for (int p = 0; p < P.n_pos; p++) {
    const int f = P.pos_free[p];
    for (int i = 0; i < 36; i++) { D[36 * p + i] = f >= 0 ? node_blocks[36 * P.free_node[f] + i] : 0.0; C[36 * p + i] = 0.0; }
    for (int i = 0; i < 6; i++) b[6 * p + i] = f >= 0 ? b_nodes[6 * P.free_node[f] + i] : 0.0;
    for (int q = P.cpl_ptr[p]; q < P.cpl_ptr[p + 1]; q++) coupling(P.cpl[q] >> 1, P.cpl[q] & 1, &C[36 * p]);
  }
  for (int lv = 0; lv < P.n_levels; lv++) {
    for (int q = P.elim_ptr[lv]; q < P.elim_ptr[lv + 1]; q++) {
      const int pl = P.elim[3 * q], p = P.elim[3 * q + 1];
      if (!pg_elim(&D[36 * p], &C[36 * pl], &C[36 * p], &b[6 * p], &Lf[36 * p], &Wl[36 * p], &Wr[36 * p], &y[6 * p])) return -1;
    }
    for (int q = P.upd_ptr[lv]; q < P.upd_ptr[lv + 1]; q++) {
      const int s = P.upd[3 * q], l = P.upd[3 * q + 1], r = P.upd[3 * q + 2];
      pg_update(&D[36 * s], &b[6 * s], &C[36 * s], l >= 0 ? &Wr[36 * l] : nullptr, l >= 0 ? &y[6 * l] : nullptr, r >= 0 ? &Wl[36 * r] : nullptr,
                r >= 0 ? &Wr[36 * r] : nullptr, r >= 0 ? &y[6 * r] : nullptr);
    }
  }
  const int n = 6 * P.nb;
  std::vector<double> Bm((size_t)n * n, 0.0), Bv(n, 0.0);
  for (int i = 0; i < P.nb; i++) for (int j = i; j < P.nb; j++) {
    const int pair = i * P.nb + j;
    for (int ent = 0; ent < 36; ent++) {
      double v = 0.0;
      for (int q = P.bd_ptr[pair]; q < P.bd_ptr[pair + 1]; q++) {
        const int kind = P.bd[3 * q], idx = P.bd[3 * q + 1], tr = P.bd[3 * q + 2];
        if (kind == 0) v += node_blocks[36 * P.free_node[idx] + ent];
        else if (kind == 1) { double acc[36] = {}; coupling(idx, tr, acc); v += acc[ent]; }
        else if (kind == 2) v += D[36 * idx + ent];
        else v += C[36 * idx + ent];
      }
      Bm[(size_t)(6 * j + ent % 6) * n + 6 * i + ent / 6] = v;
    }
  }
  for (int i = 0; i < P.nb; i++) for (int r = 0; r < 6; r++) {
    double v = 0.0;
    for (int q = P.bb_ptr[i]; q < P.bb_ptr[i + 1]; q++) v += P.bb[2 * q] == 0 ? b_nodes[6 * P.free_node[P.bb[2 * q + 1]] + r] : b[6 * P.bb[2 * q + 1] + r];
    Bv[6 * i + r] = v;
  }
  for (int k = 0; k < n; k++) {   // the kernel's right-looking Cholesky, serially
    const double d = Bm[(size_t)k * n + k]; if (!(d > 0.0)) return -1;
    Bm[(size_t)k * n + k] = std::sqrt(d);
    for (int i = k + 1; i < n; i++) Bm[(size_t)i * n + k] /= Bm[(size_t)k * n + k];
    for (int i = k + 1; i < n; i++) for (int j = k + 1; j <= i; j++) Bm[(size_t)i * n + j] -= Bm[(size_t)i * n + k] * Bm[(size_t)j * n + k];
  }
  for (int k = 0; k < n; k++) { Bv[k] /= Bm[(size_t)k * n + k]; for (int i = k + 1; i < n; i++) Bv[i] -= Bm[(size_t)i * n + k] * Bv[k]; }
  for (int k = n - 1; k >= 0; k--) { Bv[k] /= Bm[(size_t)k * n + k]; for (int i = 0; i < k; i++) Bv[i] -= Bm[(size_t)k * n + i] * Bv[k]; }
  for (int p = 0; p < P.n_pos; p++) if (P.pos_free[p] < 0) for (int i = 0; i < 6; i++) xs[6 * p + i] = P.pos_border[p] >= 0 ? Bv[6 * P.pos_border[p] + i] : 0.0;
  for (int lv = P.n_levels - 1; lv >= 0; lv--)
    for (int q = P.elim_ptr[lv]; q < P.elim_ptr[lv + 1]; q++) {
      const int pl = P.elim[3 * q], p = P.elim[3 * q + 1], pr = P.elim[3 * q + 2];
      pg_backsub(&Lf[36 * p], &Wl[36 * p], &Wr[36 * p], &y[6 * p], &xs[6 * pl], &xs[6 * pr], &xs[6 * p]);
    }
  for (int i = 0; i < 6 * N; i++) x[i] = 0.0;
  for (int f = 0; f < P.F; f++) {
    const double* v = P.free_border[f] >= 0 ? &Bv[6 * P.free_border[f]] : &xs[6 * P.free_pos[f]];
    for (int i = 0; i < 6; i++) x[6 * P.free_node[f] + i] = v[i];
  }
  return P.nb;
}

}
