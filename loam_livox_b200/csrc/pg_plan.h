// Pose graph (posegraph.cu): the elimination plan of the LM step's normal equations, built on the host from the graph's topology alone.
// Plain C++: posegraph.cu builds it for every solve and tests/cpp/pg_host.cpp builds it for the host test of the elimination.
//
// The free nodes are the ones an edge touches, except node 0 (held constant).  The border S is the set of free endpoints of every edge whose two
// endpoints are free and not consecutive (|a - b| != 1: a "loop" edge).  The other free nodes form runs of consecutive indices, the segments.
// A segment couples only to itself and to the S nodes just before and after it, so its system is block-tridiagonal: positions
// [left end, its nodes..., right end], where an end is an S node or, when the neighbour is not in S, a virtual node without couplings.
// Block cyclic reduction eliminates every other interior position of the current list per level (level lists below); what stays at the end is
// the two ends, whose accumulated blocks are the segment's contribution to the Schur complement on S.
#pragma once
#include <algorithm>
#include <vector>

struct PgPlan {
  int N = 0, M = 0, F = 0, nb = 0, n_pos = 0, n_seg = 0, n_levels = 0;
  std::vector<int> free_of_node;    // [N] free index, -1 for node 0 and nodes without edges
  std::vector<int> free_node;       // [F] node of a free index (ascending)
  std::vector<int> inc_ptr, inc;    // [F + 1], [..]: edges incident to a free node, ascending edge order, as edge * 2 + (1 if the node is its end)
  std::vector<int> border;          // [nb] free index of each S node (ascending)
  std::vector<int> free_border;     // [F] S index of a free node, -1 outside S
  std::vector<int> free_pos;        // [F] position of a segment node, -1 for S nodes
  std::vector<int> pos_free;        // [n_pos] free index of an interior position, -1 for a segment end
  std::vector<int> pos_border;      // [n_pos] S index of a segment end, -1 for interior positions and virtual ends
  std::vector<int> cpl_ptr, cpl;    // [n_pos + 1], [..]: edges coupling a position to the next one, ascending, as edge * 2 + (1 if stored transposed)
  std::vector<int> seg_first;       // [n_seg + 1] first position of each segment (its left end); the right end is seg_first[s + 1] - 1
  std::vector<int> elim_ptr, elim;  // [n_levels + 1], triples (left, eliminated, right) positions per level
  std::vector<int> upd_ptr, upd;    // [n_levels + 1], triples (survivor, eliminated on its left or -1, eliminated on its right or -1)
  // the border system, in blocks of S x S (upper triangle, block pair i * nb + j, i <= j) and per S node for the right-hand side.
  // Items (kind, index, transposed): 0 the assembled diagonal block / rhs of free node `index`, 1 the coupling of edge `index`, 2 the end
  // block / rhs at position `index`, 3 the coupling left end -> right end at position `index`.
  std::vector<int> bd_ptr, bd;      // [nb * nb + 1], triples
  std::vector<int> bb_ptr, bb;      // [nb + 1], pairs (kind, index)
};

// Builds the plan.  ea / eb: edge endpoints, already checked to lie in 0 .. N-1 and to differ.  Returns the border size (the caller refuses
// more than it supports before using the rest).
inline int pg_build_plan(int N, int M, const int* ea, const int* eb, PgPlan& P) {
  P = PgPlan(); P.N = N; P.M = M;
  P.free_of_node.assign(N, -1);
  std::vector<char> touched(N, 0);
  for (int e = 0; e < M; e++) { touched[ea[e]] = 1; touched[eb[e]] = 1; }
  for (int n = 1; n < N; n++) if (touched[n]) { P.free_of_node[n] = P.F++; P.free_node.push_back(n); }
  // incidence (ascending edge order per node)
  P.inc_ptr.assign(P.F + 1, 0);
  for (int e = 0; e < M; e++) for (int s = 0; s < 2; s++) { const int f = P.free_of_node[s ? eb[e] : ea[e]]; if (f >= 0) P.inc_ptr[f + 1]++; }
  for (int f = 0; f < P.F; f++) P.inc_ptr[f + 1] += P.inc_ptr[f];
  P.inc.resize(P.inc_ptr[P.F]);
  { std::vector<int> fill(P.inc_ptr.begin(), P.inc_ptr.end() - 1);
    for (int e = 0; e < M; e++) for (int s = 0; s < 2; s++) { const int f = P.free_of_node[s ? eb[e] : ea[e]]; if (f >= 0) P.inc[fill[f]++] = 2 * e + s; } }
  // border
  std::vector<int> sidx(P.F, -1);
  std::vector<char> in_s(P.F, 0);
  for (int e = 0; e < M; e++) {
    const int fa = P.free_of_node[ea[e]], fb = P.free_of_node[eb[e]];
    if (fa >= 0 && fb >= 0 && std::abs(ea[e] - eb[e]) != 1) { in_s[fa] = 1; in_s[fb] = 1; }
  }
  for (int f = 0; f < P.F; f++) if (in_s[f]) { sidx[f] = P.nb++; P.border.push_back(f); }
  P.free_border = sidx;
  // segments: maximal runs of consecutive node indices, all free and outside S
  P.free_pos.assign(P.F, -1);
  P.seg_first.push_back(0);
  for (int f = 0; f < P.F;) {
    if (in_s[f]) { f++; continue; }
    int g = f; while (g + 1 < P.F && !in_s[g + 1] && P.free_node[g + 1] == P.free_node[g] + 1) g++;
    const int left = P.free_node[f] - 1, right = P.free_node[g] + 1;
    const int fl = left >= 0 ? P.free_of_node[left] : -1, fr = right < N ? P.free_of_node[right] : -1;
    P.pos_free.push_back(-1); P.pos_border.push_back(fl >= 0 ? sidx[fl] : -1);
    for (int k = f; k <= g; k++) { P.free_pos[k] = (int)P.pos_free.size(); P.pos_free.push_back(k); P.pos_border.push_back(-1); }
    P.pos_free.push_back(-1); P.pos_border.push_back(fr >= 0 ? sidx[fr] : -1);
    P.seg_first.push_back((int)P.pos_free.size());
    P.n_seg++; f = g + 1;
  }
  P.n_pos = (int)P.pos_free.size();
  // couplings: a free-free edge between consecutive nodes goes to the position of its lower node (a segment node, or the left end of the
  // segment that starts after an S node); every other free-free edge couples two S nodes
  std::vector<std::vector<int>> cp(P.n_pos);
  std::vector<std::vector<int>> bitems((size_t)P.nb * P.nb);
  std::vector<int> left_end_of(P.F, -1);   // S free index -> position of the left end of the segment right after it
  for (int s = 0; s < P.n_seg; s++) { const int p = P.seg_first[s]; if (P.pos_border[p] >= 0) left_end_of[P.border[P.pos_border[p]]] = p; }
  for (int e = 0; e < M; e++) {
    const int fa = P.free_of_node[ea[e]], fb = P.free_of_node[eb[e]];
    if (fa < 0 || fb < 0) continue;
    const bool a_lo = ea[e] < eb[e]; const int lo = a_lo ? fa : fb, hi = a_lo ? fb : fa;
    if (in_s[lo] && in_s[hi]) {   // block row lo, column hi (border order is node order): J_a^T J_b, transposed when a is the higher node
      bitems[(size_t)sidx[lo] * P.nb + sidx[hi]].insert(bitems[(size_t)sidx[lo] * P.nb + sidx[hi]].end(), {1, e, a_lo ? 0 : 1});
    } else {
      const int p = in_s[lo] ? left_end_of[lo] : P.free_pos[lo];
      cp[p].push_back(2 * e + (a_lo ? 0 : 1));
    }
  }
  P.cpl_ptr.assign(P.n_pos + 1, 0);
  for (int p = 0; p < P.n_pos; p++) { P.cpl_ptr[p + 1] = P.cpl_ptr[p] + (int)cp[p].size(); P.cpl.insert(P.cpl.end(), cp[p].begin(), cp[p].end()); }
  // levels of cyclic reduction, all segments side by side
  std::vector<std::vector<int>> el, up;
  for (int s = 0; s < P.n_seg; s++) {
    std::vector<int> cur; for (int p = P.seg_first[s]; p < P.seg_first[s + 1]; p++) cur.push_back(p);
    for (int lv = 0; cur.size() > 2; lv++) {
      if ((int)el.size() <= lv) { el.emplace_back(); up.emplace_back(); }
      const int n = (int)cur.size();
      for (int i = 1; i <= n - 2; i += 2) el[lv].insert(el[lv].end(), {cur[i - 1], cur[i], cur[i + 1]});
      std::vector<int> next;
      for (int j = 0; j < n; j++) {
        if ((j & 1) && j != n - 1) continue;
        const int l = (j >= 1 && ((j - 1) & 1)) ? cur[j - 1] : -1, r = (j + 1 <= n - 2 && ((j + 1) & 1)) ? cur[j + 1] : -1;
        if (l >= 0 || r >= 0) up[lv].insert(up[lv].end(), {cur[j], l, r});
        next.push_back(cur[j]);
      }
      cur.swap(next);
    }
  }
  P.n_levels = (int)el.size();
  P.elim_ptr.assign(1, 0); P.upd_ptr.assign(1, 0);
  for (int lv = 0; lv < P.n_levels; lv++) {
    P.elim.insert(P.elim.end(), el[lv].begin(), el[lv].end()); P.elim_ptr.push_back((int)P.elim.size() / 3);
    P.upd.insert(P.upd.end(), up[lv].begin(), up[lv].end()); P.upd_ptr.push_back((int)P.upd.size() / 3);
  }
  // the border system: node blocks, then edge couplings (ascending), then the segments' contributions (ascending segment order)
  for (int i = 0; i < P.nb; i++) {
    std::vector<int>& d = bitems[(size_t)i * P.nb + i];
    d.insert(d.begin(), {0, P.border[i], 0});
  }
  std::vector<std::vector<int>> rhs(P.nb);
  for (int i = 0; i < P.nb; i++) rhs[i].insert(rhs[i].end(), {0, P.border[i]});
  for (int s = 0; s < P.n_seg; s++) {
    const int pl = P.seg_first[s], pr = P.seg_first[s + 1] - 1, sl = P.pos_border[pl], sr = P.pos_border[pr];
    if (sl >= 0) { bitems[(size_t)sl * P.nb + sl].insert(bitems[(size_t)sl * P.nb + sl].end(), {2, pl, 0}); rhs[sl].insert(rhs[sl].end(), {2, pl}); }
    if (sr >= 0) { bitems[(size_t)sr * P.nb + sr].insert(bitems[(size_t)sr * P.nb + sr].end(), {2, pr, 0}); rhs[sr].insert(rhs[sr].end(), {2, pr}); }
    if (sl >= 0 && sr >= 0) bitems[(size_t)sl * P.nb + sr].insert(bitems[(size_t)sl * P.nb + sr].end(), {3, pl, 0});
  }
  P.bd_ptr.assign((size_t)P.nb * P.nb + 1, 0);
  for (size_t k = 0; k < bitems.size(); k++) { P.bd.insert(P.bd.end(), bitems[k].begin(), bitems[k].end()); P.bd_ptr[k + 1] = (int)P.bd.size() / 3; }
  P.bb_ptr.assign(P.nb + 1, 0);
  for (int i = 0; i < P.nb; i++) { P.bb.insert(P.bb.end(), rhs[i].begin(), rhs[i].end()); P.bb_ptr[i + 1] = (int)P.bb.size() / 2; }
  return P.nb;
}
