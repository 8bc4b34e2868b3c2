// nd_precond.cpp -- host side of the sparse exact preconditioner: nested dissection of the pose graph, macro levels,
// dense block algebra of the setup, the static work plan of the apply phases, and a host emulation of that plan
// (verification only).  See nd_precond.h for the design.  Host code only (g++), no CUDA here.
#include "nd_precond.h"

#include <algorithm>
#include <cmath>
#include <cstdio>
#include <cstring>
#include <functional>
#include <numeric>
#include <sstream>
#include <stdexcept>

namespace dpgo {
namespace nd {

namespace {

// ---------------------------------------------------------------------------------------------------------------
// pose-graph adjacency from the block-CSR pattern
// ---------------------------------------------------------------------------------------------------------------
struct Graph {
  int n = 0;
  std::vector<int> ptr, adj;
};

Graph make_graph(const BsrView &Q) {
  Graph g;
  g.n = Q.n;
  std::vector<std::vector<int>> nb((size_t)Q.n);
  for (int j = 0; j < Q.n; ++j)
    for (int b = Q.rowptr[j]; b < Q.rowptr[j + 1]; ++b) {
      const int i = Q.bcol[b];
      if (i < 0 || i >= Q.n) throw std::runtime_error("nd: block column index out of range");
      if (i != j) { nb[(size_t)j].push_back(i); nb[(size_t)i].push_back(j); }
    }
  g.ptr.assign((size_t)Q.n + 1, 0);
  for (int j = 0; j < Q.n; ++j) {
    auto &v = nb[(size_t)j];
    std::sort(v.begin(), v.end());
    v.erase(std::unique(v.begin(), v.end()), v.end());
    g.ptr[(size_t)j + 1] = g.ptr[(size_t)j] + (int)v.size();
  }
  g.adj.reserve((size_t)g.ptr[(size_t)Q.n]);
  for (int j = 0; j < Q.n; ++j) g.adj.insert(g.adj.end(), nb[(size_t)j].begin(), nb[(size_t)j].end());
  return g;
}

// ---------------------------------------------------------------------------------------------------------------
// nested dissection by BFS level structures (George): the separator is one level set of a BFS from a
// pseudo-peripheral vertex, chosen small and balanced, then thinned.
// ---------------------------------------------------------------------------------------------------------------
struct NdNode {
  int parent = -1, level = 0;
  int child[2] = {-1, -1};
  std::vector<int> own;          // separator poses (inner node) or all poses (leaf)
  std::vector<int> bnd;          // ancestors' poses adjacent to the subtree
  std::vector<int> cum;          // cum[l - level] = own poses of the subtree at dissection levels <= l
};

struct Dissector {
  const Graph &g;
  int leaf_size;
  std::vector<NdNode> tree;
  std::vector<int> stamp, lvl;   // membership stamp / BFS level
  int cur = 0;

  Dissector(const Graph &gg, int ls) : g(gg), leaf_size(std::max(1, ls)), stamp((size_t)gg.n, -1), lvl((size_t)gg.n, -1) {}

  // BFS inside the vertices stamped `id`; fills order / lvl, returns number of levels
  int bfs(int start, int id, std::vector<int> &order) {
    order.clear();
    order.push_back(start);
    lvl[(size_t)start] = 0;
    stamp[(size_t)start] = id + 1;               // id + 1 = visited in this sweep
    size_t head = 0;
    int maxl = 0;
    while (head < order.size()) {
      const int u = order[head++];
      for (int q = g.ptr[(size_t)u]; q < g.ptr[(size_t)u + 1]; ++q) {
        const int v = g.adj[(size_t)q];
        if (stamp[(size_t)v] == id) {
          stamp[(size_t)v] = id + 1;
          lvl[(size_t)v] = lvl[(size_t)u] + 1;
          maxl = std::max(maxl, lvl[(size_t)v]);
          order.push_back(v);
        }
      }
    }
    return maxl + 1;
  }

  void restamp(const std::vector<int> &nodes, int id) {
    for (int v : nodes) stamp[(size_t)v] = id;
  }

  // returns false if the set cannot be split (too small / diameter < 2)
  bool bisect(const std::vector<int> &nodes, std::vector<int> &A, std::vector<int> &B, std::vector<int> &S) {
    A.clear(); B.clear(); S.clear();
    const int n = (int)nodes.size();
    cur += 2;
    const int id = cur;
    restamp(nodes, id);
    // connected components
    std::vector<int> order;
    std::vector<std::vector<int>> comps;
    for (int s : nodes)
      if (stamp[(size_t)s] == id) {
        bfs(s, id, order);
        comps.push_back(order);
      }
    if (comps.size() > 1) {
      std::stable_sort(comps.begin(), comps.end(), [](const std::vector<int> &x, const std::vector<int> &y) { return x.size() > y.size(); });
      for (auto &c : comps) {
        std::vector<int> &dst = (A.size() <= B.size()) ? A : B;
        dst.insert(dst.end(), c.begin(), c.end());
      }
      return true;
    }
    // pseudo-peripheral start vertex
    int s = nodes[0];
    int nl = 0;
    for (int it = 0; it < 4; ++it) {
      cur += 2;
      restamp(nodes, cur);
      nl = bfs(s, cur, order);
      const int far = order.back();
      if (far == s) break;
      if (it < 3) s = far;
    }
    if (nl < 3) return false;
    std::vector<int> cnt((size_t)nl, 0);
    for (int v : order) cnt[(size_t)lvl[(size_t)v]]++;
    std::vector<int> cum((size_t)nl, 0);
    std::partial_sum(cnt.begin(), cnt.end(), cum.begin());
    int bk = -1;
    double best = 1e300;
    for (int pass = 0; pass < 2 && bk < 0; ++pass) {
      const double minside = (pass == 0) ? 0.25 * n : 1.0;
      for (int k = 1; k < nl - 1; ++k) {
        const int a = cum[(size_t)k - 1], b = n - cum[(size_t)k];
        if (std::min(a, b) < minside) continue;
        const double score = cnt[(size_t)k] + 0.02 * std::abs(a - b) + (pass ? 0.5 * std::abs(a - b) : 0.0);
        if (score < best) { best = score; bk = k; }
      }
    }
    if (bk < 0) return false;
    std::vector<int> cand;
    for (int v : order) {
      const int l = lvl[(size_t)v];
      if (l < bk) A.push_back(v);
      else if (l > bk) B.push_back(v);
      else cand.push_back(v);
    }
    // thin the separator: a vertex without neighbours on one side joins the other side
    cur += 2;
    const int idA = cur, idB = cur + 1;
    for (int v : A) stamp[(size_t)v] = idA;
    for (int v : B) stamp[(size_t)v] = idB;
    for (int v : cand) stamp[(size_t)v] = -1;
    for (int v : cand) {
      bool na = false, nb = false;
      for (int q = g.ptr[(size_t)v]; q < g.ptr[(size_t)v + 1]; ++q) {
        const int u = g.adj[(size_t)q];
        if (stamp[(size_t)u] == idA) na = true;
        else if (stamp[(size_t)u] == idB) nb = true;
      }
      if (na && nb) S.push_back(v);
      else if (nb && !na) { B.push_back(v); stamp[(size_t)v] = idB; }
      else { A.push_back(v); stamp[(size_t)v] = idA; }
    }
    cur += 2;
    return !A.empty() && !B.empty();
  }

  void dissect(std::vector<int> nodes, int parent, int level, int which) {
    const int idx = (int)tree.size();
    tree.emplace_back();
    tree[(size_t)idx].parent = parent;
    tree[(size_t)idx].level = level;
    if (parent >= 0) tree[(size_t)parent].child[which] = idx;
    std::vector<int> A, B, S;
    if ((int)nodes.size() <= leaf_size || level >= 60 || !bisect(nodes, A, B, S)) {
      std::sort(nodes.begin(), nodes.end());
      tree[(size_t)idx].own = std::move(nodes);
      return;
    }
    std::sort(S.begin(), S.end());
    tree[(size_t)idx].own = S;
    nodes.clear();
    nodes.shrink_to_fit();
    dissect(std::move(A), idx, level + 1, 0);
    dissect(std::move(B), idx, level + 1, 1);
  }
};

// merge-unique of sorted vectors keeping only entries accepted by `keep`
template <class F> std::vector<int> merge_filter(const std::vector<int> &a, const std::vector<int> &b, F keep) {
  std::vector<int> out;
  out.reserve(a.size() + b.size());
  size_t i = 0, j = 0;
  while (i < a.size() || j < b.size()) {
    int v;
    if (j >= b.size() || (i < a.size() && a[i] <= b[j])) {
      v = a[i];
      if (j < b.size() && b[j] == v) ++j;
      ++i;
    } else {
      v = b[j++];
    }
    if (keep(v)) out.push_back(v);
  }
  return out;
}

// ---------------------------------------------------------------------------------------------------------------
// small dense algebra (row-major); OpenMP over independent rows / column slices where it pays
// ---------------------------------------------------------------------------------------------------------------
bool chol_lower(double *A, int s) {     // A = L L^T in place (lower triangle holds L)
  const int NB = 64;
  for (int kb = 0; kb < s; kb += NB) {
    const int ke = std::min(s, kb + NB);
    for (int i = kb; i < ke; ++i) {                                   // diagonal block, row-dot form
      for (int j = kb; j <= i; ++j) {
        double sum = A[(size_t)i * s + j];
        for (int k = kb; k < j; ++k) sum -= A[(size_t)i * s + k] * A[(size_t)j * s + k];
        if (i == j) {
          if (!(sum > 0.0)) return false;
          A[(size_t)i * s + i] = std::sqrt(sum);
        } else {
          A[(size_t)i * s + j] = sum / A[(size_t)j * s + j];
        }
      }
    }
#pragma omp parallel for schedule(static) if (s - ke > 256)
    for (int i = ke; i < s; ++i) {                                     // panel below the diagonal block
      for (int j = kb; j < ke; ++j) {
        double sum = A[(size_t)i * s + j];
        for (int k = kb; k < j; ++k) sum -= A[(size_t)i * s + k] * A[(size_t)j * s + k];
        A[(size_t)i * s + j] = sum / A[(size_t)j * s + j];
      }
    }
#pragma omp parallel for schedule(dynamic, 16) if (s - ke > 256)
    for (int i = ke; i < s; ++i) {                                     // trailing update (lower part)
      const double *li = A + (size_t)i * s + kb;
      for (int j = ke; j <= i; ++j) {
        const double *lj = A + (size_t)j * s + kb;
        double sum = 0.0;
        for (int k = 0; k < ke - kb; ++k) sum += li[k] * lj[k];
        A[(size_t)i * s + j] -= sum;
      }
    }
  }
  return true;
}

// B (s x m, row-major) <- (L L^T)^-1 B
void chol_solve(const double *L, int s, double *B, int m) {
  const int CH = 256;
  const int nch = (m + CH - 1) / CH;
#pragma omp parallel for schedule(dynamic, 1) if (nch > 1 && (double)s * s * m > 1e7)
  for (int ch = 0; ch < nch; ++ch) {
    const int c0 = ch * CH, c1 = std::min(m, c0 + CH);
    for (int i = 0; i < s; ++i) {
      double *bi = B + (size_t)i * m;
      for (int k = 0; k < i; ++k) {
        const double l = L[(size_t)i * s + k];
        if (l == 0.0) continue;
        const double *bk = B + (size_t)k * m;
        for (int c = c0; c < c1; ++c) bi[c] -= l * bk[c];
      }
      const double inv = 1.0 / L[(size_t)i * s + i];
      for (int c = c0; c < c1; ++c) bi[c] *= inv;
    }
    for (int i = s - 1; i >= 0; --i) {
      double *bi = B + (size_t)i * m;
      const double inv = 1.0 / L[(size_t)i * s + i];
      for (int c = c0; c < c1; ++c) bi[c] *= inv;
      for (int k = 0; k < i; ++k) {
        const double l = L[(size_t)i * s + k];
        if (l == 0.0) continue;
        double *bk = B + (size_t)k * m;
        for (int c = c0; c < c1; ++c) bk[c] -= l * bi[c];
      }
    }
  }
}

// dense algebra of one node.  in: Foo (s x s, row-major, SPD), Fob (s x b), Fbb (b x b);
// out: W = Foo^-1 (s x s), Fm = W Fob (s x b), Fbb -= Fob^T Fm
void host_factor(int s, int b, double *Foo, double *Fob, double *Fbb) {
  std::vector<double> L(Foo, Foo + (size_t)s * s);
  if (!chol_lower(L.data(), s)) throw std::runtime_error("nd: Schur complement not positive definite");
  for (int i = 0; i < s; ++i)
    for (int j = i + 1; j < s; ++j) L[(size_t)i * s + j] = 0.0;
  // W = Foo^-1 : solve with the identity
  std::fill(Foo, Foo + (size_t)s * s, 0.0);
  for (int i = 0; i < s; ++i) Foo[(size_t)i * s + i] = 1.0;
  chol_solve(L.data(), s, Foo, s);
  for (int i = 0; i < s; ++i)                                          // symmetrise (rounding)
    for (int j = 0; j < i; ++j) {
      const double v = 0.5 * (Foo[(size_t)i * s + j] + Foo[(size_t)j * s + i]);
      Foo[(size_t)i * s + j] = Foo[(size_t)j * s + i] = v;
    }
  if (b > 0) {
    std::vector<double> E(Fob, Fob + (size_t)s * b);                   // E = Fob (s x b)
    chol_solve(L.data(), s, Fob, b);                                   // Fm = W E
#pragma omp parallel for schedule(static) if ((double)s * b * b > 1e7)
    for (int p = 0; p < b; ++p) {                                      // Fbb -= E^T Fm
      double *row = Fbb + (size_t)p * b;
      for (int k = 0; k < s; ++k) {
        const double e = E[(size_t)k * b + p];
        if (e == 0.0) continue;
        const double *fm = Fob + (size_t)k * b;
        for (int q = 0; q < b; ++q) row[q] -= e * fm[q];
      }
    }
  }
}

inline int ceil_div(int a, int b) { return (a + b - 1) / b; }

}  // namespace

// =================================================================================================================
// 1. hierarchy
// =================================================================================================================
void build_hierarchy(const BsrView &Q, const Options &opt, Hierarchy &H) {
  if (Q.n < 1 || (Q.dh != 3 && Q.dh != 4)) throw std::runtime_error("nd: bad problem dimensions");
  const Graph g = make_graph(Q);
  Dissector dis(g, opt.leaf_size);
  {
    std::vector<int> all((size_t)Q.n);
    std::iota(all.begin(), all.end(), 0);
    dis.dissect(std::move(all), -1, 0, 0);
  }
  std::vector<NdNode> &T = dis.tree;
  const int nt = (int)T.size();
  int depth = 0;
  for (const NdNode &t : T) depth = std::max(depth, t.level + 1);
  std::vector<int> ndof((size_t)Q.n, -1);
  for (int i = 0; i < nt; ++i)
    for (int p : T[(size_t)i].own) ndof[(size_t)p] = i;
  for (int p = 0; p < Q.n; ++p)
    if (ndof[(size_t)p] < 0) throw std::runtime_error("nd: dissection lost a pose");
  // subtree boundary sets and per-level own counts, children before parents (children have larger indices)
  for (int i = nt - 1; i >= 0; --i) {
    NdNode &t = T[(size_t)i];
    std::vector<int> direct;
    for (int p : t.own)
      for (int q = g.ptr[(size_t)p]; q < g.ptr[(size_t)p + 1]; ++q) {
        const int u = g.adj[(size_t)q];
        if (T[(size_t)ndof[(size_t)u]].level < t.level) direct.push_back(u);     // an ancestor's pose (separator property)
      }
    std::sort(direct.begin(), direct.end());
    direct.erase(std::unique(direct.begin(), direct.end()), direct.end());
    auto keep = [&](int u) { return T[(size_t)ndof[(size_t)u]].level < t.level; };
    std::vector<int> acc = direct;
    for (int c = 0; c < 2; ++c)
      if (t.child[c] >= 0) acc = merge_filter(acc, T[(size_t)t.child[c]].bnd, keep);
    t.bnd = std::move(acc);
    t.cum.assign((size_t)(depth - t.level), 0);
    t.cum[0] = (int)t.own.size();
    for (int c = 0; c < 2; ++c)
      if (t.child[c] >= 0) {
        const NdNode &ch = T[(size_t)t.child[c]];
        for (size_t l = 0; l < ch.cum.size(); ++l) t.cum[l + 1] += ch.cum[l];
      }
  }
  for (NdNode &t : T)                                                   // exact-level counts -> cumulative
    for (size_t l = 1; l < t.cum.size(); ++l) t.cum[l] += t.cum[l - 1];

  // ---- choose the macro levels: enumerate cut sets, cost = phases * t_phase + bytes / bandwidth -----------------
  std::vector<std::vector<int>> at_level((size_t)depth);
  for (int i = 0; i < nt; ++i) at_level[(size_t)T[(size_t)i].level].push_back(i);
  const int dh = Q.dh;
  // cost of one application in microseconds: every phase pays a fixed part (grid barrier + dependent L2 round trips of
  // the gather / job / epilogue stages), a part proportional to the largest input vector a CTA has to stage (every CTA
  // that works on a node gathers the node's whole input: own tiles going up, boundary tiles coming down), and its share
  // of the streamed matrix bytes.  Checked on an H100 SXM (400 W) on sphere2500, the bench workload: the model's choice,
  // 3 macro levels, is the fastest of 1-4 levels (0.545 ms per RTR step against 0.607 with 2 and 0.591 with 4 levels)
  // and stays the choice for t_phase_us 2.0-5.0 and bw_gbs 2000.
  auto eval = [&](const std::vector<int> &cuts, double &bytes_out) {
    double bytes = 0.0, us = 0.0;
    for (size_t k = 0; k < cuts.size(); ++k) {
      const int c0 = cuts[k], c1 = (k + 1 < cuts.size()) ? cuts[k + 1] : depth;
      double stage_bytes_f = 0.0, stage_bytes_b = 0.0;
      int max_own = 0, max_bnd = 0;
      for (int i : at_level[(size_t)c0]) {
        const NdNode &t = T[(size_t)i];
        const int last = std::min<int>((int)t.cum.size() - 1, c1 - 1 - c0);
        const double s = (double)dh * t.cum[(size_t)last], b = (double)dh * t.bnd.size();
        stage_bytes_f += s * (s + b) * 8.0;
        stage_bytes_b += s * b * 8.0;
        max_own = std::max(max_own, t.cum[(size_t)last]);
        max_bnd = std::max(max_bnd, (int)t.bnd.size());
      }
      // leaves of the dissection tree that end above this cut level belong to the fragment of their ancestor: counted there
      bytes += stage_bytes_f + stage_bytes_b;
      us += opt.t_phase_us + opt.t_tile_us * max_own + stage_bytes_f / (opt.bw_gbs * 1e3);
      if (k > 0) us += opt.t_phase_us + opt.t_tile_us * max_bnd + stage_bytes_b / (opt.bw_gbs * 1e3);
    }
    bytes_out = bytes;
    return us;
  };
  struct Cand { std::vector<int> cuts; double cost, bytes; };
  std::vector<Cand> cands;
  {
    std::vector<int> cuts = {0};
    std::function<void(int, int)> rec = [&](int start, int left) {
      if (opt.force_ncuts < 0 || (int)cuts.size() - 1 == opt.force_ncuts) {
        double bytes;
        const double c = eval(cuts, bytes);
        cands.push_back({cuts, c, bytes});
      }
      if (left == 0) return;
      for (int l = start; l < depth; ++l) {
        if (at_level[(size_t)l].empty()) continue;
        cuts.push_back(l);
        rec(l + 1, left - 1);
        cuts.pop_back();
      }
    };
    rec(1, opt.force_ncuts >= 0 ? opt.force_ncuts : opt.max_cuts);
    if (cands.empty()) {                                   // fewer dissection levels than the forced cut count
      double bytes;
      const double c = eval(cuts, bytes);
      cands.push_back({cuts, c, bytes});
    }
  }
  const double byte_cap = 24e9;
  const Cand *bestc = nullptr;
  for (const Cand &c : cands)
    if (c.bytes <= byte_cap && (!bestc || c.cost < bestc->cost)) bestc = &c;
  if (!bestc) throw std::runtime_error("nd: exact preconditioner would need more than 24 GB for this graph");
  const std::vector<int> best_cuts = bestc->cuts;

  // ---- macro nodes -------------------------------------------------------------------------------------------
  H = Hierarchy();
  H.n = Q.n;
  H.dh = dh;
  H.cuts = best_cuts;
  H.nd_depth = depth;
  H.nstages = (int)best_cuts.size();
  std::vector<int> macro_of((size_t)nt, -1);
  for (size_t k = 0; k < best_cuts.size(); ++k) {
    const int c0 = best_cuts[k];
    for (int i : at_level[(size_t)c0]) {
      MacroNode m;
      m.stage = H.nstages - 1 - (int)k;
      macro_of[(size_t)i] = (int)H.nodes.size();
      H.nodes.push_back(std::move(m));
    }
  }
  for (int i = 0; i < nt; ++i) {                                        // parents precede children in T
    if (macro_of[(size_t)i] < 0) macro_of[(size_t)i] = macro_of[(size_t)T[(size_t)i].parent];
  }
  for (int i = 0; i < nt; ++i) {
    const int m = macro_of[(size_t)i];
    MacroNode &mn = H.nodes[(size_t)m];
    const bool is_root_of_fragment = (T[(size_t)i].parent < 0) || (macro_of[(size_t)T[(size_t)i].parent] != m);
    if (is_root_of_fragment) {
      mn.bnd = T[(size_t)i].bnd;
      mn.parent = (T[(size_t)i].parent < 0) ? -1 : macro_of[(size_t)T[(size_t)i].parent];
      if (mn.parent >= 0) H.nodes[(size_t)mn.parent].children.push_back(m);
    }
  }
  // own lists: deeper dissection nodes first inside a fragment (any order is valid for the dense inverse)
  for (int i = nt - 1; i >= 0; --i) {
    MacroNode &mn = H.nodes[(size_t)macro_of[(size_t)i]];
    mn.own.insert(mn.own.end(), T[(size_t)i].own.begin(), T[(size_t)i].own.end());
  }
  H.node_of.assign((size_t)Q.n, -1);
  H.perm.clear();
  H.iperm.assign((size_t)Q.n, -1);
  // permuted order: stage by stage (deepest first), node by node
  int64_t blob = 0;
  int cb = 0;
  std::vector<int> order((size_t)H.nodes.size());
  std::iota(order.begin(), order.end(), 0);
  std::stable_sort(order.begin(), order.end(), [&](int a, int b) { return H.nodes[(size_t)a].stage < H.nodes[(size_t)b].stage; });
  for (int m : order) {
    MacroNode &mn = H.nodes[(size_t)m];
    mn.perm0 = (int)H.perm.size();
    for (int p : mn.own) {
      H.node_of[(size_t)p] = m;
      H.iperm[(size_t)p] = (int)H.perm.size();
      H.perm.push_back(p);
    }
    const int s = dh * (int)mn.own.size(), b = dh * (int)mn.bnd.size();
    const int nfr = (int)mn.own.size() + (int)mn.bnd.size();
    mn.gf_off = blob;
    blob += (int64_t)ceil_div(nfr, 2) * PANEL_ROWS * s;
    mn.gb_off = blob;
    blob += (int64_t)ceil_div((int)mn.own.size(), 2) * PANEL_ROWS * b;
    mn.cbuf0 = cb;
    cb += (int)mn.bnd.size();
  }
  if ((int)H.perm.size() != Q.n) throw std::runtime_error("nd: permutation incomplete");
  // every boundary pose must be owned by a proper ancestor
  for (size_t m = 0; m < H.nodes.size(); ++m)
    for (int p : H.nodes[m].bnd) {
      int a = H.nodes[m].parent;
      const int owner = H.node_of[(size_t)p];
      while (a >= 0 && a != owner) a = H.nodes[(size_t)a].parent;
      if (a < 0) throw std::runtime_error("nd: boundary pose not owned by an ancestor");
    }
  H.cbuf_tiles = std::max(cb, 1);
  H.blob_doubles = blob;
}

// =================================================================================================================
// 2. numeric
// =================================================================================================================
void build_numeric(const BsrView &Q, const Options &opt, Hierarchy &H, std::vector<double> &blob) {
  const int dh = H.dh;
  blob.assign((size_t)H.blob_doubles, 0.0);
  const size_t nn = H.nodes.size();
  std::vector<std::vector<double>> U(nn);            // Schur update of every node on its boundary (b x b), freed by the parent
  std::vector<int> pos((size_t)H.n, -1);             // pose -> position in the current front
  std::vector<int> order(nn);
  std::iota(order.begin(), order.end(), 0);
  std::stable_sort(order.begin(), order.end(), [&](int a, int b) { return H.nodes[(size_t)a].stage < H.nodes[(size_t)b].stage; });
  for (int m : order) {
    MacroNode &mn = H.nodes[(size_t)m];
    const int no = (int)mn.own.size(), nb = (int)mn.bnd.size();
    const int s = dh * no, b = dh * nb;
    for (int k = 0; k < no; ++k) pos[(size_t)mn.own[(size_t)k]] = k;
    for (int k = 0; k < nb; ++k) pos[(size_t)mn.bnd[(size_t)k]] = no + k;
    std::vector<double> Foo((size_t)s * s, 0.0), Fob((size_t)s * std::max(b, 1), 0.0), Fbb((size_t)std::max(b, 1) * std::max(b, 1), 0.0);
    auto add = [&](int fi, int fj, int k, int c, double v) {          // front pose positions fi, fj; scalar offsets k, c
      const int gi = fi * dh + k, gj = fj * dh + c;
      if (fi < no && fj < no) Foo[(size_t)gi * s + gj] += v;
      else if (fi < no) Fob[(size_t)gi * b + (gj - s)] += v;
      // (bnd, own) is the transpose of (own, bnd); (bnd, bnd) belongs to the ancestors' own blocks
    };
    for (int kj = 0; kj < no; ++kj) {
      const int j = mn.own[(size_t)kj];
      for (int bb = Q.rowptr[j]; bb < Q.rowptr[j + 1]; ++bb) {
        const int i = Q.bcol[bb];
        const int owner = H.node_of[(size_t)i];
        int fi = -1;
        if (owner == m) fi = pos[(size_t)i];
        else if (H.nodes[(size_t)owner].stage > mn.stage) fi = pos[(size_t)i];       // an ancestor's pose -> boundary position
        else continue;                                                                  // a descendant's pose: inside a child's update
        if (fi < 0) throw std::runtime_error("nd: pose adjacent to a node is missing from its front");
        const double *blk = Q.bval + (size_t)bb * 16;
        for (int k = 0; k < dh; ++k)
          for (int c = 0; c < dh; ++c) {
            // blk[k][c] = Q[dh i + k, dh j + c]; by symmetry also Q[dh j + c, dh i + k]: fill (own j, front i)
            add(kj, fi, c, k, blk[k * 4 + c]);
          }
      }
    }
    for (int k = 0; k < s; ++k) Foo[(size_t)k * s + k] += opt.shift;
    // children's updates
    for (int c : mn.children) {
      const MacroNode &ch = H.nodes[(size_t)c];
      const int cb = dh * (int)ch.bnd.size();
      const std::vector<double> &Uc = U[(size_t)c];
      for (int p = 0; p < (int)ch.bnd.size(); ++p) {
        const int fp = pos[(size_t)ch.bnd[(size_t)p]];
        for (int q = 0; q < (int)ch.bnd.size(); ++q) {
          const int fq = pos[(size_t)ch.bnd[(size_t)q]];
          for (int k = 0; k < dh; ++k)
            for (int cc = 0; cc < dh; ++cc) {
              const double v = Uc[(size_t)(p * dh + k) * cb + (q * dh + cc)];
              const int gi = fp * dh + k, gj = fq * dh + cc;
              if (fp < no && fq < no) Foo[(size_t)gi * s + gj] += v;
              else if (fp < no) Fob[(size_t)gi * b + (gj - s)] += v;
              else if (fq >= no) Fbb[(size_t)(gi - s) * b + (gj - s)] += v;
            }
        }
      }
      U[(size_t)c].clear();
      U[(size_t)c].shrink_to_fit();
    }
    host_factor(s, b, Foo.data(), Fob.data(), Fbb.data());
    if (b > 0) {
      U[(size_t)m].assign(Fbb.begin(), Fbb.begin() + (size_t)b * b);
    }
    // panels.  forward matrix rows: front poses (own then bnd), cols: own scalars
    {
      double *gf = blob.data() + mn.gf_off;
      const int nfr = no + nb;
      for (int fr = 0; fr < nfr; ++fr) {
        const int panel = fr / 2, half = fr % 2;
        for (int c = 0; c < dh; ++c) {
          const int prow = half * dh + c;
          double *dst = gf + (size_t)panel * PANEL_ROWS * s + prow;
          if (fr < no) {
            const double *src = Foo.data() + (size_t)(fr * dh + c) * s;        // W row
            for (int j = 0; j < s; ++j) dst[(size_t)j * PANEL_ROWS] = src[j];
          } else {
            const int col = (fr - no) * dh + c;                                 // (F^T)[col][j] = Fm[j][col]
            for (int j = 0; j < s; ++j) dst[(size_t)j * PANEL_ROWS] = Fob[(size_t)j * b + col];
          }
        }
      }
      double *gb = blob.data() + mn.gb_off;
      for (int fr = 0; fr < no; ++fr) {
        const int panel = fr / 2, half = fr % 2;
        for (int c = 0; c < dh; ++c) {
          const int prow = half * dh + c;
          double *dst = gb + (size_t)panel * PANEL_ROWS * b + prow;
          const double *src = Fob.data() + (size_t)(fr * dh + c) * b;
          for (int j = 0; j < b; ++j) dst[(size_t)j * PANEL_ROWS] = src[j];
        }
      }
    }
    for (int p : mn.own) pos[(size_t)p] = -1;
    for (int p : mn.bnd) pos[(size_t)p] = -1;
  }
}

void build_refactor(const Hierarchy &H, Refactor &R) {
  const int dh = H.dh;
  const size_t nn = H.nodes.size();
  R = Refactor();
  std::vector<int> order(nn);
  std::iota(order.begin(), order.end(), 0);
  std::stable_sort(order.begin(), order.end(), [&](int a, int b) { return H.nodes[(size_t)a].stage < H.nodes[(size_t)b].stage; });
  std::vector<int> idx(nn);
  for (size_t q = 0; q < nn; ++q) idx[(size_t)order[q]] = (int)q;
  R.stage0.assign((size_t)H.nstages + 1, 0);
  R.max_nfr.assign((size_t)H.nstages, 0);
  R.max_s.assign((size_t)H.nstages, 0);
  R.max_blob.assign((size_t)H.nstages, 0);
  std::vector<int64_t> stage_front((size_t)H.nstages, 0), stage_ws((size_t)H.nstages, 0);
  std::vector<int> where((size_t)H.n, -1);                   // pose -> position in the child's bnd list
  for (int m : order) {
    const MacroNode &mn = H.nodes[(size_t)m];
    const int st = mn.stage, no = (int)mn.own.size(), nb = (int)mn.bnd.size(), nfr = no + nb;
    const int64_t M = (int64_t)dh * nfr, s = (int64_t)dh * no, b = (int64_t)dh * nb;
    RefactorNode rn = {};
    rn.front = stage_front[(size_t)st];
    rn.ws = stage_ws[(size_t)st];
    rn.gf = mn.gf_off;
    rn.gb = mn.gb_off;
    rn.no = no;
    rn.nb = nb;
    rn.pose0 = (int)R.poses.size();
    rn.ch0 = (int)R.child.size();
    rn.nch = (int)mn.children.size();
    R.poses.insert(R.poses.end(), mn.own.begin(), mn.own.end());
    R.poses.insert(R.poses.end(), mn.bnd.begin(), mn.bnd.end());
    for (int c : mn.children) {
      const MacroNode &ch = H.nodes[(size_t)c];
      if (ch.stage != st - 1) throw std::runtime_error("nd: a child two stages below its parent");
      R.child.push_back({idx[(size_t)c], (int)R.cmap.size()});
      for (size_t k = 0; k < ch.bnd.size(); ++k) where[(size_t)ch.bnd[k]] = (int)k;
      for (int q = 0; q < nfr; ++q) R.cmap.push_back(where[(size_t)R.poses[(size_t)rn.pose0 + q]]);
      for (int p : ch.bnd) where[(size_t)p] = -1;
    }
    stage_front[(size_t)st] += M * M;
    stage_ws[(size_t)st] += (int64_t)REFACTOR_PIVOT_BLOCK * (REFACTOR_PIVOT_BLOCK + 2 * M);
    R.max_nfr[(size_t)st] = std::max(R.max_nfr[(size_t)st], nfr);
    R.max_s[(size_t)st] = std::max(R.max_s[(size_t)st], (int)s);
    R.max_blob[(size_t)st] = std::max<int64_t>(R.max_blob[(size_t)st], (int64_t)ceil_div(nfr, 2) * PANEL_ROWS * s +
                                                                         (int64_t)ceil_div(no, 2) * PANEL_ROWS * b);
    R.stage0[(size_t)st + 1]++;
    R.nodes.push_back(rn);
  }
  for (int st = 0; st < H.nstages; ++st) R.stage0[(size_t)st + 1] += R.stage0[(size_t)st];
  int64_t even = 0, odd = 0, ws = 0;
  for (int st = 0; st < H.nstages; ++st) {
    (st % 2 ? odd : even) = std::max(st % 2 ? odd : even, stage_front[(size_t)st]);
    ws = std::max(ws, stage_ws[(size_t)st]);
  }
  for (RefactorNode &rn : R.nodes) {
    const int st = H.nodes[(size_t)order[(size_t)(&rn - R.nodes.data())]].stage;
    if (st % 2) rn.front += even;
  }
  R.arena_even = even;
  R.arena_doubles = std::max<int64_t>(even + odd, 1);
  R.ws_doubles = std::max<int64_t>(ws, 1);
}

void build_selinv(const Hierarchy &H, const Refactor &R, Selinv &S) {
  const size_t nn = R.nodes.size();
  S = Selinv();
  std::vector<int> order(H.nodes.size());
  std::iota(order.begin(), order.end(), 0);
  std::stable_sort(order.begin(), order.end(), [&](int a, int b) { return H.nodes[(size_t)a].stage < H.nodes[(size_t)b].stage; });
  std::vector<int> idx(H.nodes.size());
  for (size_t q = 0; q < nn; ++q) idx[(size_t)order[q]] = (int)q;
  S.macro = order;
  S.parent.assign(nn, -1);
  S.pmap0.assign(nn, 0);
  S.max_b.assign((size_t)H.nstages, 0);
  std::vector<int> where((size_t)H.n, -1);
  for (size_t q = 0; q < nn; ++q) {
    const MacroNode &mn = H.nodes[(size_t)order[q]];
    S.max_b[(size_t)mn.stage] = std::max(S.max_b[(size_t)mn.stage], H.dh * (int)mn.bnd.size());
    S.pmap0[q] = (int)S.pmap.size();
    if (mn.parent < 0) {
      if (!mn.bnd.empty()) throw std::runtime_error("nd: a root node with boundary poses");
      continue;
    }
    const int pq = idx[(size_t)mn.parent];
    S.parent[q] = pq;
    const RefactorNode &pn = R.nodes[(size_t)pq];
    for (int k = 0; k < pn.no + pn.nb; ++k) where[(size_t)R.poses[(size_t)pn.pose0 + k]] = k;
    for (int p : mn.bnd) {
      if (where[(size_t)p] < 0) throw std::runtime_error("nd: boundary pose outside the parent front");
      S.pmap.push_back(where[(size_t)p]);
    }
    for (int k = 0; k < pn.no + pn.nb; ++k) where[(size_t)R.poses[(size_t)pn.pose0 + k]] = -1;
  }
  if (S.pmap.empty()) S.pmap.push_back(0);
}

void emulate_selinv(const Hierarchy &H, const Refactor &R, const Selinv &S, const std::vector<double> &blob,
                    std::vector<std::vector<double>> &front) {
  const int dh = H.dh;
  const size_t nn = R.nodes.size();
  front.assign(nn, {});
  for (size_t qq = nn; qq-- > 0;) {                       // root stage first (R is ordered deepest first)
    const RefactorNode &rn = R.nodes[qq];
    const int64_t s = (int64_t)dh * rn.no, b = (int64_t)dh * rn.nb, M = s + b;
    std::vector<double> &F = front[qq];
    F.assign((size_t)(M * M), 0.0);
    const double *gf = blob.data() + rn.gf, *gb = blob.data() + rn.gb;
    auto W = [&](int64_t r, int64_t j) { return gf[(r / dh / 2) * PANEL_ROWS * s + j * PANEL_ROWS + (r / dh % 2) * dh + r % dh]; };
    auto Fm = [&](int64_t i, int64_t k) { return gb[(i / dh / 2) * PANEL_ROWS * b + k * PANEL_ROWS + (i / dh % 2) * dh + i % dh]; };
    for (int64_t c = 0; c < s; ++c)
      for (int64_t r = 0; r < s; ++r) F[(size_t)(r + M * c)] = W(r, c);
    if (b > 0) {
      const std::vector<double> &Pf = front[(size_t)S.parent[qq]];
      const RefactorNode &pn = R.nodes[(size_t)S.parent[qq]];
      const int64_t Mp = (int64_t)dh * (pn.no + pn.nb);
      const int *pm = S.pmap.data() + S.pmap0[qq];
      for (int64_t c = 0; c < b; ++c)
        for (int64_t r = 0; r < b; ++r) {
          const int64_t pr = pm[r / dh] * dh + r % dh, pc = pm[c / dh] * dh + c % dh;
          F[(size_t)(s + r + M * (s + c))] = pr <= pc ? Pf[(size_t)(pr + Mp * pc)] : Pf[(size_t)(pc + Mp * pr)];
        }
      for (int64_t j = 0; j < b; ++j)                     // Sigma_ob = -Fm Sigma_bb
        for (int64_t i = 0; i < s; ++i) {
          double acc = 0.0;
          for (int64_t k = 0; k < b; ++k) acc = std::fma(Fm(i, k), F[(size_t)(s + k + M * (s + j))], acc);
          F[(size_t)(i + M * (s + j))] = -acc;
        }
      for (int64_t j = 0; j < s; ++j)                     // Sigma_oo = W - Sigma_ob Fm^T (upper triangle)
        for (int64_t i = 0; i <= j; ++i) {
          double acc = 0.0;
          for (int64_t k = 0; k < b; ++k) acc = std::fma(F[(size_t)(i + M * (s + k))], Fm(j, k), acc);
          F[(size_t)(i + M * j)] -= acc;
        }
    }
  }
}

// =================================================================================================================
// 3. plan
// =================================================================================================================
namespace {

struct Run { int node; int p0, p1; double cost; };
// cost of one panel besides its streamed columns, in column units: two epilogue items (record, slot sums, projection,
// stores: ~1000 cycles each on one of 16 warps) against ~2-3 cycles per streamed 64-byte column
constexpr double PANEL_FIXED_COST = 48.0;

struct PhaseBuilder {
  const Hierarchy &H;
  const Options &opt;
  Plan &P;
  int dir, stage;
  // contribution lists per (parent node, front pose position): built lazily per node
  std::vector<std::vector<std::vector<int>>> contrib;   // [node][front pose] -> cbuf tile ids

  PhaseBuilder(const Hierarchy &h, const Options &o, Plan &p) : H(h), opt(o), P(p), dir(0), stage(0), contrib(h.nodes.size()) {}

  const std::vector<std::vector<int>> &contributions(int m) {
    auto &cl = contrib[(size_t)m];
    const MacroNode &mn = H.nodes[(size_t)m];
    const size_t nfr = mn.own.size() + mn.bnd.size();
    if (cl.size() == nfr) return cl;
    cl.assign(nfr, {});
    std::vector<std::pair<int, int>> where;             // pose -> front position (sorted by pose)
    where.reserve(nfr);
    for (size_t k = 0; k < mn.own.size(); ++k) where.push_back({mn.own[k], (int)k});
    for (size_t k = 0; k < mn.bnd.size(); ++k) where.push_back({mn.bnd[k], (int)(mn.own.size() + k)});
    std::sort(where.begin(), where.end());
    for (int c : mn.children) {
      const MacroNode &ch = H.nodes[(size_t)c];
      for (size_t kb = 0; kb < ch.bnd.size(); ++kb) {
        auto it = std::lower_bound(where.begin(), where.end(), std::make_pair(ch.bnd[kb], -1));
        if (it == where.end() || it->first != ch.bnd[kb]) throw std::runtime_error("nd: child boundary outside the parent front");
        cl[(size_t)it->second].push_back(ch.cbuf0 + (int)kb);
      }
    }
    return cl;
  }

  // contribution list -> (count, inline ids, pointer to the remaining ids in csrc)
  void set_contrib(const std::vector<int> &v, int &nc, int &cext, int *ci) {
    nc = (int)v.size();
    cext = (int)P.csrc.size();
    for (int q = 0; q < INLINE_CONTRIB; ++q) ci[q] = (q < nc) ? v[(size_t)q] : 0;
    for (int q = INLINE_CONTRIB; q < nc; ++q) P.csrc.push_back(v[(size_t)q]);
  }

  void build() {
    const int G = opt.grid, dh = H.dh;
    // matrices of this phase
    std::vector<int> nodes;
    for (size_t m = 0; m < H.nodes.size(); ++m)
      if (H.nodes[m].stage == stage) nodes.push_back((int)m);
    auto rows_of = [&](const MacroNode &mn) { return dir == 0 ? (int)(mn.own.size() + mn.bnd.size()) : (int)mn.own.size(); };   // front poses
    auto cols_of = [&](const MacroNode &mn) { return dir == 0 ? (int)mn.own.size() : (int)mn.bnd.size(); };                      // tiles
    double total = 0.0;
    for (int m : nodes) {
      const MacroNode &mn = H.nodes[(size_t)m];
      total += (double)ceil_div(rows_of(mn), 2) * (cols_of(mn) * dh + PANEL_FIXED_COST);
    }
    const double target = std::max(total / G, 1.0);
    std::vector<Run> runs;
    for (int m : nodes) {
      const MacroNode &mn = H.nodes[(size_t)m];
      const int np = ceil_div(rows_of(mn), 2);
      const double pc = cols_of(mn) * dh + PANEL_FIXED_COST;   // cost of one panel: streamed columns + its two epilogues
      const double cost = np * pc;
      int k = (int)std::floor(cost / target + 0.5);
      k = std::max(1, std::min(k, np));
      for (int q = 0; q < k; ++q) {
        const int p0 = (int)((int64_t)np * q / k), p1 = (int)((int64_t)np * (q + 1) / k);
        if (p1 > p0) runs.push_back({m, p0, p1, (p1 - p0) * pc});
      }
    }
    // longest-processing-time assignment
    std::vector<int> ridx(runs.size());
    std::iota(ridx.begin(), ridx.end(), 0);
    std::stable_sort(ridx.begin(), ridx.end(), [&](int a, int b) { return runs[(size_t)a].cost > runs[(size_t)b].cost; });
    std::vector<double> load((size_t)G, 0.0);
    std::vector<std::vector<int>> mine((size_t)G);
    for (int ri : ridx) {
      int bestc = 0;
      for (int c = 1; c < G; ++c)
        if (load[(size_t)c] < load[(size_t)bestc]) bestc = c;
      load[(size_t)bestc] += runs[(size_t)ri].cost;
      mine[(size_t)bestc].push_back(ri);
    }
    P.phases.push_back({dir, stage, (int)P.cta_phase.size(), 0});
    for (int c = 0; c < G; ++c) {
      const int s0 = (int)P.steps.size();
      std::sort(mine[(size_t)c].begin(), mine[(size_t)c].end());
      emit_cta(mine[(size_t)c], runs);
      const int s1 = (int)P.steps.size();
      CtaPhase cp = {s0, s1, 0, 0, 0, 0, 0, 0};
      if (s1 > s0) {
        const Step &st = P.steps[(size_t)s0];
        cp.g0 = st.g0; cp.g1 = st.g1; cp.j0 = st.j0; cp.j1 = st.j1; cp.e0 = st.e0; cp.e1 = st.e1;
      }
      P.cta_phase.push_back(cp);
    }
  }

  // one CTA: group its runs into steps
  void emit_cta(const std::vector<int> &my, const std::vector<Run> &runs) {
    const int dh = H.dh;
    const int ycap = opt.ycap_tiles, scap = opt.slot_cap;
    auto cols_of = [&](const MacroNode &mn) { return dir == 0 ? (int)mn.own.size() : (int)mn.bnd.size(); };
    // split runs that exceed the slot capacity
    std::vector<Run> work;
    for (int ri : my) {
      Run r = runs[(size_t)ri];
      while (r.p1 - r.p0 > scap) {
        work.push_back({r.node, r.p0, r.p0 + scap, 0.0});
        r.p0 += scap;
      }
      work.push_back(r);
    }
    size_t i = 0;
    while (i < work.size()) {
      const MacroNode &mn0 = H.nodes[(size_t)work[i].node];
      const int ct0 = cols_of(mn0);
      if (ct0 > ycap) {
        // column-chunked run: dedicated steps, partial sums carried in the slots
        const Run &r = work[i];
        const int np = r.p1 - r.p0;
        const int nchunks = ceil_div(ct0, ycap);
        const int pieces = pieces_for(np, std::min(ct0, ycap) * dh);
        for (int ch = 0; ch < nchunks; ++ch) {
          const int t0 = ch * ycap, t1 = std::min(ct0, t0 + ycap);
          Step st = {};
          st.g0 = (int)P.gathers.size();
          emit_gathers(r.node, t0, t1, 0);
          st.g1 = (int)P.gathers.size();
          st.j0 = (int)P.jobs.size();
          emit_jobs(r, t0, t1, 0, 0, pieces, ch > 0);
          st.j1 = (int)P.jobs.size();
          st.e0 = (int)P.epis.size();
          if (ch == nchunks - 1) emit_epis(r, 0, pieces);
          st.e1 = (int)P.epis.size();
          P.steps.push_back(st);
          P.max_ytiles = std::max(P.max_ytiles, t1 - t0);
          P.max_slots = std::max(P.max_slots, np * pieces);
        }
        ++i;
        continue;
      }
      // greedy merge of whole-width runs
      size_t j = i;
      int ytiles = 0, panels = 0;
      std::vector<std::pair<int, int>> ybase;             // (node, first smem tile)
      while (j < work.size()) {
        const MacroNode &mn = H.nodes[(size_t)work[j].node];
        const int ct = cols_of(mn);
        if (ct > ycap) break;
        bool have = false;
        for (auto &yb : ybase) have = have || (yb.first == work[j].node);
        const int addt = have ? 0 : ct;
        const int addp = work[j].p1 - work[j].p0;
        if (j > i && (ytiles + addt > ycap || panels + addp > scap)) break;
        if (!have) { ybase.push_back({work[j].node, ytiles}); ytiles += ct; }
        panels += addp;
        ++j;
      }
      int maxcols = 0;
      for (size_t q = i; q < j; ++q) maxcols = std::max(maxcols, cols_of(H.nodes[(size_t)work[q].node]) * dh);
      int pieces = pieces_for(panels, maxcols);
      pieces = std::max(1, std::min(pieces, scap / std::max(panels, 1)));
      Step st = {};
      st.g0 = (int)P.gathers.size();
      for (auto &yb : ybase) emit_gathers(yb.first, 0, cols_of(H.nodes[(size_t)yb.first]), yb.second);
      st.g1 = (int)P.gathers.size();
      st.j0 = (int)P.jobs.size();
      std::vector<int> slot0s;
      int slot = 0;
      for (size_t q = i; q < j; ++q) {
        int yb0 = 0;
        for (auto &yb : ybase) if (yb.first == work[q].node) yb0 = yb.second;
        const int ct = cols_of(H.nodes[(size_t)work[q].node]);
        const int pc = std::max(1, std::min(pieces, std::max(1, ct * dh / 32)));
        slot0s.push_back(slot);
        emit_jobs(work[q], 0, ct, yb0, slot, pc, false);
        slot += (work[q].p1 - work[q].p0) * pc;
      }
      st.j1 = (int)P.jobs.size();
      st.e0 = (int)P.epis.size();
      for (size_t q = i; q < j; ++q) {
        const int ct = cols_of(H.nodes[(size_t)work[q].node]);
        const int pc = std::max(1, std::min(pieces, std::max(1, ct * dh / 32)));
        emit_epis(work[q], slot0s[q - i], pc);
      }
      st.e1 = (int)P.epis.size();
      P.steps.push_back(st);
      P.max_ytiles = std::max(P.max_ytiles, ytiles);
      P.max_slots = std::max(P.max_slots, slot);
      i = j;
    }
  }

  // column pieces per panel: about one job per warp (a job has a fixed cost of a few hundred issue slots), none
  // shorter than 32 columns (one full round of the DMMA loop)
  int pieces_for(int panels, int ncols) const {
    const int want = opt.warps;
    int pieces = std::max(1, want / std::max(panels, 1));
    pieces = std::min(pieces, std::max(1, ncols / 32));
    pieces = std::min(pieces, std::max(1, opt.slot_cap / std::max(panels, 1)));
    return pieces;
  }

  // tiles [t0, t1) of the node's input vector -> smem tiles ybase + (t - t0)
  void emit_gathers(int m, int t0, int t1, int ybase) {
    const MacroNode &mn = H.nodes[(size_t)m];
    for (int t = t0; t < t1; ++t) {
      Gather g = {};
      g.ytile = ybase + (t - t0);
      if (dir == 0) {
        g.src = mn.own[(size_t)t];                                    // pose id: source = V
        set_contrib(contributions(m)[(size_t)t], g.nc, g.cext, g.ci);
      } else {
        g.src = H.iperm[(size_t)mn.bnd[(size_t)t]];                   // permuted tile: source = TX (solution of the ancestors)
      }
      P.gathers.push_back(g);
    }
  }

  void emit_jobs(const Run &r, int t0, int t1, int ybase, int slot_base, int pieces, bool accum) {
    const MacroNode &mn = H.nodes[(size_t)r.node];
    const int dh = H.dh;
    const int ncols_total = (dir == 0 ? (int)mn.own.size() : (int)mn.bnd.size()) * dh;
    const int64_t mat0 = (dir == 0) ? mn.gf_off : mn.gb_off;
    const int c0 = t0 * dh, c1 = t1 * dh;
    for (int p = r.p0; p < r.p1; ++p)
      for (int q = 0; q < pieces; ++q) {
        int a = c0 + (int)((int64_t)(c1 - c0) * q / pieces), b = c0 + (int)((int64_t)(c1 - c0) * (q + 1) / pieces);
        a = c0 + ((a - c0) & ~3);
        if (q + 1 < pieces) b = c0 + ((b - c0) & ~3);
        Job jb = {};
        jb.mat = mat0 + ((int64_t)p * ncols_total + a) * PANEL_ROWS;
        jb.ncols = std::max(0, b - a);
        jb.ycol = ybase * dh + (a - c0);
        jb.slot = slot_base + (p - r.p0) * pieces + q;
        jb.accum = accum ? 1 : 0;
        P.jobs.push_back(jb);
        P.bytes_per_apply += (int64_t)jb.ncols * PANEL_ROWS * 8;
      }
  }

  void emit_epis(const Run &r, int slot_base, int pieces) {
    const MacroNode &mn = H.nodes[(size_t)r.node];
    const int no = (int)mn.own.size(), nb = (int)mn.bnd.size();
    const int nfr = (dir == 0) ? no + nb : no;
    const bool root = (mn.parent < 0);
    const bool has_cols = (dir == 0) ? true : (nb > 0);
    for (int p = r.p0; p < r.p1; ++p)
      for (int half = 0; half < 2; ++half) {
        const int fr = 2 * p + half;
        if (fr >= nfr) continue;
        Epi e = {};
        e.slot0 = slot_base + (p - r.p0) * pieces;
        e.nslots = has_cols ? pieces : 0;
        e.half = half;
        if (dir == 0) {
          if (fr < no) {
            e.kind = root ? EPI_ROOT : EPI_F_OWN;
            e.out = mn.perm0 + fr;
            e.aux = mn.own[(size_t)fr];
          } else {
            e.kind = EPI_F_BND;
            e.out = mn.cbuf0 + (fr - no);
            e.aux = -1;
            set_contrib(contributions(r.node)[(size_t)fr], e.nc, e.cext, e.ci);
          }
        } else {
          e.kind = EPI_B_OWN;
          e.out = mn.perm0 + fr;
          e.aux = mn.own[(size_t)fr];
        }
        P.epis.push_back(e);
      }
  }
};

}  // namespace

void build_plan(const Hierarchy &H, const Options &opt, Plan &P) {
  P = Plan();
  P.grid = opt.grid;
  P.r = opt.r;
  PhaseBuilder pb(H, opt, P);
  for (int st = 0; st < H.nstages; ++st) {
    pb.dir = 0;
    pb.stage = st;
    pb.build();
  }
  for (int st = H.nstages - 2; st >= 0; --st) {
    pb.dir = 1;
    pb.stage = st;
    pb.build();
  }
}

// A step's phase time is set by its slowest warp, and a round of the job loop that streams from L2 costs an L2 round
// trip where a resident round costs a shared-memory one.  So residency is handed out in rounds, per (CTA, phase): a level
// L caps the rounds every warp of every step of the phase streams, the first rounds of a warp's job sequence are the
// resident ones.  Lowering a phase's level by one saves one L2 round trip in each step that reaches it; the CTA's budget
// goes, one level at a time, to the phase where that saving costs the fewest bytes.
void assign_residency(Plan &P, int warps, int64_t budget_bytes) {
  const int G = P.grid;
  for (Job &j : P.jobs) { j.soff = 0; j.nres = 0; }
  P.resident_doubles.assign((size_t)G, 0);
  P.max_resident_doubles = 0;
  P.resident_bytes = 0;
  const int64_t budget = std::max<int64_t>(0, budget_bytes / 8);
  const int nph = (int)P.phases.size();
  auto nrounds = [](int ncols) { return (ncols + RES_ROUND - 1) / RES_ROUND; };
  for (int c = 0; c < G; ++c) {
    // per phase: the rounds (shared-memory doubles of each, in order) of every (step, warp), and the step of each
    std::vector<std::vector<std::vector<int>>> seq((size_t)nph);
    std::vector<std::vector<int>> seq_step((size_t)nph);
    std::vector<int> level((size_t)nph, 0);
    for (int ph = 0; ph < nph; ++ph) {
      const CtaPhase &cp = P.cta_phase[(size_t)P.phases[(size_t)ph].cta0 + c];
      for (int si = cp.s0; si < cp.s1; ++si) {
        const Step &st = P.steps[(size_t)si];
        for (int w = 0; w < warps && st.j0 + w < st.j1; ++w) {
          std::vector<int> rd;
          for (int ji = st.j0 + w; ji < st.j1; ji += warps) {
            const int nc = P.jobs[(size_t)ji].ncols;
            for (int k = 0; k < nrounds(nc); ++k)
              rd.push_back(resident_doubles(std::min(nc, (k + 1) * RES_ROUND)) - resident_doubles(k * RES_ROUND));
          }
          level[(size_t)ph] = std::max(level[(size_t)ph], (int)rd.size());
          seq[(size_t)ph].push_back(std::move(rd));
          seq_step[(size_t)ph].push_back(si);
        }
      }
    }
    int64_t used = 0;
    while (true) {
      int best = -1;
      int64_t best_cost = 0;
      double best_score = 0.0;
      for (int ph = 0; ph < nph; ++ph) {
        const int L = level[(size_t)ph];
        if (L == 0) continue;
        int64_t cost = 0;
        std::vector<int> steps_hit;
        for (size_t q = 0; q < seq[(size_t)ph].size(); ++q) {
          const std::vector<int> &rd = seq[(size_t)ph][q];
          if ((int)rd.size() < L) continue;
          cost += rd[rd.size() - (size_t)L];
          steps_hit.push_back(seq_step[(size_t)ph][q]);
        }
        if (used + cost > budget) continue;
        std::sort(steps_hit.begin(), steps_hit.end());
        const double saved = (double)(std::unique(steps_hit.begin(), steps_hit.end()) - steps_hit.begin());
        const double score = (double)cost / saved;
        if (best < 0 || score < best_score) { best = ph; best_cost = cost; best_score = score; }
      }
      if (best < 0) break;
      --level[(size_t)best];
      used += best_cost;
    }
    // the region: the resident rounds of every (phase, step, warp) in job order, one after the other
    int off = 0;
    for (int ph = 0; ph < nph; ++ph) {
      const CtaPhase &cp = P.cta_phase[(size_t)P.phases[(size_t)ph].cta0 + c];
      for (int si = cp.s0; si < cp.s1; ++si) {
        const Step &st = P.steps[(size_t)si];
        for (int w = 0; w < warps && st.j0 + w < st.j1; ++w) {
          int total = 0;
          for (int ji = st.j0 + w; ji < st.j1; ji += warps) total += nrounds(P.jobs[(size_t)ji].ncols);
          int left = std::max(0, total - level[(size_t)ph]);
          for (int ji = st.j0 + w; ji < st.j1 && left > 0; ji += warps) {
            Job &jb = P.jobs[(size_t)ji];
            const int take = std::min(left, nrounds(jb.ncols));
            left -= take;
            jb.nres = std::min(jb.ncols, take * RES_ROUND);
            jb.soff = off;
            off += resident_doubles(jb.nres);
            P.resident_bytes += (int64_t)jb.nres * PANEL_ROWS * 8;
          }
        }
      }
    }
    if (off > budget) throw std::runtime_error("nd: resident region exceeds its budget");
    P.resident_doubles[(size_t)c] = off;
    P.max_resident_doubles = std::max(P.max_resident_doubles, off);
  }
}

// =================================================================================================================
// host emulation of the plan (verification only)
// =================================================================================================================
static void emulate_pass(const Hierarchy &H, const Plan &P, const std::vector<double> &blob, int r, const double *V, double *Z,
                         std::vector<std::vector<double>> &region, bool fill);

void emulate_apply(const Hierarchy &H, const Plan &P, const std::vector<double> &blob, int r, const double *V, double *Z) {
  const bool resident = P.resident_bytes > 0;
  std::vector<std::vector<double>> region((size_t)P.grid);
  for (int c = 0; c < P.grid && resident; ++c) region[(size_t)c].assign((size_t)P.resident_doubles[(size_t)c], std::nan(""));
  std::vector<double> Zfill;
  if (resident) Zfill.assign((size_t)r * H.dh * H.n, 0.0);
  for (int pass = resident ? 0 : 1; pass < 2; ++pass)
    emulate_pass(H, P, blob, r, V, pass == 0 ? Zfill.data() : Z, region, resident && pass == 0);
}

// one application; fill: resident columns are read from the panels and copied to the region, else read from the region
static void emulate_pass(const Hierarchy &H, const Plan &P, const std::vector<double> &blob, int r, const double *V, double *Z,
                         std::vector<std::vector<double>> &region, bool fill) {
  const int dh = H.dh, ts = r * dh;
  std::vector<double> TX((size_t)H.n * ts, 0.0), C((size_t)H.cbuf_tiles * ts, 0.0);
  std::vector<double> ys((size_t)std::max(P.max_ytiles, 1) * ts), slots((size_t)std::max(P.max_slots, 1) * PANEL_ROWS * r);
  for (size_t ph = 0; ph < P.phases.size(); ++ph) {
    const Phase &phs = P.phases[ph];
    for (int c = 0; c < P.grid; ++c) {
      const CtaPhase &cph = P.cta_phase[(size_t)phs.cta0 + c];
      const int s0 = cph.s0, s1 = cph.s1;
      if (s1 > s0) {                                                    // the inline copy of the first step must agree
        const Step &f = P.steps[(size_t)s0];
        if (f.g0 != cph.g0 || f.g1 != cph.g1 || f.j0 != cph.j0 || f.j1 != cph.j1 || f.e0 != cph.e0 || f.e1 != cph.e1)
          throw std::runtime_error("nd: inline first step disagrees with the step table");
      }
      std::fill(slots.begin(), slots.end(), std::nan(""));            // a slot must be written before it is read
      for (int si = s0; si < s1; ++si) {
        const Step &st = P.steps[(size_t)si];
        std::fill(ys.begin(), ys.end(), std::nan(""));
        for (int gi = st.g0; gi < st.g1; ++gi) {
          const Gather &g = P.gathers[(size_t)gi];
          for (int e = 0; e < ts; ++e) {
            double v = (phs.dir == 0) ? V[(size_t)g.src * ts + e] : TX[(size_t)g.src * ts + e];
            for (int k = 0; k < g.nc; ++k) {
              const int ct = (k < INLINE_CONTRIB) ? g.ci[k] : P.csrc[(size_t)(g.cext + k - INLINE_CONTRIB)];
              v -= C[(size_t)ct * ts + e];
            }
            ys[(size_t)g.ytile * ts + e] = v;
          }
        }
        for (int ji = st.j0; ji < st.j1; ++ji) {
          const Job &jb = P.jobs[(size_t)ji];
          const double *mat = blob.data() + jb.mat;
          double *sl = slots.data() + (size_t)jb.slot * PANEL_ROWS * r;
          // column j of a resident piece: group j / 4, lane 4 row + j % 4 (dpgo_kernels.cu phase_nd)
          auto rslot = [&](int j, int row) -> double & {
            return region[(size_t)c].at((size_t)jb.soff + (size_t)(j / 4) * 32 + (size_t)(row * 4 + (j & 3)));
          };
          if (fill)
            for (int j = 0; j < jb.nres; ++j)
              for (int row = 0; row < PANEL_ROWS; ++row) rslot(j, row) = mat[(size_t)j * PANEL_ROWS + row];
          for (int row = 0; row < PANEL_ROWS; ++row)
            for (int a = 0; a < r; ++a) {
              double acc = 0.0;
              for (int j = 0; j < jb.ncols; ++j) {
                const double m = (j < jb.nres && !fill) ? rslot(j, row) : mat[(size_t)j * PANEL_ROWS + row];
                acc += m * ys[(size_t)(jb.ycol + j) * r + a];
              }
              if (jb.accum) sl[row * r + a] += acc; else sl[row * r + a] = acc;
            }
        }
        for (int ei = st.e0; ei < st.e1; ++ei) {
          const Epi &ep = P.epis[(size_t)ei];
          for (int cc = 0; cc < dh; ++cc)
            for (int a = 0; a < r; ++a) {
              const int e = cc * r + a, row = ep.half * dh + cc;
              double sum = 0.0;
              for (int k = 0; k < ep.nslots; ++k) sum += slots[(size_t)(ep.slot0 + k) * PANEL_ROWS * r + row * r + a];
              if (ep.kind == EPI_F_OWN) {
                TX[(size_t)ep.out * ts + e] = sum;
              } else if (ep.kind == EPI_F_BND) {
                for (int k = 0; k < ep.nc; ++k) {
                  const int ct = (k < INLINE_CONTRIB) ? ep.ci[k] : P.csrc[(size_t)(ep.cext + k - INLINE_CONTRIB)];
                  sum += C[(size_t)ct * ts + e];
                }
                C[(size_t)ep.out * ts + e] = sum;
              } else if (ep.kind == EPI_ROOT) {
                TX[(size_t)ep.out * ts + e] = sum;
                Z[(size_t)ep.aux * ts + e] = sum;
              } else {
                const double x = TX[(size_t)ep.out * ts + e] - sum;
                TX[(size_t)ep.out * ts + e] = x;
                Z[(size_t)ep.aux * ts + e] = x;
              }
            }
        }
      }
    }
  }
}

std::string describe(const Hierarchy &H, const Plan &P) {
  std::ostringstream os;
  os << "nd: n=" << H.n << " depth=" << H.nd_depth << " cuts=[";
  for (size_t k = 0; k < H.cuts.size(); ++k) os << (k ? "," : "") << H.cuts[k];
  os << "] stages=" << H.nstages << " nodes=" << H.nodes.size() << " blob=" << (H.blob_doubles * 8) / 1e6 << "MB phases=" << P.phases.size()
     << " bytes/apply=" << P.bytes_per_apply / 1e6 << "MB steps=" << P.steps.size() << " jobs=" << P.jobs.size() << " epis=" << P.epis.size()
     << " max_ytiles=" << P.max_ytiles << " max_slots=" << P.max_slots
     << " resident=" << (P.bytes_per_apply > 0 ? (double)P.resident_bytes / (double)P.bytes_per_apply : 0.0)
     << " max_resident_KB=" << P.max_resident_doubles * 8 / 1024.0;
  for (int st = 0; st < H.nstages; ++st) {
    int cnt = 0, smax = 0, bmax = 0;
    for (const MacroNode &m : H.nodes)
      if (m.stage == st) { ++cnt; smax = std::max(smax, (int)m.own.size()); bmax = std::max(bmax, (int)m.bnd.size()); }
    os << " | stage " << st << ": " << cnt << " nodes, own<=" << smax << " bnd<=" << bmax;
  }
  return os.str();
}

}  // namespace nd
}  // namespace dpgo
