// dpgo_capi_covariance.cu -- pose marginal covariances (dpgo_pose_covariances) and their host emulation: the host
// builds the information matrix's block pattern, the nested-dissection hierarchy over it and the list of requested 3 x 3
// blocks once; the values, the factorisation and the selected inversion run on the device (dpgo_covariance.cu,
// nd_refactor.cu).
#include <cuda_runtime.h>

#include <algorithm>
#include <cmath>
#include <memory>
#include <numeric>
#include <string>
#include <vector>

#include "dpgo_covariance.cuh"
#include "dpgo_handle.cuh"

namespace dpgo::capi {
namespace {

namespace nd = dpgo::nd;
constexpr int CDH = 3;

struct CovProblem {
  int n, d, b, ne, anchor;
  int64_t m;
  const int32_t *p1, *p2, *pairs;
  const double *R, *t, *kappa, *tau, *weight, *T;
  int64_t num_pairs;
};

// Everything the host decides once: pattern + contributions, hierarchy, selected-inversion maps, output items.
struct CovSetup {
  std::vector<int> rowptr, bcol, cptr;
  std::vector<int2> contrib, bnode;
  nd::Hierarchy H;
  nd::Refactor R;
  nd::Selinv S;
  std::vector<CovItem> items;        // stage by stage (item0)
  std::vector<int> item0;
};

int check_args(const CovProblem &P, const double *cov) {
  DPGO_REQUIRE(P.n >= 1 && (P.d == 2 || P.d == 3) && P.m >= 0 && P.num_pairs >= 0, DPGO_ERR_INVALID_ARG, "pose_covariances: bad dimensions");
  DPGO_REQUIRE(P.T && cov && (P.m == 0 || (P.p1 && P.p2 && P.R && P.t && P.kappa && P.tau)), DPGO_ERR_INVALID_ARG,
               "pose_covariances: null argument");
  DPGO_REQUIRE(P.anchor >= 0 && P.anchor < P.n, DPGO_ERR_INVALID_ARG, "pose_covariances: anchor pose out of range");
  DPGO_REQUIRE(P.num_pairs == 0 || P.pairs, DPGO_ERR_INVALID_ARG, "pose_covariances: null pair list");
  for (int64_t e = 0; e < P.m; ++e) {
    DPGO_REQUIRE(P.p1[e] >= 0 && P.p1[e] < P.n && P.p2[e] >= 0 && P.p2[e] < P.n, DPGO_ERR_INVALID_ARG,
                 "pose_covariances: edge endpoint out of range");
    DPGO_REQUIRE(P.p1[e] != P.p2[e], DPGO_ERR_INVALID_ARG, "pose_covariances: an edge joins a pose to itself");
    const double w = P.weight ? P.weight[e] : 1.0;
    DPGO_REQUIRE(std::isfinite(P.kappa[e]) && std::isfinite(P.tau[e]) && std::isfinite(w) && P.kappa[e] >= 0 && P.tau[e] >= 0 && w >= 0,
                 DPGO_ERR_INVALID_ARG, "pose_covariances: kappa, tau and weight must be finite and non-negative");
  }
  for (int64_t q = 0; q < 2 * P.num_pairs; ++q)
    DPGO_REQUIRE(P.pairs[q] >= 0 && P.pairs[q] < P.n, DPGO_ERR_INVALID_ARG, "pose_covariances: pair pose out of range");
  for (int64_t q = 0; q < (int64_t)P.d * (P.d + 1) * P.n; ++q)
    DPGO_REQUIRE(std::isfinite(P.T[q]), DPGO_ERR_INVALID_ARG, "pose_covariances: the trajectory is not finite");
  // every pose reaches the anchor through edges of positive weight (else H restricted to the free poses is singular)
  std::vector<int> up((size_t)P.n);
  std::iota(up.begin(), up.end(), 0);
  auto find = [&](int x) { while (up[(size_t)x] != x) x = up[(size_t)x] = up[(size_t)up[(size_t)x]]; return x; };
  for (int64_t e = 0; e < P.m; ++e)
    if ((P.weight ? P.weight[e] : 1.0) > 0 && (P.kappa[e] > 0 || P.tau[e] > 0)) up[(size_t)find(P.p1[e])] = find(P.p2[e]);
  const int root = find(P.anchor);
  for (int p = 0; p < P.n; ++p)
    DPGO_REQUIRE(find(p) == root, DPGO_ERR_INVALID_ARG,
                 "pose_covariances: pose " + std::to_string(p) + " is not connected to the anchor pose by an edge of positive weight");
  return DPGO_OK;
}

int setup(const CovProblem &P, nd::Options opt, CovSetup &C) {
  const int sub = P.d == 3 ? 2 : 1;           // nodes per pose
  // pose blocks (a, c) with their contributions {edge, role of a | role of c << 1}, in edge order; the anchor is decoupled;
  // requested pairs are structural blocks, so that both poses of a pair share a front of the dissection
  struct Pc { int a, c, e, code; };
  std::vector<Pc> pc;
  pc.reserve((size_t)(4 * P.m + 2 * P.num_pairs + P.n));
  for (int p = 0; p < P.n; ++p) pc.push_back({p, p, -1, 0});
  for (int64_t e = 0; e < P.m; ++e) {
    const int i = P.p1[e], j = P.p2[e];
    if (i != P.anchor) pc.push_back({i, i, (int)e, 0});
    if (j != P.anchor) pc.push_back({j, j, (int)e, 3});
    if (i != P.anchor && j != P.anchor) { pc.push_back({i, j, (int)e, 2}); pc.push_back({j, i, (int)e, 1}); }
  }
  for (int64_t q = 0; q < P.num_pairs; ++q) {
    const int i = P.pairs[2 * q], j = P.pairs[2 * q + 1];
    if (i != j && i != P.anchor && j != P.anchor) { pc.push_back({i, j, -1, 0}); pc.push_back({j, i, -1, 0}); }
  }
  std::stable_sort(pc.begin(), pc.end(), [](const Pc &x, const Pc &y) { return x.c != y.c ? x.c < y.c : x.a < y.a; });
  // block-CSR over nodes: row node jn = sub c + sc, column nodes in = sub a + sa in increasing order
  C.rowptr.assign((size_t)P.ne + 1, 0);
  C.bcol.clear(); C.cptr.assign(1, 0); C.contrib.clear(); C.bnode.clear();
  size_t g0 = 0;
  for (int c = 0; c < P.n; ++c) {
    size_t g1 = g0;
    while (g1 < pc.size() && pc[g1].c == c) ++g1;
    for (int sc = 0; sc < sub; ++sc) {
      const int jn = sub * c + sc;
      for (size_t u = g0; u < g1;) {
        size_t v = u;
        while (v < g1 && pc[v].a == pc[u].a) ++v;
        for (int sa = 0; sa < sub; ++sa) {
          const int in = sub * pc[u].a + sa;
          C.bcol.push_back(in);
          C.bnode.push_back(make_int2(in, jn));
          for (size_t w = u; w < v; ++w)
            if (pc[w].e >= 0) C.contrib.push_back(make_int2(pc[w].e, pc[w].code));
          C.cptr.push_back((int)C.contrib.size());
        }
        u = v;
      }
      C.rowptr[(size_t)jn + 1] = (int)C.bcol.size();
    }
    g0 = g1;
  }
  if (C.contrib.empty()) C.contrib.push_back(make_int2(0, 0));
  try {
    std::vector<double> zeros(C.bcol.size() * 16, 0.0);
    nd::BsrView Q{P.ne, CDH, C.rowptr.data(), C.bcol.data(), zeros.data()};
    nd::build_hierarchy(Q, opt, C.H);
    nd::build_refactor(C.H, C.R);
    nd::build_selinv(C.H, C.R, C.S);
  } catch (const std::exception &e) {
    return fail(DPGO_ERR_UNSUPPORTED, std::string("pose_covariances: ") + e.what());
  }
  if (C.R.child.empty()) C.R.child.push_back({0, 0});
  if (C.R.cmap.empty()) C.R.cmap.push_back(-1);
  // front position of every node inside each refactor node's front, looked up by binary search
  const size_t nn = C.R.nodes.size();
  std::vector<int> ridx(C.H.nodes.size());
  for (size_t q = 0; q < nn; ++q) ridx[(size_t)C.S.macro[q]] = (int)q;
  std::vector<std::vector<std::pair<int, int>>> fpos(nn);
  for (size_t q = 0; q < nn; ++q) {
    const nd::RefactorNode &rn = C.R.nodes[q];
    for (int k = 0; k < rn.no + rn.nb; ++k) fpos[q].push_back({C.R.poses[(size_t)rn.pose0 + k], k});
    std::sort(fpos[q].begin(), fpos[q].end());
  }
  auto pos_in = [&](int q, int x) {
    auto it = std::lower_bound(fpos[(size_t)q].begin(), fpos[(size_t)q].end(), std::make_pair(x, -1));
    return (it != fpos[(size_t)q].end() && it->first == x) ? it->second : -1;
  };
  // 3 x 3 block (x, y) of the inverse -> out: from the front of x's owner if it holds y, else of y's owner if it holds x
  std::vector<std::pair<int, CovItem>> staged;
  auto add = [&](int x, int y, long long out) -> bool {
    int q = ridx[(size_t)C.H.node_of[(size_t)x]];
    int px = pos_in(q, x), py = pos_in(q, y);
    if (py < 0) {
      q = ridx[(size_t)C.H.node_of[(size_t)y]];
      px = pos_in(q, x); py = pos_in(q, y);
    }
    if (px < 0 || py < 0) return false;
    staged.push_back({C.H.nodes[(size_t)C.S.macro[(size_t)q]].stage, CovItem{q, CDH * px, CDH * py, 0, out}});
    return true;
  };
  const long long bb = (long long)P.b * P.b;
  auto add_pose_pair = [&](int i, int j, long long out) -> bool {
    if (i == P.anchor || j == P.anchor) return true;           // zero block
    for (int sa = 0; sa < sub; ++sa)
      for (int sc = 0; sc < sub; ++sc)
        if (!add(sub * i + sa, sub * j + sc, out + (long long)CDH * sa * P.b + CDH * sc)) return false;
    return true;
  };
  for (int p = 0; p < P.n; ++p)
    if (!add_pose_pair(p, p, (long long)p * bb)) return fail(DPGO_ERR_UNSUPPORTED, "pose_covariances: a pose block outside its front");
  for (int64_t q = 0; q < P.num_pairs; ++q)
    if (!add_pose_pair(P.pairs[2 * q], P.pairs[2 * q + 1], ((long long)P.n + q) * bb))
      return fail(DPGO_ERR_UNSUPPORTED, "pose_covariances: a pair block outside every front");
  std::stable_sort(staged.begin(), staged.end(), [](const auto &x, const auto &y) { return x.first < y.first; });
  C.items.clear();
  C.item0.assign((size_t)C.H.nstages + 1, 0);
  for (const auto &s : staged) { C.items.push_back(s.second); C.item0[(size_t)s.first + 1]++; }
  for (int st = 0; st < C.H.nstages; ++st) C.item0[(size_t)st + 1] += C.item0[(size_t)st];
  if (C.items.empty()) C.items.push_back(CovItem{0, 0, 0, 0, 0});
  return DPGO_OK;
}

void fill_info(const CovProblem &P, const CovSetup &C, int64_t *info) {
  for (int i = 0; i < 16; ++i) info[i] = 0;
  int smax = 0, bmax = 0;
  for (const auto &m : C.H.nodes) { smax = std::max(smax, (int)m.own.size() * CDH); bmax = std::max(bmax, (int)m.bnd.size() * CDH); }
  info[0] = C.H.nstages; info[1] = (int64_t)C.H.nodes.size(); info[2] = P.ne; info[3] = (int64_t)C.bcol.size();
  info[4] = 8 * (C.H.blob_doubles + C.R.arena_doubles + C.R.ws_doubles + (int64_t)C.bcol.size() * 16);
  info[5] = smax; info[6] = bmax; info[7] = C.H.nd_depth;
  info[8] = (int64_t)C.item0.back();
  info[9] = 2 * (int64_t)C.H.nstages;                  // factor + sweep stages
  for (size_t st = 0; st + 1 < C.R.stage0.size(); ++st) info[13] = std::max(info[13], (int64_t)(C.R.stage0[st + 1] - C.R.stage0[st]));
}

nd::Options cov_options(int force_cuts, int leaf_size) {
  nd::Options opt;
  opt.shift = 0.0;
  opt.force_ncuts = force_cuts;
  if (leaf_size > 0) opt.leaf_size = leaf_size;
  return opt;
}

// b x b blocks of the item outputs: zero first (the anchor's blocks are never written)
int run_device(const CovProblem &P, int device, double *cov_host, double *pair_cov_host, int64_t *info16) {
  DPGO_TRY(require_device(device));
  DPGO_CUDA(cudaSetDevice(device));
  CovSetup C;
  DPGO_TRY(setup(P, cov_options(-1, 0), C));
  cudaStream_t st = nullptr;
  DPGO_CUDA(cudaStreamCreateWithFlags(&st, cudaStreamNonBlocking));
  const dpgo::Stream own(st);
  dpgo::Event ev[4];
  for (auto &e : ev) DPGO_CUDA(dpgo::create_event(e, cudaEventDefault));
  const size_t nT = (size_t)P.d * (P.d + 1) * P.n, m = (size_t)P.m;
  DevBuf<double> dT, dR, dt, dk, dtau, dw, bval, blob, arena, ws, out;
  DevBuf<int> p1, p2, cptr, rowptr, bcol, rposes, rcmap, fail_flag, parent, pmap0, pmap;
  DevBuf<int2> contrib, bnode;
  DevBuf<nd::RefactorNode> rnodes;
  DevBuf<nd::RefactorChild> rchild;
  DevBuf<dpgo::GjJob> rjobs;
  DevBuf<CovItem> items;
  DPGO_CUDA(dT.assign(P.T, nT, st));
  DPGO_CUDA(dR.assign(P.R, m * P.d * P.d, st));
  DPGO_CUDA(dt.assign(P.t, m * P.d, st));
  DPGO_CUDA(dk.assign(P.kappa, m, st));
  DPGO_CUDA(dtau.assign(P.tau, m, st));
  if (P.weight) DPGO_CUDA(dw.assign(P.weight, m, st));
  DPGO_CUDA(p1.assign(P.p1, m, st));
  DPGO_CUDA(p2.assign(P.p2, m, st));
  DPGO_CUDA(cptr.assign(C.cptr.data(), C.cptr.size(), st));
  DPGO_CUDA(contrib.assign(C.contrib.data(), C.contrib.size(), st));
  DPGO_CUDA(bnode.assign(C.bnode.data(), C.bnode.size(), st));
  DPGO_CUDA(rowptr.assign(C.rowptr.data(), C.rowptr.size(), st));
  DPGO_CUDA(bcol.assign(C.bcol.data(), C.bcol.size(), st));
  DPGO_CUDA(bval.alloc(C.bcol.size() * 16));
  DPGO_CUDA(rnodes.assign(C.R.nodes.data(), C.R.nodes.size(), st));
  DPGO_CUDA(rchild.assign(C.R.child.data(), C.R.child.size(), st));
  DPGO_CUDA(rposes.assign(C.R.poses.data(), C.R.poses.size(), st));
  DPGO_CUDA(rcmap.assign(C.R.cmap.data(), C.R.cmap.size(), st));
  DPGO_CUDA(parent.assign(C.S.parent.data(), C.S.parent.size(), st));
  DPGO_CUDA(pmap0.assign(C.S.pmap0.data(), C.S.pmap0.size(), st));
  DPGO_CUDA(pmap.assign(C.S.pmap.data(), C.S.pmap.size(), st));
  DPGO_CUDA(items.assign(C.items.data(), C.items.size(), st));
  DPGO_CUDA(blob.alloc((size_t)C.H.blob_doubles));
  DPGO_CUDA(cudaMemsetAsync(blob.get(), 0, sizeof(double) * (size_t)C.H.blob_doubles, st));
  DPGO_CUDA(arena.alloc((size_t)C.R.arena_doubles));
  DPGO_CUDA(ws.alloc((size_t)C.R.ws_doubles));
  const size_t nout = (size_t)(P.n + P.num_pairs) * P.b * P.b;
  DPGO_CUDA(out.alloc(nout));
  DPGO_CUDA(cudaMemsetAsync(out.get(), 0, sizeof(double) * nout, st));
  DPGO_CUDA(fail_flag.alloc(1));
  DPGO_CUDA(cudaMemsetAsync(fail_flag.get(), 0, sizeof(int), st));
  constexpr int B = nd::REFACTOR_PIVOT_BLOCK;
  std::vector<dpgo::GjJob> jobs(C.R.nodes.size());
  for (size_t q = 0; q < jobs.size(); ++q) {
    const nd::RefactorNode &rn = C.R.nodes[q];
    const int M = CDH * (rn.no + rn.nb);
    double *w = ws.get() + rn.ws;
    jobs[q] = {arena.get() + rn.front, w, w + B * B, w + B * B + (size_t)B * M, M, CDH * rn.no};
  }
  DPGO_CUDA(rjobs.assign(jobs.data(), jobs.size(), st));

  DPGO_CUDA(cudaEventRecord(ev[0].get(), st));
  dpgo::KPoseInfo ka = {P.d, P.anchor, (int64_t)C.bcol.size(), cptr.get(), contrib.get(), bnode.get(), p1.get(), p2.get(),
                        dT.get(), dR.get(), dt.get(), dk.get(), dtau.get(), P.weight ? dw.get() : nullptr, bval.get()};
  DPGO_CUDA(dpgo::launch_assemble_pose_info(ka, st));
  DPGO_CUDA(cudaEventRecord(ev[1].get(), st));
  dpgo::KRefactor kr;
  kr.dh = CDH; kr.shift = 0.0;
  kr.nodes = rnodes.get(); kr.child = rchild.get(); kr.poses = rposes.get(); kr.cmap = rcmap.get();
  kr.rowptr = rowptr.get(); kr.bcol = bcol.get(); kr.bval = bval.get();
  kr.arena = arena.get(); kr.jobs = rjobs.get(); kr.blob = blob.get(); kr.fail = fail_flag.get();
  DPGO_CUDA(dpgo::launch_nd_refactor(kr, C.R, st));
  DPGO_CUDA(cudaEventRecord(ev[2].get(), st));
  dpgo::KSelinv ks = {rnodes.get(), parent.get(), pmap0.get(), pmap.get(), blob.get(), arena.get(), items.get(), out.get(), P.b};
  DPGO_CUDA(dpgo::launch_nd_selinv(ks, C.R, C.S, C.item0, st));
  DPGO_CUDA(cudaEventRecord(ev[3].get(), st));
  int failed = 0;
  DPGO_CUDA(cudaMemcpyAsync(&failed, fail_flag.get(), sizeof(int), cudaMemcpyDeviceToHost, st));
  DPGO_CUDA(cudaStreamSynchronize(st));
  if (failed)
    return fail(DPGO_ERR_CUDA, "pose_covariances: the anchored information matrix is not positive definite (a pivot of its "
                               "factorisation was not positive): zero precisions or a degenerate trajectory");
  DPGO_CUDA(cudaMemcpy(cov_host, out.get(), sizeof(double) * (size_t)P.n * P.b * P.b, cudaMemcpyDeviceToHost));
  if (P.num_pairs > 0)
    DPGO_CUDA(cudaMemcpy(pair_cov_host, out.get() + (size_t)P.n * P.b * P.b, sizeof(double) * (size_t)P.num_pairs * P.b * P.b,
                         cudaMemcpyDeviceToHost));
  if (info16) {
    fill_info(P, C, info16);
    float ms[3] = {0, 0, 0};
    for (int k = 0; k < 3; ++k) DPGO_CUDA(cudaEventElapsedTime(&ms[k], ev[k].get(), ev[k + 1].get()));
    for (int k = 0; k < 3; ++k) info16[10 + k] = (int64_t)std::llround((double)ms[k] * 1e6);
  }
  return DPGO_OK;
}

}  // namespace
}  // namespace dpgo::capi

using namespace dpgo::capi;

extern "C" {

int dpgo_pose_covariances(int n, int d, int64_t m, const int32_t *p1, const int32_t *p2, const double *R, const double *t,
                          const double *kappa, const double *tau, const double *weight, const double *T_host, int anchor,
                          int device, int64_t num_pairs, const int32_t *pairs, double *cov_host, double *pair_cov_host,
                          int64_t *info16) {
  const int b = d == 3 ? 6 : 3;
  CovProblem P{n, d, b, d == 3 ? 2 * n : n, anchor, m, p1, p2, pairs, R, t, kappa, tau, weight, T_host, num_pairs};
  DPGO_TRY(check_args(P, cov_host));
  DPGO_REQUIRE(num_pairs == 0 || pair_cov_host, DPGO_ERR_INVALID_ARG, "pose_covariances: null pair output");
  if (info16) std::fill(info16, info16 + 16, (int64_t)0);
  if (n == 1) {                                             // the anchor alone: nothing is uncertain
    std::fill(cov_host, cov_host + (size_t)b * b, 0.0);
    if (num_pairs > 0) std::fill(pair_cov_host, pair_cov_host + (size_t)num_pairs * b * b, 0.0);
    return DPGO_OK;
  }
  return run_device(P, device, cov_host, pair_cov_host, info16);
}

int dpgo_pose_covariances_debug_emulate(int n, int d, int64_t m, const int32_t *p1, const int32_t *p2, const double *R,
                                        const double *t, const double *kappa, const double *tau, const double *weight,
                                        const double *T_host, int anchor, int force_cuts, int leaf_size, int64_t num_pairs,
                                        const int32_t *pairs, double *cov_host, double *pair_cov_host, int64_t *info16) {
  const int b = d == 3 ? 6 : 3;
  CovProblem P{n, d, b, d == 3 ? 2 * n : n, anchor, m, p1, p2, pairs, R, t, kappa, tau, weight, T_host, num_pairs};
  DPGO_TRY(check_args(P, cov_host));
  DPGO_REQUIRE(num_pairs == 0 || pair_cov_host, DPGO_ERR_INVALID_ARG, "pose_covariances: null pair output");
  CovSetup C;
  DPGO_TRY(setup(P, cov_options(force_cuts, leaf_size), C));
  // the assembly kernel's arithmetic, entry by entry
  std::vector<double> bval(C.bcol.size() * 16, 0.0);
  for (size_t blk = 0; blk < C.bcol.size(); ++blk) {
    const int2 bn = C.bnode[blk];
    for (int x = 0; x < CDH; ++x)
      for (int y = 0; y < CDH; ++y) {
        const int pa = d == 3 ? bn.x >> 1 : bn.x;
        const int qa = d == 3 ? 3 * (bn.x & 1) + x : x, qc = d == 3 ? 3 * (bn.y & 1) + y : y;
        double v = 0.0;
        if (pa == anchor) {
          v = (bn.x == bn.y && x == y) ? 1.0 : 0.0;
        } else {
          for (int q = C.cptr[blk]; q < C.cptr[blk + 1]; ++q) {
            const int2 cc = C.contrib[(size_t)q];
            const int e = cc.x;
            const double *Ri = T_host + (size_t)p1[e] * d * (d + 1), *Rj = T_host + (size_t)p2[e] * d * (d + 1);
            const double w = weight ? weight[e] : 1.0;
            v += d == 3 ? dpgo::cov::edge_info<3>(cc.y & 1, qa, cc.y >> 1, qc, Ri, Rj, R + (size_t)e * 9, t + (size_t)e * 3, kappa[e], tau[e], w)
                        : dpgo::cov::edge_info<2>(cc.y & 1, qa, cc.y >> 1, qc, Ri, Rj, R + (size_t)e * 4, t + (size_t)e * 2, kappa[e], tau[e], w);
          }
        }
        bval[blk * 16 + (size_t)x * 4 + y] = v;
      }
  }
  std::vector<double> out((size_t)(n + num_pairs) * b * b, 0.0);
  try {
    nd::BsrView Q{P.ne, CDH, C.rowptr.data(), C.bcol.data(), bval.data()};
    std::vector<double> blob;
    std::vector<std::vector<double>> front;
    nd::build_numeric(Q, cov_options(force_cuts, leaf_size), C.H, blob);
    nd::emulate_selinv(C.H, C.R, C.S, blob, front);
    for (int st = 0; st < C.H.nstages; ++st)
      for (int i = C.item0[(size_t)st]; i < C.item0[(size_t)st + 1]; ++i) {
        const dpgo::CovItem &it = C.items[(size_t)i];
        const nd::RefactorNode &rn = C.R.nodes[(size_t)it.node];
        const int64_t M = (int64_t)CDH * (rn.no + rn.nb);
        const std::vector<double> &F = front[(size_t)it.node];
        for (int x = 0; x < CDH; ++x)
          for (int y = 0; y < CDH; ++y) {
            const int64_t r = it.ra + x, c = it.rc + y;
            out[(size_t)(it.out + (long long)x * b + y)] = r <= c ? F[(size_t)(r + M * c)] : F[(size_t)(c + M * r)];
          }
      }
  } catch (const std::exception &e) {
    return fail(DPGO_ERR_CUDA, std::string("pose_covariances (host emulation): ") + e.what());
  }
  std::copy(out.begin(), out.begin() + (size_t)n * b * b, cov_host);
  if (num_pairs > 0) std::copy(out.begin() + (size_t)n * b * b, out.end(), pair_cov_host);
  if (info16) fill_info(P, C, info16);
  return DPGO_OK;
}

}  // extern "C"
