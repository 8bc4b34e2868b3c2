// dpgo_capi_edges.cu -- Q from edge records on the device and robust re-weighting: the synchronous calls refresh the
// preconditioners on the host, the stream-ordered ones refactorise them on the device.
#include <cuda_runtime.h>
#include <algorithm>
#include <cstring>
#include <utility>
#include <vector>

#include "dpgo_handle.cuh"

namespace dpgo::capi {
namespace {

// weights (and the GNC counts) of the non-fixed edges at the resident iterate, under robust cost `cost` (0..5; 5 is GNC)
int launch_reweight(dpgo_problem *p, int cost, double mu, double param) {
  DPGO_REQUIRE(cost >= 0 && cost <= 5, DPGO_ERR_INVALID_ARG, "unknown robust cost");
  DPGO_REQUIRE(cost != 5 || mu > 0, DPGO_ERR_INVALID_ARG, "GNC needs mu > 0");
  const dpgo_problem::Edges &E = p->edges;
  DPGO_CUDA(cudaMemsetAsync(E.gnc.get(), 0, 3 * sizeof(unsigned long long), p->stream));
  DPGO_CUDA(dpgo::launch_edge_weights(p->r, p->dh, E.ne, E.p1.get(), E.p2.get(), E.T.get(), E.om.get(), E.fixed.get(),
                                      p->vec[dpgo::V_X0].get(), cost, mu, param, E.w.get(), E.res.get(), E.gnc.get(), p->stream));
  return DPGO_OK;
}

// Q's values on the device from the edge records and their current weights (k_assemble_Q, stream-ordered)
int assemble_Q(dpgo_problem *p) {
  const dpgo_problem::Edges &E = p->edges;
  DPGO_CUDA(dpgo::launch_assemble_Q(p->bsr.nb, E.cptr.get(), E.contrib.get(), E.T.get(), E.om.get(), E.w.get(), E.sblk.get(),
                                    p->bsr.bval.get(), p->stream));
  return DPGO_OK;
}

int reassemble_Q(dpgo_problem *p) {
  DPGO_TRY(assemble_Q(p));
  // the host copy feeds the lazily built exact preconditioners; block-Jacobi blocks are refreshed right away
  DPGO_CUDA(cudaMemcpyAsync(p->bsr.h_bval.data(), p->bsr.bval.get(), sizeof(double) * 16 * (size_t)p->bsr.nb,
                            cudaMemcpyDeviceToHost, p->stream));
  DPGO_CUDA(cudaStreamSynchronize(p->stream));
  p->bsr.h_stale = false;
  if (p->bsr.dinv) {
    std::vector<double> dinv;
    jacobi_blocks(p->n, p->dh, p->bsr.h_rowptr, p->bsr.h_bcol, p->bsr.h_bval, dinv);
    DPGO_CUDA(p->bsr.dinv.upload(dinv.data(), dinv.size(), p->stream));
    DPGO_CUDA(cudaStreamSynchronize(p->stream));
  }
  free_nd(p);                                            // (Q + 0.1 I)^-1 changed: rebuilt on next use
  return DPGO_OK;
}

// After k_assemble_Q on the stream: block-Jacobi and the prepared exact preconditioners refactorised on the device.  Only
// the first call after the sparse exact structure was dropped (or never built) runs host work and synchronises; an
// unprepared dense one stays lazy.
int refresh_preconditioners_async(dpgo_problem *p) {
  p->bsr.h_stale = true;
  dpgo_problem::Edges &E = p->edges;
  E.fail_armed = true;
  if (p->bsr.dinv)
    DPGO_CUDA(dpgo::launch_jacobi_blocks(p->n, p->dh, p->bsr.rowptr.get(), p->bsr.bcol.get(), p->bsr.bval.get(), 0.1,
                                         p->bsr.dinv.get(), E.fail.get(), p->stream));
  if (p->bsr.precond_mask & (1u << DPGO_PRECOND_SPARSE_EXACT)) DPGO_TRY(ensure_nd(p, ND_SPARSE));
  for (int slot : {ND_SPARSE, ND_DENSE}) {
    if (!p->nd[slot].ready) continue;
    DPGO_TRY(ensure_refactor(p, slot));
    DPGO_TRY(launch_refactor(p, slot));
  }
  return DPGO_OK;
}

}  // namespace
}  // namespace dpgo::capi

using namespace dpgo::capi;

extern "C" {

// ---- Q from edge records on the device, robust re-weighting -----------------------------------------------------
int dpgo_problem_set_edges(dpgo_problem_t *p, int64_t m, const int32_t *p1, const int32_t *p2, const double *R, const double *t,
                           const double *kappa, const double *tau, const double *weight, const int32_t *fixed_weight,
                           int64_t num_static, const int32_t *static_pose, const double *static_blocks, unsigned precond_mask) {
  DPGO_CHECK_HANDLE(p);
  DPGO_REQUIRE(m >= 0 && (m == 0 || (p1 && p2 && R && t && kappa && tau)), DPGO_ERR_INVALID_ARG, "null edge arrays");
  DPGO_REQUIRE(num_static >= 0 && (num_static == 0 || (static_pose && static_blocks)), DPGO_ERR_INVALID_ARG, "null static blocks");
  const int d = p->d, dh = p->dh, n = p->n;
  for (int64_t e = 0; e < m; ++e)
    if (p1[e] < 0 || p1[e] >= n || p2[e] < 0 || p2[e] >= n) return fail(DPGO_ERR_INVALID_ARG, "edge endpoint out of range");
  for (int64_t q = 0; q < num_static; ++q)
    if (static_pose[q] < 0 || static_pose[q] >= n) return fail(DPGO_ERR_INVALID_ARG, "static block pose out of range");
  // pattern: zero-valued triplets give the block-CSR structure (and the usual launch tables) ...
  std::vector<BlockTriplet> trip;
  trip.reserve((size_t)(4 * m + num_static));
  auto add = [&](int bi, int bj) { BlockTriplet bt; bt.brow = bi; bt.bcol = bj; std::memset(bt.v, 0, sizeof(bt.v)); trip.push_back(bt); };
  for (int64_t e = 0; e < m; ++e) { add(p1[e], p1[e]); add(p2[e], p2[e]); add(p1[e], p2[e]); add(p2[e], p1[e]); }
  for (int64_t q = 0; q < num_static; ++q) add(static_pose[q], static_pose[q]);
  DPGO_TRY(build_from_triplets(p, trip, precond_mask));
  // ... and every block's contribution list in input order: block (bi, bj) = entry with bcol == bi in row bj
  const std::vector<int> &rowptr = p->bsr.h_rowptr, &bcol = p->bsr.h_bcol;
  auto find_block = [&](int bi, int bj) {
    const int *lo = bcol.data() + rowptr[(size_t)bj], *hi = bcol.data() + rowptr[(size_t)bj + 1];
    return (int)(std::lower_bound(lo, hi, bi) - bcol.data());
  };
  const int64_t nb = p->bsr.nb;
  std::vector<int> cnt((size_t)nb + 1, 0);
  std::vector<std::pair<int, int2>> items;             // (block, (index, kind))
  items.reserve((size_t)(4 * m + num_static));
  for (int64_t e = 0; e < m; ++e) {
    items.push_back({find_block(p1[e], p1[e]), make_int2((int)e, 0)});
    items.push_back({find_block(p2[e], p2[e]), make_int2((int)e, 1)});
    items.push_back({find_block(p1[e], p2[e]), make_int2((int)e, 2)});
    items.push_back({find_block(p2[e], p1[e]), make_int2((int)e, 3)});
  }
  for (int64_t q = 0; q < num_static; ++q) items.push_back({find_block(static_pose[q], static_pose[q]), make_int2((int)q, 4)});
  for (auto &it : items) cnt[(size_t)it.first + 1]++;
  for (int64_t b = 0; b < nb; ++b) cnt[(size_t)b + 1] += cnt[(size_t)b];
  std::vector<int2> contrib(items.size());
  {
    std::vector<int> fill(cnt.begin(), cnt.end() - 1);
    for (auto &it : items) contrib[(size_t)fill[(size_t)it.first]++] = it.second;     // input order inside a block
  }
  std::vector<double> eT((size_t)m * 16, 0.0), eom((size_t)m * 4, 0.0), ew((size_t)m, 1.0), sb((size_t)num_static * 16, 0.0);
  std::vector<int> fx((size_t)m, 0), q1((size_t)m), q2((size_t)m);
  for (int64_t e = 0; e < m; ++e) {
    double *T = &eT[(size_t)e * 16];
    for (int a = 0; a < d; ++a) {
      for (int b = 0; b < d; ++b) T[a * 4 + b] = R[(size_t)e * d * d + a * d + b];
      T[a * 4 + d] = t[(size_t)e * d + a];
      eom[(size_t)e * 4 + a] = kappa[e];
    }
    T[d * 4 + d] = 1.0;
    eom[(size_t)e * 4 + d] = tau[e];
    if (weight) ew[(size_t)e] = weight[e];
    if (fixed_weight) fx[(size_t)e] = fixed_weight[e] ? 1 : 0;
    q1[(size_t)e] = p1[e];
    q2[(size_t)e] = p2[e];
  }
  for (int64_t q = 0; q < num_static; ++q)
    for (int a = 0; a < dh; ++a)
      for (int b = 0; b < dh; ++b) sb[(size_t)q * 16 + a * 4 + b] = static_blocks[(size_t)q * dh * dh + a * dh + b];
  p->edges = {};
  dpgo_problem::Edges &E = p->edges;
  E.ne = m;
  DPGO_CUDA(E.p1.assign(q1.data(), q1.size(), p->stream));
  DPGO_CUDA(E.p2.assign(q2.data(), q2.size(), p->stream));
  DPGO_CUDA(E.fixed.assign(fx.data(), fx.size(), p->stream));
  DPGO_CUDA(E.cptr.assign(cnt.data(), cnt.size(), p->stream));
  DPGO_CUDA(E.contrib.assign(contrib.data(), contrib.size(), p->stream));
  DPGO_CUDA(E.T.assign(eT.data(), eT.size(), p->stream));
  DPGO_CUDA(E.om.assign(eom.data(), eom.size(), p->stream));
  DPGO_CUDA(E.w.assign(ew.data(), ew.size(), p->stream));
  DPGO_CUDA(E.sblk.assign(sb.data(), sb.size(), p->stream));
  DPGO_CUDA(E.res.alloc((size_t)m));
  DPGO_CUDA(E.gnc.alloc(3));
  DPGO_CUDA(cudaMemsetAsync(E.gnc.get(), 0, 3 * sizeof(unsigned long long), p->stream));
  DPGO_CUDA(E.fail.alloc(1));
  DPGO_CUDA(cudaMemsetAsync(E.fail.get(), 0, sizeof(int), p->stream));
  return reassemble_Q(p);
}

int dpgo_problem_set_edge_weights(dpgo_problem_t *p, const double *weights_host) {
  DPGO_CHECK_HANDLE(p);
  DPGO_REQUIRE(p->edges.cptr, DPGO_ERR_STATE, "dpgo_problem_set_edges has not been called");
  DPGO_REQUIRE(weights_host || p->edges.ne == 0, DPGO_ERR_INVALID_ARG, "null weights");
  DPGO_CUDA(p->edges.w.upload(weights_host, (size_t)p->edges.ne, p->stream));
  return reassemble_Q(p);
}

int dpgo_problem_robust_reweight(dpgo_problem_t *p, int cost, double mu, double param, double *weights_host, double *residuals2_host) {
  DPGO_CHECK_HANDLE(p);
  DPGO_REQUIRE(p->edges.cptr, DPGO_ERR_STATE, "dpgo_problem_set_edges has not been called");
  DPGO_TRY(launch_reweight(p, cost, mu, param));
  const dpgo_problem::Edges &E = p->edges;
  if (weights_host && E.ne)
    DPGO_CUDA(cudaMemcpyAsync(weights_host, E.w.get(), sizeof(double) * (size_t)E.ne, cudaMemcpyDeviceToHost, p->stream));
  if (residuals2_host && E.ne)
    DPGO_CUDA(cudaMemcpyAsync(residuals2_host, E.res.get(), sizeof(double) * (size_t)E.ne, cudaMemcpyDeviceToHost, p->stream));
  return reassemble_Q(p);
}

// ---- stream-ordered re-weighting: the preconditioners are refactorised on the device --------------------------------
int dpgo_problem_set_edge_weights_async(dpgo_problem_t *p, const double *weights_dev) {
  DPGO_CHECK_HANDLE(p);
  DPGO_REQUIRE(weights_dev || p->edges.ne == 0, DPGO_ERR_INVALID_ARG, "null weights");
  DPGO_REQUIRE(p->edges.cptr, DPGO_ERR_STATE, "dpgo_problem_set_edges has not been called");
  const dpgo_problem::Edges &E = p->edges;
  if (E.ne)
    DPGO_CUDA(cudaMemcpyAsync(E.w.get(), weights_dev, sizeof(double) * (size_t)E.ne, cudaMemcpyDeviceToDevice, p->stream));
  DPGO_TRY(assemble_Q(p));
  return refresh_preconditioners_async(p);
}

int dpgo_problem_robust_reweight_async(dpgo_problem_t *p, int cost, double mu, double param) {
  DPGO_CHECK_HANDLE(p);
  DPGO_REQUIRE(p->edges.cptr, DPGO_ERR_STATE, "dpgo_problem_set_edges has not been called");
  DPGO_TRY(launch_reweight(p, cost, mu, param));
  DPGO_TRY(assemble_Q(p));
  return refresh_preconditioners_async(p);
}

int dpgo_problem_device_edge_weights(dpgo_problem_t *p, double **w_dev, double **res2_dev) {
  DPGO_REQUIRE(p && w_dev && res2_dev, DPGO_ERR_INVALID_ARG, "null argument");
  DPGO_REQUIRE(p->edges.cptr, DPGO_ERR_STATE, "dpgo_problem_set_edges has not been called");
  *w_dev = p->edges.w.get();
  *res2_dev = p->edges.res.get();
  return DPGO_OK;
}

int dpgo_problem_gnc_counts(dpgo_problem_t *p, int64_t *out3) {
  DPGO_CHECK_HANDLE(p);
  DPGO_REQUIRE(out3, DPGO_ERR_INVALID_ARG, "null argument");
  DPGO_REQUIRE(p->edges.cptr, DPGO_ERR_STATE, "dpgo_problem_set_edges has not been called");
  unsigned long long c[3] = {0, 0, 0};
  DPGO_CUDA(cudaMemcpyAsync(c, p->edges.gnc.get(), sizeof(c), cudaMemcpyDeviceToHost, p->stream));
  DPGO_CUDA(cudaStreamSynchronize(p->stream));
  DPGO_TRY(check_refactor_fail(p));
  for (int q = 0; q < 3; ++q) out3[q] = (int64_t)c[q];
  return DPGO_OK;
}

}  // extern "C"
