// dpgo_capi_precond.cu -- the exact preconditioners of a problem handle: the nested-dissection factorisation of
// Q + 0.1 I (host ordering, symbolic analysis, plan and numbers), its device refactorisation, the host block-Jacobi blocks,
// and the C calls that report on or emulate the block solve.
#include <cuda_runtime.h>
#include <algorithm>
#include <cstdio>
#include <cstdlib>
#include <memory>
#include <string>
#include <vector>

#include "dpgo_handle.cuh"

namespace dpgo::capi {
namespace {

void nd_fill_info(const dpgo::nd::Hierarchy &H, const dpgo::nd::Plan &P, int64_t *info) {
  for (int i = 0; i < 16; ++i) info[i] = 0;
  int smax = 0, bmax = 0;
  for (const auto &m : H.nodes) { smax = std::max(smax, (int)m.own.size() * H.dh); bmax = std::max(bmax, (int)m.bnd.size() * H.dh); }
  info[0] = H.nstages; info[1] = (int64_t)H.nodes.size(); info[2] = (int64_t)P.phases.size(); info[3] = H.blob_doubles * 8;
  info[4] = P.bytes_per_apply; info[5] = smax; info[6] = bmax; info[7] = H.nd_depth; info[8] = (int64_t)P.steps.size();
  info[9] = (int64_t)P.jobs.size(); info[10] = (int64_t)P.epis.size(); info[11] = P.max_ytiles; info[12] = P.max_slots;
  info[13] = P.resident_bytes; info[14] = (int64_t)P.max_resident_doubles * 8;
}

// shared-memory sizes of the kernel's view of a plan (the staged areas the resident budget is what is left of)
void nd_kernel_sizes(const dpgo::nd::Plan &plan, dpgo::KNd &K) {
  K.max_ytiles = std::max(plan.max_ytiles, 1);
  K.max_slots = std::max(plan.max_slots, 1);
  K.max_gathers = K.max_ytiles;          // a step gathers at most what its shared-memory tiles hold
  K.resident_doubles = 0;
}

dpgo::nd::Options nd_options(int grid, int r, int dh, bool cluster = false) {
  dpgo::nd::Options opt;
  opt.grid = grid;
  opt.r = r;
  // a phase end is a hardware cluster barrier in cluster mode: deeper dissections pay off earlier (16 agents side by side
  // on one H100 SXM at 400 W: torus3D, 312 poses per agent, 7140-7260 rounds/s against 5540-5660 with the grid value
  // 3.5 us, and 1.0 us is no faster; sphere2500's 156-pose agents are best with 2.0 us as well)
  if (cluster) opt.t_phase_us = 2.0;
  opt.warps = dpgo::OPT_THREADS / 32;
  opt.ycap_tiles = dpgo::nd_ycap_tiles(r, dh);
  opt.slot_cap = dpgo::nd_slot_cap(r);
  if (const char *e = std::getenv("DPGO_ND_CUTS")) opt.force_ncuts = std::atoi(e);
  return opt;
}

// The host copy of Q's values after an asynchronous re-weight changed them on the device only: downloaded before any
// host-side use (synchronises).
int sync_host_bval(dpgo_problem *p) {
  if (!p->bsr.h_stale) return DPGO_OK;
  DPGO_CUDA(cudaMemcpyAsync(p->bsr.h_bval.data(), p->bsr.bval.get(), sizeof(double) * 16 * (size_t)p->bsr.nb,
                            cudaMemcpyDeviceToHost, p->stream));
  DPGO_CUDA(cudaStreamSynchronize(p->stream));
  p->bsr.h_stale = false;
  return DPGO_OK;
}

}  // namespace

void free_nd(dpgo_problem *p) {
  ++p->generation;
  for (dpgo_problem::Nd &F : p->nd) F = {};
}

// A factorisation's device refactorisation: scatter maps, fronts, sweep jobs of its hierarchy, built once per hierarchy on
// the host (synchronises).
int ensure_refactor(dpgo_problem *p, int slot) {
  namespace nd = dpgo::nd;
  dpgo_problem::Nd &F = p->nd[slot];
  if (F.R) return DPGO_OK;
  const std::string what = slot == ND_DENSE ? "dense exact preconditioner refactorisation" : "sparse exact preconditioner refactorisation";
  auto R = std::make_unique<nd::Refactor>();
  try {
    nd::build_refactor(*F.H, *R);
  } catch (const std::exception &e) {
    return fail(DPGO_ERR_UNSUPPORTED, what + ": " + e.what());
  }
  if (R->child.empty()) R->child.push_back({0, 0});        // one macro level: no children, nothing reads these
  if (R->cmap.empty()) R->cmap.push_back(-1);
  DPGO_CUDA(F.rnodes.assign(R->nodes.data(), R->nodes.size(), p->stream));
  DPGO_CUDA(F.rchild.assign(R->child.data(), R->child.size(), p->stream));
  DPGO_CUDA(F.rposes.assign(R->poses.data(), R->poses.size(), p->stream));
  DPGO_CUDA(F.rcmap.assign(R->cmap.data(), R->cmap.size(), p->stream));
  DPGO_CUDA(F.arena.alloc((size_t)R->arena_doubles));
  DPGO_CUDA(F.ws.alloc((size_t)R->ws_doubles));
  std::vector<dpgo::GjJob> jobs(R->nodes.size());
  constexpr int B = nd::REFACTOR_PIVOT_BLOCK;
  for (size_t q = 0; q < jobs.size(); ++q) {
    const nd::RefactorNode &rn = R->nodes[q];
    const int M = p->dh * (rn.no + rn.nb);
    double *w = F.ws.get() + rn.ws;
    jobs[q] = {F.arena.get() + rn.front, w, w + B * B, w + B * B + (size_t)B * M, M, p->dh * rn.no};
  }
  DPGO_CUDA(F.rjobs.assign(jobs.data(), jobs.size(), p->stream));
  DPGO_CUDA(cudaStreamSynchronize(p->stream));
  F.R = std::move(R);
  return DPGO_OK;
}

// The numbers of a factorisation recomputed from Q's values on the device, its panels rewritten in place: ordinary
// launches on the handle's stream, no host work, no synchronisation.
int launch_refactor(dpgo_problem *p, int slot) {
  dpgo_problem::Nd &F = p->nd[slot];
  dpgo::KRefactor k;
  k.dh = p->dh;
  k.shift = 0.1;
  k.nodes = F.rnodes.get();
  k.child = F.rchild.get();
  k.poses = F.rposes.get();
  k.cmap = F.rcmap.get();
  k.rowptr = p->bsr.rowptr.get();
  k.bcol = p->bsr.bcol.get();
  k.bval = p->bsr.bval.get();
  k.arena = F.arena.get();
  k.jobs = F.rjobs.get();
  k.blob = F.blob.get();
  k.fail = p->edges.fail.get();
  DPGO_CUDA(dpgo::launch_nd_refactor(k, *F.R, p->stream));
  return DPGO_OK;
}

// An exact preconditioner's block factorisation of Q + 0.1 I is built on first use (host: ordering, symbolic, plan).  The
// sparse one takes its numbers from the host (build_numeric); the dense one, whose single macro level is the dense inverse
// of every connected component (an O(N^3) host inverse), from the device refactorisation of Q's values.
int ensure_nd(dpgo_problem *p, int slot) {
  dpgo_problem::Nd &F = p->nd[slot];
  if (F.ready) return DPGO_OK;
  const bool dense = slot == ND_DENSE;
  const std::string what = dense ? "dense exact preconditioner" : "sparse exact preconditioner";
  if (!(p->bsr.precond_mask & (1u << nd_precond(slot))))
    return fail(DPGO_ERR_STATE, what + " was not requested in set_Q (precond_mask)");
  namespace nd = dpgo::nd;
  ++p->generation;
  F = {};
  if (!dense) DPGO_TRY(sync_host_bval(p));
  nd::Plan plan;
  std::vector<double> blob;
  auto H = std::make_unique<nd::Hierarchy>();
  try {
    nd::Options opt = nd_options(p->grid, p->r, p->dh, p->cluster);
    if (dense) opt.force_ncuts = 0;
    nd::BsrView Q{p->n, p->dh, p->bsr.h_rowptr.data(), p->bsr.h_bcol.data(), p->bsr.h_bval.data()};
    nd::build_hierarchy(Q, opt, *H);
    if (!dense) nd::build_numeric(Q, opt, *H, blob);
    nd::build_plan(*H, opt, plan);
  } catch (const std::exception &e) {
    return fail(DPGO_ERR_UNSUPPORTED, what + " setup: " + e.what());
  }
  if (plan.max_ytiles > dpgo::nd_ycap_tiles(p->r, p->dh) || plan.max_slots > dpgo::nd_slot_cap(p->r))
    return fail(DPGO_ERR_UNSUPPORTED, what + ": plan exceeds the shared-memory capacities");
  if ((int)plan.phases.size() > dpgo::nd::MAX_PHASES)
    return fail(DPGO_ERR_UNSUPPORTED, what + ": too many phases");
  dpgo::KNd &K = F.k;
  nd_kernel_sizes(plan, K);
  try {
    // grid mode only: agents stepped side by side as clusters are slower with the resident columns than with L1 (16-agent
    // sphere2500 / torus3D on one H100 80GB HBM3 at 400 W: 6818-6878 / 7689-7729 rounds/s against 7177-7222 / 7819-7855)
    nd::assign_residency(plan, dpgo::OPT_THREADS / 32, p->cluster ? 0 : dpgo::nd_resident_budget(p->r, p->dh, K));
  } catch (const std::exception &e) {
    return fail(DPGO_ERR_UNSUPPORTED, what + " setup: " + e.what());
  }
  K.resident_doubles = plan.max_resident_doubles;
  nd_fill_info(*H, plan, F.info);
  F.H = std::move(H);
  for (size_t k = 0; k < plan.phases.size(); ++k) { K.dir[k] = plan.phases[k].dir; K.cta0[k] = plan.phases[k].cta0; }
  DPGO_CUDA(F.cta_phase.assign(plan.cta_phase.data(), plan.cta_phase.size(), p->stream));
  DPGO_CUDA(F.steps.assign(plan.steps.data(), plan.steps.size(), p->stream));
  DPGO_CUDA(F.gathers.assign(plan.gathers.data(), plan.gathers.size(), p->stream));
  DPGO_CUDA(F.jobs.assign(plan.jobs.data(), plan.jobs.size(), p->stream));
  DPGO_CUDA(F.epis.assign(plan.epis.data(), plan.epis.size(), p->stream));
  DPGO_CUDA(F.csrc.assign(plan.csrc.data(), plan.csrc.size(), p->stream));
  if (dense) {
    // the refactorisation writes every panel row a front pose owns; the padding rows keep these zeros
    DPGO_CUDA(F.blob.alloc((size_t)F.H->blob_doubles));
    DPGO_CUDA(cudaMemsetAsync(F.blob.get(), 0, sizeof(double) * (size_t)F.H->blob_doubles, p->stream));
  } else {
    DPGO_CUDA(F.blob.assign(blob.data(), blob.size(), p->stream));
  }
  K.cta_phase = F.cta_phase.get(); K.steps = F.steps.get(); K.gathers = F.gathers.get(); K.jobs = F.jobs.get();
  K.epis = F.epis.get(); K.csrc = F.csrc.get(); K.blob = F.blob.get();
  const size_t tile = (size_t)p->ts;
  DPGO_CUDA(F.TX.alloc(tile * (size_t)p->n));
  DPGO_CUDA(F.C.alloc(tile * (size_t)F.H->cbuf_tiles));
  K.TX = F.TX.get();
  K.C = F.C.get();
  DPGO_CUDA(cudaMemsetAsync(K.TX, 0, sizeof(double) * tile * (size_t)p->n, p->stream));
  DPGO_CUDA(cudaMemsetAsync(K.C, 0, sizeof(double) * tile * (size_t)F.H->cbuf_tiles, p->stream));
  if (dense) {
    DPGO_TRY(ensure_refactor(p, slot));
    DPGO_TRY(launch_refactor(p, slot));
  }
  DPGO_CUDA(cudaStreamSynchronize(p->stream));
  K.nphases = (int)plan.phases.size();
  F.ready = true;
  ++p->generation;
  return DPGO_OK;
}

// block-Jacobi inverse blocks (Q_jj + 0.1 I)^-1, stored [k][c] padded
void jacobi_blocks(int n, int dh, const std::vector<int> &rowptr, const std::vector<int> &bcol, const std::vector<double> &bval,
                   std::vector<double> &dinv) {
  dinv.assign((size_t)n * 16, 0.0);
  for (int j = 0; j < n; ++j) {
    double A[4][8];
    for (int k = 0; k < 4; ++k)
      for (int c = 0; c < 8; ++c) A[k][c] = (c >= 4 && c - 4 == k) ? 1.0 : 0.0;
    for (int k = 0; k < dh; ++k) A[k][k] = 0.1;
    for (int k = dh; k < 4; ++k) A[k][k] = 1.0;
    for (int b = rowptr[j]; b < rowptr[j + 1]; ++b)
      if (bcol[b] == j)
        for (int k = 0; k < dh; ++k)
          for (int c = 0; c < dh; ++c) A[k][c] += bval[(size_t)b * 16 + k * 4 + c];
    for (int k = 0; k < 4; ++k) {          // Gauss-Jordan, SPD so no pivoting
      const double inv = 1.0 / A[k][k];
      for (int c = 0; c < 8; ++c) A[k][c] *= inv;
      for (int i = 0; i < 4; ++i)
        if (i != k) {
          const double f = A[i][k];
          for (int c = 0; c < 8; ++c) A[i][c] -= f * A[k][c];
        }
    }
    for (int k = 0; k < dh; ++k)
      for (int c = 0; c < dh; ++c) dinv[(size_t)j * 16 + k * 4 + c] = A[k][4 + c];
  }
}

}  // namespace dpgo::capi

using namespace dpgo::capi;

extern "C" {

int dpgo_nd_info(dpgo_problem_t *p, int64_t *info16) {
  DPGO_CHECK_HANDLE(p);
  DPGO_REQUIRE(info16, DPGO_ERR_INVALID_ARG, "null argument");
  DPGO_REQUIRE(p->bsr.have, DPGO_ERR_STATE, "set_Q has not been called");
  DPGO_TRY(ensure_nd(p, ND_SPARSE));
  std::copy(p->nd[ND_SPARSE].info, p->nd[ND_SPARSE].info + 16, info16);
  return DPGO_OK;
}

int dpgo_nd_node_sizes(dpgo_problem_t *p, int64_t cap, int32_t *own, int32_t *bnd, int32_t *stage, int64_t *count) {
  DPGO_CHECK_HANDLE(p);
  DPGO_REQUIRE(count && cap >= 0 && (cap == 0 || (own && bnd && stage)), DPGO_ERR_INVALID_ARG, "null argument");
  DPGO_REQUIRE(p->bsr.have, DPGO_ERR_STATE, "set_Q has not been called");
  DPGO_TRY(ensure_nd(p, ND_SPARSE));
  const auto &nodes = p->nd[ND_SPARSE].H->nodes;
  *count = (int64_t)nodes.size();
  for (size_t q = 0; q < nodes.size() && (int64_t)q < cap; ++q) {
    own[q] = (int32_t)nodes[q].own.size();
    bnd[q] = (int32_t)nodes[q].bnd.size();
    stage[q] = nodes[q].stage;
  }
  return DPGO_OK;
}

int dpgo_nd_debug_emulate(int n, int d, int r, int64_t nb, const int32_t *brow, const int32_t *bcol, const double *blocks,
                          double shift, int grid, int force_cuts, int leaf_size, const double *V_host, double *Z_host,
                          int64_t *info16) {
  DPGO_REQUIRE(n >= 1 && (d == 2 || d == 3) && r >= 1 && r <= 8 && grid >= 1, DPGO_ERR_INVALID_ARG, "bad dimensions");
  DPGO_REQUIRE(nb >= 0 && (nb == 0 || (brow && bcol && blocks)) && V_host && Z_host, DPGO_ERR_INVALID_ARG, "null argument");
  const int dh = d + 1;
  std::vector<BlockTriplet> trip;
  DPGO_TRY(blocks_to_triplets(n, dh, nb, brow, bcol, blocks, trip));
  std::vector<int> rowptr, bc;
  std::vector<double> bv;
  assemble_bsr(n, trip, rowptr, bc, bv);
  namespace nd = dpgo::nd;
  try {
    nd::Options opt = nd_options(grid, r, dh);
    opt.force_ncuts = force_cuts;
    opt.shift = shift;
    if (leaf_size > 0) opt.leaf_size = leaf_size;
    nd::BsrView Q{n, dh, rowptr.data(), bc.data(), bv.data()};
    nd::Hierarchy H;
    nd::Plan plan;
    std::vector<double> blob;
    nd::build_hierarchy(Q, opt, H);
    nd::build_numeric(Q, opt, H, blob);
    nd::build_plan(H, opt, plan);
    if (plan.max_ytiles > opt.ycap_tiles || plan.max_slots > opt.slot_cap)
      return fail(DPGO_ERR_UNSUPPORTED, "plan exceeds the shared-memory capacities");
    // residency as a launch of this plan would have it, or with DPGO_ND_RESIDENT_BYTES per CTA (verification)
    dpgo::KNd K = {};
    nd_kernel_sizes(plan, K);
    int64_t budget = dpgo::nd_resident_budget(r, dh, K);
    if (const char *e = std::getenv("DPGO_ND_RESIDENT_BYTES")) budget = std::atoll(e);
    nd::assign_residency(plan, opt.warps, budget);
    nd::emulate_apply(H, plan, blob, r, V_host, Z_host);
    if (info16) nd_fill_info(H, plan, info16);
    if (const char *dump = std::getenv("DPGO_ND_DUMP_JOBS")) {            // residency of every job, CSV
      if (FILE *fp = std::fopen(dump, "w")) {
        std::fprintf(fp, "phase,cta,step,warp,ncols,nres,soff,budget\n");
        for (size_t ph = 0; ph < plan.phases.size(); ++ph)
          for (int c = 0; c < plan.grid; ++c) {
            const nd::CtaPhase &cp = plan.cta_phase[(size_t)plan.phases[ph].cta0 + c];
            for (int si = cp.s0; si < cp.s1; ++si)
              for (int j = plan.steps[(size_t)si].j0; j < plan.steps[(size_t)si].j1; ++j) {
                const nd::Job &jb = plan.jobs[(size_t)j];
                std::fprintf(fp, "%zu,%d,%d,%d,%d,%d,%d,%lld\n", ph, c, si, (j - plan.steps[(size_t)si].j0) % opt.warps, jb.ncols,
                             jb.nres, jb.soff, (long long)budget);
              }
          }
        std::fclose(fp);
      }
    }
  } catch (const std::exception &e) {
    return fail(DPGO_ERR_UNSUPPORTED, std::string("sparse exact preconditioner: ") + e.what());
  }
  return DPGO_OK;
}

}  // extern "C"
