// dpgo_capi.cu -- implementation of the C ABI in include/dpgo_b200.h (host side of the library:
// handle management, CSR -> block-CSR conversion, preconditioner setup, H2D/D2H staging, launches).
// No CPU compute fallback exists here: every numeric entry point runs the sm_90a kernels.
#include <cuda_runtime.h>
#include <algorithm>
#include <chrono>
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <memory>
#include <numeric>
#include <string>
#include <vector>

#include "dpgo_devbuf.cuh"
#include "dpgo_kernels.cuh"

using dpgo::DevBuf;

namespace {

thread_local std::string g_last_error;

int fail(int code, const std::string &msg) {
  g_last_error = msg;
  return code;
}

#define DPGO_CUDA(call)                                                                           \
  do {                                                                                            \
    cudaError_t _e = (call);                                                                      \
    if (_e != cudaSuccess)                                                                        \
      return fail(DPGO_ERR_CUDA, std::string(#call) + ": " + cudaGetErrorString(_e));             \
  } while (0)

#define DPGO_REQUIRE(cond, code, msg) \
  do {                                \
    if (!(cond)) return fail(code, msg); \
  } while (0)

#define DPGO_TRY(expr)            \
  do {                            \
    int _s = (expr);              \
    if (_s != DPGO_OK) return _s; \
  } while (0)

// The two exact preconditioners apply the same operator P_X((Q + 0.1 I)^-1 V) with the same block solve: SPARSE_EXACT on
// the macro levels the cost model picks, DENSE_EXACT on a single one, whose root panels are the dense inverse of every
// connected component.  A launch reads the factorisation its preconditioner selects (the sparse one unless DENSE_EXACT).
enum NdSlot { ND_SPARSE = 0, ND_DENSE = 1 };
int nd_slot(int precond) { return precond == DPGO_PRECOND_DENSE_EXACT ? ND_DENSE : ND_SPARSE; }
int nd_precond(int slot) { return slot == ND_DENSE ? DPGO_PRECOND_DENSE_EXACT : DPGO_PRECOND_SPARSE_EXACT; }

}  // namespace

struct dpgo_problem {
  dpgo::Stream own_stream;       // declared first: destroyed after every buffer, event and graph below
  int n = 0, d = 0, r = 0, dh = 0, N = 0, ts = 0;
  int device = 0, sms = 0, grid = 0, max_grid = 0, max_cluster = 0;
  bool cluster = false;          // the persistent kernel runs as ONE thread-block cluster (small agents)
  cudaStream_t stream = nullptr;
  dpgo::Event ev_done, ev_fork;  // fork / join of the batched calls (fan_out)
  uint64_t generation = 0;       // bumped whenever device buffers a captured round refers to may have been replaced
  struct RoundGraph { std::vector<uint64_t> key; dpgo::GraphExec exec; int uses = 0; bool failed = false; };
  std::vector<RoundGraph> round_graphs;      // CUDA graphs of the batched round / host I/O calls, kept by the call's first agent
  template <class Job> struct JobTable { std::vector<uint64_t> key; DevBuf<Job> jobs; int ctas = 0; };
  int launch_mode = 0;           // 0: full cooperative grid, 1: one thread-block cluster
  // Q in block-CSR, its launch tables and its host copy (lazy preconditioner setup): build_from_triplets
  struct BlockQ {
    int64_t nb = 0;
    bool have = false;
    unsigned precond_mask = 0;
    DevBuf<int> rowptr, bcol, cta_rows;
    DevBuf<int2> groups;         // row groups of the TMA-fed SpMV
    int ngroups = 0;
    DevBuf<double> bval, dinv, partials;
    std::vector<int> h_rowptr, h_bcol;
    std::vector<double> h_bval;
    bool h_stale = false;        // an asynchronous re-weight changed bval on the device only (sync_host_bval)
  } bsr;
  // the exact preconditioners: one nested-dissection block factorisation of Q + 0.1 I per kind (ensure_nd), nd[ND_SPARSE]
  // on the cost model's macro levels, nd[ND_DENSE] on a single one; dropped by set_Q / a synchronous re-weight, refactorised
  // in place by an asynchronous one
  struct Nd {
    bool ready = false;
    dpgo::KNd k = {};            // kernel view of the buffers below
    DevBuf<dpgo::nd::CtaPhase> cta_phase;
    DevBuf<dpgo::nd::Step> steps;
    DevBuf<dpgo::nd::Gather> gathers;
    DevBuf<dpgo::nd::Job> jobs;
    DevBuf<dpgo::nd::Epi> epis;
    DevBuf<int> csrc;
    DevBuf<double> blob, TX, C;
    std::unique_ptr<dpgo::nd::Hierarchy> H;
    int64_t info[16] = {};
    // device refactorisation of the blob (ensure_refactor): scatter maps, fronts, sweep workspace and jobs of H
    std::unique_ptr<dpgo::nd::Refactor> R;
    DevBuf<dpgo::nd::RefactorNode> rnodes;
    DevBuf<dpgo::nd::RefactorChild> rchild;
    DevBuf<int> rposes, rcmap;
    DevBuf<double> arena, ws;
    DevBuf<dpgo::GjJob> rjobs;
  } nd[2];
  // edge records for the device-side Q assembly / robust re-weighting (dpgo_problem_set_edges)
  struct Edges {
    int64_t ne = 0;
    DevBuf<int> p1, p2, fixed, cptr;
    DevBuf<int2> contrib;
    DevBuf<double> T, om, w, sblk, res;
    DevBuf<unsigned long long> gnc;   // GNC counts of the last re-weight: weight 1, 0, in between (non-fixed edges)
    DevBuf<int> fail;                 // set by a device refactorisation whose matrix was not positive definite
    bool fail_armed = false;          // an asynchronous re-weight ran since the flag was last read
  } edges;
  // vectors
  DevBuf<double> G, vec[dpgo::V_COUNT], S[2];
  DevBuf<unsigned> bar;          // [0] arrival counter, [1] epoch
  DevBuf<unsigned long long> phase_ns;       // diagnostic phase clock (64 slots), allocated on request
  DevBuf<dpgo_opt_result_t> result;
  std::unique_ptr<dpgo_opt_result_t, dpgo::CudaFreeHost> h_result;   // pinned
  bool async_pending = false;
  std::chrono::high_resolution_clock::time_point async_t0;
  // exchange: the public poses (dpgo_agent_set_public_poses) and the shared edges (dpgo_agent_set_shared_edges)
  struct Public {
    int num = 0;
    DevBuf<int> pose, slot;      // slot: n, the public slot of each pose, -1 when the pose is not public
    bool slot_unique = true;     // no pose is listed twice (the accelerated rounds pack through slot)
  } pub;
  struct Shared {
    int num_edges = 0, num_poses = 0, max_slot = -1;
    DevBuf<int> pose_ids, pose_ptr, slot, out;
    DevBuf<double> T, om;
  } shared;
  bool G_dirty = true;           // G may hold values that dpgo_agent_build_G does not overwrite
  // distributed initialisation (dpgo_align.cu): local-frame trajectory, lift, alignment candidates, result
  DevBuf<double> Tloc, ylift;
  struct Align {
    int groups = 0, cands = 0, max_slot = -1, max_nbr = -1;
    DevBuf<int> grp_nbr, grp_ptr, cand_local, cand_slot, cand_out;
    DevBuf<double> cand_T, cand_R, cand_t, cand_w;
  } align;
  DevBuf<double> T_align;
  DevBuf<int> align_info;
  std::vector<JobTable<dpgo::AlignJob>> align_tables;   // job tables of dpgo_agents_align_async, kept by the call's first agent
  DevBuf<int> ready;
  int ready_cap = 0;
  dpgo::Event ev_align;                    // recorded on the stream of the last dpgo_agents_align_async that aligned this agent
  // team status (dpgo_status.cu): last optimising call's relative change + count, per-CTA partials, ticket of the last CTA
  struct Status {
    DevBuf<double> opt_record, part;
    DevBuf<unsigned> ticket;
    std::vector<JobTable<dpgo::StatusJob>> tables;   // job tables of dpgo_agents_status_async, kept by the call's first agent
  } status;
  DevBuf<double> anchor, traj;   // dpgo_agent_trajectory_global
  // accelerated rounds: Y, V, XPrev (allocated by accel_init); (dpgo_accel.cu) momentum record + ticket on the device; the
  // host's count of begun rounds and the restart rule of the last begin, which decide whether the agent's next
  // dpgo_agents_accel_round_async restarts
  struct Accel {
    DevBuf<double> vec[3], state;
    DevBuf<double> part;         // accel_ctas(n) per-CTA partials of the finish launch's |X - XPrev|^2
    DevBuf<unsigned> ticket;     // [0] begin launch, [1] finish launch (the finish runs on the agent's own stream)
    long long rounds = 0;
    bool restart_due = false;
    std::vector<JobTable<dpgo::AccelJob>> tables;    // job tables of dpgo_agents_accel_begin_async, kept by the call's first agent
  } acc;
  // greedy independent-set rounds (dpgo_select.cu), kept by the first agent of a runner on a GPU: the agent graph in CSR
  // form, the round's k-byte mask, and the selection log (cap rounds of k bytes; rounds issued, the device counts
  // its own rows).  A grown log retires the old buffer until the next read of the log or the handle's destruction.
  struct Select {
    int k = 0;
    DevBuf<int> ptr, adj;
    DevBuf<unsigned char> mask, log;
    DevBuf<unsigned long long> count;
    long long rounds = 0, cap = 0;
    std::vector<DevBuf<unsigned char>> retired;
  } sel;
  const unsigned char *gate = nullptr;     // set for the duration of a gated round: this agent's byte of the mask

  size_t vec_bytes() const { return sizeof(double) * (size_t)r * (size_t)N; }
};

namespace {

void fill_kparams(const dpgo_problem *p, dpgo::KParams &kp, int op, const dpgo_opt_params_t &prm) {
  kp.n = p->n;
  kp.N = p->N;
  kp.grid = p->grid;
  kp.op = op;
  kp.rowptr = p->bsr.rowptr.get();
  kp.bcol = p->bsr.bcol.get();
  kp.bval = p->bsr.bval.get();
  kp.dinv = p->bsr.dinv.get();
  kp.cta_rows = p->bsr.cta_rows.get();
  kp.G = p->G.get();
  for (int i = 0; i < dpgo::V_COUNT; ++i) kp.v[i] = p->vec[i].get();
  for (int i = 0; i < 2; ++i) kp.S[i] = p->S[i].get();
  kp.partials = p->bsr.partials.get();
  kp.bar_counter = p->bar.get();
  kp.bar_epoch = p->bar.get() + 1;
  const dpgo_problem::Nd &F = p->nd[nd_slot(prm.precond)];
  kp.nd = F.k;
  if (!F.ready) kp.nd.nphases = 0;
  kp.cluster = p->cluster ? 1 : 0;
  kp.smem_doubles = 0;
  kp.phase_ns = p->phase_ns.get();
  kp.opt_record = p->status.opt_record.get();
  kp.gate = p->gate;
  kp.prm = prm;
  kp.result = p->result.get();
}

cudaError_t run_spmv(const dpgo_problem *p, const double *X, const double *G, double *out) {
  if (p->bsr.ngroups > 0)
    return dpgo::launch_spmv_tma(p->r, p->dh, p->bsr.ngroups, p->bsr.groups.get(), p->bsr.rowptr.get(), p->bsr.bcol.get(),
                                 p->bsr.bval.get(), X, G, out, p->sms, p->stream);
  return dpgo::launch_spmv(p->r, p->dh, p->n, p->bsr.rowptr.get(), p->bsr.bcol.get(), p->bsr.bval.get(), X, G, out, p->stream);
}

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

dpgo::nd::Options nd_options(int grid, int r, bool cluster = false) {
  dpgo::nd::Options opt;
  opt.grid = grid;
  opt.r = r;
  // a phase end is a hardware cluster barrier in cluster mode: deeper dissections pay off earlier (16 agents side by side
  // on one H100 SXM at 400 W: torus3D, 312 poses per agent, 7140-7260 rounds/s against 5540-5660 with the grid value
  // 3.5 us, and 1.0 us is no faster; sphere2500's 156-pose agents are best with 2.0 us as well)
  if (cluster) opt.t_phase_us = 2.0;
  opt.warps = dpgo::OPT_THREADS / 32;
  opt.ycap_tiles = dpgo::ND_YCAP_TILES;
  opt.slot_cap = dpgo::ND_SLOT_CAP;
  if (const char *e = std::getenv("DPGO_ND_CUTS")) opt.force_ncuts = std::atoi(e);
  return opt;
}

void free_nd(dpgo_problem *p) {
  ++p->generation;
  for (dpgo_problem::Nd &F : p->nd) F = {};
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
  for (size_t st = 0; st + 1 < R->stage0.size(); ++st)
    if (R->stage0[st + 1] - R->stage0[st] > 65535) return fail(DPGO_ERR_UNSUPPORTED, what + ": more than 65535 nodes in one stage");
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
    nd::Options opt = nd_options(p->grid, p->r, p->cluster);
    if (dense) opt.force_ncuts = 0;
    nd::BsrView Q{p->n, p->dh, p->bsr.h_rowptr.data(), p->bsr.h_bcol.data(), p->bsr.h_bval.data()};
    nd::build_hierarchy(Q, opt, *H);
    if (!dense) nd::build_numeric(Q, opt, *H, blob);
    nd::build_plan(*H, opt, plan);
  } catch (const std::exception &e) {
    return fail(DPGO_ERR_UNSUPPORTED, what + " setup: " + e.what());
  }
  if (plan.max_ytiles > dpgo::ND_YCAP_TILES || plan.max_slots > dpgo::ND_SLOT_CAP)
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

int check_precond(dpgo_problem *p, int precond) {
  if (precond < 0 || precond > 3) return fail(DPGO_ERR_INVALID_ARG, "unknown preconditioner id");
  if (precond == DPGO_PRECOND_SPARSE_EXACT || precond == DPGO_PRECOND_DENSE_EXACT) return ensure_nd(p, nd_slot(precond));
  if (precond == DPGO_PRECOND_BLOCK_JACOBI && !p->bsr.dinv)
    return fail(DPGO_ERR_STATE, "block-Jacobi preconditioner was not prepared by set_Q (precond_mask)");
  return DPGO_OK;
}

int run_op(dpgo_problem *p, int op, const dpgo_opt_params_t &prm) {
  DPGO_REQUIRE(p->bsr.have, DPGO_ERR_STATE, "set_Q has not been called");
  dpgo::KParams kp;
  fill_kparams(p, kp, op, prm);
  DPGO_CUDA(dpgo::launch_optimize(p->r, p->dh, kp, p->stream));
  return DPGO_OK;
}

// ---- host-side block assembly ---------------------------------------------------------------
struct BlockTriplet {
  int brow, bcol;      // Q sub-block at rows dh*brow.., cols dh*bcol..
  double v[16];        // padded 4x4, v[k*4+c] = Q[dh*brow+k, dh*bcol+c]
};

// block triplets -> block-CSR (rows = output tiles, duplicates summed in a fixed order)
void assemble_bsr(int n, const std::vector<BlockTriplet> &trip, std::vector<int> &rowptr, std::vector<int> &bcol,
                  std::vector<double> &bval) {
  // sort by (output tile = bcol, neighbour tile = brow); stable so duplicate summation order is fixed
  std::vector<int64_t> order(trip.size());
  std::iota(order.begin(), order.end(), 0);
  std::stable_sort(order.begin(), order.end(), [&](int64_t x, int64_t y) {
    if (trip[x].bcol != trip[y].bcol) return trip[x].bcol < trip[y].bcol;
    return trip[x].brow < trip[y].brow;
  });
  rowptr.assign((size_t)n + 1, 0);
  bcol.clear();
  bval.clear();
  bcol.reserve(trip.size());
  bval.reserve(trip.size() * 16);
  int last_j = -1, last_i = -1;
  for (int64_t o : order) {
    const BlockTriplet &t = trip[o];
    if (t.bcol == last_j && t.brow == last_i) {
      double *dst = &bval[bval.size() - 16];
      for (int e = 0; e < 16; ++e) dst[e] += t.v[e];
    } else {
      bcol.push_back(t.brow);
      bval.insert(bval.end(), t.v, t.v + 16);
      rowptr[t.bcol + 1]++;
      last_j = t.bcol;
      last_i = t.brow;
    }
  }
  for (int j = 0; j < n; ++j) rowptr[j + 1] += rowptr[j];
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

int build_from_triplets(dpgo_problem *p, std::vector<BlockTriplet> &trip, unsigned precond_mask) {
  const int n = p->n, dh = p->dh;
  std::vector<int> rowptr, bcol;
  std::vector<double> bval;
  assemble_bsr(n, trip, rowptr, bcol, bval);
  const int64_t nb = (int64_t)bcol.size();

  std::vector<double> dinv;
  if (precond_mask & (1u << DPGO_PRECOND_BLOCK_JACOBI)) jacobi_blocks(n, dh, rowptr, bcol, bval, dinv);

  // persistent-kernel grid and balanced row partition
  const int sg = (p->r > 4) ? 32 : ((p->r > 2) ? 16 : 8);
  const int rows_per_pass = (dpgo::OPT_THREADS / 32) * (32 / sg);
  int grid = p->max_grid;
  const bool dense = (precond_mask & ((1u << DPGO_PRECOND_DENSE_EXACT) | (1u << DPGO_PRECOND_SPARSE_EXACT))) != 0;
  if (!dense) grid = std::max(1, std::min(grid, (n + rows_per_pass - 1) / rows_per_pass));
  // Launch mode 1 (dpgo_problem_set_launch_mode): the step kernel runs as ONE thread-block cluster (<= 16 CTAs) whose
  // phase ends are hardware cluster barriers instead of the atomic-counter grid barrier.  For one agent alone this is
  // SLOWER than the full grid (10-16 SMs stream the preconditioner blocks more slowly than all of them;
  // scripts/phase_times.py --agents 8 / 16 compares the two); its point is that a cluster launch is not cooperative, so
  // the agents of a colour class run side by side on one GPU and the round captures into a CUDA graph
  // (dpgo_agents_round_async).
  p->cluster = false;
  if (p->max_cluster >= 8 && p->launch_mode == 1) {
    // (one CTA per 16 poses is enough: always taking 16 CTAs makes small agents slower)
    grid = std::max(1, std::min(p->max_cluster, (n + rows_per_pass - 1) / rows_per_pass));
    p->cluster = true;
  }
  std::vector<int> cta_rows(grid + 1, 0);
  {
    // cost model: blocks + constant epilogue weight per row
    const double wrow = 4.0;
    double total = 0.0;
    for (int j = 0; j < n; ++j) total += (rowptr[j + 1] - rowptr[j]) + wrow;
    double accw = 0.0;
    int ci = 1;
    for (int j = 0; j < n; ++j) {
      accw += (rowptr[j + 1] - rowptr[j]) + wrow;
      while (ci < grid && accw >= total * ci / grid) cta_rows[ci++] = j + 1;
    }
    while (ci <= grid) cta_rows[ci++] = n;
  }

  // upload
  cudaSetDevice(p->device);
  p->bsr = {};
  free_nd(p);
  dpgo_problem::BlockQ &B = p->bsr;
  B.h_rowptr = rowptr;
  B.h_bcol = bcol;
  B.h_bval = bval;
  // +8 ints of slack: the bulk-TMA windows are rounded out to 16 bytes
  DPGO_CUDA(B.rowptr.alloc((size_t)n + 1 + 8));
  DPGO_CUDA(B.bcol.alloc((size_t)std::max<int64_t>(nb, 1) + 8));
  DPGO_CUDA(cudaMemsetAsync(B.rowptr.get(), 0, sizeof(int) * (n + 1 + 8), p->stream));
  DPGO_CUDA(cudaMemsetAsync(B.bcol.get(), 0, sizeof(int) * (std::max<int64_t>(nb, 1) + 8), p->stream));
  DPGO_CUDA(B.bval.alloc(16 * (size_t)std::max<int64_t>(nb, 1)));
  DPGO_CUDA(B.cta_rows.assign(cta_rows.data(), cta_rows.size(), p->stream));
  DPGO_CUDA(B.partials.alloc((size_t)2 * grid * dpgo::NRED));
  DPGO_CUDA(B.rowptr.upload(rowptr.data(), (size_t)n + 1, p->stream));
  DPGO_CUDA(B.bcol.upload(bcol.data(), (size_t)nb, p->stream));
  DPGO_CUDA(B.bval.upload(bval.data(), 16 * (size_t)nb, p->stream));
  DPGO_CUDA(cudaMemsetAsync(B.partials.get(), 0, sizeof(double) * 2 * grid * dpgo::NRED, p->stream));
  if (!dinv.empty()) DPGO_CUDA(B.dinv.assign(dinv.data(), dinv.size(), p->stream));
  // row groups for the TMA-fed SpMV: consecutive rows, <= SPMV_GROUP_BLOCKS blocks and rows each
  {
    const int BT = dpgo::spmv_group_blocks();
    std::vector<int2> groups;
    bool ok = true;
    int rr = 0;
    while (rr < n) {
      const int start = rr;
      int blocks = 0;
      while (rr < n && (rr - start) < BT && blocks + (rowptr[rr + 1] - rowptr[rr]) <= BT) {
        blocks += rowptr[rr + 1] - rowptr[rr];
        ++rr;
      }
      if (rr == start) { ok = false; break; }        // a single row exceeds the stage: fall back to the gather kernel
      groups.push_back(make_int2(start, rowptr[start]));
    }
    if (ok && nb > 0) {
      groups.push_back(make_int2(n, (int)nb));
      DPGO_CUDA(B.groups.assign(groups.data(), groups.size(), p->stream));
      B.ngroups = (int)groups.size() - 1;
    }
  }
  DPGO_CUDA(cudaStreamSynchronize(p->stream));
  B.nb = nb;
  p->grid = grid;
  B.precond_mask = precond_mask;

  B.have = true;
  return DPGO_OK;
}

int upload_vec(dpgo_problem *p, int id, const double *host) {
  DPGO_CUDA(cudaMemcpyAsync(p->vec[id].get(), host, p->vec_bytes(), cudaMemcpyHostToDevice, p->stream));
  return DPGO_OK;
}
int download_vec(dpgo_problem *p, int id, double *host) {
  DPGO_CUDA(cudaMemcpyAsync(host, p->vec[id].get(), p->vec_bytes(), cudaMemcpyDeviceToHost, p->stream));
  return DPGO_OK;
}
// After the stream has been synchronised: report (once) a device refactorisation that met a matrix that was not positive
// definite.  Only read when an asynchronous re-weight ran since the last read.
int check_refactor_fail(dpgo_problem *p) {
  dpgo_problem::Edges &E = p->edges;
  if (!E.fail_armed) return DPGO_OK;
  E.fail_armed = false;
  int flag = 0;
  DPGO_CUDA(cudaMemcpy(&flag, E.fail.get(), sizeof(int), cudaMemcpyDeviceToHost));
  if (!flag) return DPGO_OK;
  DPGO_CUDA(cudaMemset(E.fail.get(), 0, sizeof(int)));
  return fail(DPGO_ERR_CUDA, "device refactorisation: Q + 0.1 I is not positive definite (negative edge weight?)");
}

int fetch_result(dpgo_problem *p) {
  DPGO_CUDA(cudaMemcpyAsync(p->h_result.get(), p->result.get(), sizeof(dpgo_opt_result_t), cudaMemcpyDeviceToHost, p->stream));
  DPGO_CUDA(cudaStreamSynchronize(p->stream));
  return check_refactor_fail(p);
}

#define DPGO_CHECK_HANDLE(p)                                                         \
  do {                                                                               \
    if (!(p)) return fail(DPGO_ERR_INVALID_ARG, "null problem handle");              \
    cudaError_t _e = cudaSetDevice((p)->device);                                     \
    if (_e != cudaSuccess) return fail(DPGO_ERR_CUDA, cudaGetErrorString(_e));       \
  } while (0)

}  // namespace

extern "C" {

int dpgo_abi_version(void) { return DPGO_B200_ABI_VERSION; }
const char *dpgo_last_error(void) { return g_last_error.c_str(); }

int dpgo_device_count(int *count) {
  DPGO_REQUIRE(count, DPGO_ERR_INVALID_ARG, "null count");
  int c = 0;
  cudaError_t e = cudaGetDeviceCount(&c);
  if (e != cudaSuccess) {
    *count = 0;
    return fail(DPGO_ERR_NO_DEVICE, std::string("cudaGetDeviceCount: ") + cudaGetErrorString(e));
  }
  *count = c;
  return DPGO_OK;
}

void dpgo_opt_params_default(dpgo_opt_params_t *p) {
  if (!p) return;
  p->algorithm = DPGO_ALG_RTR;        // ref: src/QuadraticOptimizer.cpp:22-28
  p->tr_iterations = 1;
  p->tr_max_inner = 50;
  p->precond = DPGO_PRECOND_SPARSE_EXACT;
  p->rgd_stepsize = 1e-3;
  p->tr_tolerance = 1e-2;
  p->tr_initial_radius = 1e1;
}

int dpgo_problem_create(int n, int d, int r, int device, dpgo_problem_t **out) {
  DPGO_REQUIRE(out, DPGO_ERR_INVALID_ARG, "null output handle");
  *out = nullptr;
  DPGO_REQUIRE(n >= 1, DPGO_ERR_INVALID_ARG, "n must be >= 1");
  DPGO_REQUIRE(n <= 100000000, DPGO_ERR_UNSUPPORTED, "n above 1e8 poses: element offsets are 32-bit in the kernels");
  DPGO_REQUIRE(d == 2 || d == 3, DPGO_ERR_UNSUPPORTED, "d must be 2 or 3");
  DPGO_REQUIRE(r >= d, DPGO_ERR_INVALID_ARG, "r must be >= d (ref: assert(r >= d), src/QuadraticProblem.cpp:19)");
  DPGO_REQUIRE((d == 3 && r <= 5) || (d == 2 && (r <= 3 || r == 5)), DPGO_ERR_UNSUPPORTED,
               "unsupported rank (compiled instantiations: d=3: r in 3..5; d=2: r in {2,3,5})");
  int count = 0;
  cudaError_t e = cudaGetDeviceCount(&count);
  if (e != cudaSuccess || count == 0)
    return fail(DPGO_ERR_NO_DEVICE, "no CUDA device available: the GPU path has no CPU fallback");
  DPGO_REQUIRE(device >= 0 && device < count, DPGO_ERR_NO_DEVICE, "device index out of range");
  DPGO_CUDA(cudaSetDevice(device));
  dpgo_problem *p = new (std::nothrow) dpgo_problem();
  if (!p) return fail(DPGO_ERR_ALLOC, "host allocation failed");
  p->n = n; p->d = d; p->r = r; p->dh = d + 1; p->N = (d + 1) * n; p->ts = r * (d + 1);
  {
    static uint64_t serial = 0;             // handles are created from one thread at a time (as the rest of this API)
    p->generation = (++serial) << 24;       // a recycled address never matches the key of a captured round
  }
  p->device = device;
  auto bail = [&](int code, const std::string &m) { dpgo_problem_destroy(p); return fail(code, m); };
  if (cudaDeviceGetAttribute(&p->sms, cudaDevAttrMultiProcessorCount, device) != cudaSuccess)
    return bail(DPGO_ERR_CUDA, "cudaDeviceGetAttribute failed");
  cudaStream_t own = nullptr;
  const cudaError_t se = cudaStreamCreateWithFlags(&own, cudaStreamNonBlocking);
  p->own_stream.reset(own);
  if (se != cudaSuccess) return bail(DPGO_ERR_CUDA, "cudaStreamCreate failed");
  p->stream = own;
  p->max_grid = dpgo::optimize_max_grid(r, d + 1, device);
  p->max_cluster = dpgo::optimize_max_cluster(r, d + 1, device);
  if (p->max_grid <= 0) return bail(DPGO_ERR_CUDA, "persistent kernel cannot be made resident on this device");
  const size_t vb = p->vec_bytes();
  for (int i = 0; i < dpgo::V_COUNT; ++i) {
    if (p->vec[i].alloc((size_t)r * p->N) != cudaSuccess) return bail(DPGO_ERR_ALLOC, "device allocation failed (vectors)");
    cudaMemsetAsync(p->vec[i].get(), 0, vb, p->stream);
  }
  if (p->G.alloc((size_t)r * p->N) != cudaSuccess) return bail(DPGO_ERR_ALLOC, "device allocation failed (G)");
  cudaMemsetAsync(p->G.get(), 0, vb, p->stream);
  for (int i = 0; i < 2; ++i) {
    if (p->S[i].alloc(9 * (size_t)n) != cudaSuccess) return bail(DPGO_ERR_ALLOC, "device allocation failed (S)");
    cudaMemsetAsync(p->S[i].get(), 0, sizeof(double) * 9 * (size_t)n, p->stream);
  }
  if (p->bar.alloc(2) != cudaSuccess) return bail(DPGO_ERR_ALLOC, "device allocation failed");
  cudaMemsetAsync(p->bar.get(), 0, 2 * sizeof(unsigned), p->stream);
  if (p->result.alloc(1) != cudaSuccess) return bail(DPGO_ERR_ALLOC, "device allocation failed");
  if (p->status.opt_record.alloc(2) != cudaSuccess || p->status.part.alloc(3 * (size_t)dpgo::status_ctas(n)) != cudaSuccess ||
      p->status.ticket.alloc(1) != cudaSuccess)
    return bail(DPGO_ERR_ALLOC, "device allocation failed (status)");
  cudaMemsetAsync(p->status.opt_record.get(), 0, 2 * sizeof(double), p->stream);
  cudaMemsetAsync(p->status.ticket.get(), 0, sizeof(unsigned), p->stream);
  dpgo_opt_result_t *pinned = nullptr;
  const cudaError_t he = cudaMallocHost(&pinned, sizeof(dpgo_opt_result_t));
  p->h_result.reset(pinned);
  if (he != cudaSuccess) return bail(DPGO_ERR_ALLOC, "pinned allocation failed");
  if (cudaStreamSynchronize(p->stream) != cudaSuccess) return bail(DPGO_ERR_CUDA, "device initialisation failed");
  // empty Q (ref: ctor calls setQ(SparseMatrix(N,N)), src/QuadraticProblem.cpp:23)
  std::vector<BlockTriplet> none;
  int s = build_from_triplets(p, none, 1u << DPGO_PRECOND_BLOCK_JACOBI);
  if (s != DPGO_OK) { std::string m = g_last_error; dpgo_problem_destroy(p); return fail(s, m); }
  *out = p;
  return DPGO_OK;
}

int dpgo_problem_destroy(dpgo_problem_t *p) {
  if (!p) return DPGO_OK;
  cudaSetDevice(p->device);
  if (p->stream) cudaStreamSynchronize(p->stream);
  delete p;
  return DPGO_OK;
}

int dpgo_problem_set_stream(dpgo_problem_t *p, void *cuda_stream) {
  DPGO_CHECK_HANDLE(p);
  DPGO_CUDA(cudaStreamSynchronize(p->stream));
  p->stream = cuda_stream ? (cudaStream_t)cuda_stream : p->own_stream.get();
  return DPGO_OK;
}

int dpgo_problem_sync(dpgo_problem_t *p) {
  DPGO_CHECK_HANDLE(p);
  DPGO_CUDA(cudaStreamSynchronize(p->stream));
  return check_refactor_fail(p);
}

int dpgo_problem_set_launch_mode(dpgo_problem_t *p, int mode) {
  DPGO_CHECK_HANDLE(p);
  DPGO_REQUIRE(mode >= -1 && mode <= 1, DPGO_ERR_INVALID_ARG, "launch mode must be -1 (default), 0 (grid) or 1 (cluster)");
  DPGO_REQUIRE(mode != 1 || p->max_cluster >= 8, DPGO_ERR_UNSUPPORTED, "this device cannot co-schedule a cluster of >= 8 CTAs of the step kernel");
  p->launch_mode = mode;
  return DPGO_OK;
}

int dpgo_problem_launch_info(const dpgo_problem_t *p, int *grid, int *cluster) {
  DPGO_REQUIRE(p, DPGO_ERR_INVALID_ARG, "null problem handle");
  if (grid) *grid = p->grid;
  if (cluster) *cluster = p->cluster ? 1 : 0;
  return DPGO_OK;
}

int dpgo_problem_dims(const dpgo_problem_t *p, int *n, int *d, int *r, int64_t *num_blocks) {
  DPGO_REQUIRE(p, DPGO_ERR_INVALID_ARG, "null problem handle");
  if (n) *n = p->n;
  if (d) *d = p->d;
  if (r) *r = p->r;
  if (num_blocks) *num_blocks = p->bsr.nb;
  return DPGO_OK;
}

int dpgo_problem_set_Q_csr(dpgo_problem_t *p, int nrows, const int32_t *rowptr, const int32_t *colind,
                           const double *values, unsigned precond_mask) {
  DPGO_CHECK_HANDLE(p);
  DPGO_REQUIRE(nrows == p->N, DPGO_ERR_INVALID_ARG, "Q must be (d+1)n x (d+1)n");
  DPGO_REQUIRE(rowptr, DPGO_ERR_INVALID_ARG, "null CSR row pointer");
  DPGO_REQUIRE(rowptr[0] == 0, DPGO_ERR_INVALID_ARG, "CSR row pointer must start at 0");
  for (int i = 0; i < nrows; ++i)
    if (rowptr[i + 1] < rowptr[i]) return fail(DPGO_ERR_INVALID_ARG, "CSR row pointer is not non-decreasing");
  DPGO_REQUIRE(rowptr[nrows] == 0 || (colind && values), DPGO_ERR_INVALID_ARG, "null CSR arrays");
  const int dh = p->dh;
  std::vector<BlockTriplet> trip;
  trip.reserve((size_t)rowptr[nrows] / (dh * dh) + 16);
  for (int ib = 0; ib < p->n; ++ib) {
    const size_t first = trip.size();
    for (int k = 0; k < dh; ++k) {
      const int rr = ib * dh + k;
      for (int q = rowptr[rr]; q < rowptr[rr + 1]; ++q) {
        const int cc = colind[q];
        if (cc < 0 || cc >= p->N) return fail(DPGO_ERR_INVALID_ARG, "column index out of range");
        const int jb = cc / dh, c = cc - jb * dh;
        size_t t = first;
        for (; t < trip.size(); ++t)
          if (trip[t].bcol == jb) break;
        if (t == trip.size()) {
          BlockTriplet bt;
          bt.brow = ib;
          bt.bcol = jb;
          std::memset(bt.v, 0, sizeof(bt.v));
          trip.push_back(bt);
        }
        trip[t].v[k * 4 + c] += values[q];
      }
    }
  }
  return build_from_triplets(p, trip, precond_mask);
}

int dpgo_problem_set_Q_blocks(dpgo_problem_t *p, int64_t nb, const int32_t *brow, const int32_t *bcol,
                              const double *blocks, unsigned precond_mask) {
  DPGO_CHECK_HANDLE(p);
  DPGO_REQUIRE(nb >= 0 && (nb == 0 || (brow && bcol && blocks)), DPGO_ERR_INVALID_ARG, "null block arrays");
  const int dh = p->dh;
  std::vector<BlockTriplet> trip((size_t)nb);
  for (int64_t q = 0; q < nb; ++q) {
    if (brow[q] < 0 || brow[q] >= p->n || bcol[q] < 0 || bcol[q] >= p->n)
      return fail(DPGO_ERR_INVALID_ARG, "block index out of range");
    trip[q].brow = brow[q];
    trip[q].bcol = bcol[q];
    std::memset(trip[q].v, 0, sizeof(trip[q].v));
    for (int k = 0; k < dh; ++k)
      for (int c = 0; c < dh; ++c) trip[q].v[k * 4 + c] = blocks[(size_t)q * dh * dh + k * dh + c];
  }
  return build_from_triplets(p, trip, precond_mask);
}

int dpgo_problem_set_G_dense(dpgo_problem_t *p, const double *G_host) {
  DPGO_CHECK_HANDLE(p);
  p->G_dirty = true;
  if (!G_host) {
    DPGO_CUDA(cudaMemsetAsync(p->G.get(), 0, p->vec_bytes(), p->stream));
  } else {
    DPGO_CUDA(cudaMemcpyAsync(p->G.get(), G_host, p->vec_bytes(), cudaMemcpyHostToDevice, p->stream));
  }
  DPGO_CUDA(cudaStreamSynchronize(p->stream));
  return DPGO_OK;
}

int dpgo_problem_set_G_csr(dpgo_problem_t *p, const int32_t *rowptr, const int32_t *colind, const double *values) {
  DPGO_CHECK_HANDLE(p);
  if (!rowptr) return dpgo_problem_set_G_dense(p, nullptr);
  std::vector<double> G((size_t)p->r * p->N, 0.0);
  for (int a = 0; a < p->r; ++a)
    for (int q = rowptr[a]; q < rowptr[a + 1]; ++q) {
      if (colind[q] < 0 || colind[q] >= p->N) return fail(DPGO_ERR_INVALID_ARG, "G column index out of range");
      G[(size_t)colind[q] * p->r + a] += values[q];
    }
  return dpgo_problem_set_G_dense(p, G.data());
}

// ---- evaluation ---------------------------------------------------------------------------------
static int eval_at(dpgo_problem_t *p, const double *X_host) {
  DPGO_REQUIRE(X_host, DPGO_ERR_INVALID_ARG, "null X");
  DPGO_TRY(upload_vec(p, dpgo::V_X0, X_host));
  dpgo_opt_params_t prm;
  dpgo_opt_params_default(&prm);
  prm.precond = DPGO_PRECOND_NONE;
  DPGO_TRY(run_op(p, dpgo::OP_EVAL, prm));
  return DPGO_OK;
}

int dpgo_problem_f(dpgo_problem_t *p, const double *X_host, double *f_out) {
  DPGO_CHECK_HANDLE(p);
  DPGO_REQUIRE(f_out, DPGO_ERR_INVALID_ARG, "null output");
  DPGO_TRY(eval_at(p, X_host));
  DPGO_TRY(fetch_result(p));
  *f_out = p->h_result->f_init;
  return DPGO_OK;
}

int dpgo_problem_egrad(dpgo_problem_t *p, const double *X_host, double *out_host) {
  DPGO_CHECK_HANDLE(p);
  DPGO_REQUIRE(out_host, DPGO_ERR_INVALID_ARG, "null output");
  DPGO_TRY(eval_at(p, X_host));
  DPGO_TRY(download_vec(p, dpgo::V_EG0, out_host));
  DPGO_CUDA(cudaStreamSynchronize(p->stream));
  return DPGO_OK;
}

int dpgo_problem_ehess(dpgo_problem_t *p, const double *V_host, double *out_host) {
  DPGO_CHECK_HANDLE(p);
  DPGO_REQUIRE(V_host && out_host, DPGO_ERR_INVALID_ARG, "null argument");
  DPGO_REQUIRE(p->bsr.have, DPGO_ERR_STATE, "set_Q has not been called");
  DPGO_TRY(upload_vec(p, dpgo::V_AUX, V_host));
  DPGO_CUDA(run_spmv(p, p->vec[dpgo::V_AUX].get(), nullptr, p->vec[dpgo::V_HD].get()));
  DPGO_TRY(download_vec(p, dpgo::V_HD, out_host));
  DPGO_CUDA(cudaStreamSynchronize(p->stream));
  return DPGO_OK;
}

int dpgo_problem_rgrad(dpgo_problem_t *p, const double *X_host, double *out_host, double *norm_out) {
  DPGO_CHECK_HANDLE(p);
  DPGO_TRY(eval_at(p, X_host));
  if (out_host) DPGO_TRY(download_vec(p, dpgo::V_RG0, out_host));
  DPGO_TRY(fetch_result(p));
  if (norm_out) *norm_out = p->h_result->gradnorm_init;
  return DPGO_OK;
}

int dpgo_problem_f_rgradnorm(dpgo_problem_t *p, const double *X_host, double *f_out, double *norm_out) {
  DPGO_CHECK_HANDLE(p);
  DPGO_TRY(eval_at(p, X_host));
  DPGO_TRY(fetch_result(p));
  if (f_out) *f_out = p->h_result->f_init;
  if (norm_out) *norm_out = p->h_result->gradnorm_init;
  return DPGO_OK;
}

int dpgo_problem_rhess(dpgo_problem_t *p, const double *X_host, const double *V_host, double *out_host) {
  DPGO_CHECK_HANDLE(p);
  DPGO_REQUIRE(X_host && V_host && out_host, DPGO_ERR_INVALID_ARG, "null argument");
  DPGO_TRY(upload_vec(p, dpgo::V_X0, X_host));
  DPGO_TRY(upload_vec(p, dpgo::V_AUX, V_host));
  dpgo_opt_params_t prm;
  dpgo_opt_params_default(&prm);
  prm.precond = DPGO_PRECOND_NONE;
  DPGO_TRY(run_op(p, dpgo::OP_RHESS, prm));
  DPGO_TRY(download_vec(p, dpgo::V_HD, out_host));
  DPGO_CUDA(cudaStreamSynchronize(p->stream));
  return DPGO_OK;
}

int dpgo_problem_precon(dpgo_problem_t *p, int precond, const double *X_host, const double *V_host, double *out_host) {
  DPGO_CHECK_HANDLE(p);
  DPGO_REQUIRE(X_host && V_host && out_host, DPGO_ERR_INVALID_ARG, "null argument");
  DPGO_TRY(check_precond(p, precond));
  DPGO_TRY(upload_vec(p, dpgo::V_X0, X_host));
  DPGO_TRY(upload_vec(p, dpgo::V_AUX, V_host));
  dpgo_opt_params_t prm;
  dpgo_opt_params_default(&prm);
  prm.precond = precond;
  DPGO_TRY(run_op(p, dpgo::OP_PRECON, prm));
  DPGO_TRY(download_vec(p, dpgo::V_Z, out_host));
  DPGO_CUDA(cudaStreamSynchronize(p->stream));
  return DPGO_OK;
}

int dpgo_manifold_tangent_project(dpgo_problem_t *p, const double *X_host, const double *Z_host, double *out_host) {
  return dpgo_problem_precon(p, DPGO_PRECOND_NONE, X_host, Z_host, out_host);
}

int dpgo_manifold_retract(dpgo_problem_t *p, const double *X_host, const double *eta_host, double *out_host) {
  DPGO_CHECK_HANDLE(p);
  DPGO_REQUIRE(X_host && eta_host && out_host, DPGO_ERR_INVALID_ARG, "null argument");
  DPGO_TRY(upload_vec(p, dpgo::V_X0, X_host));
  DPGO_TRY(upload_vec(p, dpgo::V_AUX, eta_host));
  dpgo_opt_params_t prm;
  dpgo_opt_params_default(&prm);
  prm.precond = DPGO_PRECOND_NONE;
  DPGO_TRY(run_op(p, dpgo::OP_RETRACT, prm));
  DPGO_TRY(download_vec(p, dpgo::V_X1, out_host));
  DPGO_CUDA(cudaStreamSynchronize(p->stream));
  return DPGO_OK;
}

int dpgo_manifold_project(dpgo_problem_t *p, const double *M_host, double *out_host) {
  DPGO_CHECK_HANDLE(p);
  DPGO_REQUIRE(M_host && out_host, DPGO_ERR_INVALID_ARG, "null argument");
  DPGO_TRY(upload_vec(p, dpgo::V_AUX, M_host));
  DPGO_CUDA(dpgo::launch_stiefel_project(p->r, p->dh, p->n, p->vec[dpgo::V_AUX].get(), p->vec[dpgo::V_T].get(), p->stream));
  DPGO_TRY(download_vec(p, dpgo::V_T, out_host));
  DPGO_CUDA(cudaStreamSynchronize(p->stream));
  return DPGO_OK;
}

// ---- optimiser -----------------------------------------------------------------------------------
static int check_params(dpgo_problem_t *p, const dpgo_opt_params_t *prm) {
  DPGO_REQUIRE(prm, DPGO_ERR_INVALID_ARG, "null params");
  DPGO_REQUIRE(prm->algorithm == DPGO_ALG_RTR || prm->algorithm == DPGO_ALG_RGD, DPGO_ERR_INVALID_ARG, "unknown algorithm");
  DPGO_REQUIRE(prm->tr_iterations >= 1 && prm->tr_max_inner >= 1, DPGO_ERR_INVALID_ARG, "iteration counts must be >= 1");
  DPGO_REQUIRE(prm->tr_initial_radius > 0 && prm->tr_tolerance >= 0, DPGO_ERR_INVALID_ARG, "bad radius / tolerance");
  if (prm->algorithm == DPGO_ALG_RTR) DPGO_TRY(check_precond(p, prm->precond));
  return DPGO_OK;
}

int dpgo_optimize(dpgo_problem_t *p, const dpgo_opt_params_t *params, const double *X_in_host, double *X_out_host,
                  dpgo_opt_result_t *result) {
  DPGO_CHECK_HANDLE(p);
  DPGO_REQUIRE(X_in_host && X_out_host, DPGO_ERR_INVALID_ARG, "null X");
  DPGO_TRY(check_params(p, params));
  const auto t0 = std::chrono::high_resolution_clock::now();
  DPGO_TRY(upload_vec(p, dpgo::V_X0, X_in_host));
  DPGO_TRY(run_op(p, dpgo::OP_OPTIMIZE, *params));
  DPGO_TRY(download_vec(p, dpgo::V_X0, X_out_host));
  DPGO_TRY(fetch_result(p));
  const auto t1 = std::chrono::high_resolution_clock::now();
  p->h_result->elapsed_ms = std::chrono::duration<double, std::milli>(t1 - t0).count();
  if (result) *result = *p->h_result;
  return DPGO_OK;
}

int dpgo_problem_upload_X(dpgo_problem_t *p, const double *X_host) {
  DPGO_CHECK_HANDLE(p);
  DPGO_REQUIRE(X_host, DPGO_ERR_INVALID_ARG, "null X");
  DPGO_TRY(upload_vec(p, dpgo::V_X0, X_host));
  DPGO_CUDA(cudaStreamSynchronize(p->stream));
  return DPGO_OK;
}

int dpgo_problem_download_X(dpgo_problem_t *p, double *X_host) {
  DPGO_CHECK_HANDLE(p);
  DPGO_REQUIRE(X_host, DPGO_ERR_INVALID_ARG, "null X");
  DPGO_TRY(download_vec(p, dpgo::V_X0, X_host));
  DPGO_CUDA(cudaStreamSynchronize(p->stream));
  return DPGO_OK;
}

int dpgo_problem_upload_X_async(dpgo_problem_t *p, const double *X_host) {
  DPGO_CHECK_HANDLE(p);
  DPGO_REQUIRE(X_host, DPGO_ERR_INVALID_ARG, "null X");
  return upload_vec(p, dpgo::V_X0, X_host);
}

int dpgo_problem_download_X_async(dpgo_problem_t *p, double *X_host) {
  DPGO_CHECK_HANDLE(p);
  DPGO_REQUIRE(X_host, DPGO_ERR_INVALID_ARG, "null X");
  return download_vec(p, dpgo::V_X0, X_host);
}

int dpgo_problem_copy_X_from_device(dpgo_problem_t *p, const double *X_dev) {
  DPGO_CHECK_HANDLE(p);
  DPGO_REQUIRE(X_dev, DPGO_ERR_INVALID_ARG, "null X");
  DPGO_CUDA(cudaMemcpyAsync(p->vec[dpgo::V_X0].get(), X_dev, p->vec_bytes(), cudaMemcpyDeviceToDevice, p->stream));
  return DPGO_OK;
}

int dpgo_problem_device_X(dpgo_problem_t *p, double **X_dev) {
  DPGO_REQUIRE(p && X_dev, DPGO_ERR_INVALID_ARG, "null argument");
  *X_dev = p->vec[dpgo::V_X0].get();
  return DPGO_OK;
}

int dpgo_problem_device_G(dpgo_problem_t *p, double **G_dev) {
  DPGO_REQUIRE(p && G_dev, DPGO_ERR_INVALID_ARG, "null argument");
  *G_dev = p->G.get();
  p->G_dirty = true;             // the caller may write G directly
  return DPGO_OK;
}

int dpgo_optimize_resident_async(dpgo_problem_t *p, const dpgo_opt_params_t *params) {
  DPGO_CHECK_HANDLE(p);
  DPGO_TRY(check_params(p, params));
  p->async_t0 = std::chrono::high_resolution_clock::now();
  DPGO_TRY(run_op(p, dpgo::OP_OPTIMIZE, *params));
  p->async_pending = true;
  return DPGO_OK;
}

int dpgo_optimize_result(dpgo_problem_t *p, dpgo_opt_result_t *result) {
  DPGO_CHECK_HANDLE(p);
  DPGO_TRY(fetch_result(p));
  if (p->async_pending) {
    const auto t1 = std::chrono::high_resolution_clock::now();
    p->h_result->elapsed_ms = std::chrono::duration<double, std::milli>(t1 - p->async_t0).count();
    p->async_pending = false;
  }
  if (result) *result = *p->h_result;
  return DPGO_OK;
}

int dpgo_debug_phase_latency(dpgo_problem_t *p, int phases, double *us_per_phase, double *us_launch) {
  DPGO_CHECK_HANDLE(p);
  DPGO_REQUIRE(phases >= 1 && us_per_phase, DPGO_ERR_INVALID_ARG, "bad arguments");
  dpgo_opt_params_t prm;
  dpgo_opt_params_default(&prm);
  prm.precond = DPGO_PRECOND_NONE;
  dpgo::Event e0, e1;
  DPGO_CUDA(dpgo::create_event(e0, cudaEventDefault));
  DPGO_CUDA(dpgo::create_event(e1, cudaEventDefault));
  float ms[2] = {0, 0};
  const int counts[2] = {1, phases + 1};
  for (int rep = 0; rep < 2; ++rep) {
    prm.tr_max_inner = counts[rep];
    for (int w = 0; w < 3; ++w) DPGO_TRY(run_op(p, dpgo::OP_PHASE_BENCH, prm));
    DPGO_CUDA(cudaEventRecord(e0.get(), p->stream));
    for (int w = 0; w < 10; ++w) DPGO_TRY(run_op(p, dpgo::OP_PHASE_BENCH, prm));
    DPGO_CUDA(cudaEventRecord(e1.get(), p->stream));
    DPGO_CUDA(cudaEventSynchronize(e1.get()));
    DPGO_CUDA(cudaEventElapsedTime(&ms[rep], e0.get(), e1.get()));
  }
  *us_per_phase = 1e3 * (ms[1] - ms[0]) / 10.0 / phases;
  if (us_launch) *us_launch = 1e3 * ms[0] / 10.0 - *us_per_phase;
  return DPGO_OK;
}

int dpgo_debug_phase_times64(dpgo_problem_t *p, int enable, double *ms_by_kind) {
  DPGO_CHECK_HANDLE(p);
  if (enable && !p->phase_ns) {
    DPGO_CUDA(p->phase_ns.alloc(64));
    DPGO_CUDA(cudaMemsetAsync(p->phase_ns.get(), 0, 64 * sizeof(unsigned long long), p->stream));
  }
  if (p->phase_ns) {
    unsigned long long ns[64];
    DPGO_CUDA(cudaStreamSynchronize(p->stream));
    DPGO_CUDA(cudaMemcpy(ns, p->phase_ns.get(), sizeof(ns), cudaMemcpyDeviceToHost));
    if (ms_by_kind)
      for (int i = 0; i < 64; ++i) ms_by_kind[i] = 1e-6 * (double)ns[i];
    DPGO_CUDA(cudaMemset(p->phase_ns.get(), 0, sizeof(ns)));
    if (!enable) p->phase_ns = {};
  } else if (ms_by_kind) {
    for (int i = 0; i < 64; ++i) ms_by_kind[i] = 0.0;
  }
  return DPGO_OK;
}

int dpgo_spmv_device(dpgo_problem_t *p, const double *X_dev, double *out_dev, int add_G) {
  DPGO_CHECK_HANDLE(p);
  DPGO_REQUIRE(X_dev && out_dev, DPGO_ERR_INVALID_ARG, "null argument");
  DPGO_REQUIRE(p->bsr.have, DPGO_ERR_STATE, "set_Q has not been called");
  DPGO_CUDA(run_spmv(p, X_dev, add_G ? p->G.get() : nullptr, out_dev));
  return DPGO_OK;
}

int64_t dpgo_spmv_algorithmic_bytes(const dpgo_problem_t *p, int add_G) {
  if (!p) return 0;
  // SURVEY 8(d): nb*((d+1)^2*8 + 4) + (n+1)*4 + 2*r*(d+1)*n*8 (+ r*(d+1)*n*8 if G is read)
  const int64_t dh = p->dh;
  int64_t b = p->bsr.nb * (dh * dh * 8 + 4) + ((int64_t)p->n + 1) * 4 + 2 * (int64_t)p->r * dh * p->n * 8;
  if (add_G) b += (int64_t)p->r * dh * p->n * 8;
  return b;
}

int64_t dpgo_precond_algorithmic_bytes(const dpgo_problem_t *p, int preconditioner) {
  if (!p) return 0;
  const int64_t N = (int64_t)p->dh * p->n, vec = (int64_t)p->r * N * 8;
  if (preconditioner == DPGO_PRECOND_BLOCK_JACOBI) return (int64_t)p->n * 16 * 8 + 2 * vec;
  if (preconditioner != DPGO_PRECOND_SPARSE_EXACT && preconditioner != DPGO_PRECOND_DENSE_EXACT) return 0;
  const dpgo_problem::Nd &F = p->nd[nd_slot(preconditioner)];
  return F.ready ? F.info[4] + 2 * vec : 0;
}

int dpgo_nd_info(dpgo_problem_t *p, int64_t *info16) {
  DPGO_CHECK_HANDLE(p);
  DPGO_REQUIRE(info16, DPGO_ERR_INVALID_ARG, "null argument");
  DPGO_REQUIRE(p->bsr.have, DPGO_ERR_STATE, "set_Q has not been called");
  DPGO_TRY(ensure_nd(p, ND_SPARSE));
  std::copy(p->nd[ND_SPARSE].info, p->nd[ND_SPARSE].info + 16, info16);
  return DPGO_OK;
}

int dpgo_nd_debug_emulate(int n, int d, int r, int64_t nb, const int32_t *brow, const int32_t *bcol, const double *blocks,
                          double shift, int grid, int force_cuts, int leaf_size, const double *V_host, double *Z_host,
                          int64_t *info16) {
  DPGO_REQUIRE(n >= 1 && (d == 2 || d == 3) && r >= 1 && r <= 8 && grid >= 1, DPGO_ERR_INVALID_ARG, "bad dimensions");
  DPGO_REQUIRE(nb >= 0 && (nb == 0 || (brow && bcol && blocks)) && V_host && Z_host, DPGO_ERR_INVALID_ARG, "null argument");
  const int dh = d + 1;
  std::vector<BlockTriplet> trip((size_t)nb);
  for (int64_t q = 0; q < nb; ++q) {
    if (brow[q] < 0 || brow[q] >= n || bcol[q] < 0 || bcol[q] >= n) return fail(DPGO_ERR_INVALID_ARG, "block index out of range");
    trip[(size_t)q].brow = brow[q];
    trip[(size_t)q].bcol = bcol[q];
    std::memset(trip[(size_t)q].v, 0, sizeof(trip[(size_t)q].v));
    for (int k = 0; k < dh; ++k)
      for (int c = 0; c < dh; ++c) trip[(size_t)q].v[k * 4 + c] = blocks[(size_t)q * dh * dh + k * dh + c];
  }
  std::vector<int> rowptr, bc;
  std::vector<double> bv;
  assemble_bsr(n, trip, rowptr, bc, bv);
  namespace nd = dpgo::nd;
  try {
    nd::Options opt = nd_options(grid, r);
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

// ---- Q from edge records on the device, robust re-weighting -----------------------------------------------------
// weights (and the GNC counts) of the non-fixed edges at the resident iterate
static int launch_reweight(dpgo_problem *p, int cost, double mu, double param) {
  const dpgo_problem::Edges &E = p->edges;
  DPGO_CUDA(cudaMemsetAsync(E.gnc.get(), 0, 3 * sizeof(unsigned long long), p->stream));
  DPGO_CUDA(dpgo::launch_edge_weights(p->r, p->dh, E.ne, E.p1.get(), E.p2.get(), E.T.get(), E.om.get(), E.fixed.get(),
                                      p->vec[dpgo::V_X0].get(), cost, mu, param, E.w.get(), E.res.get(), E.gnc.get(), p->stream));
  return DPGO_OK;
}

static int reassemble_Q(dpgo_problem *p) {
  const dpgo_problem::Edges &E = p->edges;
  DPGO_CUDA(dpgo::launch_assemble_Q(p->bsr.nb, E.cptr.get(), E.contrib.get(), E.T.get(), E.om.get(), E.w.get(), E.sblk.get(),
                                    p->bsr.bval.get(), p->stream));
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
  DPGO_REQUIRE(cost >= 0 && cost <= 5, DPGO_ERR_INVALID_ARG, "unknown robust cost");
  DPGO_REQUIRE(cost != 5 || mu > 0, DPGO_ERR_INVALID_ARG, "GNC needs mu > 0");
  DPGO_TRY(launch_reweight(p, cost, mu, param));
  const dpgo_problem::Edges &E = p->edges;
  if (weights_host && E.ne)
    DPGO_CUDA(cudaMemcpyAsync(weights_host, E.w.get(), sizeof(double) * (size_t)E.ne, cudaMemcpyDeviceToHost, p->stream));
  if (residuals2_host && E.ne)
    DPGO_CUDA(cudaMemcpyAsync(residuals2_host, E.res.get(), sizeof(double) * (size_t)E.ne, cudaMemcpyDeviceToHost, p->stream));
  return reassemble_Q(p);
}

// ---- stream-ordered re-weighting: the preconditioners are refactorised on the device --------------------------------
// After k_assemble_Q on the stream: block-Jacobi and the prepared exact preconditioners refactorised on the device.  Only
// the first call after the sparse exact structure was dropped (or never built) runs host work and synchronises; an
// unprepared dense one stays lazy.
static int refresh_preconditioners_async(dpgo_problem *p) {
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

int dpgo_problem_set_edge_weights_async(dpgo_problem_t *p, const double *weights_dev) {
  DPGO_CHECK_HANDLE(p);
  DPGO_REQUIRE(weights_dev || p->edges.ne == 0, DPGO_ERR_INVALID_ARG, "null weights");
  DPGO_REQUIRE(p->edges.cptr, DPGO_ERR_STATE, "dpgo_problem_set_edges has not been called");
  const dpgo_problem::Edges &E = p->edges;
  if (E.ne)
    DPGO_CUDA(cudaMemcpyAsync(E.w.get(), weights_dev, sizeof(double) * (size_t)E.ne, cudaMemcpyDeviceToDevice, p->stream));
  DPGO_CUDA(dpgo::launch_assemble_Q(p->bsr.nb, E.cptr.get(), E.contrib.get(), E.T.get(), E.om.get(), E.w.get(), E.sblk.get(),
                                    p->bsr.bval.get(), p->stream));
  return refresh_preconditioners_async(p);
}

int dpgo_problem_robust_reweight_async(dpgo_problem_t *p, int cost, double mu, double param) {
  DPGO_CHECK_HANDLE(p);
  DPGO_REQUIRE(p->edges.cptr, DPGO_ERR_STATE, "dpgo_problem_set_edges has not been called");
  DPGO_REQUIRE(cost >= 0 && cost <= 5, DPGO_ERR_INVALID_ARG, "unknown robust cost");
  DPGO_REQUIRE(cost != 5 || mu > 0, DPGO_ERR_INVALID_ARG, "GNC needs mu > 0");
  DPGO_TRY(launch_reweight(p, cost, mu, param));
  const dpgo_problem::Edges &E = p->edges;
  DPGO_CUDA(dpgo::launch_assemble_Q(p->bsr.nb, E.cptr.get(), E.contrib.get(), E.T.get(), E.om.get(), E.w.get(), E.sblk.get(),
                                    p->bsr.bval.get(), p->stream));
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

// ---- plain device helpers ----------------------------------------------------------------------
int dpgo_device_set(int device) {
  DPGO_CUDA(cudaSetDevice(device));
  return DPGO_OK;
}
int dpgo_device_malloc(int device, size_t bytes, void **ptr) {
  DPGO_REQUIRE(ptr, DPGO_ERR_INVALID_ARG, "null argument");
  *ptr = nullptr;
  DPGO_CUDA(cudaSetDevice(device));
  DPGO_CUDA(cudaMalloc(ptr, std::max<size_t>(bytes, 8)));
  DPGO_CUDA(cudaMemset(*ptr, 0, std::max<size_t>(bytes, 8)));
  return DPGO_OK;
}
int dpgo_device_free(int device, void *ptr) {
  DPGO_CUDA(cudaSetDevice(device));
  if (ptr) DPGO_CUDA(cudaFree(ptr));
  return DPGO_OK;
}
int dpgo_stream_create(int device, void **cuda_stream) {
  DPGO_REQUIRE(cuda_stream, DPGO_ERR_INVALID_ARG, "null argument");
  DPGO_CUDA(cudaSetDevice(device));
  cudaStream_t s;
  DPGO_CUDA(cudaStreamCreateWithFlags(&s, cudaStreamNonBlocking));
  *cuda_stream = (void *)s;
  return DPGO_OK;
}
int dpgo_stream_destroy(int device, void *cuda_stream) {
  DPGO_CUDA(cudaSetDevice(device));
  if (cuda_stream) DPGO_CUDA(cudaStreamDestroy((cudaStream_t)cuda_stream));
  return DPGO_OK;
}
int dpgo_stream_synchronize(int device, void *cuda_stream) {
  DPGO_CUDA(cudaSetDevice(device));
  DPGO_CUDA(cudaStreamSynchronize((cudaStream_t)cuda_stream));
  return DPGO_OK;
}

// ---- boundary-pose exchange --------------------------------------------------------------------
int dpgo_agent_set_public_poses(dpgo_problem_t *p, int num_public, const int32_t *public_pose) {
  DPGO_CHECK_HANDLE(p);
  ++p->generation;
  DPGO_REQUIRE(num_public >= 0 && (num_public == 0 || public_pose), DPGO_ERR_INVALID_ARG, "bad public pose list");
  for (int s = 0; s < num_public; ++s)
    if (public_pose[s] < 0 || public_pose[s] >= p->n) return fail(DPGO_ERR_INVALID_ARG, "public pose index out of range");
  p->pub = {};
  std::vector<int> pub_slot((size_t)p->n, -1);
  for (int s = 0; s < num_public; ++s) {
    if (pub_slot[(size_t)public_pose[s]] >= 0) p->pub.slot_unique = false;
    else pub_slot[(size_t)public_pose[s]] = s;
  }
  p->pub.num = num_public;
  if (num_public) DPGO_CUDA(p->pub.pose.assign(public_pose, (size_t)num_public, p->stream));
  DPGO_CUDA(p->pub.slot.assign(pub_slot.data(), pub_slot.size(), p->stream));
  DPGO_CUDA(cudaStreamSynchronize(p->stream));
  return DPGO_OK;
}

int dpgo_agent_pack_public(dpgo_problem_t *p, double *send_dev) {
  DPGO_CHECK_HANDLE(p);
  DPGO_REQUIRE(send_dev || p->pub.num == 0, DPGO_ERR_INVALID_ARG, "null send buffer");
  DPGO_CUDA(dpgo::launch_pack_tiles(p->ts, p->pub.num, p->pub.pose.get(), p->vec[dpgo::V_X0].get(), send_dev, p->stream, p->gate));
  return DPGO_OK;
}

int dpgo_agent_set_shared_edges(dpgo_problem_t *p, int num_edges, const int32_t *local_pose, const int32_t *nbr_slot,
                                const int32_t *outgoing, const double *T, const double *omega) {
  DPGO_CHECK_HANDLE(p);
  ++p->generation;
  DPGO_REQUIRE(num_edges >= 0 && (num_edges == 0 || (local_pose && nbr_slot && outgoing && T && omega)),
               DPGO_ERR_INVALID_ARG, "bad shared edge arrays");
  const int dh = p->dh;
  for (int e = 0; e < num_edges; ++e)
    if (local_pose[e] < 0 || local_pose[e] >= p->n || nbr_slot[e] < 0)
      return fail(DPGO_ERR_INVALID_ARG, "shared edge index out of range");
  // group edges by local pose, keeping input order inside a pose (= reference accumulation order)
  std::vector<int> order(num_edges);
  std::iota(order.begin(), order.end(), 0);
  std::stable_sort(order.begin(), order.end(), [&](int x, int y) { return local_pose[x] < local_pose[y]; });
  std::vector<int> pose_ids, pose_ptr, slot(num_edges), outg(num_edges);
  std::vector<double> Ts((size_t)num_edges * dh * dh), oms((size_t)num_edges * dh);
  for (int q = 0; q < num_edges; ++q) {
    const int e = order[q];
    if (pose_ids.empty() || pose_ids.back() != local_pose[e]) {
      pose_ids.push_back(local_pose[e]);
      pose_ptr.push_back(q);
    }
    slot[q] = nbr_slot[e];
    outg[q] = outgoing[e] ? 1 : 0;
    std::memcpy(&Ts[(size_t)q * dh * dh], T + (size_t)e * dh * dh, sizeof(double) * dh * dh);
    std::memcpy(&oms[(size_t)q * dh], omega + (size_t)e * dh, sizeof(double) * dh);
  }
  pose_ptr.push_back(num_edges);
  p->shared = {};
  p->shared.num_edges = num_edges;
  p->G_dirty = true;
  p->shared.num_poses = (int)pose_ids.size();
  for (int e = 0; e < num_edges; ++e) p->shared.max_slot = std::max(p->shared.max_slot, (int)nbr_slot[e]);
  if (num_edges) {
    DPGO_CUDA(p->shared.pose_ids.assign(pose_ids.data(), pose_ids.size(), p->stream));
    DPGO_CUDA(p->shared.pose_ptr.assign(pose_ptr.data(), pose_ptr.size(), p->stream));
    DPGO_CUDA(p->shared.slot.assign(slot.data(), slot.size(), p->stream));
    DPGO_CUDA(p->shared.out.assign(outg.data(), outg.size(), p->stream));
    DPGO_CUDA(p->shared.T.assign(Ts.data(), Ts.size(), p->stream));
    DPGO_CUDA(p->shared.om.assign(oms.data(), oms.size(), p->stream));
  }
  DPGO_CUDA(cudaStreamSynchronize(p->stream));
  return DPGO_OK;
}

int dpgo_agent_build_G(dpgo_problem_t *p, const double *gathered_dev, int64_t num_slots) {
  DPGO_CHECK_HANDLE(p);
  DPGO_REQUIRE(gathered_dev || p->shared.num_edges == 0, DPGO_ERR_INVALID_ARG, "null gathered buffer");
  DPGO_REQUIRE((int64_t)p->shared.max_slot < num_slots || p->shared.num_edges == 0, DPGO_ERR_INVALID_ARG,
               "a shared edge refers to a slot beyond the gathered buffer (exchange plan / slot table mismatch)");
  // k_build_G assigns every tile of a pose with shared edges; the other tiles of G are zero and stay zero, so G is cleared
  // only when something else may have written it (set_G, a new edge table)
  if (p->G_dirty) {
    DPGO_CUDA(cudaMemsetAsync(p->G.get(), 0, p->vec_bytes(), p->stream));
    p->G_dirty = false;
  }
  const dpgo_problem::Shared &S = p->shared;
  if (S.num_edges)
    DPGO_CUDA(dpgo::launch_build_G(p->r, p->dh, S.num_poses, S.pose_ids.get(), S.pose_ptr.get(), S.slot.get(), S.out.get(),
                                   S.T.get(), S.om.get(), gathered_dev, p->G.get(), p->stream, p->gate));
  return DPGO_OK;
}

// ---- Nesterov acceleration on the resident iterate ----------------------------------------------------
#define DPGO_ACC_READY(p) DPGO_REQUIRE((p)->acc.vec[0], DPGO_ERR_STATE, "dpgo_agent_accel_init has not been called")
int dpgo_agent_accel_init(dpgo_problem_t *p) {
  DPGO_CHECK_HANDLE(p);
  // allocated once: captured round graphs keep these addresses
  for (int i = 0; i < 3; ++i) {
    if (!p->acc.vec[i]) DPGO_CUDA(p->acc.vec[i].alloc((size_t)p->r * p->N));
    DPGO_CUDA(cudaMemcpyAsync(p->acc.vec[i].get(), p->vec[dpgo::V_X0].get(), p->vec_bytes(), cudaMemcpyDeviceToDevice, p->stream));
  }
  if (!p->acc.state) DPGO_CUDA(p->acc.state.alloc(dpgo::ACCEL_STATE_DOUBLES));
  if (!p->acc.part) DPGO_CUDA(p->acc.part.alloc((size_t)dpgo::accel_ctas(p->n)));
  if (!p->acc.ticket) DPGO_CUDA(p->acc.ticket.alloc(2));
  DPGO_CUDA(cudaMemsetAsync(p->acc.state.get(), 0, sizeof(double) * dpgo::ACCEL_STATE_DOUBLES, p->stream));
  DPGO_CUDA(cudaMemsetAsync(p->acc.ticket.get(), 0, 2 * sizeof(unsigned), p->stream));
  p->acc.rounds = 0;
  p->acc.restart_due = false;
  return DPGO_OK;
}
int dpgo_agent_accel_begin(dpgo_problem_t *p, double alpha) {
  DPGO_CHECK_HANDLE(p);
  DPGO_ACC_READY(p);
  double *X = p->vec[dpgo::V_X0].get(), *Y = p->acc.vec[0].get(), *V = p->acc.vec[1].get(), *XP = p->acc.vec[2].get();
  DPGO_CUDA(cudaMemcpyAsync(XP, X, p->vec_bytes(), cudaMemcpyDeviceToDevice, p->stream));
  DPGO_CUDA(dpgo::launch_stiefel_project(p->r, p->dh, p->n, X, Y, p->stream, 1.0 - alpha, V, alpha));
  return DPGO_OK;
}
int dpgo_agent_accel_end(dpgo_problem_t *p, double gamma, int optimized) {
  DPGO_CHECK_HANDLE(p);
  DPGO_ACC_READY(p);
  double *X = p->vec[dpgo::V_X0].get(), *Y = p->acc.vec[0].get(), *V = p->acc.vec[1].get();
  if (!optimized) DPGO_CUDA(cudaMemcpyAsync(X, Y, p->vec_bytes(), cudaMemcpyDeviceToDevice, p->stream));
  DPGO_CUDA(dpgo::launch_stiefel_project(p->r, p->dh, p->n, V, V, p->stream, 1.0, X, gamma, Y, -gamma));
  return DPGO_OK;
}
int dpgo_agent_accel_restart_begin(dpgo_problem_t *p) {
  DPGO_CHECK_HANDLE(p);
  DPGO_ACC_READY(p);
  DPGO_CUDA(cudaMemcpyAsync(p->vec[dpgo::V_X0].get(), p->acc.vec[2].get(), p->vec_bytes(), cudaMemcpyDeviceToDevice, p->stream));
  return DPGO_OK;
}
int dpgo_agent_accel_restart_end(dpgo_problem_t *p) {
  DPGO_CHECK_HANDLE(p);
  DPGO_ACC_READY(p);
  for (int i = 0; i < 2; ++i)
    DPGO_CUDA(cudaMemcpyAsync(p->acc.vec[i].get(), p->vec[dpgo::V_X0].get(), p->vec_bytes(), cudaMemcpyDeviceToDevice, p->stream));
  return DPGO_OK;
}
int dpgo_agent_pack_public_aux(dpgo_problem_t *p, double *send_dev) {
  DPGO_CHECK_HANDLE(p);
  DPGO_ACC_READY(p);
  DPGO_REQUIRE(send_dev || p->pub.num == 0, DPGO_ERR_INVALID_ARG, "null send buffer");
  DPGO_CUDA(dpgo::launch_pack_tiles(p->ts, p->pub.num, p->pub.pose.get(), p->acc.vec[0].get(), send_dev, p->stream));
  return DPGO_OK;
}

}  // extern "C"

namespace {

int require_device() {
  int count = 0;
  if (cudaGetDeviceCount(&count) != cudaSuccess || count == 0) {
    cudaGetLastError();
    return fail(DPGO_ERR_NO_DEVICE, "no CUDA device available: the GPU path has no CPU fallback");
  }
  return DPGO_OK;
}

// The agent list of a batched call: at least one handle, none null, all on the first one's device (made current) and, for
// the calls that serve every agent with one launch (same_shape), all with its d and r.  The handles must be distinct: the
// batched calls keep per-agent device state (ticket counters, partial sums, momentum records, alignment buffers) that one
// call must not touch twice; an agent listed twice would share its ticket between two jobs and could leave it non-zero
// for good.
int check_agents(dpgo_problem_t *const *agents, int count, bool same_shape) {
  DPGO_TRY(require_device());
  DPGO_REQUIRE(agents && count >= 1, DPGO_ERR_INVALID_ARG, "no agents");
  const dpgo_problem *lead = agents[0];
  for (int i = 0; i < count; ++i) {
    const dpgo_problem *p = agents[i];
    DPGO_REQUIRE(p, DPGO_ERR_INVALID_ARG, "null problem handle");
    DPGO_REQUIRE(p->device == lead->device, DPGO_ERR_INVALID_ARG, "the agents of one call must live on one device");
    DPGO_REQUIRE(!same_shape || (p->d == lead->d && p->r == lead->r), DPGO_ERR_INVALID_ARG,
                 "the agents of one call must share d and r");
  }
  std::vector<const dpgo_problem_t *> h(agents, agents + count);
  std::sort(h.begin(), h.end());
  DPGO_REQUIRE(std::adjacent_find(h.begin(), h.end()) == h.end(), DPGO_ERR_INVALID_ARG, "an agent is listed twice");
  DPGO_CUDA(cudaSetDevice(lead->device));
  return DPGO_OK;
}

// The stream a batched call works on: `stream`, or for NULL the stream the first agent is set to.
cudaStream_t call_stream(const dpgo_problem *lead, void *stream) { return stream ? (cudaStream_t)stream : lead->stream; }

// What a call that fans out over its agents (fan_out) needs: its stream, the first agent's fork event and every agent's
// join event; and whether the call may be replayed as a CUDA graph: not on the legacy default stream, which cannot be
// captured, nor with DPGO_ROUND_GRAPH=0.
int fan_out_stream(dpgo_problem_t *const *agents, int count, void *stream, cudaStream_t &main, bool &graph) {
  static const bool enabled = [] { const char *e = std::getenv("DPGO_ROUND_GRAPH"); return !e || std::atoi(e) != 0; }();
  dpgo_problem *lead = agents[0];
  main = call_stream(lead, stream);
  graph = enabled && main != cudaStreamLegacy && main != nullptr;
  if (!lead->ev_fork) DPGO_CUDA(dpgo::create_event(lead->ev_fork));
  for (int i = 0; i < count; ++i)
    if (!agents[i]->ev_done) DPGO_CUDA(dpgo::create_event(agents[i]->ev_done));
  return DPGO_OK;
}

struct StreamSwap {                        // the handle's work goes to another stream for the duration of a call
  dpgo_problem *p; cudaStream_t saved;
  StreamSwap(dpgo_problem *q, cudaStream_t to) : p(q), saved(q->stream) { q->stream = to; }
  ~StreamSwap() { p->stream = saved; }
};

// Issues body(i, agents[i]) for every agent with the handle set to stream_of(agent): an agent on a stream of its own works
// between a fork from `main` and a join into it, side by side with the others; an agent on `main` works in list order.
template <class StreamOf, class Body>
int fan_out(dpgo_problem_t *const *agents, int count, cudaStream_t main, StreamOf stream_of, Body body) {
  dpgo_problem *lead = agents[0];
  DPGO_CUDA(cudaEventRecord(lead->ev_fork.get(), main));
  for (int i = 0; i < count; ++i) {
    dpgo_problem *p = agents[i];
    StreamSwap swap(p, stream_of(p));
    if (p->stream != main) DPGO_CUDA(cudaStreamWaitEvent(p->stream, lead->ev_fork.get(), 0));
    DPGO_TRY(body(i, p));
    if (p->stream != main) {
      DPGO_CUDA(cudaEventRecord(p->ev_done.get(), p->stream));
      DPGO_CUDA(cudaStreamWaitEvent(main, p->ev_done.get(), 0));
    }
  }
  return DPGO_OK;
}

// Replay a repeated multi-launch sequence as a CUDA graph.  The graphs live with `lead` (the first agent of the call),
// keyed by everything the captured launches depend on.  First use: eager (warms every lazily created resource);
// second use: captured while it is issued, instantiated and launched; later: one cudaGraphLaunch.
template <class Issue> int replay_or_issue(dpgo_problem *lead, const std::vector<uint64_t> &key, cudaStream_t main, Issue issue) {
  dpgo_problem::RoundGraph *entry = nullptr;
  for (auto &g : lead->round_graphs)
    if (g.key == key) { entry = &g; break; }
  if (!entry) {
    if (lead->round_graphs.size() >= 48) return issue();      // e.g. the greedy schedule on many agents: stay eager
    lead->round_graphs.emplace_back();
    entry = &lead->round_graphs.back();
    entry->key = key;
  }
  if (entry->exec) {
    DPGO_CUDA(cudaGraphLaunch(entry->exec.get(), main));
    return DPGO_OK;
  }
  if (entry->failed || entry->uses++ == 0) return issue();
  cudaGraph_t graph = nullptr;
  if (cudaStreamBeginCapture(main, cudaStreamCaptureModeThreadLocal) != cudaSuccess) {
    cudaGetLastError();
    entry->failed = true;
    return issue();
  }
  const int rc = issue();
  const cudaError_t ce = cudaStreamEndCapture(main, &graph);
  if (rc != DPGO_OK || ce != cudaSuccess || !graph) {
    cudaGetLastError();
    if (graph) cudaGraphDestroy(graph);
    entry->failed = true;
    return issue();
  }
  cudaGraphExec_t exec = nullptr;
  const cudaError_t ie = cudaGraphInstantiate(&exec, graph, 0);
  cudaGraphDestroy(graph);
  if (ie != cudaSuccess) {
    cudaGetLastError();
    entry->failed = true;
    return issue();
  }
  entry->exec.reset(exec);
  DPGO_CUDA(cudaGraphLaunch(exec, main));
  return DPGO_OK;
}

constexpr size_t JOB_TABLES_MAX = 32;

// The job table of an agent list is filled (fill(jobs) returns the CTA count) and uploaded once, stream-ordered, and kept in
// `tables` under `key`; a repeated call finds it, so the call is its kernel launches and nothing else and can be captured
// into a CUDA graph.  Past JOB_TABLES_MAX tables the oldest is freed.
template <class Job, class Fill>
int job_table(std::vector<dpgo_problem::JobTable<Job>> &tables, std::vector<uint64_t> &key, int count, cudaStream_t st,
              Fill fill, const dpgo_problem::JobTable<Job> *&tab) {
  for (const auto &t : tables)
    if (t.key == key) { tab = &t; return DPGO_OK; }
  if (tables.size() >= JOB_TABLES_MAX) {                   // a table may still be read by a launch in flight
    DPGO_CUDA(cudaDeviceSynchronize());
    tables.erase(tables.begin());
  }
  std::vector<Job> jobs((size_t)count);
  const int ctas = fill(jobs);
  DevBuf<Job> d_jobs;
  DPGO_CUDA(d_jobs.assign(jobs.data(), jobs.size(), st));
  tables.push_back({std::move(key), std::move(d_jobs), ctas});
  tab = &tables.back();
  return DPGO_OK;
}

// What the round calls prepare alike after check_agents: valid parameters for every agent, the call's stream and events,
// and whether the round may be replayed as a CUDA graph.
int round_preamble(dpgo_problem_t *const *agents, int num_active, const dpgo_opt_params_t *params, void *main_stream,
                   cudaStream_t &main, bool &graph) {
  bool capturable = true;
  for (int i = 0; i < num_active; ++i) {
    dpgo_problem *p = agents[i];
    DPGO_TRY(check_params(p, params));
    // a cooperative launch does not capture; a pending G clear or an unbuilt factorisation must run eagerly first
    const int slot = nd_slot(params->precond);
    if (!p->cluster || p->G_dirty || p->phase_ns || ((p->bsr.precond_mask & (1u << nd_precond(slot))) && !p->nd[slot].ready))
      capturable = false;
  }
  DPGO_TRY(fan_out_stream(agents, num_active, main_stream, main, graph));
  graph = graph && capturable;
  return DPGO_OK;
}

// The start of every key a batched call keeps a CUDA graph or a job table under: a tag that keeps the keys of different
// calls apart, then every agent's handle and generation.  The caller appends whatever else its cached work depends on.
std::vector<uint64_t> call_key(uint64_t tag, dpgo_problem_t *const *agents, int count) {
  std::vector<uint64_t> key{tag};
  for (int i = 0; i < count; ++i) {
    key.push_back((uint64_t)(uintptr_t)agents[i]);
    key.push_back(agents[i]->generation);
  }
  return key;
}

// The start of a round graph's key: call_key, the stream, the slot count and the parameters.  The caller appends the
// buffers its launches capture.
std::vector<uint64_t> round_key(uint64_t tag, dpgo_problem_t *const *agents, int num_active, const dpgo_opt_params_t *params,
                                cudaStream_t main, int64_t num_slots) {
  uint64_t w[(sizeof(*params) + 7) / 8] = {};
  std::memcpy(w, params, sizeof(*params));
  std::vector<uint64_t> key = call_key(tag, agents, num_active);
  key.push_back((uint64_t)(uintptr_t)main);
  key.push_back((uint64_t)num_slots);
  key.insert(key.end(), w, w + sizeof(w) / 8);
  return key;
}

// The stream_of of the round calls' fan_out: cluster agents step side by side on their own streams, full-grid agents in
// order on main.
auto round_streams(cudaStream_t main) {
  return [main](const dpgo_problem *p) { return p->cluster ? p->own_stream.get() : main; };
}

}  // namespace

extern "C" {

static int issue_round(dpgo_problem_t *const *agents, int num_active, const dpgo_opt_params_t *params,
                       const double *gathered_dev, int64_t num_slots, double *const *send_dev, cudaStream_t main,
                       int pack_after_join) {
  const int passes = pack_after_join ? 2 : 1;
  for (int pass = 0; pass < passes; ++pass) {
    DPGO_TRY(fan_out(agents, num_active, main, round_streams(main), [&](int i, dpgo_problem *p) -> int {
      if (pass == 0) {
        DPGO_TRY(dpgo_agent_build_G(p, gathered_dev, num_slots));
        DPGO_TRY(dpgo_optimize_resident_async(p, params));
      }
      return pass == passes - 1 ? dpgo_agent_pack_public(p, send_dev[i]) : DPGO_OK;
    }));
  }
  return DPGO_OK;
}

// One RBCD round of the agents of one GPU, issued with one call.  Per active agent: G rebuild from the gathered tiles -> RTR
// step -> pack of its public tiles.  Agents launched as single thread-block clusters (dpgo_problem_set_launch_mode(p, 1))
// work on their own streams between a fork from and a join into main, so up to 8 clusters of 16 CTAs share the GPU;
// full-grid agents run in order on main.  Agents of one colour class are never neighbours, so a pack into the (aliased)
// gathered buffer cannot race with another active agent's G rebuild; with pack_after_join != 0 (every agent active on the
// previous round's poses) the packs are issued in a second pass instead.
// A cluster round with the same agents, buffers and parameters as an earlier one is replayed as a CUDA graph (the cluster
// launches are ordinary launches, so the fork/join captures): 1 driver call per round instead of ~7 per agent, which is
// what bounds 8 agents x ~100 us of GPU work otherwise.  A round with a full-grid agent stays eager.
int dpgo_agents_round_async(dpgo_problem_t *const *agents, int num_active, const dpgo_opt_params_t *params,
                            const double *gathered_dev, int64_t num_slots, double *const *send_dev, void *main_stream,
                            int pack_after_join) {
  DPGO_REQUIRE(num_active >= 0 && (num_active == 0 || send_dev) && params, DPGO_ERR_INVALID_ARG, "bad arguments");
  if (num_active == 0) return DPGO_OK;
  DPGO_TRY(check_agents(agents, num_active, false));
  cudaStream_t main = nullptr;
  bool graph = false;
  DPGO_TRY(round_preamble(agents, num_active, params, main_stream, main, graph));
  auto issue = [&]() { return issue_round(agents, num_active, params, gathered_dev, num_slots, send_dev, main, pack_after_join); };
  if (!graph) return issue();
  std::vector<uint64_t> key = round_key(0x726e640000ull, agents, num_active, params, main, num_slots);   // "rnd"
  for (int i = 0; i < num_active; ++i) key.push_back((uint64_t)(uintptr_t)send_dev[i]);
  key.push_back((uint64_t)(uintptr_t)gathered_dev);
  key.push_back((uint64_t)pack_after_join);
  return replay_or_issue(agents[0], key, main, issue);
}

// The host boundary of a round with one call per direction (the end-to-end path of DistributedPGO.step_host):
//   direction 0: X of every listed agent from (pinned) host memory, then its public tiles packed into send_dev[i]
//   direction 1: X of every listed agent back to host memory
// all on `stream`; a repeated call (same agents, buffers, stream) is replayed as a CUDA graph of memcpy / kernel nodes.
int dpgo_agents_host_io_async(dpgo_problem_t *const *agents, int count, double *const *X_host, double *const *send_dev,
                              int direction, void *stream) {
  DPGO_REQUIRE(count >= 0 && (count == 0 || X_host) && (direction == 0 || direction == 1), DPGO_ERR_INVALID_ARG,
               "bad arguments");
  if (count == 0) return DPGO_OK;
  DPGO_TRY(check_agents(agents, count, false));
  for (int i = 0; i < count; ++i) DPGO_REQUIRE(X_host[i], DPGO_ERR_INVALID_ARG, "null host buffer");
  cudaStream_t main = nullptr;
  bool graph = false;
  DPGO_TRY(fan_out_stream(agents, count, stream, main, graph));
  // every agent's copy (+ pack) on its own stream: the copies of different agents overlap each other and the packs
  auto issue = [&]() {
    return fan_out(agents, count, main, [](dpgo_problem *p) { return p->own_stream.get(); }, [&](int i, dpgo_problem *p) -> int {
      if (direction == 1) return download_vec(p, dpgo::V_X0, X_host[i]);
      DPGO_TRY(upload_vec(p, dpgo::V_X0, X_host[i]));
      return send_dev && send_dev[i] ? dpgo_agent_pack_public(p, send_dev[i]) : DPGO_OK;
    });
  };
  if (!graph) return issue();
  std::vector<uint64_t> key = call_key(0x696f0000ull + (uint64_t)direction, agents, count);   // "io"
  for (int i = 0; i < count; ++i) {
    key.push_back((uint64_t)(uintptr_t)X_host[i]);
    key.push_back((uint64_t)(uintptr_t)((send_dev && direction == 0) ? send_dev[i] : nullptr));
  }
  key.push_back((uint64_t)(uintptr_t)main);
  return replay_or_issue(agents[0], key, main, issue);
}

int dpgo_agent_f_rgradnorm_resident(dpgo_problem_t *p, double *f_out, double *norm_out) {
  DPGO_CHECK_HANDLE(p);
  dpgo_opt_params_t prm;
  dpgo_opt_params_default(&prm);
  prm.precond = DPGO_PRECOND_NONE;
  DPGO_TRY(run_op(p, dpgo::OP_EVAL, prm));
  DPGO_TRY(fetch_result(p));
  if (f_out) *f_out = p->h_result->f_init;
  if (norm_out) *norm_out = p->h_result->gradnorm_init;
  return DPGO_OK;
}


// ---- distributed initialisation: frame alignment -------------------------------------------------------
namespace {
// Every buffer an AlignJob points to is allocated once, except the candidate table's: dpgo_agent_set_align_candidates
// replaces those and bumps the handle's generation, so a kept job table never points to freed memory.
dpgo::AlignJob align_job(const dpgo_problem *p) {
  const dpgo_problem::Align &A = p->align;
  dpgo::AlignJob J = {};
  J.ngroups = A.groups;
  J.n = p->n;
  J.grp_nbr = A.grp_nbr.get(); J.grp_ptr = A.grp_ptr.get();
  J.cand_local = A.cand_local.get(); J.cand_slot = A.cand_slot.get(); J.cand_out = A.cand_out.get(); J.cand_T = A.cand_T.get();
  J.kappa = nullptr;
  J.cand_R = A.cand_R.get(); J.cand_t = A.cand_t.get(); J.w = A.cand_w.get();
  J.Tloc = p->Tloc.get(); J.ylift = p->ylift.get(); J.X = p->vec[dpgo::V_X0].get();
  J.T_align = p->T_align.get(); J.info = p->align_info.get();
  return J;
}
}  // namespace

int dpgo_agent_set_local_trajectory(dpgo_problem_t *p, const double *T_host, const double *YLift_host) {
  DPGO_CHECK_HANDLE(p);
  DPGO_REQUIRE(T_host && YLift_host, DPGO_ERR_INVALID_ARG, "null trajectory or lifting matrix");
  const size_t tn = (size_t)p->d * p->dh * p->n, yn = (size_t)p->r * p->d;
  if (!p->Tloc) DPGO_CUDA(p->Tloc.alloc(tn));
  if (!p->ylift) DPGO_CUDA(p->ylift.alloc(yn));
  DPGO_CUDA(p->Tloc.upload(T_host, tn, p->stream));
  DPGO_CUDA(p->ylift.upload(YLift_host, yn, p->stream));
  dpgo::AlignJob J = align_job(p);
  J.T_align = nullptr;                     // identity: X = YLift T
  J.info = nullptr;
  DevBuf<dpgo::AlignJob> job;
  DPGO_CUDA(job.assign(&J, 1, p->stream));
  DPGO_CUDA(dpgo::launch_frame_lift(p->d, p->r, 1, p->n, job.get(), p->stream));
  DPGO_CUDA(cudaStreamSynchronize(p->stream));
  return DPGO_OK;
}

int dpgo_agent_set_align_candidates(dpgo_problem_t *p, int num_groups, const int32_t *group_neighbor, const int32_t *group_ptr,
                                    const int32_t *local_pose, const int32_t *nbr_slot, const int32_t *outgoing, const double *T) {
  DPGO_CHECK_HANDLE(p);
  DPGO_REQUIRE(num_groups >= 0 && (num_groups == 0 || (group_neighbor && group_ptr)), DPGO_ERR_INVALID_ARG, "bad candidate groups");
  const int m = num_groups ? group_ptr[num_groups] : 0;
  DPGO_REQUIRE(!num_groups || group_ptr[0] == 0, DPGO_ERR_INVALID_ARG, "group_ptr must start at 0");
  for (int g = 0; g < num_groups; ++g) {
    DPGO_REQUIRE(group_ptr[g + 1] > group_ptr[g], DPGO_ERR_INVALID_ARG, "every candidate group needs a candidate");
    DPGO_REQUIRE(group_neighbor[g] >= 0 && (g == 0 || group_neighbor[g] > group_neighbor[g - 1]), DPGO_ERR_INVALID_ARG,
                 "candidate groups must be in increasing neighbour id");
  }
  DPGO_REQUIRE(m == 0 || (local_pose && nbr_slot && outgoing && T), DPGO_ERR_INVALID_ARG, "null candidate arrays");
  int max_slot = -1;
  for (int q = 0; q < m; ++q) {
    DPGO_REQUIRE(local_pose[q] >= 0 && local_pose[q] < p->n && nbr_slot[q] >= 0, DPGO_ERR_INVALID_ARG,
                 "candidate index out of range");
    max_slot = std::max(max_slot, (int)nbr_slot[q]);
  }
  ++p->generation;                         // the job tables of dpgo_agents_align_async point into the old candidate table
  p->align = {};
  p->align.groups = num_groups;
  p->align.cands = m;
  p->align.max_slot = max_slot;
  p->align.max_nbr = num_groups ? group_neighbor[num_groups - 1] : -1;
  if (!p->T_align) DPGO_CUDA(p->T_align.alloc((size_t)p->d * p->dh));
  if (!p->align_info) DPGO_CUDA(p->align_info.alloc(4));
  if (!num_groups) return DPGO_OK;
  const int dh = p->dh;
  std::vector<int> outg(m);
  for (int q = 0; q < m; ++q) outg[q] = outgoing[q] ? 1 : 0;
  DPGO_CUDA(p->align.grp_nbr.assign(group_neighbor, (size_t)num_groups, p->stream));
  DPGO_CUDA(p->align.grp_ptr.assign(group_ptr, (size_t)num_groups + 1, p->stream));
  DPGO_CUDA(p->align.cand_local.assign(local_pose, (size_t)m, p->stream));
  DPGO_CUDA(p->align.cand_slot.assign(nbr_slot, (size_t)m, p->stream));
  DPGO_CUDA(p->align.cand_out.assign(outg.data(), outg.size(), p->stream));
  DPGO_CUDA(p->align.cand_T.assign(T, (size_t)m * dh * dh, p->stream));
  DPGO_CUDA(p->align.cand_R.alloc((size_t)m * p->d * p->d));
  DPGO_CUDA(p->align.cand_t.alloc((size_t)m * p->d));
  DPGO_CUDA(p->align.cand_w.alloc((size_t)m));
  DPGO_CUDA(cudaStreamSynchronize(p->stream));
  return DPGO_OK;
}

int dpgo_agents_align_async(dpgo_problem_t *const *agents, int count, const double *gathered_dev, int64_t num_slots,
                            const int32_t *ready_host, int num_agents, void *stream) {
  DPGO_TRY(check_agents(agents, count, true));
  DPGO_REQUIRE(ready_host && num_agents >= 1, DPGO_ERR_INVALID_ARG, "null ready flags");
  dpgo_problem *lead = agents[0];
  int max_cands = 0, max_poses = 0;
  for (int i = 0; i < count; ++i) {
    dpgo_problem *p = agents[i];
    DPGO_REQUIRE(p->Tloc && p->T_align, DPGO_ERR_STATE,
                 "dpgo_agent_set_local_trajectory and dpgo_agent_set_align_candidates must be called first");
    DPGO_REQUIRE(p->align.cands == 0 || (gathered_dev && p->align.max_slot < num_slots), DPGO_ERR_INVALID_ARG,
                 "a candidate refers to a slot beyond the gathered buffer");
    DPGO_REQUIRE(p->align.max_nbr < num_agents, DPGO_ERR_INVALID_ARG, "a candidate group names an agent beyond the ready flags");
    if (!p->ev_align) DPGO_CUDA(dpgo::create_event(p->ev_align));
    max_cands = std::max(max_cands, p->align.cands);
    max_poses = std::max(max_poses, p->n);
  }
  const cudaStream_t st = call_stream(lead, stream);
  std::vector<uint64_t> key = call_key(0x616c6e0000ull, agents, count);   // "aln"
  const dpgo_problem::JobTable<dpgo::AlignJob> *tab = nullptr;
  DPGO_TRY(job_table(lead->align_tables, key, count, st, [&](std::vector<dpgo::AlignJob> &jobs) {
    for (int i = 0; i < count; ++i) jobs[(size_t)i] = align_job(agents[i]);
    return 0;                              // the align launches size their grids by count, max_cands and max_poses
  }, tab));
  if (num_agents > lead->ready_cap) {
    DPGO_CUDA(lead->ready.alloc((size_t)num_agents));
    lead->ready_cap = num_agents;
  }
  DPGO_CUDA(lead->ready.upload(ready_host, (size_t)num_agents, st));   // the flags change every wave
  DPGO_CUDA(dpgo::launch_align_candidates(lead->d, lead->r, count, max_cands, tab->jobs.get(), gathered_dev, st));
  DPGO_CUDA(dpgo::launch_robust_rotation_average(lead->d, count, tab->jobs.get(), lead->ready.get(),
                                                 2.0 * std::sqrt(2.0) * std::sin(0.25), st));
  DPGO_CUDA(dpgo::launch_frame_lift(lead->d, lead->r, count, max_poses, tab->jobs.get(), st));
  for (int i = 0; i < count; ++i) DPGO_CUDA(cudaEventRecord(agents[i]->ev_align.get(), st));   // dpgo_agent_align_result waits on it
  return DPGO_OK;
}

int dpgo_agent_align_result(dpgo_problem_t *p, double *T_align_host, int32_t *info4) {
  DPGO_CHECK_HANDLE(p);
  DPGO_REQUIRE(p->T_align, DPGO_ERR_STATE, "dpgo_agent_set_align_candidates has not been called");
  DPGO_REQUIRE(info4, DPGO_ERR_INVALID_ARG, "null info");
  if (p->ev_align) DPGO_CUDA(cudaEventSynchronize(p->ev_align.get()));     // the align call may have run on another stream
  if (T_align_host)
    DPGO_CUDA(cudaMemcpyAsync(T_align_host, p->T_align.get(), sizeof(double) * p->d * p->dh, cudaMemcpyDeviceToHost, p->stream));
  DPGO_CUDA(cudaMemcpyAsync(info4, p->align_info.get(), sizeof(int) * 4, cudaMemcpyDeviceToHost, p->stream));
  DPGO_CUDA(cudaStreamSynchronize(p->stream));
  return DPGO_OK;
}

int dpgo_robust_single_rotation_averaging(int device, int d, int m, const double *R_host, const double *kappa_host,
                                          double threshold, double *R_out, int32_t *inlier_flags, int32_t *iterations) {
  DPGO_REQUIRE(d == 2 || d == 3, DPGO_ERR_UNSUPPORTED, "d must be 2 or 3");
  DPGO_REQUIRE(m >= 1 && R_host && R_out, DPGO_ERR_INVALID_ARG, "need m >= 1 rotations and an output");
  DPGO_REQUIRE(threshold > 0, DPGO_ERR_INVALID_ARG, "threshold must be positive");
  int count = 0;
  if (cudaGetDeviceCount(&count) != cudaSuccess || device < 0 || device >= count)
    return fail(DPGO_ERR_NO_DEVICE, "no such CUDA device: the GPU path has no CPU fallback");
  DPGO_CUDA(cudaSetDevice(device));
  // everything on the legacy default stream: the synchronous reads at the end follow the launch
  DevBuf<double> R, k, w, T;
  DevBuf<int> grp, info;
  DevBuf<dpgo::AlignJob> job;
  DPGO_CUDA(R.assign(R_host, (size_t)m * d * d, nullptr));
  DPGO_CUDA(w.alloc((size_t)m));
  DPGO_CUDA(T.alloc((size_t)d * (d + 1)));
  DPGO_CUDA(info.alloc(4));
  if (kappa_host) DPGO_CUDA(k.assign(kappa_host, (size_t)m, nullptr));
  const int grp_host[4] = {0, 0, m, 1};    // neighbour 0, candidates [0, m), ready flag of neighbour 0
  DPGO_CUDA(grp.assign(grp_host, 4, nullptr));
  dpgo::AlignJob J = {};
  J.ngroups = 1;
  J.grp_nbr = grp.get(); J.grp_ptr = grp.get() + 1;
  J.kappa = k.get(); J.cand_R = R.get(); J.w = w.get();
  J.T_align = T.get(); J.info = info.get();
  DPGO_CUDA(job.assign(&J, 1, nullptr));
  DPGO_CUDA(dpgo::launch_robust_rotation_average(d, 1, job.get(), grp.get() + 3, threshold, nullptr));
  std::vector<double> T_host((size_t)d * (d + 1)), w_host((size_t)m);
  int info_host[4];
  DPGO_CUDA(cudaMemcpy(T_host.data(), T.get(), sizeof(double) * T_host.size(), cudaMemcpyDeviceToHost));
  DPGO_CUDA(cudaMemcpy(w_host.data(), w.get(), sizeof(double) * m, cudaMemcpyDeviceToHost));
  DPGO_CUDA(cudaMemcpy(info_host, info.get(), sizeof(info_host), cudaMemcpyDeviceToHost));
  for (int a = 0; a < d; ++a)
    for (int c = 0; c < d; ++c) R_out[a * d + c] = T_host[(size_t)c * d + a];
  if (inlier_flags)
    for (int q = 0; q < m; ++q) inlier_flags[q] = w_host[(size_t)q] > 1.0 - 1e-8 ? 1 : 0;
  if (iterations) *iterations = info_host[3];
  return DPGO_OK;
}

}  // extern "C"

// ---- team status and rounding (dpgo_status.cu) ---------------------------------------------------------------------------
extern "C" {

int dpgo_agents_status_async(dpgo_problem_t *const *agents, int count, const int32_t *slot, double *status_dev, void *stream) {
  DPGO_TRY(check_agents(agents, count, true));
  DPGO_REQUIRE(slot && status_dev, DPGO_ERR_INVALID_ARG, "null slots or status buffer");
  dpgo_problem *lead = agents[0];
  std::vector<int32_t> sorted(slot, slot + count);
  std::sort(sorted.begin(), sorted.end());
  DPGO_REQUIRE(sorted[0] >= 0, DPGO_ERR_INVALID_ARG, "negative status slot");
  DPGO_REQUIRE(std::adjacent_find(sorted.begin(), sorted.end()) == sorted.end(), DPGO_ERR_INVALID_ARG, "duplicate status slot");
  std::vector<uint64_t> key = call_key(0x7374730000ull, agents, count);   // "sts"
  key.insert(key.end(), slot, slot + count);
  key.push_back((uint64_t)(uintptr_t)status_dev);
  const cudaStream_t st = call_stream(lead, stream);
  const dpgo_problem::JobTable<dpgo::StatusJob> *tab = nullptr;
  DPGO_TRY(job_table(lead->status.tables, key, count, st, [&](std::vector<dpgo::StatusJob> &jobs) {
    int ctas = 0;
    for (int i = 0; i < count; ++i) {
      const dpgo_problem *p = agents[i];
      dpgo::StatusJob &J = jobs[(size_t)i];
      J.n = p->n;
      J.cta0 = ctas;
      J.rowptr = p->bsr.rowptr.get(); J.bcol = p->bsr.bcol.get(); J.bval = p->bsr.bval.get();
      J.X = p->vec[dpgo::V_X0].get(); J.G = p->G.get();
      J.opt_record = p->status.opt_record.get();
      J.partials = p->status.part.get();
      J.ticket = p->status.ticket.get();
      J.out = status_dev + (size_t)slot[i] * DPGO_STATUS_DOUBLES;
      ctas += dpgo::status_ctas(p->n);
    }
    return ctas;
  }, tab));
  DPGO_CUDA(dpgo::launch_agents_status(lead->r, lead->dh, count, tab->ctas, tab->jobs.get(), st));
  return DPGO_OK;
}

int dpgo_agent_trajectory_global(dpgo_problem_t *p, const double *anchor_host, double *T_host) {
  DPGO_TRY(require_device());
  DPGO_REQUIRE(anchor_host && T_host, DPGO_ERR_INVALID_ARG, "null anchor or trajectory");
  DPGO_CHECK_HANDLE(p);
  if (!p->anchor) DPGO_CUDA(p->anchor.alloc((size_t)p->ts));
  if (!p->traj) DPGO_CUDA(p->traj.alloc((size_t)p->d * p->N));
  DPGO_CUDA(p->anchor.upload(anchor_host, (size_t)p->ts, p->stream));
  DPGO_CUDA(dpgo::launch_trajectory_global(p->r, p->dh, p->n, p->anchor.get(), p->vec[dpgo::V_X0].get(), p->traj.get(), p->stream));
  DPGO_CUDA(cudaMemcpyAsync(T_host, p->traj.get(), sizeof(double) * (size_t)p->d * p->N, cudaMemcpyDeviceToHost, p->stream));
  DPGO_CUDA(cudaStreamSynchronize(p->stream));
  return DPGO_OK;
}

int dpgo_host_alloc_pinned(size_t bytes, void **ptr) {
  DPGO_TRY(require_device());
  DPGO_REQUIRE(ptr && bytes > 0, DPGO_ERR_INVALID_ARG, "null output or zero size");
  DPGO_CUDA(cudaMallocHost(ptr, bytes));
  return DPGO_OK;
}

int dpgo_host_free_pinned(void *ptr) {
  if (ptr) DPGO_CUDA(cudaFreeHost(ptr));
  return DPGO_OK;
}

int dpgo_copy_to_host_async(int device, void *dst_host, const void *src_dev, size_t bytes, void *stream) {
  DPGO_TRY(require_device());
  DPGO_REQUIRE(dst_host && src_dev, DPGO_ERR_INVALID_ARG, "null buffer");
  DPGO_CUDA(cudaSetDevice(device));
  DPGO_CUDA(cudaMemcpyAsync(dst_host, src_dev, bytes, cudaMemcpyDeviceToHost, (cudaStream_t)stream));
  return DPGO_OK;
}

// ---- accelerated rounds (dpgo_accel.cu) ------------------------------------------------------------------------------------
int dpgo_agents_accel_begin_async(dpgo_problem_t *const *agents, int count, const int32_t *active_flags, double momentum_N,
                                  int restart_interval, double *const *send_dev, double *const *send_aux_dev, void *stream) {
  DPGO_TRY(check_agents(agents, count, true));
  DPGO_REQUIRE(active_flags && send_dev && send_aux_dev, DPGO_ERR_INVALID_ARG, "null active flags or send buffers");
  DPGO_REQUIRE(momentum_N >= 1.0 && restart_interval >= 1, DPGO_ERR_INVALID_ARG,
               "momentum_N must be >= 1 and restart_interval >= 1");
  dpgo_problem *lead = agents[0];
  std::vector<uint64_t> key = call_key(0x6163620000ull, agents, count);   // "acb"
  for (int i = 0; i < count; ++i) {
    const dpgo_problem *p = agents[i];
    DPGO_ACC_READY(p);
    DPGO_REQUIRE(p->pub.slot && p->pub.slot_unique, DPGO_ERR_STATE,
                 "the agent needs a public pose list without duplicates (dpgo_agent_set_public_poses)");
    DPGO_REQUIRE(p->pub.num == 0 || (send_dev[i] && send_aux_dev[i]), DPGO_ERR_INVALID_ARG, "null send buffer");
    key.push_back((uint64_t)(active_flags[i] != 0));
    key.push_back((uint64_t)(uintptr_t)send_dev[i]);
    key.push_back((uint64_t)(uintptr_t)send_aux_dev[i]);
  }
  const cudaStream_t st = call_stream(lead, stream);
  const dpgo_problem::JobTable<dpgo::AccelJob> *tab = nullptr;
  DPGO_TRY(job_table(lead->acc.tables, key, count, st, [&](std::vector<dpgo::AccelJob> &jobs) {
    int ctas = 0;
    for (int i = 0; i < count; ++i) {
      const dpgo_problem *p = agents[i];
      dpgo::AccelJob &J = jobs[(size_t)i];
      J.n = p->n;
      J.cta0 = ctas;
      J.active = active_flags[i] != 0;
      J.X = p->vec[dpgo::V_X0].get(); J.Y = p->acc.vec[0].get(); J.V = p->acc.vec[1].get(); J.XP = p->acc.vec[2].get();
      J.state = p->acc.state.get();
      J.opt_record = p->status.opt_record.get();
      J.pub_slot = p->pub.slot.get();
      J.send_x = send_dev[i]; J.send_y = send_aux_dev[i];
      J.ticket = p->acc.ticket.get();
      ctas += dpgo::accel_ctas(p->n);
    }
    return ctas;
  }, tab));
  DPGO_CUDA(dpgo::launch_accel_agents(lead->r, lead->dh, count, tab->ctas, tab->jobs.get(), momentum_N, restart_interval, st));
  for (int i = 0; i < count; ++i) {
    dpgo_problem *p = agents[i];
    ++p->acc.rounds;
    p->acc.restart_due = (p->acc.rounds + 1) % restart_interval == 0;
  }
  return DPGO_OK;
}

static int issue_accel_round(dpgo_problem_t *const *agents, int num_active, const dpgo_opt_params_t *params,
                             const double *gathered_dev, const double *gathered_aux_dev, int64_t num_slots, cudaStream_t main) {
  return fan_out(agents, num_active, main, round_streams(main), [&](int, dpgo_problem *p) -> int {
    double *X = p->vec[dpgo::V_X0].get(), *Y = p->acc.vec[0].get(), *V = p->acc.vec[1].get(), *XP = p->acc.vec[2].get();
    DPGO_TRY(dpgo_agent_build_G(p, gathered_aux_dev, num_slots));
    DPGO_CUDA(cudaMemcpyAsync(X, Y, p->vec_bytes(), cudaMemcpyDeviceToDevice, p->stream));
    DPGO_TRY(dpgo_optimize_resident_async(p, params));
    DPGO_CUDA(dpgo::launch_accel_finish(p->r, p->dh, p->n, X, Y, V, XP, p->acc.state.get(),
                                        p->acc.restart_due ? dpgo::ACCEL_FINISH_V_RESTART : dpgo::ACCEL_FINISH_V, p->acc.part.get(),
                                        p->acc.ticket.get() + 1, p->status.opt_record.get(), p->stream));
    if (p->acc.restart_due) {
      DPGO_TRY(dpgo_agent_build_G(p, gathered_dev, num_slots));
      DPGO_TRY(dpgo_optimize_resident_async(p, params));
      DPGO_CUDA(dpgo::launch_accel_finish(p->r, p->dh, p->n, X, Y, V, XP, p->acc.state.get(), dpgo::ACCEL_FINISH_RESTART_END,
                                          p->acc.part.get(), p->acc.ticket.get() + 1, p->status.opt_record.get(), p->stream));
    }
    return DPGO_OK;
  });
}

int dpgo_agents_accel_round_async(dpgo_problem_t *const *agents, int num_active, const dpgo_opt_params_t *params,
                                  const double *gathered_dev, const double *gathered_aux_dev, int64_t num_slots,
                                  void *main_stream) {
  DPGO_REQUIRE(num_active >= 0 && params, DPGO_ERR_INVALID_ARG, "bad arguments");
  if (num_active == 0) return DPGO_OK;
  DPGO_TRY(check_agents(agents, num_active, false));
  for (int i = 0; i < num_active; ++i) {
    DPGO_ACC_READY(agents[i]);
    DPGO_REQUIRE(agents[i]->acc.state && agents[i]->acc.rounds > 0, DPGO_ERR_STATE,
                 "dpgo_agents_accel_begin_async has not been called");
    DPGO_REQUIRE(gathered_aux_dev || agents[i]->shared.num_edges == 0, DPGO_ERR_INVALID_ARG, "null gathered buffer");
  }
  cudaStream_t main = nullptr;
  bool graph = false;
  DPGO_TRY(round_preamble(agents, num_active, params, main_stream, main, graph));
  auto issue = [&]() { return issue_accel_round(agents, num_active, params, gathered_dev, gathered_aux_dev, num_slots, main); };
  if (!graph) return issue();
  std::vector<uint64_t> key = round_key(0x6163630000ull, agents, num_active, params, main, num_slots);   // "acc"
  for (int i = 0; i < num_active; ++i)
    key.push_back((uint64_t)agents[i]->acc.restart_due);    // two variants per active set: plain and restart rounds
  key.push_back((uint64_t)(uintptr_t)gathered_dev);
  key.push_back((uint64_t)(uintptr_t)gathered_aux_dev);
  return replay_or_issue(agents[0], key, main, issue);
}

// ---- greedy independent-set rounds (dpgo_select.cu) -----------------------------------------------------------------------
int dpgo_agents_set_agent_graph(dpgo_problem_t *lead, int num_agents, const int32_t *adj_ptr, const int32_t *adj) {
  DPGO_TRY(require_device());
  DPGO_CHECK_HANDLE(lead);
  DPGO_REQUIRE(num_agents >= 1 && num_agents <= dpgo::SELECT_MAX_AGENTS && adj_ptr, DPGO_ERR_INVALID_ARG,
               "the agent graph needs 1 to 1024 agents and a row pointer");
  DPGO_REQUIRE(adj_ptr[0] == 0 && (adj_ptr[num_agents] == 0 || adj), DPGO_ERR_INVALID_ARG, "bad agent graph arrays");
  for (int a = 0; a < num_agents; ++a) {
    DPGO_REQUIRE(adj_ptr[a + 1] >= adj_ptr[a], DPGO_ERR_INVALID_ARG, "the agent graph's row pointer must not decrease");
    for (int e = adj_ptr[a]; e < adj_ptr[a + 1]; ++e)
      DPGO_REQUIRE(adj[e] >= 0 && adj[e] < num_agents && adj[e] != a, DPGO_ERR_INVALID_ARG,
                   "agent graph neighbour out of range or a self loop");
  }
  DPGO_CUDA(cudaSetDevice(lead->device));
  DPGO_CUDA(cudaDeviceSynchronize());                       // the old buffers may still be read by a round in flight
  lead->sel = {};
  dpgo_problem::Select &S = lead->sel;
  const int m = adj_ptr[num_agents];
  DPGO_CUDA(S.ptr.assign(adj_ptr, (size_t)num_agents + 1, lead->stream));
  DPGO_CUDA(S.adj.assign(adj, (size_t)m, lead->stream));
  DPGO_CUDA(S.mask.alloc((size_t)num_agents));
  DPGO_CUDA(S.count.alloc(1));
  DPGO_CUDA(cudaMemsetAsync(S.count.get(), 0, sizeof(unsigned long long), lead->stream));
  DPGO_CUDA(cudaStreamSynchronize(lead->stream));
  S.k = num_agents;
  ++lead->generation;
  return DPGO_OK;
}

namespace {
struct GateSet {                           // every agent of a round reads its byte of the mask for the duration of a call
  dpgo_problem_t *const *agents; int count;
  GateSet(dpgo_problem_t *const *a, int n, const unsigned char *mask, const int32_t *index) : agents(a), count(n) {
    for (int i = 0; i < n; ++i) a[i]->gate = mask + index[i];
  }
  ~GateSet() { for (int i = 0; i < count; ++i) agents[i]->gate = nullptr; }
};
}  // namespace

// One greedy independent-set round of the agents of one GPU: the selection from the gathered status records, then every
// listed agent's G rebuild -> step -> pack, each kernel gated by the agent's byte of the mask.  The selected agents share
// no edge, so packs into an aliased gathered buffer cannot race with another selected agent's G rebuild.
int dpgo_agents_select_round_async(dpgo_problem_t *const *agents, int count, const int32_t *agent_index,
                                   const dpgo_opt_params_t *params, const double *records_dev, const double *gathered_dev,
                                   int64_t num_slots, double *const *send_dev, void *stream) {
  DPGO_TRY(check_agents(agents, count, false));
  DPGO_REQUIRE(agent_index && params && records_dev && send_dev, DPGO_ERR_INVALID_ARG, "bad arguments");
  dpgo_problem *lead = agents[0];
  DPGO_REQUIRE(lead->sel.k > 0, DPGO_ERR_STATE, "dpgo_agents_set_agent_graph has not been called for the first agent");
  std::vector<char> seen((size_t)lead->sel.k, 0);
  for (int i = 0; i < count; ++i) {
    DPGO_REQUIRE(agent_index[i] >= 0 && agent_index[i] < lead->sel.k && !seen[(size_t)agent_index[i]], DPGO_ERR_INVALID_ARG,
                 "agent indices must be distinct and below the agent graph's size");
    seen[(size_t)agent_index[i]] = 1;
  }
  cudaStream_t main = nullptr;
  bool graph = false;
  DPGO_TRY(round_preamble(agents, count, params, stream, main, graph));
  dpgo_problem::Select &S = lead->sel;
  if (S.rounds == S.cap) {                                  // the log doubles; the old buffer is freed after the next read
    const long long cap = std::max(64LL, 2 * S.cap);
    DevBuf<unsigned char> grown;
    DPGO_CUDA(grown.alloc((size_t)cap * S.k));
    if (S.log) {
      DPGO_CUDA(cudaMemcpyAsync(grown.get(), S.log.get(), (size_t)S.rounds * S.k, cudaMemcpyDeviceToDevice, main));
      S.retired.push_back(std::move(S.log));
    }
    S.log = std::move(grown);
    S.cap = cap;
  }
  auto issue = [&]() -> int {
    DPGO_CUDA(dpgo::launch_select_independent(S.k, records_dev, S.ptr.get(), S.adj.get(), S.mask.get(), S.log.get(),
                                              S.count.get(), main));
    GateSet gates(agents, count, S.mask.get(), agent_index);
    return issue_round(agents, count, params, gathered_dev, num_slots, send_dev, main, 0);
  };
  int rc = DPGO_OK;
  if (!graph) {
    rc = issue();
  } else {
    std::vector<uint64_t> key = round_key(0x73656c0000ull, agents, count, params, main, num_slots);   // "sel"
    for (int i = 0; i < count; ++i) {
      key.push_back((uint64_t)(uintptr_t)send_dev[i]);
      key.push_back((uint64_t)agent_index[i]);
    }
    key.push_back((uint64_t)(uintptr_t)gathered_dev);
    key.push_back((uint64_t)(uintptr_t)records_dev);
    key.push_back((uint64_t)(uintptr_t)S.log.get());
    rc = replay_or_issue(lead, key, main, issue);
  }
  if (rc == DPGO_OK) ++S.rounds;
  return rc;
}

int dpgo_agents_selection_log(dpgo_problem_t *lead, int64_t first_round, int64_t max_rounds, uint8_t *out_host,
                              int64_t *total_rounds) {
  DPGO_TRY(require_device());
  DPGO_CHECK_HANDLE(lead);
  DPGO_REQUIRE(lead->sel.k > 0, DPGO_ERR_STATE, "dpgo_agents_set_agent_graph has not been called for this agent");
  DPGO_REQUIRE(first_round >= 0 && max_rounds >= 0 && (max_rounds == 0 || out_host), DPGO_ERR_INVALID_ARG, "bad log range");
  DPGO_CUDA(cudaSetDevice(lead->device));
  DPGO_CUDA(cudaDeviceSynchronize());                       // the log is written on the streams of the round calls
  lead->sel.retired.clear();
  if (total_rounds) *total_rounds = lead->sel.rounds;
  const int64_t rows = std::max<int64_t>(0, std::min<int64_t>(max_rounds, lead->sel.rounds - first_round));
  if (rows > 0)
    DPGO_CUDA(cudaMemcpy(out_host, lead->sel.log.get() + (size_t)first_round * lead->sel.k, (size_t)rows * lead->sel.k,
                         cudaMemcpyDeviceToHost));
  return DPGO_OK;
}

int dpgo_agent_accel_state(dpgo_problem_t *p, double *out3) {
  DPGO_TRY(require_device());
  DPGO_REQUIRE(out3, DPGO_ERR_INVALID_ARG, "null output");
  DPGO_CHECK_HANDLE(p);
  DPGO_REQUIRE(p->acc.state, DPGO_ERR_STATE, "dpgo_agent_accel_init has not been called");
  DPGO_CUDA(cudaDeviceSynchronize());                       // the record is written on the stream of the begin calls
  DPGO_CUDA(cudaMemcpy(out3, p->acc.state.get(), 3 * sizeof(double), cudaMemcpyDeviceToHost));
  return DPGO_OK;
}

}  // extern "C"
