// dpgo_capi_agents.cu -- the multi-agent side of the C ABI: the per-agent setup calls (boundary-pose exchange, Nesterov
// acceleration, distributed initialisation) and the batched calls that serve every agent of a GPU with one call, with
// their fork/join, CUDA-graph replay and job-table plumbing.
#include <cuda_runtime.h>
#include <algorithm>
#include <cmath>
#include <cstdlib>
#include <cstring>
#include <numeric>
#include <vector>

#include "dpgo_handle.cuh"

namespace dpgo::capi {
namespace {

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

int issue_round(dpgo_problem_t *const *agents, int num_active, const dpgo_opt_params_t *params,
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

int issue_accel_round(dpgo_problem_t *const *agents, int num_active, const dpgo_opt_params_t *params,
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

struct GateSet {                           // every agent of a round reads its byte of the mask for the duration of a call
  dpgo_problem_t *const *agents; int count;
  GateSet(dpgo_problem_t *const *a, int n, const unsigned char *mask, const int32_t *index) : agents(a), count(n) {
    for (int i = 0; i < n; ++i) a[i]->gate = mask + index[i];
  }
  ~GateSet() { for (int i = 0; i < count; ++i) agents[i]->gate = nullptr; }
};

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
}  // namespace dpgo::capi

using namespace dpgo::capi;

extern "C" {

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

// ---- batched rounds and host I/O ---------------------------------------------------------------------------------------
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

// ---- distributed initialisation: frame alignment -------------------------------------------------------

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
  DPGO_TRY(require_device(device));
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

// ---- team status and rounding (dpgo_status.cu) ---------------------------------------------------------------------------

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

int dpgo_agent_accel_state(dpgo_problem_t *p, double *out3) {
  DPGO_TRY(require_device());
  DPGO_REQUIRE(out3, DPGO_ERR_INVALID_ARG, "null output");
  DPGO_CHECK_HANDLE(p);
  DPGO_REQUIRE(p->acc.state, DPGO_ERR_STATE, "dpgo_agent_accel_init has not been called");
  DPGO_CUDA(cudaDeviceSynchronize());                       // the record is written on the stream of the begin calls
  DPGO_CUDA(cudaMemcpy(out3, p->acc.state.get(), 3 * sizeof(double), cudaMemcpyDeviceToHost));
  return DPGO_OK;
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

}  // extern "C"
