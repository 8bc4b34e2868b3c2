// dpgo_handle.cuh -- the problem handle behind the C ABI and what the C API translation units (dpgo_capi*.cu) share: the
// error macros and the helpers more than one of them calls.  Private to those files and never installed; the library
// builds with -fvisibility=hidden, so nothing declared here is exported.
#pragma once
#include <cuda_runtime.h>
#include <chrono>
#include <cstdint>
#include <memory>
#include <string>
#include <vector>

#include "dpgo_devbuf.cuh"
#include "dpgo_kernels.cuh"

using dpgo::DevBuf;

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

namespace dpgo::capi {

// Records msg as the calling thread's last error (dpgo_last_error) and returns code.
int fail(int code, const std::string &msg);

#define DPGO_CUDA(call)                                                                             \
  do {                                                                                              \
    cudaError_t _e = (call);                                                                        \
    if (_e != cudaSuccess)                                                                          \
      return ::dpgo::capi::fail(DPGO_ERR_CUDA, std::string(#call) + ": " + cudaGetErrorString(_e)); \
  } while (0)

#define DPGO_REQUIRE(cond, code, msg)                  \
  do {                                                 \
    if (!(cond)) return ::dpgo::capi::fail(code, msg); \
  } while (0)

#define DPGO_TRY(expr)            \
  do {                            \
    int _s = (expr);              \
    if (_s != DPGO_OK) return _s; \
  } while (0)

#define DPGO_CHECK_HANDLE(p)                                                                 \
  do {                                                                                       \
    if (!(p)) return ::dpgo::capi::fail(DPGO_ERR_INVALID_ARG, "null problem handle");        \
    cudaError_t _e = cudaSetDevice((p)->device);                                             \
    if (_e != cudaSuccess) return ::dpgo::capi::fail(DPGO_ERR_CUDA, cudaGetErrorString(_e)); \
  } while (0)



#define DPGO_ACC_READY(p) DPGO_REQUIRE((p)->acc.vec[0], DPGO_ERR_STATE, "dpgo_agent_accel_init has not been called")

// The two exact preconditioners apply the same operator P_X((Q + 0.1 I)^-1 V) with the same block solve: SPARSE_EXACT on
// the macro levels the cost model picks, DENSE_EXACT on a single one, whose root panels are the dense inverse of every
// connected component.  A launch reads the factorisation its preconditioner selects (the sparse one unless DENSE_EXACT).
enum NdSlot { ND_SPARSE = 0, ND_DENSE = 1 };
inline int nd_slot(int precond) { return precond == DPGO_PRECOND_DENSE_EXACT ? ND_DENSE : ND_SPARSE; }
inline int nd_precond(int slot) { return slot == ND_DENSE ? DPGO_PRECOND_DENSE_EXACT : DPGO_PRECOND_SPARSE_EXACT; }

struct BlockTriplet {
  int brow, bcol;      // Q sub-block at rows dh*brow.., cols dh*bcol..
  double v[16];        // padded 4x4, v[k*4+c] = Q[dh*brow+k, dh*bcol+c]
};

// ---- dpgo_capi.cu ----
// A CUDA device exists (the GPU path has no CPU fallback) and `device` is one of them; DPGO_ERR_NO_DEVICE otherwise.
int require_device(int device = 0);
// nb dense dh x dh blocks (row-major, block q at (brow[q], bcol[q]), both in [0, n)) as padded triplets.
int blocks_to_triplets(int n, int dh, int64_t nb, const int32_t *brow, const int32_t *bcol, const double *blocks,
                       std::vector<BlockTriplet> &trip);
void assemble_bsr(int n, const std::vector<BlockTriplet> &trip, std::vector<int> &rowptr, std::vector<int> &bcol,
                  std::vector<double> &bval);
int build_from_triplets(dpgo_problem *p, std::vector<BlockTriplet> &trip, unsigned precond_mask);
int check_params(dpgo_problem *p, const dpgo_opt_params_t *prm);
int upload_vec(dpgo_problem *p, int id, const double *host);
int download_vec(dpgo_problem *p, int id, double *host);
int check_refactor_fail(dpgo_problem *p);

// ---- dpgo_capi_precond.cu ----
void jacobi_blocks(int n, int dh, const std::vector<int> &rowptr, const std::vector<int> &bcol, const std::vector<double> &bval,
                   std::vector<double> &dinv);
void free_nd(dpgo_problem *p);
int ensure_nd(dpgo_problem *p, int slot);
int ensure_refactor(dpgo_problem *p, int slot);
int launch_refactor(dpgo_problem *p, int slot);

}  // namespace dpgo::capi
