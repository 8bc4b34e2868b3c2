// dpgo_kernels.cuh -- kernel-side parameter block shared by dpgo_kernels.cu and the C API (dpgo_capi*.cu)
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include "../../include/dpgo_b200.h"
#include "nd_precond.h"

namespace dpgo {

// work vectors, each r x (d+1)n fp64 in HBM
enum VecId {
  V_X0 = 0, V_X1,        // iterate double buffer (X0 is the externally visible one)
  V_EG0, V_EG1,          // Euclidean gradient at X0 / X1
  V_RG0, V_RG1,          // Riemannian gradient
  V_Z00, V_Z01,          // preconditioned gradient M^-1 g at X0 / X1
  V_ETA, V_RES, V_Z,     // tCG: step, residual, preconditioned residual
  V_D0, V_D1,            // tCG: search direction double buffer
  V_HD,                  // H[delta]
  V_T,                   // scratch (Stiefel projection output)
  V_XIN,                 // copy of the input iterate (relative change)
  V_AUX,                 // operand of the single-operation entry points
  V_COUNT
};

enum OpCode {
  OP_OPTIMIZE = 0,   // full RTR / RGD call
  OP_EVAL = 1,       // f, EG, RG, |RG| at X0
  OP_RHESS = 2,      // HD = Hess f(X0)[AUX]
  OP_PRECON = 3,     // Z  = P_X0( M^-1 AUX )
  OP_RETRACT = 4,    // X1 = R_X0(AUX)
  OP_PHASE_BENCH = 9, // diagnostic: empty phases
};

constexpr int NRED = 4;            // scalars reduced per phase
constexpr int OPT_THREADS = 512;   // persistent kernel block size
constexpr int SPMV_GROUP_BLOCKS = 192;  // blocks per row group of the TMA-fed SpMV (24 KB of Q per smem stage)
// Shared-memory capacities of one step of the block solve (sparse and dense exact preconditioners): pose tiles of a phase's
// input vector staged per step (r x (d+1) doubles each), and partial-sum slots (8 rows x r doubles each).  Both areas grow
// with r, so above r (d+1) = 20 and r = 5 the counts shrink in proportion: a plan at the capacities never stages more than
// one at (r, d+1) = (5, 4) does, and what it leaves to the resident panel columns stays above 30 KB.  The planner honours
// smaller capacities with smaller steps (more of them, or column-chunked ones).
constexpr int nd_ycap_tiles(int r, int dh) { return r * dh <= 20 ? 600 : 12000 / (r * dh); }
constexpr int nd_slot_cap(int r) { return r <= 5 ? 240 : 1200 / r; }
constexpr int OPT_SMEM_LIMIT = 227 * 1024;  // dynamic shared memory one CTA of an H100 may ask for (checked by optimize_max_grid)
constexpr int SP_CACHE_INTS = 2048;  // shared-memory copy of a CTA's block-CSR structure (row pointers + block columns), 8 KB

// exact preconditioner (nd_precond.h): the static plan and the panel blob in HBM / L2
struct KNd {
  int nphases;
  int max_ytiles, max_slots;       // shared-memory tiles / partial-sum slots the plan needs per step
  int max_gathers;                 // gather records staged per step (<= max_ytiles)
  int resident_doubles;            // shared-memory region of the resident panel columns (largest over the CTAs)
  int dir[nd::MAX_PHASES];         // per phase: 0 forward (input = residual), 1 backward (input = ancestors' solution)
  int cta0[nd::MAX_PHASES];        // per phase: first (phase, CTA) record
  const nd::CtaPhase *cta_phase;
  const nd::Step *steps;
  const nd::Gather *gathers;
  const nd::Job *jobs;
  const nd::Epi *epis;
  const int *csrc;
  const double *blob;
  double *TX;            // n tiles, permuted order: t (forward) then x (backward), unprojected
  double *C;             // contribution tiles of the forward sweep
};

struct KParams {
  int n;                 // poses
  int N;                 // (d+1) n
  int grid;              // CTAs of the persistent kernel
  int op;
  const int *rowptr;     // n+1
  const int *bcol;       // nb
  const double *bval;    // nb*16
  const double *dinv;    // n*16   block-Jacobi inverse blocks, may be null
  const int *cta_rows;   // grid+1 balanced row partition
  const double *G;       // linear term r x N
  double *v[V_COUNT];
  double *S[2];          // n*9   sym(Y^T EG_Y) per pose at X0 / X1
  double *partials;      // 2 * grid * NRED
  unsigned *bar_counter;
  unsigned *bar_epoch;
  dpgo_opt_params_t prm;
  dpgo_opt_result_t *result;   // device copy of the result record
  KNd nd;                // the exact preconditioner prm.precond selects (nd.nphases == 0: not prepared)
  int cluster;           // 1: the whole grid is ONE thread-block cluster (<= 16 CTAs): phase ends use barrier.cluster
  int smem_doubles;      // dynamic shared memory of this launch, in doubles
  unsigned long long *phase_ns; // diagnostic (nullable): per phase kind, ns seen by CTA 0 (dpgo_debug_phase_times64)
  double *opt_record;    // 2 doubles: relative change of the last optimising call, optimising calls so far (OP_OPTIMIZE only)
  const unsigned char *gate;   // nullable: the agent's byte of a selection mask; 0 = the launch returns at entry
};

// Instantiations of the compiled (r, d+1) pairs, every d <= r <= DPGO_MAX_RANK (the pairs dpgo_problem_create accepts); R and
// DH are constexpr in the body.
#define DPGO_DISPATCH(R_, DH_, ...)                                    \
  do {                                                                   \
    if ((DH_) == 4) {                                                    \
      switch (R_) {                                                      \
        case 3: { constexpr int R = 3, DH = 4; __VA_ARGS__; } break;     \
        case 4: { constexpr int R = 4, DH = 4; __VA_ARGS__; } break;     \
        case 5: { constexpr int R = 5, DH = 4; __VA_ARGS__; } break;     \
        case 6: { constexpr int R = 6, DH = 4; __VA_ARGS__; } break;     \
        case 7: { constexpr int R = 7, DH = 4; __VA_ARGS__; } break;     \
        case 8: { constexpr int R = 8, DH = 4; __VA_ARGS__; } break;     \
        default: break;                                                  \
      }                                                                  \
    } else if ((DH_) == 3) {                                             \
      switch (R_) {                                                      \
        case 2: { constexpr int R = 2, DH = 3; __VA_ARGS__; } break;     \
        case 3: { constexpr int R = 3, DH = 3; __VA_ARGS__; } break;     \
        case 4: { constexpr int R = 4, DH = 3; __VA_ARGS__; } break;     \
        case 5: { constexpr int R = 5, DH = 3; __VA_ARGS__; } break;     \
        case 6: { constexpr int R = 6, DH = 3; __VA_ARGS__; } break;     \
        case 7: { constexpr int R = 7, DH = 3; __VA_ARGS__; } break;     \
        case 8: { constexpr int R = 8, DH = 3; __VA_ARGS__; } break;     \
        default: break;                                                  \
      }                                                                  \
    }                                                                    \
  } while (0)

// launchers (dpgo_kernels.cu)
cudaError_t launch_optimize(int r, int dh, const KParams &kp, cudaStream_t stream);
cudaError_t launch_spmv(int r, int dh, int n, const int *rowptr, const int *bcol, const double *bval,
                        const double *X, const double *G, double *out, cudaStream_t stream);
cudaError_t launch_spmv_tma(int r, int dh, int ngroups, const int2 *groups, const int *rowptr, const int *bcol,
                            const double *bval, const double *X, const double *G, double *out, int sms,
                            cudaStream_t stream);
int spmv_group_blocks();                            // blocks per row group of the TMA-fed SpMV in use
int optimize_max_grid(int r, int dh, int device);   // co-resident CTA count for the persistent kernel
// bytes of resident panel columns (nd::assign_residency) a CTA may keep next to what the sparse plan stages
int64_t nd_resident_budget(int r, int dh, const KNd &nd);
int optimize_max_cluster(int r, int dh, int device); // largest single-cluster grid (16, 8 or 0) the kernel can be launched with
cudaError_t launch_stiefel_project(int r, int dh, int n, const double *M, double *out, cudaStream_t stream, double c0 = 1.0,
                                   const double *B = nullptr, double c1 = 0.0, const double *C = nullptr, double c2 = 0.0);
// gate (nullable): the agent's byte of a selection mask; the launch does nothing when it is 0
cudaError_t launch_pack_tiles(int ts, int count, const int *pose, const double *X, double *out, cudaStream_t stream,
                              const unsigned char *gate = nullptr);
cudaError_t launch_build_G(int r, int dh, int nposes, const int *pose_ids, const int *pose_ptr, const int *edge_slot,
                           const int *edge_out, const double *edge_T, const double *edge_om, const double *gathered,
                           double *G, cudaStream_t stream, const unsigned char *gate = nullptr);
cudaError_t launch_assemble_Q(int64_t nb, const int *cptr, const int2 *contrib, const double *eT, const double *eom, const double *ew,
                              const double *sblk, double *bval, cudaStream_t stream);
// gnc (nullable, zeroed by the caller): counts over the non-fixed edges of weight exactly 1, exactly 0, and in between
cudaError_t launch_edge_weights(int r, int dh, int64_t m, const int *p1, const int *p2, const double *eT, const double *eom,
                                const int *fixed, const double *X, int cost, double mu, double param, double *w, double *resid,
                                unsigned long long *gnc, cudaStream_t stream);

// One matrix of a batched Gauss-Jordan sweep (dense_inverse.cu): A is M x M column-major (ld = M), swept over its pivots
// [0, s); piv (32 x 32), Rw (32 x M) and C (M x 32) are its workspace.
struct GjJob {
  double *A, *piv, *Rw, *C;
  int M, s;
};
// gridDim.y and gridDim.z are at most 65535: the batched launches that put one CTA set per matrix or per node there
// (gj_sweep_batch, launch_nd_refactor, launch_nd_selinv) take a longer batch in consecutive slices of this many.
constexpr int MAX_GRID_YZ = 65535;
// Sweeps every job of jobs_dev (max_M / max_s bound the jobs' sizes): 3 launches per 32 pivots and slice of
// MAX_GRID_YZ jobs, no synchronisation.  A non-positive pivot sets *fail (nullable).
cudaError_t gj_sweep_batch(const GjJob *jobs_dev, int njobs, int max_M, int max_s, int *fail, cudaStream_t stream);

// ---- numeric refactorisation of the exact preconditioners on the device (nd_refactor.cu) ----
// Device view of an nd::Refactor plus the buffers it fills; see nd_precond.h.
struct KRefactor {
  int dh;
  double shift;
  const nd::RefactorNode *nodes;
  const nd::RefactorChild *child;
  const int *poses, *cmap;
  const int *rowptr, *bcol;          // block-CSR pattern of Q
  const double *bval;                // Q values
  double *arena;                     // fronts (nd::Refactor::arena_doubles)
  const GjJob *jobs;                 // one sweep job per node, nodes order
  double *blob;                      // the panel blob, rewritten in place
  int *fail;                         // set when a front is not positive definite
};
// Every stage of R (deepest first): assemble the fronts, sweep them, pack the panels.  Ordinary launches on `stream`, none
// synchronising; the sequence captures into a CUDA graph.
cudaError_t launch_nd_refactor(const KRefactor &k, const nd::Refactor &R, cudaStream_t stream);
// block-Jacobi inverse blocks (Q_jj + shift I)^-1 of every pose, 4x4 padded (the host's jacobi_blocks in dpgo_capi_precond.cu);
// a non-positive pivot sets *fail (nullable)
cudaError_t launch_jacobi_blocks(int n, int dh, const int *rowptr, const int *bcol, const double *bval, double shift, double *dinv,
                                 int *fail, cudaStream_t stream);

// ---- pose covariances (dpgo_covariance.cu) ----
// The Gauss-Newton information H of a trajectory in block-CSR form over 3-scalar nodes (d = 2: one per pose; d = 3: two,
// w_i then v_i), blocks padded to 4 x 4 as the factorisation reads them: bval[b][k][c] = H[3 node.x + k, 3 node.y + c].
// Block b sums its contributions contrib[cptr[b] .. cptr[b+1]) = {edge, role of node.x | role of node.y << 1} in that
// order; the anchor's nodes are identity blocks without coupling.
struct KPoseInfo {
  int d, anchor;
  int64_t nb;
  const int *cptr;
  const int2 *contrib, *bnode;       // bnode[b] = {column node, row node}
  const int *p1, *p2;
  const double *T, *R, *t, *kappa, *tau, *w;   // T: d x (d+1)n column-major; R, t, kappa, tau as in dpgo_pose_covariances; w nullable
  double *bval;
};
cudaError_t launch_assemble_pose_info(const KPoseInfo &k, cudaStream_t stream);
// One 3 x 3 block of a front inverse: rows ra.., columns rc.. of refactor node `node`'s front -> out[x * ld + y].
struct CovItem { int node, ra, rc, pad; long long out; };
// Selected inversion over the fronts of a factorisation with shift 0 (nd::Selinv), root stage first; the items of stage st
// are items[item0[st] .. item0[st+1]).
struct KSelinv {
  const nd::RefactorNode *nodes;
  const int *parent, *pmap0, *pmap;
  const double *blob;
  double *arena;                     // front inverses, in the refactorisation's arena layout
  const CovItem *items;
  double *out;
  int ld;
};
cudaError_t launch_nd_selinv(const KSelinv &k, const nd::Refactor &R, const nd::Selinv &S, const std::vector<int> &item0,
                             cudaStream_t stream);

// ---- frame alignment of the distributed initialisation (dpgo_align.cu) ----
// One aligning agent.  Its candidates are grouped per neighbour (group g = candidates [grp_ptr[g], grp_ptr[g+1]) against
// agent grp_nbr[g], groups in increasing neighbour id); candidate q pairs local pose cand_local[q] with the gathered tile
// cand_slot[q] through the shared edge cand_T[q] ((d+1) x (d+1) row-major), cand_out[q] != 0 when the agent owns its tail.
struct AlignJob {
  int ngroups;
  int n;                                   // poses of the agent
  const int *grp_nbr, *grp_ptr;
  const int *cand_local, *cand_slot, *cand_out;
  const double *cand_T;
  const double *kappa;                     // per candidate rotation weight; nullptr = 1
  double *cand_R, *cand_t, *w;             // candidate rotations (d x d row-major), translations (d; nullptr: none), weights
  const double *Tloc;                      // d x (d+1)n local-frame trajectory, column-major
  const double *ylift;                     // r x d, column-major
  double *X;                               // r x (d+1)n resident iterate
  double *T_align;                         // out: d x (d+1) column-major [R t]; nullptr in a lift job = identity
  int *info;                               // out: neighbour used (-1: none), candidates, inliers, GNC iterations
};
constexpr int ALIGN_THREADS = 256;         // block of k_robust_rotation_average (one CTA per aligning agent)
cudaError_t launch_align_candidates(int d, int r, int njobs, int max_cands, const AlignJob *jobs, const double *gathered,
                                    cudaStream_t stream);
cudaError_t launch_robust_rotation_average(int d, int njobs, const AlignJob *jobs, const int *ready, double cbar,
                                           cudaStream_t stream);
// X = YLift (T_align T) for every pose of every job whose info reports inliers (info == nullptr: always)
cudaError_t launch_frame_lift(int d, int r, int njobs, int max_poses, const AlignJob *jobs, cudaStream_t stream);

// ---- team status and rounding (dpgo_status.cu) ----
// One agent of a status launch: CTAs [cta0, cta0 + status_ctas(n)) own STATUS_ROWS consecutive rows of its block-CSR Q each.
struct StatusJob {
  int n, cta0;
  const int *rowptr, *bcol;
  const double *bval, *X, *G;
  const double *opt_record;                // KParams::opt_record of the agent
  double *partials;                        // status_ctas(n) x 3 per-CTA partial sums
  unsigned *ticket;                        // CTAs of the agent done in this launch (the last one resets it to 0)
  double *out;                             // DPGO_STATUS_DOUBLES
};
constexpr int STATUS_THREADS = 256;
constexpr int STATUS_ROWS = 32;
__host__ __device__ inline int status_ctas(int n) { return (n + STATUS_ROWS - 1) / STATUS_ROWS; }
cudaError_t launch_agents_status(int r, int dh, int njobs, int total_ctas, const StatusJob *jobs, cudaStream_t stream);
// T = [proj_SO(d)(Ya^T X_i R-block), Ya^T X_i t - Ya^T pa] per pose (d x (d+1)n column-major); anchor = [Ya pa], r x (d+1)
cudaError_t launch_trajectory_global(int r, int dh, int n, const double *anchor, const double *X, double *T, cudaStream_t stream);

// ---- greedy independent-set selection (dpgo_select.cu) ----
// One CTA: rank of every agent by records[a * DPGO_STATUS_DOUBLES + 2] (|rgrad|^2) decreasing, ties by lower id; then the
// greedy walk in that order over the agent graph (CSR adj_ptr / adj): an agent is taken unless a neighbour already is.
// mask[a] = 1 for a taken agent; the mask is also appended to log + (*log_count) * k, and *log_count is incremented.
constexpr int SELECT_MAX_AGENTS = 1024;
cudaError_t launch_select_independent(int k, const double *records, const int *adj_ptr, const int *adj, unsigned char *mask,
                                      unsigned char *log, unsigned long long *log_count, cudaStream_t stream);

// ---- accelerated rounds (dpgo_accel.cu) ----
// Momentum record of an agent: {gamma, alpha, iterations, gamma of the last round, optimising calls at the last begin}; slot
// 3 is the gamma the round's V update uses, which a restart has already cleared from slot 0; slot 4 is KParams::opt_record[1]
// as the round began, from which the finish launch counts the round as one optimising call.
constexpr int ACCEL_STATE_DOUBLES = 5;
// One agent of an accelerated begin launch: CTAs [cta0, cta0 + accel_ctas(n)) own ACCEL_THREADS consecutive poses each.
struct AccelJob {
  int n, cta0, active;
  double *X, *Y, *V, *XP;
  double *state;                           // ACCEL_STATE_DOUBLES
  const double *opt_record;                // KParams::opt_record of the agent (its count is snapshot into state[4])
  const int *pub_slot;                     // n: public slot of the pose, -1 when it is not public
  double *send_x, *send_y;                 // the agent's public tiles of X and of Y
  unsigned *ticket;                        // CTAs of the agent done in this launch (the last one resets it to 0)
};
constexpr int ACCEL_THREADS = 128;
__host__ __device__ inline int accel_ctas(int n) { return (n + ACCEL_THREADS - 1) / ACCEL_THREADS; }
cudaError_t launch_accel_agents(int r, int dh, int njobs, int total_ctas, const AccelJob *jobs, double momentum_n,
                                int restart_interval, cudaStream_t stream);
// ACCEL_FINISH_V and ACCEL_FINISH_RESTART_END end a round: they also write opt_record = {sqrt(|X - XP|^2 / n), state[4] + 1},
// reducing through partials (accel_ctas(n) doubles) and ticket (the last CTA resets it to 0).
enum AccelFinish { ACCEL_FINISH_V = 0, ACCEL_FINISH_V_RESTART = 1, ACCEL_FINISH_RESTART_END = 2 };
cudaError_t launch_accel_finish(int r, int dh, int n, double *X, double *Y, double *V, const double *XP, const double *state,
                                int mode, double *partials, unsigned *ticket, double *opt_record, cudaStream_t stream);

}  // namespace dpgo
