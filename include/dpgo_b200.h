/*
 * dpgo_b200.h -- C ABI of the GPU-native (H100, sm_90a) pose-graph-optimisation hot path.
 *
 * This is the drop-in boundary: every entry point replaces one piece of the reference's
 * (tjcunhao/dpo, fork of mit-acl/dpgo) C++ interface for the per-iteration path.  The
 * reference has no C ABI of its own; the C++ mirror under include/DPGO/ (same class names and
 * signatures as the reference) and the Python mirror dpo_b200/ are thin hosts over this file.
 * "ref:" comments cite the reference interface each function stands in for (paths relative
 * to the reference root).
 *
 * Conventions
 *   - plain pointers and sizes only; no C++/torch types; all functions return a status code
 *     (DPGO_OK == 0) and never throw or abort.  dpgo_last_error() gives a thread-local message.
 *   - dense arrays are COLUMN-MAJOR r x (d+1)n doubles; pose i is the contiguous r x (d+1)
 *     tile at columns [(d+1)i, (d+1)(i+1)) (layout pinned by ref tests/testEigenMap.cpp:12-36).
 *   - "host" pointers are caller-owned CPU memory (the library copies in/out);
 *     "dev" pointers are CUDA device memory on the problem's device.
 *   - one opaque handle <-> one GPU <-> one CUDA stream; a handle is used by one thread at a
 *     time (ref: a QuadraticProblem is used by one thread at a time, src/PGOAgent.cpp:676-682).
 *   - all arithmetic is fp64.  There is NO CPU fallback: without a usable CUDA device
 *     dpgo_problem_create() fails with DPGO_ERR_NO_DEVICE.
 */
#ifndef DPGO_B200_H
#define DPGO_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define DPGO_B200_ABI_VERSION 1

/* Largest relaxation rank r: a pose tile's r lifted rows are the rows of the 8 x 4 A fragment of the fp64 tensor op
   (mma.sync m8n8k4) in the product with Q and in the block solve. */
#define DPGO_MAX_RANK 8

#if defined(__GNUC__)
#define DPGO_API __attribute__((visibility("default")))
#else
#define DPGO_API
#endif

/* ---- status codes ------------------------------------------------------------------ */
enum {
  DPGO_OK = 0,
  DPGO_ERR_INVALID_ARG = 1, /* shape / pointer / range violation (ref: assert() on shapes,
                               src/QuadraticProblem.cpp:32-33,51-52) */
  DPGO_ERR_NO_DEVICE = 2,   /* no CUDA device / device index out of range */
  DPGO_ERR_CUDA = 3,        /* a CUDA runtime call or kernel failed, or a numerical solve failed (the chordal
                               initialisation's conjugate gradients broke down or did not converge in max_iter) */
  DPGO_ERR_STATE = 4,       /* call order violation (e.g. optimise before set_Q) */
  DPGO_ERR_UNSUPPORTED = 5, /* d not in {2,3}; r above DPGO_MAX_RANK (every d <= r <= 8 is compiled); an exact
                               preconditioner whose blocks would exceed 24 GB (DENSE_EXACT: N above about 54k) */
  DPGO_ERR_ALLOC = 6
};

/* ---- enums mirrored from the reference ----------------------------------------------- */
/* ref: include/DPGO/DPGO_types.h:29-35 (ROPTALG) */
enum { DPGO_ALG_RTR = 0, DPGO_ALG_RGD = 1 };

/* Preconditioner used inside truncated CG.
 * ref: src/QuadraticProblem.cpp:31-42,75-87: exact solve with Q + 0.1 I (CHOLMOD) followed by
 * tangent projection.  SPARSE_EXACT applies it through a nested-dissection block factorisation (dense
 * Schur-complement blocks on 2-4 macro levels, L2-resident for sphere2500-sized agents; O(n log n)-ish memory instead
 * of O(n^2)): the default, and what "exact" means everywhere below.  DENSE_EXACT applies the same operator with the
 * same block solve on a single macro level: the dense inverse of every connected component, 8 N^2 bytes in HBM
 * streamed per application (an A/B reference for the default).  BLOCK_JACOBI is the SpMV-only throughput mode (same
 * fixed points, different inner iterates); NONE is projection only. */
enum { DPGO_PRECOND_NONE = 0, DPGO_PRECOND_BLOCK_JACOBI = 1, DPGO_PRECOND_DENSE_EXACT = 2, DPGO_PRECOND_SPARSE_EXACT = 3 };

/* ref: ROPTLIB tCGstatusSet as recorded by src/QuadraticOptimizer.cpp:115 */
enum {
  DPGO_TCG_NEGCURVTURE = 0, DPGO_TCG_EXCREGION = 1, DPGO_TCG_LCON = 2, DPGO_TCG_SCON = 3,
  DPGO_TCG_MAXITER = 4, DPGO_TCG_NOT_RUN = -1
};

typedef struct dpgo_problem dpgo_problem_t; /* opaque: QuadraticProblem + manifold + device state */

/* Solver knobs.  ref: include/DPGO/QuadraticOptimizer.h:36-70 setters; defaults
 * src/QuadraticOptimizer.cpp:20-29 (RTR, step 1e-3, 1 iteration, tol 1e-2, radius 10, 50 inner). */
typedef struct dpgo_opt_params {
  int32_t algorithm;          /* DPGO_ALG_* */
  int32_t tr_iterations;      /* setTrustRegionIterations */
  int32_t tr_max_inner;       /* setTrustRegionMaxInnerIterations */
  int32_t precond;            /* DPGO_PRECOND_* (must have been prepared by set_Q) */
  double rgd_stepsize;        /* setGradientDescentStepsize */
  double tr_tolerance;        /* setTrustRegionTolerance */
  double tr_initial_radius;   /* setTrustRegionInitialRadius */
} dpgo_opt_params_t;

/* ref: include/DPGO/DPGO_types.h:40-59 (ROPTResult) + bookkeeping counters. */
typedef struct dpgo_opt_result {
  int32_t success;
  int32_t tcg_status;        /* status of the last tCG solve (after a give-up: that of the last rejected attempt;
                                the reference returns before recording one) */
  int32_t tcg_iterations;    /* inner iterations summed over all attempts */
  int32_t outer_iterations;  /* RTR attempts executed (accepted + rejected) */
  int32_t rejections;        /* rejected attempts */
  int32_t spmv_passes;       /* passes over Q executed inside the call */
  int32_t precond_applies;   /* applications of the tCG preconditioner M^-1: one z0 per attempt, a z0 reused
                                after a rejection included, plus one per inner iteration that did not stop */
  int32_t reserved0;
  double f_init, gradnorm_init, f_opt, gradnorm_opt, relative_change, elapsed_ms;
  double quad_init, lin_init; /* <XQ,X> and <X,G> at the input point: f = quad/2 + lin; summed over agents,
                                 (quad + lin)/2 is the centralised cost (shared-edge cross terms count once) */
} dpgo_opt_result_t;

/* ---- library / device ---------------------------------------------------------------- */
DPGO_API int dpgo_abi_version(void);
DPGO_API const char *dpgo_last_error(void);
DPGO_API int dpgo_device_count(int *count);
DPGO_API void dpgo_opt_params_default(dpgo_opt_params_t *p);

/* ---- problem lifetime.  ref: QuadraticProblem ctor/dtor, include/DPGO/QuadraticProblem.h:33-35 */
DPGO_API int dpgo_problem_create(int n, int d, int r, int device, dpgo_problem_t **out);
DPGO_API int dpgo_problem_destroy(dpgo_problem_t *p);
/* Run the handle's work on a caller-provided cudaStream_t (e.g. torch's current stream). NULL
 * restores the handle's own stream. */
DPGO_API int dpgo_problem_set_stream(dpgo_problem_t *p, void *cuda_stream);
DPGO_API int dpgo_problem_sync(dpgo_problem_t *p);
DPGO_API int dpgo_problem_dims(const dpgo_problem_t *p, int *n, int *d, int *r, int64_t *num_blocks);
/* How the persistent step kernel of this handle is launched; takes effect at the next set_Q (it sizes the row partition
 * and the block-solve plan).  0: cooperative grid over all SMs (default:
 * one agent owns the GPU, as in the reference's one-agent-per-machine deployment, examples/MultiRobotExample.cpp:229-334);
 * 1: ONE thread-block cluster of <= 16 CTAs (non-cooperative launch; hardware cluster barriers end the phases), so that the
 * steps of several small agents of one colour class run side by side on one GPU (dpgo_agents_round_async); -1: default. */
DPGO_API int dpgo_problem_set_launch_mode(dpgo_problem_t *p, int mode);
DPGO_API int dpgo_problem_launch_info(const dpgo_problem_t *p, int *grid, int *cluster);

/* ---- cost matrices ------------------------------------------------------------------- */
/* ref: QuadraticProblem::setQ(const SparseMatrix&), src/QuadraticProblem.cpp:31-42.
 * Q is the scalar row-major CSR exactly as Eigen::SparseMatrix<double,RowMajor> exposes it
 * (outerIndexPtr / innerIndexPtr / valuePtr), (d+1)n x (d+1)n, symmetric.  The library converts
 * it to (d+1)x(d+1) block-CSR in HBM and prepares the preconditioners named in precond_mask
 * (bit i = DPGO_PRECOND_i). */
DPGO_API int dpgo_problem_set_Q_csr(dpgo_problem_t *p, int nrows, const int32_t *rowptr, const int32_t *colind,
                           const double *values, unsigned precond_mask);
/* Same from block triplets: nb blocks, block k at (brow[k], bcol[k]) holds the (d+1)x(d+1)
 * sub-matrix Q[(d+1)brow.., (d+1)bcol..] row-major in blocks[k*(d+1)^2 ..]; duplicates are summed
 * (what ref constructConnectionLaplacianSE / PGOAgent::constructQMatrix produce,
 * src/DPGO_utils.cpp:264-271, src/PGOAgent.cpp:720-781). */
DPGO_API int dpgo_problem_set_Q_blocks(dpgo_problem_t *p, int64_t nb, const int32_t *brow, const int32_t *bcol,
                              const double *blocks, unsigned precond_mask);
/* Q assembled ON THE DEVICE from raw edge records (ref constructConnectionLaplacianSE, src/DPGO_utils.cpp:199-271, and the
 * shared-edge diagonal terms of PGOAgent::constructQMatrix, src/PGOAgent.cpp:720-781).  m private edges p1 -> p2 (local pose
 * ids), R: m x d x d row-major, t: m x d, kappa / tau / weight: m (weight NULL = 1), fixed_weight: m flags (NULL = none; a
 * fixed edge keeps its weight in dpgo_problem_robust_reweight: the reference's isKnownInlier, e.g. odometry); plus
 * num_static blocks added at (static_pose, static_pose), (d+1)x(d+1) row-major each (already weighted).  The block pattern
 * is built on the host once, the values by k_assemble_Q; re-assembly after a weight change keeps the pattern. */
DPGO_API int dpgo_problem_set_edges(dpgo_problem_t *p, int64_t m, const int32_t *p1, const int32_t *p2, const double *R,
                                    const double *t, const double *kappa, const double *tau, const double *weight,
                                    const int32_t *fixed_weight, int64_t num_static, const int32_t *static_pose,
                                    const double *static_blocks, unsigned precond_mask);
/* Robust re-weighting at the resident iterate (ref PGOAgent::updateLoopClosuresWeights, src/PGOAgent.cpp:1181-1245;
 * RobustCost::weight, src/DPGO_robust.cpp:23-66): w_e = weight(sqrt(kappa |Y_i R - Y_j|^2 + tau |p_j - p_i - Y_i t|^2)) for
 * every non-fixed edge, then Q is re-assembled on the device and the preconditioners are refreshed.
 * cost: 0 L2, 1 L1, 2 Huber(param), 3 TLS(param), 4 Geman-McClure, 5 GNC_TLS(mu, param = cbar).
 * weights_host / residuals2_host (nullable): the new weights and the squared residuals, m each. */
DPGO_API int dpgo_problem_robust_reweight(dpgo_problem_t *p, int cost, double mu, double param, double *weights_host,
                                          double *residuals2_host);
/* replace the edge weights (m values) and re-assemble Q on the device */
DPGO_API int dpgo_problem_set_edge_weights(dpgo_problem_t *p, const double *weights_host);
/* Stream-ordered re-weighting: the reference re-weights the loop closures and rebuilds Q and its factorisation every
 * robustOptInnerIters iterations (PGOAgent::iterate / updateLoopClosuresWeights / constructQMatrix + setQ,
 * src/PGOAgent.cpp:653-667, 1109-1112, 1174-1289).  These calls do it without a host copy or a synchronisation, on the
 * handle's stream: the same weights and the same k_assemble_Q as the synchronous calls above, then every prepared
 * preconditioner is refactorised ON THE DEVICE -- block-Jacobi (one 4x4 SPD inverse per pose) and the exact ones (the
 * multifrontal factorisation of each hierarchy, written into its panels in place; a dense exact one not prepared yet is
 * built on its first use).  Device buffers keep their addresses and the handle's generation is not bumped, so a round
 * graph captured before stays valid, and the calls can themselves be captured into a CUDA graph, with one exception that
 * synchronises (and so cannot be captured): the first call after the sparse exact preconditioner's structure was dropped
 * (set_edges, a synchronous re-weight) or never built builds its hierarchy and plan on the host, as its first use does.
 * A front that is not positive definite (impossible for weights >= 0) sets a device flag that the next synchronising call
 * (dpgo_problem_sync, dpgo_optimize_result, dpgo_problem_gnc_counts, ...) reports as DPGO_ERR_CUDA.
 * weights_dev: m doubles in device memory on the handle's device, read in stream order. */
DPGO_API int dpgo_problem_set_edge_weights_async(dpgo_problem_t *p, const double *weights_dev);
DPGO_API int dpgo_problem_robust_reweight_async(dpgo_problem_t *p, int cost, double mu, double param);
/* The device arrays of the edge weights and of the squared residuals of the last re-weight (m doubles each), for reading
 * or for writing weights in place before dpgo_problem_set_edge_weights_async(p, *w_dev). */
DPGO_API int dpgo_problem_device_edge_weights(dpgo_problem_t *p, double **w_dev, double **res2_dev);
/* Counts of the last re-weight over the non-fixed edges: out3 = {weight exactly 1, exactly 0, in between} -- what the
 * reference's PGOAgent::computeConvergedLoopClosureRatio counts (src/PGOAgent.cpp:1247-1289).  Synchronises. */
DPGO_API int dpgo_problem_gnc_counts(dpgo_problem_t *p, int64_t *out3);
/* ref: QuadraticProblem::setG, src/QuadraticProblem.cpp:44-48.  Dense r x (d+1)n column-major,
 * or the reference's sparse form (row-major CSR with r rows).  NULL / nnz == 0 clears G. */
DPGO_API int dpgo_problem_set_G_dense(dpgo_problem_t *p, const double *G_host);
DPGO_API int dpgo_problem_set_G_csr(dpgo_problem_t *p, const int32_t *rowptr, const int32_t *colind,
                           const double *values);

/* ---- evaluation (host in / host out) --------------------------------------------------- */
/* ref: QuadraticProblem::f, src/QuadraticProblem.cpp:50-60 */
DPGO_API int dpgo_problem_f(dpgo_problem_t *p, const double *X_host, double *f_out);
/* ref: QuadraticProblem::EucGrad, :62-66  (Out = X Q + G) */
DPGO_API int dpgo_problem_egrad(dpgo_problem_t *p, const double *X_host, double *out_host);
/* ref: QuadraticProblem::EucHessianEta, :68-73  (Out = V Q) */
DPGO_API int dpgo_problem_ehess(dpgo_problem_t *p, const double *V_host, double *out_host);
/* ref: QuadraticProblem::RieGrad / RieGradNorm, :89-101.  Either output may be NULL. */
DPGO_API int dpgo_problem_rgrad(dpgo_problem_t *p, const double *X_host, double *out_host, double *norm_out);
/* f, Riemannian gradient norm in ONE pass over Q (what optimize() needs before/after) */
DPGO_API int dpgo_problem_f_rgradnorm(dpgo_problem_t *p, const double *X_host, double *f_out, double *norm_out);
/* Riemannian Hessian-vector product at X: ROPTLIB Problem::HessianEta = EucHessianEta +
 * Stiefel::EucHvToHv + projection (call site src/QuadraticOptimizer.cpp:76-119). */
DPGO_API int dpgo_problem_rhess(dpgo_problem_t *p, const double *X_host, const double *V_host, double *out_host);
/* ref: QuadraticProblem::PreConditioner, :75-87 */
DPGO_API int dpgo_problem_precon(dpgo_problem_t *p, int precond, const double *X_host, const double *V_host,
                        double *out_host);

/* ---- manifold (St(d,r) x R^r)^n ------------------------------------------------------- */
/* ROPTLIB ProductManifold::Projection (tangent projection at X), call sites
 * src/QuadraticProblem.cpp:82,95, src/QuadraticOptimizer.cpp:139 */
DPGO_API int dpgo_manifold_tangent_project(dpgo_problem_t *p, const double *X_host, const double *Z_host,
                                  double *out_host);
/* ROPTLIB ProductManifold::Retraction (QF per pose), src/QuadraticOptimizer.cpp:146 */
DPGO_API int dpgo_manifold_retract(dpgo_problem_t *p, const double *X_host, const double *eta_host,
                          double *out_host);
/* ref: LiftedSEManifold::project, src/manifold/LiftedSEManifold.cpp:34-45 (polar factor per pose) */
DPGO_API int dpgo_manifold_project(dpgo_problem_t *p, const double *M_host, double *out_host);

/* ---- optimiser ------------------------------------------------------------------------ */
/* ref: QuadraticOptimizer::optimize(const Matrix&), src/QuadraticOptimizer.cpp:34-59: one
 * RTR (Riemannian trust region, truncated-CG inner solve) or RGD call, the whole loop on the
 * device in one persistent kernel; host sees only X_out and the result record. */
DPGO_API int dpgo_optimize(dpgo_problem_t *p, const dpgo_opt_params_t *params, const double *X_in_host,
                  double *X_out_host, dpgo_opt_result_t *result);

/* ---- device-resident path (iterate lives in HBM between calls) --------------------------- */
DPGO_API int dpgo_problem_upload_X(dpgo_problem_t *p, const double *X_host);
DPGO_API int dpgo_problem_download_X(dpgo_problem_t *p, double *X_host);
/* the same without the closing synchronisation (pinned host buffers; order with dpgo_problem_sync): one round of a
 * multi-agent run = upload_X_async, exchange, optimize_resident_async, download_X_async, sync */
DPGO_API int dpgo_problem_upload_X_async(dpgo_problem_t *p, const double *X_host);
DPGO_API int dpgo_problem_download_X_async(dpgo_problem_t *p, double *X_host);
/* resident iterate <- device buffer (asynchronous device-to-device copy on the handle's stream) */
DPGO_API int dpgo_problem_copy_X_from_device(dpgo_problem_t *p, const double *X_dev);
DPGO_API int dpgo_problem_device_X(dpgo_problem_t *p, double **X_dev);     /* r x (d+1)n, read/write */
DPGO_API int dpgo_problem_device_G(dpgo_problem_t *p, double **G_dev);
/* optimise the resident iterate in place; asynchronous on the handle's stream */
DPGO_API int dpgo_optimize_resident_async(dpgo_problem_t *p, const dpgo_opt_params_t *params);
/* wait for the last async optimise and fetch its result record */
DPGO_API int dpgo_optimize_result(dpgo_problem_t *p, dpgo_opt_result_t *result);
/* the Q.X product kernel alone on device buffers (the roofline kernel): Out = X Q (+ G) */
DPGO_API int dpgo_spmv_device(dpgo_problem_t *p, const double *X_dev, double *out_dev, int add_G);
DPGO_API int64_t dpgo_spmv_algorithmic_bytes(const dpgo_problem_t *p, int add_G);
/* bytes one application of the preconditioner (ref: QuadraticProblem::PreConditioner, src/QuadraticProblem.cpp:75-87)
 * has to move: the operator's blocks + input and output vector.  An exact preconditioner reports 0 until it has been
 * prepared (its first use); DENSE_EXACT then streams 8 N^2 bytes of blocks for a connected graph with an even n. */
DPGO_API int64_t dpgo_precond_algorithmic_bytes(const dpgo_problem_t *p, int preconditioner);
/* ---- sparse exact preconditioner: diagnostics ------------------------------------------------------------------ */
/* info[16] of the prepared hierarchy (prepares it if needed): 0 macro levels, 1 macro nodes, 2 phases per application,
 * 3 bytes of all blocks, 4 matrix bytes streamed per application, 5 largest own block (scalars), 6 largest boundary
 * (scalars), 7 dissection depth, 8 steps, 9 jobs, 10 epilogues, 11.. reserved */
DPGO_API int dpgo_nd_info(dpgo_problem_t *p, int64_t *info16);
/* Sizes of the hierarchy's macro nodes (prepares it if needed): *count nodes; the first min(cap, count) get their own and
 * boundary pose counts and their stage (0 = deepest).  The work of a refactorisation follows from them. */
DPGO_API int dpgo_nd_node_sizes(dpgo_problem_t *p, int64_t cap, int32_t *own, int32_t *bnd, int32_t *stage, int64_t *count);
/* HOST ONLY, verification of the planning code on machines without a GPU (never used by a product path): builds the
 * hierarchy, the blocks and the phase plan for the block matrix given as in dpgo_problem_set_Q_blocks and runs a host
 * emulation of the plan exactly as the kernel interprets it:  Z = (Q + shift I)^-1 V  (no projection), V and Z
 * r x (d+1)n column-major.  force_cuts < 0 lets the cost model choose the macro levels.  info16 as in dpgo_nd_info. */
DPGO_API int dpgo_nd_debug_emulate(int n, int d, int r, int64_t nb, const int32_t *brow, const int32_t *bcol,
                                   const double *blocks, double shift, int grid, int force_cuts, int leaf_size,
                                   const double *V_host, double *Z_host, int64_t *info16);
/* diagnostic: cost of one empty phase of the persistent kernel (grid barrier + scalar reduction) and of its launch */
DPGO_API int dpgo_debug_phase_latency(dpgo_problem_t *p, int phases, double *us_per_phase, double *us_launch);
/* diagnostic: phase clock of the persistent kernel.  enable != 0 switches it on (subsequent optimise calls
 * accumulate, per phase kind, the nanoseconds CTA 0 spent up to the closing grid barrier); every call returns the
 * accumulated milliseconds in ms_by_kind[64] and resets them; enable == 0 switches it off.  Slots: 0 eval pass,
 * 3 Hessian product, 4 tCG update, 5 retraction, 6 final; 8 + k = phase k of an exact preconditioner's application
 * (k < 16; DENSE_EXACT has phase 0 only), 24 / 25 / 26 = gathers / panel jobs / epilogues of those phases as seen by
 * CTA 0; 32 + 3 k + {0, 1, 2} = gathers / panel jobs / epilogues of phase k (k < 10) as seen by CTA 0; others unused. */
DPGO_API int dpgo_debug_phase_times64(dpgo_problem_t *p, int enable, double *ms_by_kind);

/* ---- chordal initialisation on the GPU ------------------------------------------------------------------------
 * ref: chordalInitialization, src/DPGO_utils.cpp:273-461 (two sparse least-squares problems, SPQR there; gauge R_0 = I,
 * t_0 = 0) + projectToRotationGroup :463-477.  Both normal systems are 3 x 3-block connection Laplacians, solved by
 * Jacobi-preconditioned conjugate gradients whose product is the TMA-fed block-CSR kernel of the hot path.
 * m edges p1 -> p2 (pose ids), R: m x d x d row-major, t: m x d, kappa / tau: m.  T_host: d x (d+1)n column-major
 * ([R_p t_p] per pose, the layout of the reference's Matrix).  tol: relative residual in the Jacobi-scaled norm (<= 0:
 * 1e-11); max_iter: CG iteration cap per solve (<= 0: 50000).  A solve that does not reach tol within max_iter iterations,
 * or whose residual turns NaN, fails with DPGO_ERR_CUDA; poses outside the connected component of pose 0 get R = I.
 * iterations2[2] (nullable) receives the CG iteration counts of the two solves.  Arguments are checked before any device
 * call; n = 1 needs no device.  dpgo_chordal_last_error() for the message. */
DPGO_API int dpgo_chordal_initialization(int n, int d, int64_t m, const int32_t *p1, const int32_t *p2, const double *R,
                                         const double *t, const double *kappa, const double *tau, int device, double tol,
                                         int max_iter, double *T_host, int32_t *iterations2);
DPGO_API const char *dpgo_chordal_last_error(void);

/* ---- pose marginal covariances on the GPU ----------------------------------------------------------------------
 * The uncertainty of a trajectory T (d x (d+1)n column-major, [R_p t_p] per pose: a rounded solution) under the
 * Gauss-Newton information of the edges (p1, p2, R, t, kappa, tau as in dpgo_chordal_initialization; weight: m, nullable =
 * all 1; every edge joins two different poses):
 *   perturbation   right (body frame), R_p exp([w_p]x) and t_p + R_p v_p; tangent x_p = (w_p, v_p) of dimension
 *                  b = 6 (d = 3) or b = 3 (d = 2, w_p the angle), in that order;
 *   residuals      R_j - R_i R_ij (weight kappa) and t_j - t_i - R_i t_ij (weight tau) of every edge i -> j, scaled so
 *                  that sum_e 1/2 r^T Om_e r (Om_e = weight diag(kappa .., tau ..)) is f = 1/2 <Q, T^T T> with Q the
 *                  connection Laplacian;
 *   information    H = sum_e J_e^T Om_e J_e at T (Gauss-Newton: positive semidefinite at any trajectory, with a null
 *                  space of dimension b on a connected graph: the gauge);
 *   covariance     Sigma = H_anchored^-1, the anchor pose's b rows and columns dropped (its blocks are reported as 0).
 * cov_host receives the b x b diagonal block of every pose (n b b doubles, row-major blocks); pair_cov_host the b x b
 * block Sigma[x_i, x_j] of each of the num_pairs pairs (i, j) = (pairs[2q], pairs[2q+1]).  Nothing dense: H is assembled,
 * factored and selectively inverted on the device over the nested-dissection fronts of its block pattern, in fixed
 * summation orders (two calls are bitwise equal).  The requested pairs join that pattern as structural blocks, so both
 * poses of a pair share a front and every pair block is read from one.  That has a cost: each pair is an extra edge for
 * the dissection, so many long-range pairs (loop-closure gating over a whole map) enlarge the separators, and the
 * factorisation's work and device memory (info16[4]) grow with them, up to dense fronts; requesting pairs also changes
 * the hierarchy, so the diagonal blocks of a call with pairs may differ in the last bits from one without.  Arguments
 * (ranges, finite non-negative precisions and weights, a finite trajectory, every pose connected to the anchor by edges
 * of positive weight and a positive kappa or tau) are checked before any device call (DPGO_ERR_INVALID_ARG).  That
 * check is on the graph only: information that is still singular (a pose whose edges all have tau = 0, so its
 * translation is free) fails in the factorisation with a pivot that is not positive (DPGO_ERR_CUDA), and information
 * that is merely ill-conditioned returns its (large, fp64-accurate to about cond(H) eps) inverse.  info16 (nullable): 0 macro levels, 1 macro nodes, 2 3-scalar nodes of H (d = 2: n, d = 3: 2n),
 * 3 blocks of H, 4 device bytes of H + factor + fronts, 5 largest own block (scalars), 6 largest boundary (scalars),
 * 7 dissection depth, 8 3 x 3 output blocks, 9 stages (factor + sweep), 10 / 11 / 12 assembly / factorisation /
 * selected-inversion nanoseconds (device events), 13 largest number of macro nodes in one stage (a stage of more than
 * 65535 runs in several launches), others 0.  n = 1 needs no device.  Messages: dpgo_last_error(). */
DPGO_API int dpgo_pose_covariances(int n, int d, int64_t m, const int32_t *p1, const int32_t *p2, const double *R,
                                   const double *t, const double *kappa, const double *tau, const double *weight,
                                   const double *T_host, int anchor, int device, int64_t num_pairs, const int32_t *pairs,
                                   double *cov_host, double *pair_cov_host, int64_t *info16);
/* HOST ONLY, verification on machines without a GPU (never used by a product path): the same pattern, hierarchy and
 * output blocks as dpgo_pose_covariances, the assembly kernel's arithmetic on the host, the host factorisation
 * (nd build_numeric, shift 0) and a host emulation of the selected-inversion sweep.  force_cuts < 0 lets the cost model
 * choose the macro levels, leaf_size <= 0 keeps the default.  info16 as above without the times. */
DPGO_API int dpgo_pose_covariances_debug_emulate(int n, int d, int64_t m, const int32_t *p1, const int32_t *p2,
                                                 const double *R, const double *t, const double *kappa, const double *tau,
                                                 const double *weight, const double *T_host, int anchor, int force_cuts,
                                                 int leaf_size, int64_t num_pairs, const int32_t *pairs, double *cov_host,
                                                 double *pair_cov_host, int64_t *info16);

/* ---- plain device helpers for hosts that drive several GPUs without linking the CUDA runtime themselves (the C++
 *      multi-GPU runner: exchange buffers + one stream per GPU, NCCL calls on those streams) ---------------------- */
DPGO_API int dpgo_device_set(int device);                                /* cudaSetDevice for the calling thread */
DPGO_API int dpgo_device_malloc(int device, size_t bytes, void **ptr);   /* zero-initialised */
DPGO_API int dpgo_device_free(int device, void *ptr);
DPGO_API int dpgo_stream_create(int device, void **cuda_stream);
DPGO_API int dpgo_stream_destroy(int device, void *cuda_stream);
DPGO_API int dpgo_stream_synchronize(int device, void *cuda_stream);

/* ---- boundary-pose exchange (multi-agent, one agent per GPU) ----------------------------- */
/* ref: PGOAgent::getSharedPoseDict, src/PGOAgent.cpp:95-105: register which local poses are
 * public; pack gathers their r x (d+1) tiles into a contiguous device buffer (the NCCL
 * all-gather send buffer), slot s <- pose public_pose[s]. */
DPGO_API int dpgo_agent_set_public_poses(dpgo_problem_t *p, int num_public, const int32_t *public_pose);
DPGO_API int dpgo_agent_pack_public(dpgo_problem_t *p, double *send_dev);
/* ref: PGOAgent::constructGMatrix, src/PGOAgent.cpp:783-859.  Shared edge e touches local pose
 * local_pose[e]; its neighbour pose is tile nbr_slot[e] of the gathered buffer; outgoing[e]!=0
 * means this agent owns the edge tail (G_p1 += -X_j Om T^T) else the head (G_p2 += -X_i T Om).
 * T is (d+1)x(d+1) row-major per edge, omega the (d+1) diagonal weights (kappa..,tau)*weight. */
DPGO_API int dpgo_agent_set_shared_edges(dpgo_problem_t *p, int num_edges, const int32_t *local_pose,
                                const int32_t *nbr_slot, const int32_t *outgoing, const double *T,
                                const double *omega);
/* rebuild G in HBM from the gathered neighbour tiles (deterministic: edges grouped per pose) */
DPGO_API int dpgo_agent_build_G(dpgo_problem_t *p, const double *gathered_dev, int64_t num_slots);
/* ---- Nesterov-accelerated RBCD on the resident iterate (ref src/PGOAgent.cpp:685-695 iterate, :1040-1091 updateGamma /
 *      updateAlpha / updateY / updateV / restart; the scalars gamma, alpha stay with the host, which follows the reference's
 *      recurrences).  All calls are asynchronous on the handle's stream. */
DPGO_API int dpgo_agent_accel_init(dpgo_problem_t *p);                     /* V = Y = XPrev = X        (ref :60-62, :1040-1052) */
DPGO_API int dpgo_agent_accel_begin(dpgo_problem_t *p, double alpha);       /* XPrev = X; Y = proj((1 - alpha) X + alpha V)  (ref :1077-1083) */
/* optimized == 0: X = Y (ref updateX(false, true), :1095-1098); then V = proj(V + gamma (X - Y))  (ref :1085-1091) */
DPGO_API int dpgo_agent_accel_end(dpgo_problem_t *p, double gamma, int optimized);
DPGO_API int dpgo_agent_accel_restart_begin(dpgo_problem_t *p);             /* X = XPrev  (then the caller takes a plain step) */
DPGO_API int dpgo_agent_accel_restart_end(dpgo_problem_t *p);               /* V = Y = X */
/* public tiles of the auxiliary iterate Y (ref getAuxSharedPoseDict, :107-118) */
DPGO_API int dpgo_agent_pack_public_aux(dpgo_problem_t *p, double *send_dev);
/* One RBCD round of the active agents of one GPU with one call (ref: the body of the round loop,
 * examples/MultiRobotExample.cpp:229-334: updateNeighborPoses -> iterate() -> getSharedPoseDict per selected agent).
 * Per agent: G rebuild from gathered_dev -> RTR step -> pack of its public tiles into send_dev[i] (thread-block cluster
 * agents on their own streams between a fork from and a join into main_stream, full-grid agents in order on main_stream).
 * main_stream NULL = the stream the first handle is set to.  pack_after_join != 0 issues the packs in a second pass,
 * after every agent's step (needed when neighbouring agents are active in the same round and send_dev aliases
 * gathered_dev).  A repeated round of cluster agents is replayed as a CUDA graph; a round with a full-grid agent is issued
 * eagerly (a cooperative launch does not capture).  DPGO_ROUND_GRAPH=0 keeps the eager launches.  A handle listed twice
 * is refused with DPGO_ERR_INVALID_ARG. */
DPGO_API int dpgo_agents_round_async(dpgo_problem_t *const *agents, int num_active, const dpgo_opt_params_t *params,
                            const double *gathered_dev, int64_t num_slots, double *const *send_dev, void *main_stream,
                            int pack_after_join);
/* The host boundary of a round with one call per direction (ref: the host matrices PGOAgent::setX / getX move,
 * src/PGOAgent.cpp:66-93): direction 0 = X of every listed agent from (pinned) host memory, then its public tiles packed
 * into send_dev[i] (send_dev may be NULL); direction 1 = X back to host memory.  Asynchronous on `stream` (NULL: the
 * stream the first handle is set to); a repeated call is replayed as a CUDA graph.  A handle listed twice is refused with
 * DPGO_ERR_INVALID_ARG. */
DPGO_API int dpgo_agents_host_io_async(dpgo_problem_t *const *agents, int count, double *const *X_host,
                              double *const *send_dev, int direction, void *stream);
/* ---- accelerated rounds with one call per GPU (ref src/PGOAgent.cpp:685-695,1033-1091; examples/MultiRobotExample.cpp:
 *      236-279): the momentum record {gamma, alpha, iterations} of each agent lives on the device ---------------------- */
/* Begins a round for `count` agents of one device (after dpgo_agent_accel_init and dpgo_agent_set_public_poses): advances
 * every agent's record, gamma' = (1 + sqrt(1 + ((4 N) N) (gamma gamma))) / (2 N), alpha = 1 / (gamma' N) with N = momentum_N,
 * bit for bit in this operation order; XPrev = X; Y = proj((1 - alpha) X + alpha V).  An agent with active_flags[i] == 0
 * finishes its iterate(false): X = Y, V = proj(V + gamma (X - Y)), and on a restart round ((iterations + 1) %
 * restart_interval == 0) X = XPrev, V = Y = X, gamma = alpha = 0.  Then every agent's public tiles of X and Y go to
 * send_dev[i] and send_aux_dev[i].  One launch on `stream` (NULL: the first agent's).  Calls that share an agent must be
 * ordered (one ticket counter per agent), and a handle listed twice in one call is refused with DPGO_ERR_INVALID_ARG.
 * Job tables are kept per agent list, active set and send buffers, as for dpgo_agents_status_async. */
DPGO_API int dpgo_agents_accel_begin_async(dpgo_problem_t *const *agents, int count, const int32_t *active_flags,
                                           double momentum_N, int restart_interval, double *const *send_dev,
                                           double *const *send_aux_dev, void *stream);
/* The active agents' part of the round begun by dpgo_agents_accel_begin_async, once the X tiles are in gathered_dev and
 * the Y tiles in gathered_aux_dev.  Per agent: G from the Y tiles -> X = Y -> one step (thread-block cluster agents on
 * their own streams between a fork from and a join into main_stream, full-grid agents in order on main_stream) ->
 * V = proj(V + gamma (X - Y)); on a restart round then X = XPrev -> G from the X tiles -> one plain step -> V = Y = X.
 * The round then counts as ONE optimising call of the agent, as the reference's iterate() (src/PGOAgent.cpp:673,703-716):
 * its status record (dpgo_agents_status_async) gets [3] = sqrt(|X - XPrev|^2 / n), X the iterate after the V update and
 * any restart, XPrev the iterate at the round's begin, and [4] = the count at the begin + 1, on plain and restart rounds
 * alike.  Agents idle in the round keep their fields [3] and [4].  Nothing is packed.  A repeated round is replayed as a CUDA graph (two variants per active set: plain and restart);
 * DPGO_ROUND_GRAPH=0 keeps the eager launches.  A handle listed twice is refused with DPGO_ERR_INVALID_ARG. */
DPGO_API int dpgo_agents_accel_round_async(dpgo_problem_t *const *agents, int num_active, const dpgo_opt_params_t *params,
                                           const double *gathered_dev, const double *gathered_aux_dev, int64_t num_slots,
                                           void *main_stream);
/* the agent's momentum record {gamma, alpha, iterations} after every call issued so far (synchronises the device) */
DPGO_API int dpgo_agent_accel_state(dpgo_problem_t *p, double *out3);
/* per-agent Riemannian gradient norm / cost of the resident iterate (greedy selection input) */
DPGO_API int dpgo_agent_f_rgradnorm_resident(dpgo_problem_t *p, double *f_out, double *norm_out);

/* ---- distributed initialisation: every agent starts from the chordal initialisation of its private graph, in its own
 *      frame, and joins the global frame through a robust average of the frame transforms its shared loop closures give
 *      with an initialised neighbour.  ref: PGOAgent::initializeInGlobalFrame, src/PGOAgent.cpp:369-440 ------------- */
/* ref PGOAgent::setPoseGraph, src/PGOAgent.cpp:182-185: the agent's local-frame trajectory T (d x (d+1)n column-major,
 * [R_i t_i] per pose) and the lifting matrix YLift (r x d column-major) stay resident; X = YLift T (agent 0's start). */
DPGO_API int dpgo_agent_set_local_trajectory(dpgo_problem_t *p, const double *T_host, const double *YLift_host);
/* ref computeNeighborTransform / findSharedLoopClosureWithNeighbor, src/PGOAgent.cpp:250-288,922-934: the candidate table.
 * Group g (neighbours in increasing id group_neighbor[g]) holds candidates [group_ptr[g], group_ptr[g+1]), one per public
 * pose of that neighbour the agent shares an edge with, in increasing pose id.  Candidate q: local pose local_pose[q],
 * the neighbour's tile nbr_slot[q] of the gathered buffer, the shared edge's T ((d+1) x (d+1) row-major) and
 * outgoing[q] != 0 when the agent owns the edge tail. */
DPGO_API int dpgo_agent_set_align_candidates(dpgo_problem_t *p, int num_groups, const int32_t *group_neighbor,
                                             const int32_t *group_ptr, const int32_t *local_pose, const int32_t *nbr_slot,
                                             const int32_t *outgoing, const double *T);
/* ref updateNeighborPoses -> initializeInGlobalFrame -> computeRobustNeighborTransformTwoStage, src/PGOAgent.cpp:290-331,
 * 369-440: one call per GPU and wave aligns `count` agents of one device against the gathered public tiles.  Per agent
 * the groups whose neighbour has ready_host[neighbour] != 0 are tried in order (GNC-TLS rotation averaging at the
 * threshold 2 sqrt(2) sin(0.25), ~30 degrees, then the mean translation of the inliers); the first with inliers moves
 * the trajectory into the global frame: X = YLift (T_align T).  Asynchronous on `stream` (NULL: the first agent's).
 * A handle listed twice is refused with DPGO_ERR_INVALID_ARG.  Job tables are kept per agent list, as for
 * dpgo_agents_status_async; the ready flags are uploaded on every call. */
DPGO_API int dpgo_agents_align_async(dpgo_problem_t *const *agents, int count, const double *gathered_dev, int64_t num_slots,
                                     const int32_t *ready_host, int num_agents, void *stream);
/* the agent's last alignment (waits for the stream of the align call that included the agent): T_align (d x (d+1) column-major, nullable) and info4 =
 * {neighbour used (-1: no ready neighbour), candidates, inliers (0: not aligned), GNC iterations} */
DPGO_API int dpgo_agent_align_result(dpgo_problem_t *p, double *T_align_host, int32_t *info4);
/* ref robustSingleRotationAveraging, src/DPGO_utils.cpp:567-629: the same kernel on m host rotations R_host (m x d x d
 * row-major), kappa_host (m, NULL = 1), GNC-TLS threshold `threshold` (chordal).  R_out: d x d row-major; inlier_flags
 * (m, nullable); iterations (nullable): GNC iterations run (0: GNC skipped, every residual small).  Synchronous. */
DPGO_API int dpgo_robust_single_rotation_averaging(int device, int d, int m, const double *R_host, const double *kappa_host,
                                                   double threshold, double *R_out, int32_t *inlier_flags, int32_t *iterations);

/* ---- team status and rounding of the device runners (ref PGOAgentStatus / shouldTerminate, src/PGOAgent.cpp:703-716,
 *      1007-1031; getTrajectoryInGlobalFrame, :500-519) ------------------------------------------------------------ */
/* doubles per agent record of dpgo_agents_status_async:
 *   [0] <XQ, X>   [1] <X, G>   [2] |P_X(XQ + G)|^2 (the same quantities as quad_init, lin_init, gradnorm_init^2 of an
 *   evaluation)   [3] relative change sqrt(|X - XPrev|^2 / n) of the agent's most recent optimising call (RTR or RGD;
 *   evaluations leave it alone)   [4] optimising calls since the handle was created.  An accelerated round of
 *   dpgo_agents_accel_round_async is one optimising call measured from the round's XPrev (see there). */
#define DPGO_STATUS_DOUBLES 5
/* One launch for every listed agent (all on one device, one d and r): agent i's record goes to
 * status_dev + slot[i] * DPGO_STATUS_DOUBLES (device memory; slots distinct).  An agent's record depends only on that
 * agent (fixed work split and reduction order), bit for bit.  Asynchronous on `stream` (NULL: the first agent's).
 * Each agent has one partial-sum buffer and one ticket counter: two status calls that include the same agent must be
 * ordered (one stream, or an event between them), as the round calls of one agent must be.  For the same reason a handle
 * listed twice in one call (under two slots) is refused with DPGO_ERR_INVALID_ARG: its two jobs would share the ticket.
 * The first call with a given agent list (and status_dev) uploads its job table and keeps it with the first agent; a
 * repeated call is a single kernel launch, which a CUDA graph can capture.  A first call cannot be captured.  Up to 32
 * tables are kept per first agent; a 33rd list synchronises the device and frees the oldest table, so a graph that
 * captured a status call stays valid only while its agent list is among the last 32 used with that first agent. */
DPGO_API int dpgo_agents_status_async(dpgo_problem_t *const *agents, int count, const int32_t *slot, double *status_dev,
                                      void *stream);
/* ref getTrajectoryInGlobalFrame: anchor_host = [Ya pa] (r x (d+1) column-major, the driver broadcasts agent 0's pose 0);
 * T_host (d x (d+1)n column-major) gets, per pose, [proj_SO(d)(Ya^T Y_i)  Ya^T p_i - Ya^T pa].  Synchronous. */
DPGO_API int dpgo_agent_trajectory_global(dpgo_problem_t *p, const double *anchor_host, double *T_host);
/* page-locked host memory (the destination of the status records of a C++ host) and a stream-ordered copy into it */
DPGO_API int dpgo_host_alloc_pinned(size_t bytes, void **ptr);
DPGO_API int dpgo_host_free_pinned(void *ptr);
DPGO_API int dpgo_copy_to_host_async(int device, void *dst_host, const void *src_dev, size_t bytes, void *stream);

/* ---- greedy independent-set rounds (schedule "greedy_set" of the device runners): every round steps a maximal set of
 *      agents that share no edge, chosen on the device by block gradient norm (ref examples/MultiRobotExample.cpp:308-325
 *      chooses the single largest) ---------------------------------------------------------------------------------- */
/* The agent graph of a runner's num_agents agents (1..1024) in CSR form: the neighbours of agent a are
 * adj[adj_ptr[a] .. adj_ptr[a+1]).  Kept by `lead`, the first agent of the runner's agents on its GPU; once per runner and
 * GPU.  Empties lead's selection log.  Synchronises the device. */
DPGO_API int dpgo_agents_set_agent_graph(dpgo_problem_t *lead, int num_agents, const int32_t *adj_ptr, const int32_t *adj);
/* One greedy independent-set round of `count` agents of one device (agents[0] = the lead of dpgo_agents_set_agent_graph;
 * agent_index[i] = agents[i]'s id in the agent graph).  One launch on `stream` (NULL: the lead's) selects from the status
 * records of ALL num_agents agents in records_dev (device memory, agent-major, DPGO_STATUS_DOUBLES each, as
 * dpgo_agents_status_async writes them): agents in decreasing |rgrad|^2 (field 2), ties to the lower id, each taken unless a
 * neighbour already is.  The k-byte mask is appended to lead's selection log.  Then, as dpgo_agents_round_async with
 * pack_after_join = 0, every listed agent's G rebuild -> step -> pack into send_dev[i]; the kernels of an agent left out
 * return at entry and touch nothing (iterate, G, tiles, result record, status fields 3 and 4).  The exception is a G clear
 * still pending from dpgo_problem_set_G_*, dpgo_agent_set_shared_edges or dpgo_problem_device_G: it is issued from the
 * host, before the mask exists, so it runs for a left-out agent too.
 * Ordering: the records must be complete on `stream` before the call (e.g. the status launch, or the all-gather of the
 * records, issued earlier on the same stream); the calls that share a lead must be ordered.  A repeated call of cluster
 * agents with the same buffers is replayed as a CUDA graph (the selection is device data, so one graph serves every set;
 * the log's doubling starts a new one); a call with a full-grid agent is issued eagerly, and a left-out full-grid agent
 * still costs its launches.  This call is itself never captured by the caller's graph: the log can grow on the host.
 * Agent indices must be distinct, and so must the handles: either repeated is refused with DPGO_ERR_INVALID_ARG. */
DPGO_API int dpgo_agents_select_round_async(dpgo_problem_t *const *agents, int count, const int32_t *agent_index,
                                            const dpgo_opt_params_t *params, const double *records_dev,
                                            const double *gathered_dev, int64_t num_slots, double *const *send_dev,
                                            void *stream);
/* lead's selection log: *total_rounds = rounds issued since dpgo_agents_set_agent_graph; rounds [first_round,
 * first_round + max_rounds) that exist are copied to out_host, num_agents bytes per round (1 = selected).  Synchronises the
 * device. */
DPGO_API int dpgo_agents_selection_log(dpgo_problem_t *lead, int64_t first_round, int64_t max_rounds, uint8_t *out_host,
                                       int64_t *total_rounds);

#ifdef __cplusplus
}
#endif
#endif /* DPGO_B200_H */
