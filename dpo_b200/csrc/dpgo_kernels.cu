// dpgo_kernels.cu -- sm_90a (H100) kernels of the pose-graph hot path.
//
//  k_optimize<R,DH> : ONE persistent cooperative kernel per QuadraticOptimizer::optimize() call
//                     (ref: src/QuadraticOptimizer.cpp:34-149 + ROPTLIB RTRNewton/tCG).  All phases
//                     -- fused [X.Q + G, f, tangent projection, |g|, preconditioner] passes,
//                     Riemannian Hessian-vector products of the truncated-CG loop, vector updates,
//                     QF retraction -- run inside it, separated by grid barriers; scalar
//                     reductions are fixed-order (deterministic) and every CTA replays the same
//                     scalar control flow.  The host sees only the result record.
//  k_spmv<R,DH>     : the Q.X product alone (Out = X Q [+ G]) -- the roofline kernel.
//  small kernels    : Stiefel (polar) projection, public-pose packing, G assembly.
#include "dpgo_device.cuh"
#include "dpgo_kernels.cuh"
#include "dpgo_rotation.cuh"
#include <cooperative_groups.h>
#include <algorithm>

namespace dpgo {

// ---------------------------------------------------------------------------------------------
// phase-end reduction: block partials -> global partials -> grid barrier -> every CTA sums all
// partials in the same fixed order, so all CTAs hold bit-identical scalars.
// ---------------------------------------------------------------------------------------------
struct BlockCtx {
  double *sm_warp;    // [nwarps * NRED]
  double *sm_out;     // [2 * NRED]  totals of the phase, double-buffered by parity
  unsigned epoch;
  int parity;
};

// The reduction steps around the barrier are kept short (they are pure latency, ~80 times per step): the 16 warp
// partials are combined by a shuffle tree in warp 0 (fixed order), lane 0 stores the CTA's partials and arrives at the
// barrier right behind them (the release covers the store), the whole of warp 0 polls the counter (one broadcast request)
// and goes straight on to fetch all CTAs' partials; the totals are published through a parity-double-buffered shared slot,
// so a phase end has two bar.syncs, not four.  (A fused variant -- 16-byte {value, phase} packets polled all-to-all, barrier
// and all-reduce in one round trip -- is not faster: scripts/barrier_bench3.cu compares the two; with gpu-scope "strong"
// 16-byte accesses it is much slower.)
// `update(totals)` runs in thread 0 between the two bar.syncs: it advances the CTA's SolverState (below), which every
// thread reads after the second one.
struct NoUpdate {
  __device__ void operator()(const double *) const {}
};

template <int NUSED = NRED, class Update = NoUpdate>
__device__ __forceinline__ void phase_end(const KParams &kp, BlockCtx &bc, double (&acc)[NRED], const Update &update = Update()) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nwarps = blockDim.x >> 5;
#pragma unroll
  for (int q = 0; q < NUSED; ++q) {
    double v = warp_sum(acc[q]);
    if (lane == 0) bc.sm_warp[warp * NRED + q] = v;
  }
  __syncthreads();                                       // also: every write of this phase is ordered before the release below
  bc.epoch += gridDim.x;
  double *slot = kp.partials + (size_t)bc.parity * kp.grid * NRED;
  double *outp = bc.sm_out + bc.parity * NRED;
  if (warp == 0) {
    if (NUSED > 0) {
      double s[NUSED > 0 ? NUSED : 1];
#pragma unroll
      for (int q = 0; q < NUSED; ++q) {
        double v = (lane < nwarps) ? bc.sm_warp[lane * NRED + q] : 0.0;
        s[q] = warp_sum(v);                              // fixed shuffle tree over the warps' partials
      }
      if (lane == 0) {
#pragma unroll
        for (int q = 0; q < NUSED; ++q) slot[(size_t)blockIdx.x * NRED + q] = s[q];
      }
    }
    if (!kp.cluster) {
      if (lane == 0) asm volatile("red.release.gpu.global.add.u32 [%0], 1;" ::"l"(kp.bar_counter) : "memory");
      while ((int)(ld_relaxed_u32(kp.bar_counter) - bc.epoch) < 0) { }
    }
  }
  if (kp.cluster) {
    // the grid is one thread-block cluster: the hardware cluster barrier (every thread arrives; release at cluster scope
    // publishes the CTA's global writes to the other CTAs of the cluster, which read them from L2) replaces the
    // atomic counter and its polling round trips, a fraction of the cost of a grid-wide phase end
    asm volatile("barrier.cluster.arrive.release.aligned;" ::: "memory");
    asm volatile("barrier.cluster.wait.aligned;" ::: "memory");
  }
  if (warp == 0) {
    if (NUSED > 0) {
      double t[NUSED > 0 ? NUSED : 1];
#pragma unroll
      for (int q = 0; q < NUSED; ++q) t[q] = 0.0;
      for (int c = lane; c < kp.grid; c += 32) {
#pragma unroll
        for (int q = 0; q < NUSED; ++q) t[q] += __ldcg(slot + (size_t)c * NRED + q);
      }
#pragma unroll
      for (int q = 0; q < NUSED; ++q) {
        const double v = warp_sum(t[q]);
        if (lane == 0) outp[q] = v;
      }
    }
    if (lane == 0) update(outp);
  }
  __syncthreads();
#pragma unroll
  for (int q = 0; q < NUSED; ++q) acc[q] = outp[q];
  bc.parity ^= 1;
}

// The scalar state of the solver's control flow: trust region, tCG recurrences, the result record.  It is the same in
// every thread of every CTA, so it lives once per CTA in shared memory rather than in registers of all 512 threads, where
// it would stay live across every phase.  Thread 0 advances it inside phase_end (`update`) with the totals of the phase;
// every thread reads it, and the branch it decided, after the phase end.
struct SolverState {
  dpgo_opt_result_t res;
  double f1, gn, zr0;                      // cost, |RG| and <z0, RG> at the base point
  double Delta, Delta_max;                 // trust-region radius
  double z_r, d_Pd, e_Pd, e_Pe, n0, alpha, beta, tau;   // tCG recurrences
  double denom;                            // model decrease of the candidate
  int cb;                                  // base buffer
  int pd;                                  // delta_old lives in V_D0 + pd
  int zsrc_z;                              // the Hessian's operand is V_Z (else the base point's V_Z00)
  int eta_zero, z0_valid, status, iter, total_steps;
  int brk;                                 // the last update leaves its loop
  unsigned long long tick_last;            // phase clock (CLOCK): thread 0 of CTA 0 only
};
constexpr int STATE_DOUBLES = (int)((sizeof(SolverState) + 15) / 16) * 2;   // keeps the following blocks 16-byte aligned

// The CTA's row range and (when it fits) a shared-memory copy of its block-CSR structure, set up once per launch: the
// sparse phases then start their X gathers without first waiting for two dependent global loads (row pointer, indices).
struct CtaRows {
  int r0, r1;
  const int *rowptr;      // indexable by the global row j (shared copy: local block offsets; else the global array)
  const int *bcol;        // indexable by those block offsets
  const double *bval;     // rebased to match
};

template <int R> struct RowIter {
  static constexpr int SG = SubGroup<R>::SG;
  int r0, r1, stride, jb, sgw, a, c;
  __device__ RowIter(const CtaRows &cr) {
    r0 = cr.r0;
    r1 = cr.r1;
    const int lane = threadIdx.x & 31;
    constexpr int SGW = 32 / SG;                 // sub-groups per warp
    sgw = lane / SG;
    stride = (blockDim.x >> 5) * SGW;
    jb = r0 + (threadIdx.x >> 5) * SGW;
    const int l = lane & (SG - 1);
    a = l >> 2;
    c = l & 3;
  }
};

// ---------------------------------------------------------------------------------------------
// Phase E: everything that is needed at a base point in ONE pass over Q
//   EG = X Q + G, f = 0.5 <XQ, X> + <X, G>, S = sym(Y^T EG_Y), RG = P_X(EG), |RG|^2,
//   Z0 = P_X(M^-1 RG) for the pose-local preconditioners, <Z0, RG>.
// (ref: QuadraticProblem::f / EucGrad / RieGrad, src/QuadraticProblem.cpp:50-66,89-101; the reference
//  spends 5 separate X.Q products on these values per optimize() call.)
// acc: [0] <XQ,X>  [1] <X,G>  [2] |RG|^2  [3] <Z0,RG>
// ---------------------------------------------------------------------------------------------
template <int R, int DH>
__device__ void phase_eval(const KParams &kp, const CtaRows &cr, int cb, bool save_xin, int precond, double (&acc)[NRED]) {
  constexpr int TS = R * DH;
  const double *X = kp.v[V_X0 + cb];
  double *EG = kp.v[V_EG0 + cb], *RG = kp.v[V_RG0 + cb], *Z0 = kp.v[V_Z00 + cb], *S = kp.S[cb];
  RowIter<R> it(cr);
  const bool valid = (it.a < R) && (it.c < DH);
  const int e = it.c * R + it.a;
  for (int jb = it.jb; jb < it.r1; jb += it.stride) {
    const int j = jb + it.sgw;
    const bool act = (j < it.r1);
    const int js = act ? j : it.r1 - 1;
    const bool ld = act && valid;
    double xq = gather_tile<R, DH, true, false>(cr.rowptr, cr.bcol, cr.bval, X, nullptr, 0.0, js, it.a, it.c);
    const size_t idx = (size_t)js * TS + e;
    const double x = ld ? __ldcg(X + idx) : 0.0;
    const double g = ld ? __ldcg(kp.G + idx) : 0.0;
    if (!ld) xq = 0.0;
    const double eg = xq + g;
    acc[0] = fma(xq, x, acc[0]);
    acc[1] = fma(x, g, acc[1]);
    double ya[3], sym[3];
    const double rg = tangent_project_elem<R, DH>(x, eg, it.a, it.c, ya, sym);
    if (ld) {
      EG[idx] = eg;
      RG[idx] = rg;
      if (save_xin) kp.v[V_XIN][idx] = x;
      acc[2] = fma(rg, rg, acc[2]);
    }
    if (act && it.a == 0 && it.c < 3) {
      double *s = S + (size_t)js * 9 + it.c * 3;
      s[0] = sym[0]; s[1] = sym[1]; s[2] = sym[2];
    }
    if (precond != DPGO_PRECOND_DENSE_EXACT && precond != DPGO_PRECOND_SPARSE_EXACT) {
      double z0 = rg;
      if (precond == DPGO_PRECOND_BLOCK_JACOBI) {
        double t = jacobi_elem<R, DH>(kp.dinv, js, ld ? rg : 0.0, it.a, it.c);
        double ya2[3], sym2[3];
        z0 = tangent_project_elem<R, DH>(x, t, it.a, it.c, ya2, sym2);
      }
      if (ld) {
        Z0[idx] = z0;
        acc[3] = fma(z0, rg, acc[3]);
      }
    }
  }
}

// ---------------------------------------------------------------------------------------------
// Phase H: Riemannian Hessian-vector product of the tCG direction (ref: QuadraticProblem::
// EucHessianEta, src/QuadraticProblem.cpp:68-73, + ROPTLIB Stiefel::EucHvToHv + projection):
//   delta_new = -zsrc + beta * delta_old      (formed on the fly for neighbour tiles, stored for own)
//   HD = P_X( delta_new Q - [delta_new_Y S]_pose ),   acc[0] = <delta_new, HD>
// If onfly == false the operand is read as is from `zsrc` (single-operation entry point).
// ---------------------------------------------------------------------------------------------
template <int R, int DH, bool CLOCK>
__device__ void phase_hess(const KParams &kp, const CtaRows &cr, int cb, const double *zsrc, const double *dold, double *dnew,
                           double beta, bool onfly, double (&acc)[NRED]) {
  constexpr int TS = R * DH;
  constexpr int D = DH - 1;
  const double *X = kp.v[V_X0 + cb];
  const double *S = kp.S[cb];
  double *HD = kp.v[V_HD];
  RowIter<R> it(cr);
  const bool valid = (it.a < R) && (it.c < DH);
  const int e = it.c * R + it.a;
  const bool ticking = CLOCK && (kp.phase_ns != nullptr) && blockIdx.x == 0 && threadIdx.x == 0;
  unsigned long long th0 = 0, th1 = 0;
  if (ticking) asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(th0));
  for (int jb = it.jb; jb < it.r1; jb += it.stride) {
    const int j = jb + it.sgw;
    const bool act = (j < it.r1);
    const int js = act ? j : it.r1 - 1;
    const bool ld = act && valid;
    // the row's own operands first: these loads are independent of the gather and overlap its round trips
    const size_t idx = (size_t)js * TS + e;
    double dl = 0.0, dprev = 0.0;
    if (ld) {
      dl = __ldcg(zsrc + idx);
      if (onfly && beta != 0.0) dprev = __ldcg(dold + idx);
    }
    const double x = ld ? __ldcg(X + idx) : 0.0;
    const bool rot = ld && (it.c < D);
    double s0 = 0, s1 = 0, s2 = 0;
    if (rot) {
      const double *s = S + (size_t)js * 9 + it.c * 3;
      s0 = __ldcg(s); s1 = __ldcg(s + 1); s2 = __ldcg(s + 2);
    }
    double hq;
    if (onfly) hq = gather_tile<R, DH, true, true>(cr.rowptr, cr.bcol, cr.bval, zsrc, dold, beta, js, it.a, it.c);
    else hq = gather_tile<R, DH, true, false>(cr.rowptr, cr.bcol, cr.bval, zsrc, nullptr, 0.0, js, it.a, it.c);
    if (ticking && jb == it.jb) { asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(th1)); kp.phase_ns[27] += th1 - th0; }
    if (ld && onfly) {
      dl = -dl;
      if (beta != 0.0) dl = fma(beta, dprev, dl);
      dnew[idx] = dl;
    }
    const double dr = rot ? dl : 0.0;
    const double d0 = quad_get(dr, 0), d1 = quad_get(dr, 1), d2 = (D > 2) ? quad_get(dr, 2) : 0.0;
    double w = ld ? hq : 0.0;
    if (rot) w -= (d0 * s0 + d1 * s1 + d2 * s2);
    double ya[3], sym[3];
    const double hd = tangent_project_elem<R, DH>(x, w, it.a, it.c, ya, sym);
    if (ld) {
      HD[idx] = hd;
      acc[0] = fma(dl, hd, acc[0]);
    }
  }
  if (ticking) { asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(th1)); kp.phase_ns[28] += th1 - th0; }
}

// ---------------------------------------------------------------------------------------------
// Phase U: eta += alpha delta, res += alpha HD, |res|^2 and (pose-local preconditioners)
// z = P_X(M^-1 res), <z,res>.   acc: [0] |res|^2  [1] <z,res>
// ---------------------------------------------------------------------------------------------
template <int R, int DH>
__device__ void phase_update(const KParams &kp, const CtaRows &cr, int cb, const double *dcur, double alpha, bool first, int precond,
                             double (&acc)[NRED]) {
  constexpr int TS = R * DH;
  const double *X = kp.v[V_X0 + cb];
  const double *RG = kp.v[V_RG0 + cb];
  double *ETA = kp.v[V_ETA], *RES = kp.v[V_RES], *Z = kp.v[V_Z];
  const double *HD = kp.v[V_HD];
  RowIter<R> it(cr);
  const bool valid = (it.a < R) && (it.c < DH);
  const int e = it.c * R + it.a;
  for (int jb = it.jb; jb < it.r1; jb += it.stride) {
    const int j = jb + it.sgw;
    const bool act = (j < it.r1);
    const int js = act ? j : it.r1 - 1;
    const bool ld = act && valid;
    const size_t idx = (size_t)js * TS + e;
    double res = 0.0, x = 0.0;
    if (ld) {
      const double dl = __ldcg(dcur + idx), hd = __ldcg(HD + idx);
      const double eta0 = first ? 0.0 : __ldcg(ETA + idx);
      const double res0 = first ? __ldcg(RG + idx) : __ldcg(RES + idx);
      res = fma(alpha, hd, res0);
      ETA[idx] = fma(alpha, dl, eta0);
      RES[idx] = res;
      acc[0] = fma(res, res, acc[0]);
      x = __ldcg(X + idx);
    }
    if (precond != DPGO_PRECOND_DENSE_EXACT && precond != DPGO_PRECOND_SPARSE_EXACT) {
      double z = res;
      if (precond == DPGO_PRECOND_BLOCK_JACOBI) {
        double t = jacobi_elem<R, DH>(kp.dinv, js, res, it.a, it.c);
        double ya[3], sym[3];
        z = tangent_project_elem<R, DH>(x, t, it.a, it.c, ya, sym);
      }
      if (ld) {
        Z[idx] = z;
        acc[1] = fma(z, res, acc[1]);
      }
    }
  }
}

// DMMA m8n8k4 (fp64 tensor op): D (8 x 8, two per lane) += A (8 x 4, one per lane) * B (4 x 8, one per lane)
__device__ __forceinline__ void dmma884(double &d0, double &d1, double a, double b) {
  asm volatile("mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 {%0,%1}, {%2}, {%3}, {%0,%1};" : "+d"(d0), "+d"(d1) : "d"(a), "d"(b));
}

// ---------------------------------------------------------------------------------------------
// Exact preconditioners (ref: QuadraticProblem::PreConditioner, src/QuadraticProblem.cpp:75-87 = CHOLMOD solve with
// Q + 0.1 I, then projection).  One phase of the nested-dissection block solve (nd_precond.h; DENSE_EXACT: its single
// macro level, one phase): the CTA walks its steps of the host-built plan:
//   gathers   : tiles of the phase's input vector -> shared memory (forward: residual minus the children's
//               contributions; backward: the ancestors' solution), one sub-group per tile
//   jobs      : one warp = one 8-row panel x a column piece; lane (row = lane & 7, cp = lane >> 3) reads columns
//               cp, cp + 4, ... : 256 contiguous bytes per warp load; r accumulators per lane; 2 shuffle steps
//   epilogues : one sub-group per pose: sums the panel's partial slots in fixed order, writes t / contribution / x;
//               solution tiles are projected onto the tangent space at X and dotted with V on the fly.
// acc[0] accumulates <Z, V> over the phases of one application.
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ int4 ld_int4(const void *p) { return __ldg(reinterpret_cast<const int4 *>(p)); }

template <int R, int DH, bool CLOCK>
__device__ void phase_nd(const KParams &kp, int ph, const double *V, int cb, double *Zout, double *ys, double *slots,
                         int4 *grec, double *sres, bool fill, double (&acc)[NRED]) {
  constexpr int TS = R * DH;
  constexpr int SG = SubGroup<R>::SG;
  constexpr int SGW = 32 / SG;
  constexpr int SLOT = nd::PANEL_ROWS * R;
  constexpr int NC = nd::INLINE_CONTRIB;
  const KNd &N = kp.nd;
  const int dir = N.dir[ph];
  const int4 ca = ld_int4(N.cta_phase + N.cta0[ph] + blockIdx.x),
             cbq = ld_int4(reinterpret_cast<const int4 *>(N.cta_phase + N.cta0[ph] + blockIdx.x) + 1);
  const int s0 = ca.x, s1 = ca.y;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nwarps = blockDim.x >> 5;
  const int sgw = lane / SG, l = lane & (SG - 1), a = l >> 2, c = l & 3;
  const bool valid = (a < R) && (c < DH);
  const int e = c * R + a;
  const int nsub = nwarps * SGW;
  const double *X = kp.v[V_X0 + cb];
  const double *src = (dir == 0) ? V : N.TX;
  const bool ticking = CLOCK && (kp.phase_ns != nullptr) && blockIdx.x == 0 && threadIdx.x == 0;
  for (int si = s0; si < s1; ++si) {
    int g0 = ca.z, g1 = ca.w, j0 = cbq.x, j1 = cbq.y, e0 = cbq.z, e1 = cbq.w;      // the first step sits in the CTA record
    if (si != s0) {
      const int4 sa = ld_int4(N.steps + si), sb = ld_int4(reinterpret_cast<const int4 *>(N.steps + si) + 1);
      g0 = sa.x; g1 = sa.y; j0 = sa.z; j1 = sa.w; e0 = sb.x; e1 = sb.y;
    }
    unsigned long long tg0 = 0, tg1 = 0, tg2 = 0;
    if (ticking) asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(tg0));
    // ---- gathers: the step's records are staged in shared memory with one coalesced sweep (one L2 round trip), then
    //      the loop is flat over (tile, element) with 4 independent elements per thread and round ----
    {
      const int ng = g1 - g0;
      const int4 *gsrc = reinterpret_cast<const int4 *>(N.gathers + g0);
      for (int q = threadIdx.x; q < 2 * ng; q += blockDim.x) grec[q] = __ldg(gsrc + q);
      __syncthreads();
      constexpr int GU = 4;
      const int total = ng * TS, nthr = blockDim.x;
      for (int base = threadIdx.x; base < total; base += GU * nthr) {
        int t[GU], el[GU];
        bool ok[GU];
        double v[GU], cv[GU][NC];
#pragma unroll
        for (int u = 0; u < GU; ++u) {
          const int idx = base + u * nthr;
          ok[u] = idx < total;
          t[u] = ok[u] ? idx / TS : 0;
          el[u] = idx - t[u] * TS;
          const int4 ra = grec[2 * t[u]], rb = grec[2 * t[u] + 1];             // (ytile, src, nc, cext), first contribution tiles
          v[u] = ok[u] ? __ldcg(src + (size_t)ra.y * TS + el[u]) : 0.0;
          const int ci[NC] = {rb.x, rb.y, rb.z, rb.w};
#pragma unroll
          for (int q = 0; q < NC; ++q) cv[u][q] = (ok[u] && q < ra.z) ? __ldcg(N.C + (size_t)ci[q] * TS + el[u]) : 0.0;
        }
#pragma unroll
        for (int u = 0; u < GU; ++u) {
          const int4 ra = grec[2 * t[u]];
#pragma unroll
          for (int q = 0; q < NC; ++q) v[u] -= cv[u][q];
          for (int k = NC; k < ra.z && ok[u]; ++k)
            v[u] -= __ldcg(N.C + (size_t)ld_const(N.csrc + ra.w + k - NC) * TS + el[u]);
          if (ok[u]) ys[(size_t)ra.x * TS + el[u]] = v[u];
        }
      }
    }
    __syncthreads();
    if (ticking) asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(tg1));
    // ---- jobs: DMMA m8n8k4 -- A = 8 panel rows x 4 columns (one coalesced 256-byte warp load), B = 4 columns x r
    //      right-hand sides from shared memory, D = 8 x 8 accumulators (r columns used): 1 LDG + 1 LDS + 1 DMMA per
    //      4 columns instead of 1 LDG + r LDS + r DFMA per lane, and no shuffle reduction.  Two accumulator chains;
    //      the next job's record is fetched ahead.  The rounds of the job's resident columns (nd::Job) read A from the
    //      CTA's region in shared memory, one 256-byte group per load in lane order; the launch's first application
    //      (fill) still streams them and leaves them there.  Either way every DMMA gets the same operands.
    {
      const int r8 = lane >> 2, k4 = lane & 3;
      const bool bval_lane = (r8 < R);
      int ji = j0 + warp;
      int4 ja = make_int4(0, 0, 0, 0), jb = make_int4(0, 0, 0, 0);
      if (ji < j1) { ja = ld_int4(N.jobs + ji); jb = ld_int4(reinterpret_cast<const int4 *>(N.jobs + ji) + 1); }
      while (ji < j1) {
        const int jn = ji + nwarps;
        int4 na = make_int4(0, 0, 0, 0), nb = make_int4(0, 0, 0, 0);
        if (jn < j1) { na = ld_int4(N.jobs + jn); nb = ld_int4(reinterpret_cast<const int4 *>(N.jobs + jn) + 1); }
        const long long mat = ((long long)(unsigned)ja.x) | ((long long)ja.y << 32);
        const int ncols = ja.z, ycol = ja.w, slot = jb.x, accum = jb.y, nres = jb.w;
        const double *mp = N.blob + mat + (size_t)k4 * nd::PANEL_ROWS + r8;      // A[r8][k4] of the first column group
        const double *yp = ys + (size_t)(ycol + k4) * R + (bval_lane ? r8 : 0);    // B[k4][r8]
        double *rp = sres + jb.z + lane;                                           // A[r8][k4] of resident group 0
        double d0 = 0.0, d1 = 0.0, f0 = 0.0, f1 = 0.0;
        for (int j = 0; j < ncols; j += 32) {                                        // 8 column groups (32 columns) per round
          double am[8], bm[8];
          const bool res = j < nres;                                                 // whole rounds are resident
          if (res && !fill) {
#pragma unroll
            for (int u = 0; u < 8; ++u) am[u] = (j + 4 * u < ncols) ? rp[(size_t)(j + 4 * u) * nd::PANEL_ROWS] : 0.0;
#pragma unroll
            for (int u = 0; u < 8; ++u) bm[u] = (bval_lane && j + 4 * u + k4 < ncols) ? yp[(size_t)(j + 4 * u) * R] : 0.0;
          } else if (j + 32 <= ncols) {
#pragma unroll
            for (int u = 0; u < 8; ++u) am[u] = ld_stream(mp + (size_t)(j + 4 * u) * nd::PANEL_ROWS);
#pragma unroll
            for (int u = 0; u < 8; ++u) bm[u] = bval_lane ? yp[(size_t)(j + 4 * u) * R] : 0.0;
          } else {                                                                   // last, ragged round: same 8 independent loads, predicated
#pragma unroll
            for (int u = 0; u < 8; ++u) am[u] = (j + 4 * u + k4 < ncols) ? ld_stream(mp + (size_t)(j + 4 * u) * nd::PANEL_ROWS) : 0.0;
#pragma unroll
            for (int u = 0; u < 8; ++u) bm[u] = (bval_lane && j + 4 * u + k4 < ncols) ? yp[(size_t)(j + 4 * u) * R] : 0.0;
          }
          if (res && fill) {
#pragma unroll
            for (int u = 0; u < 8; ++u)
              if (j + 4 * u < ncols) rp[(size_t)(j + 4 * u) * nd::PANEL_ROWS] = am[u];
          }
#pragma unroll
          for (int u = 0; u < 8; u += 2) {
            dmma884(d0, d1, am[u], bm[u]);
            dmma884(f0, f1, am[u + 1], bm[u + 1]);
          }
        }
        d0 += f0;
        d1 += f1;
        {
          double *sl = slots + (size_t)slot * SLOT + r8 * R + 2 * k4;              // D[r8][2 k4], D[r8][2 k4 + 1]
          if (2 * k4 < R) sl[0] = accum ? sl[0] + d0 : d0;
          if (2 * k4 + 1 < R) sl[1] = accum ? sl[1] + d1 : d1;
        }
        ji = jn; ja = na; jb = nb;
      }
    }
    __syncthreads();
    if (ticking) asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(tg2));
    // ---- epilogues (warp-uniform trip count: the projection uses full-warp shuffles); global loads first, the next
    //      item's record is fetched ahead ----
    {
      int eb = e0 + warp * SGW;
      int4 ea = make_int4(-1, 0, 0, 0), ec = make_int4(0, 0, 0, 0), ed = make_int4(0, 0, 0, 0);
      if (eb + sgw < e1) {
        const int4 *rp = reinterpret_cast<const int4 *>(N.epis + eb + sgw);
        ea = __ldg(rp); ec = __ldg(rp + 1); ed = __ldg(rp + 2);
      }
      while (eb < e1) {
        const int en = eb + nsub;
        int4 fa = make_int4(-1, 0, 0, 0), fc = make_int4(0, 0, 0, 0), fd = make_int4(0, 0, 0, 0);
        if (en + sgw < e1) {
          const int4 *rp = reinterpret_cast<const int4 *>(N.epis + en + sgw);
          fa = __ldg(rp); fc = __ldg(rp + 1); fd = __ldg(rp + 2);
        }
        const bool act = (eb + sgw < e1);
        const int kind = ea.x, slot0 = ea.y, nslots = ea.z, half = ea.w, out = ec.x, aux = ec.y, nc = ec.z, cext = ec.w;
        const bool ld = act && valid;
        const bool sol = (kind == nd::EPI_ROOT) || (kind == nd::EPI_B_OWN);
        // independent global loads: t (backward), X and V tiles (solution poses), contributions (boundary rows)
        double tval = 0.0, xq = 0.0, vv = 0.0, cv[NC] = {0.0, 0.0, 0.0, 0.0};
        if (ld) {
          if (kind == nd::EPI_B_OWN) tval = __ldcg(N.TX + (size_t)out * TS + e);
          if (sol) { xq = __ldcg(X + (size_t)aux * TS + e); vv = __ldcg(V + (size_t)aux * TS + e); }
          if (kind == nd::EPI_F_BND) {
            const int ci[NC] = {ed.x, ed.y, ed.z, ed.w};
#pragma unroll
            for (int q = 0; q < NC; ++q) cv[q] = (q < nc) ? __ldcg(N.C + (size_t)ci[q] * TS + e) : 0.0;
          }
        }
        double sum = 0.0;
        if (ld) {
          const double *sl = slots + (size_t)slot0 * SLOT + (half * DH + c) * R + a;
          for (int k = 0; k < nslots; ++k) sum += sl[(size_t)k * SLOT];
        }
        double x = 0.0;
        if (ld) {
          if (kind == nd::EPI_F_OWN) {
            N.TX[(size_t)out * TS + e] = sum;
          } else if (kind == nd::EPI_F_BND) {
#pragma unroll
            for (int q = 0; q < NC; ++q) sum += cv[q];
            for (int k = NC; k < nc; ++k) sum += __ldcg(N.C + (size_t)ld_const(N.csrc + cext + k - NC) * TS + e);
            N.C[(size_t)out * TS + e] = sum;
          } else if (sol) {
            x = (kind == nd::EPI_ROOT) ? sum : tval - sum;
            N.TX[(size_t)out * TS + e] = x;
          }
        }
        if (__any_sync(FULL, sol)) {                      // forward sweeps below the root have nothing to project
          double ya[3], sym[3];
          const double z = tangent_project_elem<R, DH>(sol ? xq : 0.0, x, a, c, ya, sym);
          if (ld && sol) {
            Zout[(size_t)aux * TS + e] = z;
            acc[0] = fma(z, vv, acc[0]);
          }
        }
        eb = en; ea = fa; ec = fc; ed = fd;
      }
    }
    if (ticking) {
      unsigned long long tg3;
      asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(tg3));
      kp.phase_ns[24] += tg1 - tg0; kp.phase_ns[25] += tg2 - tg1; kp.phase_ns[26] += tg3 - tg2;
      unsigned long long *pp = kp.phase_ns + 32 + 3 * min(ph, 9);
      pp[0] += tg1 - tg0; pp[1] += tg2 - tg1; pp[2] += tg3 - tg2;
    }
    // the next step's gathers / jobs rewrite ys / slots only after every warp is past its epilogues
    if (si + 1 < s1) __syncthreads();
  }
}

// ---------------------------------------------------------------------------------------------
// Phase RT: candidate X' = R_X(eta_final) with eta_final = eta + tau * delta (tau = 0 unless tCG
// stopped on the trust-region boundary / negative curvature), and the model-decrease dots
//   acc[0] = <eta, g>, acc[1] = <eta, H eta> with H eta = (res - g) + tau * HD (tCG recurrences).
// mode 1 (RGD, ref src/QuadraticOptimizer.cpp:124-149): eta = -step * RG.
// mode 2: eta read as is from V_AUX (single-operation entry point).
// ---------------------------------------------------------------------------------------------
template <int R, int DH>
__device__ void phase_retract(const KParams &kp, const CtaRows &cr, int cb, int mode, const double *dcur, double tau, bool eta_zero,
                              double step, double (&acc)[NRED]) {
  constexpr int TS = R * DH;
  const double *X = kp.v[V_X0 + cb];
  const double *RG = kp.v[V_RG0 + cb];
  double *X2 = kp.v[V_X0 + (1 - cb)];
  RowIter<R> it(cr);
  const bool valid = (it.a < R) && (it.c < DH);
  const int e = it.c * R + it.a;
  for (int jb = it.jb; jb < it.r1; jb += it.stride) {
    const int j = jb + it.sgw;
    const bool act = (j < it.r1);
    const int js = act ? j : it.r1 - 1;
    const bool ld = act && valid;
    const size_t idx = (size_t)js * TS + e;
    double w = 0.0;
    if (ld) {
      const double x = __ldcg(X + idx);
      double eta;
      if (mode == 1) {
        eta = -step * __ldcg(RG + idx);
      } else if (mode == 2) {
        eta = __ldcg(kp.v[V_AUX] + idx);
      } else {
        const double g = __ldcg(RG + idx);
        eta = eta_zero ? 0.0 : __ldcg(kp.v[V_ETA] + idx);
        double heta = eta_zero ? 0.0 : (__ldcg(kp.v[V_RES] + idx) - g);
        if (tau != 0.0) {
          eta = fma(tau, __ldcg(dcur + idx), eta);
          heta = fma(tau, __ldcg(kp.v[V_HD] + idx), heta);
        }
        acc[0] = fma(eta, g, acc[0]);
        acc[1] = fma(eta, heta, acc[1]);
      }
      w = x + eta;
    }
    const double q = qf_retract_elem<R, DH>(w, it.a, it.c);
    if (ld) X2[idx] = q;
  }
}

// Final phase: make X0 hold the result and accumulate |X_out - X_in|^2 (ref: relativeChange,
// src/QuadraticOptimizer.cpp:54).
template <int R, int DH> __device__ void phase_final(const KParams &kp, const CtaRows &cr, int cur, double (&acc)[NRED]) {
  constexpr int TS = R * DH;
  RowIter<R> it(cr);
  const bool valid = (it.a < R) && (it.c < DH);
  const int e = it.c * R + it.a;
  for (int jb = it.jb; jb < it.r1; jb += it.stride) {
    const int j = jb + it.sgw;
    if (j < it.r1 && valid) {
      const size_t idx = (size_t)j * TS + e;
      const double x = __ldcg(kp.v[V_X0 + cur] + idx);
      const double d = x - __ldcg(kp.v[V_XIN] + idx);
      acc[0] = fma(d, d, acc[0]);
      if (cur != 0) kp.v[V_X0][idx] = x;
    }
  }
}

__device__ __forceinline__ void zero(double (&acc)[NRED]) {
#pragma unroll
  for (int q = 0; q < NRED; ++q) acc[q] = 0.0;
}

// ---------------------------------------------------------------------------------------------
// The persistent kernel.  CLOCK = false is the variant every launch uses unless it asks for the phase clock (see
// launch_optimize_t): without the clock's timestamps the register allocator has room at the 128-register cap of
// launch_bounds(512, 1), and no phase spills.  Both variants compute the same values in the same order.
// ---------------------------------------------------------------------------------------------
template <int R, int DH, bool CLOCK> __global__ void __launch_bounds__(OPT_THREADS, 1) k_optimize(const KParams kp) {
  // a gated-off agent (selection of dpgo_agents_select_round_async): every CTA reads the same flag before anything else,
  // so the whole grid returns and no barrier, result or opt_record is touched
  if (kp.gate != nullptr && __ldg(kp.gate) == 0) return;
  extern __shared__ double smem[];
  BlockCtx bc;
  bc.sm_warp = smem;
  bc.sm_out = smem + (OPT_THREADS / 32) * NRED;
  SolverState &S = *reinterpret_cast<SolverState *>(bc.sm_out + 2 * NRED);
  if (threadIdx.x == 0) {                       // ordered before any read by the barrier below
    dpgo_opt_result_t &res = S.res;
    res.success = 0; res.tcg_status = DPGO_TCG_NOT_RUN; res.tcg_iterations = 0; res.outer_iterations = 0;
    res.rejections = 0; res.spmv_passes = 0; res.precond_applies = 0; res.reserved0 = 0;
    res.f_init = res.gradnorm_init = res.f_opt = res.gradnorm_opt = res.relative_change = res.elapsed_ms = 0.0;
    res.quad_init = res.lin_init = 0.0;
  }
  // the CTA's rows and, when they fit, its slice of the block-CSR structure in shared memory (SP_CACHE_INTS ints)
  int *sp_ints = reinterpret_cast<int *>(bc.sm_out + 2 * NRED + STATE_DOUBLES);
  CtaRows cr;
  cr.r0 = ld_const(kp.cta_rows + blockIdx.x);
  cr.r1 = ld_const(kp.cta_rows + blockIdx.x + 1);
  cr.rowptr = kp.rowptr;
  cr.bcol = kp.bcol;
  cr.bval = kp.bval;
  {
    const int nrows = cr.r1 - cr.r0;
    const int blk0 = (nrows > 0) ? ld_const(kp.rowptr + cr.r0) : 0, blk1 = (nrows > 0) ? ld_const(kp.rowptr + cr.r1) : 0;
    if (nrows > 0 && nrows + 1 + (blk1 - blk0) <= SP_CACHE_INTS) {
      for (int q = threadIdx.x; q <= nrows; q += blockDim.x) sp_ints[q] = ld_const(kp.rowptr + cr.r0 + q) - blk0;
      for (int q = threadIdx.x; q < blk1 - blk0; q += blockDim.x) sp_ints[nrows + 1 + q] = ld_const(kp.bcol + blk0 + q);
      cr.rowptr = sp_ints - cr.r0;              // indexed by the global row
      cr.bcol = sp_ints + nrows + 1;            // indexed by the local block offset
      cr.bval = kp.bval + (size_t)blk0 * 16;
    }
    __syncthreads();
  }
  double *sV = reinterpret_cast<double *>(sp_ints + SP_CACHE_INTS);   // the exact preconditioner's plan areas
  bc.epoch = *kp.bar_epoch;
  bc.parity = 0;
  // diagnostic phase clock: CTA 0 / thread 0 charges the time since the previous tick to a phase kind
  // (0 eval, 3 Hessian product, 4 tCG update, 5 retraction, 6 final, 8 + k phase k of an exact preconditioner's application)
  auto tick = [&](int kind) {
    if (CLOCK && kp.phase_ns != nullptr && blockIdx.x == 0 && threadIdx.x == 0) {
      unsigned long long t;
      asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
      if (kind >= 0) kp.phase_ns[kind] += t - S.tick_last;
      S.tick_last = t;
    }
  };
  tick(-1);
  const int precond = kp.prm.precond;
  const bool exact = (precond == DPGO_PRECOND_DENSE_EXACT) || (precond == DPGO_PRECOND_SPARSE_EXACT);
  double acc[NRED];
  // exact preconditioner: shared memory = gathered input tiles + partial-sum slots
  double *nd_ys = sV;
  double *nd_slots = sV + (size_t)kp.nd.max_ytiles * R * DH;
  int4 *nd_grec = reinterpret_cast<int4 *>((reinterpret_cast<uintptr_t>(nd_slots + (size_t)kp.nd.max_slots * nd::PANEL_ROWS * R) + 15) & ~(uintptr_t)15);
  // the CTA's resident panel columns, aliased by nothing; the launch's first application (no application counted yet:
  // z0 of the first outer iteration, or the single-operation entry point) fills them
  double *nd_res = reinterpret_cast<double *>(nd_grec + 2 * (size_t)kp.nd.max_gathers);
  // Z = P_X( (Q + 0.1 I)^-1 V ), <Z, V> in acc[0] and to `update`; every phase ends with a grid barrier
  auto apply_exact = [&](const double *Vv, int cbx, double *Zout, const auto &update) {
    zero(acc);
    for (int ph = 0; ph < kp.nd.nphases; ++ph) {
      phase_nd<R, DH, CLOCK>(kp, ph, Vv, cbx, Zout, nd_ys, nd_slots, nd_grec, nd_res, S.res.precond_applies == 0, acc);
      if (ph + 1 < kp.nd.nphases) { phase_end<0>(kp, bc, acc); tick(8 + min(ph, 15)); }
    }
    phase_end<1>(kp, bc, acc, update);
    tick(8 + min(kp.nd.nphases - 1, 15));
  };

  int cur = 0;   // which X buffer holds the current iterate

  // ---- single-operation entry points -------------------------------------------------------
  if (kp.op == OP_PHASE_BENCH) {          // diagnostic: tr_max_inner empty phases (barrier + 1-scalar reduction)
    for (int i = 0; i < kp.prm.tr_max_inner; ++i) { zero(acc); acc[0] = 1.0; phase_end<1>(kp, bc, acc); }
    if (blockIdx.x == 0 && threadIdx.x == 0) { S.res.f_init = acc[0]; *kp.result = S.res; *kp.bar_epoch = bc.epoch; }
    return;
  }
  if (kp.op == OP_PRECON) {
    if (exact) {
      apply_exact(kp.v[V_AUX], 0, kp.v[V_Z], NoUpdate());
    } else {
      // reuse phase_update with res := AUX (first = false, alpha = 0 would need RES); do it directly
      constexpr int TS = R * DH;
      RowIter<R> it(cr);
      const bool valid = (it.a < R) && (it.c < DH);
      const int e = it.c * R + it.a;
      for (int jb = it.jb; jb < it.r1; jb += it.stride) {
        const int j = jb + it.sgw;
        const bool act = (j < it.r1);
        const int js = act ? j : it.r1 - 1;
        const bool ld = act && valid;
        const size_t idx = (size_t)js * TS + e;
        const double x = ld ? __ldcg(kp.v[V_X0] + idx) : 0.0;
        double t = ld ? __ldcg(kp.v[V_AUX] + idx) : 0.0;
        if (precond == DPGO_PRECOND_BLOCK_JACOBI) t = jacobi_elem<R, DH>(kp.dinv, js, t, it.a, it.c);
        double ya[3], sym[3];
        const double z = tangent_project_elem<R, DH>(x, t, it.a, it.c, ya, sym);
        if (ld) kp.v[V_Z][idx] = z;
      }
      zero(acc); phase_end(kp, bc, acc);
    }
    if (blockIdx.x == 0 && threadIdx.x == 0) *kp.bar_epoch = bc.epoch;
    return;
  }
  if (kp.op == OP_RETRACT) {
    zero(acc);
    phase_retract<R, DH>(kp, cr, 0, 2, nullptr, 0.0, false, 0.0, acc);
    phase_end(kp, bc, acc);
    if (blockIdx.x == 0 && threadIdx.x == 0) *kp.bar_epoch = bc.epoch;
    return;
  }

  // ---- statistics at the input point (ref: src/QuadraticOptimizer.cpp:36-37) -------------------
  const bool single = (kp.prm.tr_iterations == 1);      // ref :92-110 shrink-until-accepted mode
  // thread 0: start a truncated CG solve (ROPTLIB SolversTR::tCG_TR; theta = 1, kappa = 0.1, Min_Inner_Iter = 0)
  auto tcg_begin = [&]() {
    S.z_r = S.zr0; S.d_Pd = S.zr0; S.e_Pd = 0.0; S.e_Pe = 0.0;
    S.n0 = S.gn;
    S.res.precond_applies++;                           // z0 = M^-1 g
    S.beta = 0.0; S.tau = 0.0;
    S.zsrc_z = 0; S.pd = 0; S.eta_zero = 1; S.status = DPGO_TCG_MAXITER;
  };
  // thread 0: the next tCG direction from the new <z, res>
  auto tcg_next = [&](double zr_new) {
    S.res.precond_applies++;
    const double beta = zr_new / S.z_r;
    S.beta = beta;
    S.z_r = zr_new;
    S.zsrc_z = 1;
    S.e_Pd = beta * (S.e_Pd + S.alpha * S.d_Pd);
    S.d_Pd = S.z_r + beta * beta * S.d_Pd;
  };
  zero(acc);
  phase_eval<R, DH>(kp, cr, 0, true, precond, acc);
  phase_end(kp, bc, acc, [&](const double *t) {
    dpgo_opt_result_t &res = S.res;
    res.spmv_passes++;
    const double f1 = 0.5 * t[0] + t[1];
    const double gn = sqrt(t[2]);
    S.f1 = f1; S.gn = gn; S.zr0 = t[3];
    res.f_init = f1;
    res.gradnorm_init = gn;
    res.quad_init = t[0];
    res.lin_init = t[1];
    res.f_opt = f1;
    res.gradnorm_opt = gn;
    // the trust region's start (ref :80-81, :96-97); its first tCG solve starts here unless z0 is still to be applied
    S.Delta = kp.prm.tr_initial_radius;
    S.Delta_max = single ? S.Delta : 5.0 * kp.prm.tr_initial_radius;
    S.total_steps = 0; S.cb = 0; S.iter = 0;
    S.z0_valid = !exact;
    if (kp.op != OP_EVAL && kp.op != OP_RHESS && kp.prm.algorithm != DPGO_ALG_RGD && gn >= kp.prm.tr_tolerance && !exact)
      tcg_begin();
  });
  tick(0);

  if (kp.op == OP_EVAL) {
    if (blockIdx.x == 0 && threadIdx.x == 0) { S.res.success = 1; *kp.result = S.res; *kp.bar_epoch = bc.epoch; }
    return;
  }
  if (kp.op == OP_RHESS) {
    zero(acc);
    phase_hess<R, DH, CLOCK>(kp, cr, 0, kp.v[V_AUX], nullptr, nullptr, 0.0, false, acc);
    phase_end(kp, bc, acc);
    if (blockIdx.x == 0 && threadIdx.x == 0) { *kp.result = S.res; *kp.bar_epoch = bc.epoch; }
    return;
  }

  if (kp.prm.algorithm == DPGO_ALG_RGD) {
    // ---- one fixed-step Riemannian gradient-descent step (ref :124-149) ----------------------
    zero(acc);
    phase_retract<R, DH>(kp, cr, 0, 1, nullptr, 0.0, false, kp.prm.rgd_stepsize, acc);
    phase_end(kp, bc, acc);
    zero(acc);
    phase_eval<R, DH>(kp, cr, 1, false, DPGO_PRECOND_NONE, acc);
    phase_end(kp, bc, acc, [&](const double *t) {
      S.res.spmv_passes++;
      S.res.f_opt = 0.5 * t[0] + t[1];
      S.res.gradnorm_opt = sqrt(t[2]);
      S.res.outer_iterations = 1;
    });
    cur = 1;
  } else if (S.gn >= kp.prm.tr_tolerance) {      // ref :67-70 early exit otherwise
    // ---- Riemannian trust region ------------------------------------------------------------
    while (true) {
      // -- z0 = M^-1 g for the exact preconditioners (pose-local ones were fused into phase E)
      if (!S.z0_valid) {
        const int cb = S.cb;
        apply_exact(kp.v[V_RG0 + cb], cb, kp.v[V_Z00 + cb], [&](const double *t) {
          S.zr0 = t[0];
          S.z0_valid = 1;
          tcg_begin();
        });
      }
      // -- truncated CG
      for (int j = 0; j < kp.prm.tr_max_inner; ++j) {
        {
          const int cb = S.cb, pd = S.pd;
          zero(acc);
          phase_hess<R, DH, CLOCK>(kp, cr, cb, S.zsrc_z ? kp.v[V_Z] : kp.v[V_Z00 + cb], kp.v[V_D0 + pd], kp.v[V_D0 + (1 - pd)],
                                  S.beta, true, acc);
        }
        phase_end<1>(kp, bc, acc, [&](const double *t) {
          S.res.spmv_passes++;
          S.res.tcg_iterations++;
          S.pd = 1 - S.pd;                               // delta_new becomes delta_old
          const double d_Hd = t[0];
          const double Delta = S.Delta, e_Pd = S.e_Pd, d_Pd = S.d_Pd, e_Pe = S.e_Pe;
          const double alpha = S.z_r / d_Hd;
          const double e_new = e_Pe + 2.0 * alpha * e_Pd + alpha * alpha * d_Pd;
          S.alpha = alpha;
          S.brk = d_Hd <= 0.0 || e_new >= Delta * Delta;
          if (S.brk) {
            S.tau = (-e_Pd + sqrt(e_Pd * e_Pd + d_Pd * (Delta * Delta - e_Pe))) / d_Pd;
            S.status = (d_Hd <= 0.0) ? DPGO_TCG_NEGCURVTURE : DPGO_TCG_EXCREGION;
          } else {
            S.e_Pe = e_new;
          }
        });
        tick(3);
        if (S.brk) break;
        zero(acc);
        phase_update<R, DH>(kp, cr, S.cb, kp.v[V_D0 + S.pd], S.alpha, S.eta_zero, precond, acc);
        phase_end<2>(kp, bc, acc, [&](const double *t) {
          S.eta_zero = 0;
          const double nr = sqrt(t[0]);
          const double n0 = S.n0;
          const double n0t = n0;                         // n0^theta, theta = 1
          S.brk = nr <= n0 * fmin(n0t, 0.1);
          if (S.brk) S.status = (0.1 < n0t) ? DPGO_TCG_LCON : DPGO_TCG_SCON;
          else if (!exact) tcg_next(t[1]);
        });
        tick(4);
        if (S.brk) break;
        if (exact) apply_exact(kp.v[V_RES], S.cb, kp.v[V_Z], [&](const double *t) { tcg_next(t[0]); });
      }
      // -- candidate point, model decrease, actual decrease
      zero(acc);
      phase_retract<R, DH>(kp, cr, S.cb, 0, kp.v[V_D0 + S.pd], S.tau, S.eta_zero, 0.0, acc);   // delta: read when tau != 0
      phase_end<2>(kp, bc, acc, [&](const double *t) {
        S.res.tcg_status = S.status;
        S.res.outer_iterations++;
        S.denom = -t[0] - 0.5 * t[1];
      });
      tick(5);
      zero(acc);
      phase_eval<R, DH>(kp, cr, 1 - S.cb, false, precond, acc);
      phase_end(kp, bc, acc, [&](const double *t) {
        dpgo_opt_result_t &res = S.res;
        res.spmv_passes++;
        const double f2 = 0.5 * t[0] + t[1];
        const double gn2 = sqrt(t[2]);
        const double denom = S.denom;
        const double rho = (denom != 0.0) ? (S.f1 - f2) / denom : -1.0;
        const bool accepted = rho > 0.1;                 // ROPTLIB Acceptence_Rho
        if (single) {
          if (accepted) {
            S.cb = 1 - S.cb; res.f_opt = f2; res.gradnorm_opt = gn2;
            S.brk = 1;
          } else {
            res.rejections++;
            S.brk = S.total_steps > 10;                  // ref :101-103 return the initial guess
            if (!S.brk) {
              S.Delta *= 0.25;                           // ref :104-107
              S.total_steps++;
            }
          }
        } else {
          // ROPTLIB SolversTR radius update (Shrinked_tau = 0.25, Magnified_tau = 2)
          if (rho < 0.25) S.Delta *= 0.25;
          else if (rho > 0.75 && (S.status == DPGO_TCG_NEGCURVTURE || S.status == DPGO_TCG_EXCREGION))
            S.Delta = fmin(2.0 * S.Delta, S.Delta_max);
          if (accepted) {
            S.cb = 1 - S.cb; S.f1 = f2; S.gn = gn2; S.zr0 = t[3];
            res.f_opt = f2; res.gradnorm_opt = gn2;
            S.z0_valid = !exact;
          } else {
            res.rejections++;
          }
          ++S.iter;
          S.brk = S.gn < kp.prm.tr_tolerance || S.iter >= kp.prm.tr_iterations;
        }
        if (!S.brk && S.z0_valid) tcg_begin();
      });
      tick(0);
      if (S.brk) break;
    }
    cur = S.cb;
  }

  zero(acc);
  phase_final<R, DH>(kp, cr, cur, acc);
  phase_end<1>(kp, bc, acc, [&](const double *t) {
    S.res.relative_change = sqrt(t[0] / (double)kp.n);
    S.res.success = 1;
  });
  tick(6);
  if (blockIdx.x == 0 && threadIdx.x == 0) {
    *kp.result = S.res;
    *kp.bar_epoch = bc.epoch;
    // the team status reads the relative change from here: the result record is overwritten by every OP_EVAL
    if (kp.opt_record) { kp.opt_record[0] = S.res.relative_change; kp.opt_record[1] += 1.0; }
  }
}

// ---------------------------------------------------------------------------------------------
// Stand-alone Q.X product: Out = X Q (+ G).  One sub-group per pose tile, plain grid.
// ---------------------------------------------------------------------------------------------
constexpr int SPMV_THREADS = 256;

template <int R, int DH>
__global__ void __launch_bounds__(SPMV_THREADS) k_spmv(int n, const int *__restrict__ rowptr,
                                                       const int *__restrict__ bcol,
                                                       const double *__restrict__ bval,
                                                       const double *__restrict__ X,
                                                       const double *__restrict__ G, double *__restrict__ out) {
  constexpr int SG = SubGroup<R>::SG;
  constexpr int TS = R * DH;
  const int lane = threadIdx.x & 31;
  const int l = lane & (SG - 1), a = l >> 2, c = l & 3;
  const int sg_global = (blockIdx.x * SPMV_THREADS + threadIdx.x) / SG;
  const int j = sg_global;
  const bool act = j < n;
  const int js = act ? j : n - 1;
  double v = gather_tile<R, DH, false, false>(rowptr, bcol, bval, X, nullptr, 0.0, js, a, c);
  if (act && a < R && c < DH) {
    const size_t idx = (size_t)js * TS + c * R + a;
    if (G != nullptr) v += __ldg(G + idx);
    out[idx] = v;
  }
}

// ---------------------------------------------------------------------------------------------
// Stiefel (polar-factor) projection per pose (stiefel_project_tile, dpgo_rotation.cuh), one thread per pose.
// The input is the linear combination c0 A + c1 B + c2 C (B, C optional): the Nesterov updates of the accelerated RBCD,
// Y = proj((1 - alpha) X + alpha V) and V = proj(V + gamma (X - Y)) (ref src/PGOAgent.cpp:1077-1091), are one launch each.
// (M and out may be the same buffer: a thread reads its whole tile before it writes it -- hence no __restrict__.)
// ---------------------------------------------------------------------------------------------
template <int R, int DH> __global__ void k_stiefel_project(int n, const double *M, double *out, double c0, const double *B, double c1,
                                                            const double *Cc, double c2) {
  constexpr int TS = R * DH;
  const int j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= n) return;
  stiefel_project_tile<R, DH>(
      [&](int e) {
        double v = c0 * M[(size_t)j * TS + e];
        if (B) v = fma(c1, B[(size_t)j * TS + e], v);
        if (Cc) v = fma(c2, Cc[(size_t)j * TS + e], v);
        return v;
      },
      [&](int e, double v) { out[(size_t)j * TS + e] = v; });
}

// ---------------------------------------------------------------------------------------------
// Boundary-pose exchange helpers (ref: PGOAgent::getSharedPoseDict src/PGOAgent.cpp:95-105,
// PGOAgent::constructGMatrix :783-859)
// ---------------------------------------------------------------------------------------------
__global__ void k_pack_tiles(int ts, int count, const int *__restrict__ pose, const double *__restrict__ X,
                             double *__restrict__ out, const unsigned char *__restrict__ gate) {
  const int t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= count * ts || (gate != nullptr && *gate == 0)) return;
  const int s = t / ts, e = t - s * ts;
  out[t] = X[(size_t)pose[s] * ts + e];
}

// One thread per (pose with shared edges, element): walks that pose's edges in a fixed order
// (deterministic sum).  outgoing: G_p += -(X_j Om) T^T ; incoming: G_p += -(X_i T) Om.
template <int R, int DH>
__global__ void k_build_G(int nposes, const int *__restrict__ pose_ids, const int *__restrict__ pose_ptr,
                          const int *__restrict__ edge_slot, const int *__restrict__ edge_out,
                          const double *__restrict__ edge_T, const double *__restrict__ edge_om,
                          const double *__restrict__ gathered, double *__restrict__ G,
                          const unsigned char *__restrict__ gate) {
  constexpr int TS = R * DH;
  const int t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= nposes * TS || (gate != nullptr && *gate == 0)) return;
  const int pi = t / TS, e = t - pi * TS;
  const int c = e / R, a = e - c * R;          // element (a, c) of the tile
  double acc = 0.0;
  for (int k = pose_ptr[pi]; k < pose_ptr[pi + 1]; ++k) {
    const double *Xn = gathered + (size_t)edge_slot[k] * TS;     // neighbour tile
    const double *T = edge_T + (size_t)k * DH * DH;              // row-major DH x DH
    const double *om = edge_om + (size_t)k * DH;
    double s = 0.0;
    if (edge_out[k]) {        // L[a,c] = -sum_q Xn[a,q] om[q] T[c][q]
#pragma unroll
      for (int q = 0; q < DH; ++q) s = fma(Xn[q * R + a] * om[q], T[c * DH + q], s);
    } else {                  // L[a,c] = -sum_q Xn[a,q] T[q][c] om[c]
#pragma unroll
      for (int q = 0; q < DH; ++q) s = fma(Xn[q * R + a], T[q * DH + c], s);
      s *= om[c];
    }
    acc -= s;
  }
  G[(size_t)pose_ids[pi] * TS + e] = acc;
}

// ---------------------------------------------------------------------------------------------
// Q from edge records on the device (ref: constructConnectionLaplacianSE, src/DPGO_utils.cpp:199-271, and the diagonal terms
// of PGOAgent::constructQMatrix, src/PGOAgent.cpp:720-781): one thread per block entry walks the block's contribution
// list in input order (deterministic).  Per edge i -> j with T = [R t; 0 1], Om = w diag(kappa.., tau):
//   kind 0  Q_ii += T Om T^T     kind 1  Q_jj += Om     kind 2  Q_ij = -T Om     kind 3  Q_ji = -Om T^T     kind 4  static block
// ---------------------------------------------------------------------------------------------
__global__ void k_assemble_Q(int64_t nb, const int *__restrict__ cptr, const int2 *__restrict__ contrib, const double *__restrict__ eT,
                             const double *__restrict__ eom, const double *__restrict__ ew, const double *__restrict__ sblk,
                             double *__restrict__ bval) {
  const int64_t tid = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (tid >= nb * 16) return;
  const int64_t b = tid >> 4;
  const int k = (int)((tid >> 2) & 3), c = (int)(tid & 3);
  double v = 0.0;
  for (int q = cptr[b]; q < cptr[b + 1]; ++q) {
    const int2 cc = contrib[q];
    if (cc.y == 4) { v += sblk[(size_t)cc.x * 16 + k * 4 + c]; continue; }
    const double *T = eT + (size_t)cc.x * 16, *om = eom + (size_t)cc.x * 4;
    const double w = ew[cc.x];
    if (cc.y == 0) {
      double s = 0.0;
#pragma unroll
      for (int u = 0; u < 4; ++u) s = fma(T[k * 4 + u] * (om[u] * w), T[c * 4 + u], s);
      v += s;
    } else if (cc.y == 1) {
      if (k == c) v += om[k] * w;
    } else if (cc.y == 2) {
      v -= T[k * 4 + c] * (om[c] * w);
    } else {
      v -= (om[k] * w) * T[c * 4 + k];
    }
  }
  bval[tid] = v;
}

// Robust re-weighting (ref: PGOAgent::updateLoopClosuresWeights, src/PGOAgent.cpp:1181-1245; computeMeasurementError,
// src/DPGO_utils.cpp:494-500; RobustCost::weight, src/DPGO_robust.cpp:23-66): one thread per private edge evaluates
// r^2 = kappa |Y_i R - Y_j|^2 + tau |p_j - p_i - Y_i t|^2 at the resident iterate and the weight of the chosen loss.
// cost: 0 L2, 1 L1, 2 Huber(param), 3 TLS(param), 4 Geman-McClure, 5 GNC_TLS(mu, param = cbar)
template <int R, int DH>
__global__ void k_edge_weights(int64_t m, const int *__restrict__ p1, const int *__restrict__ p2, const double *__restrict__ eT,
                               const double *__restrict__ eom, const int *__restrict__ fixed, const double *__restrict__ X, int cost,
                               double mu, double param, double *__restrict__ w, double *__restrict__ resid,
                               unsigned long long *__restrict__ gnc) {
  constexpr int D = DH - 1, TS = R * DH;
  const int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= m) return;
  const double *T = eT + (size_t)e * 16, *om = eom + (size_t)e * 4;
  const double *X1 = X + (size_t)p1[e] * TS, *X2 = X + (size_t)p2[e] * TS;
  double rot = 0.0, tra = 0.0;
  for (int a = 0; a < R; ++a) {
    for (int c = 0; c < D; ++c) {
      double s = -X2[c * R + a];
      for (int q = 0; q < D; ++q) s = fma(X1[q * R + a], T[q * 4 + c], s);
      rot = fma(s, s, rot);
    }
    double s = X2[D * R + a] - X1[D * R + a];
    for (int q = 0; q < D; ++q) s = fma(-X1[q * R + a], T[q * 4 + D], s);
    tra = fma(s, s, tra);
  }
  const double r2 = om[0] * rot + om[D] * tra;
  if (resid) resid[e] = r2;
  if (fixed && fixed[e]) return;
  // the reference passes r = sqrt(r^2) to RobustCost::weight, which squares it again: every weight is a function of r
  const double r = sqrt(r2);
  double wt = 1.0;
  if (cost == 1) wt = 1.0 / r;
  else if (cost == 2) wt = (r < param) ? 1.0 : param / r;
  else if (cost == 3) wt = (r < param) ? 1.0 : 0.0;
  else if (cost == 4) { const double s = 1.0 + __dmul_rn(r, r); wt = 1.0 / (s * s); }    // r*r rounded, not fused
  else if (cost == 5) wt = gnc_tls_weight(r, mu, param);
  w[e] = wt;
  // the counts of the reference's computeConvergedLoopClosureRatio (src/PGOAgent.cpp:1247-1289); integers, so deterministic
  if (gnc) atomicAdd(gnc + (wt == 1.0 ? 0 : (wt == 0.0 ? 1 : 2)), 1ULL);
}

// ---------------------------------------------------------------------------------------------
// launchers
// ---------------------------------------------------------------------------------------------
// Dynamic shared memory of one launch: the reduction scratch, plus what the launch's exact preconditioner stages (the
// plan's tiles, slots and resident panel columns).  Launches without an exact preconditioner ask for no more than they
// stage and leave the rest of the SM's 228 KB to L1; the plan's resident columns take what it leaves.
// (reduction scratch, the solver state and the block-CSR copy: the prefix every launch has)
constexpr size_t OPT_SMEM_BASE_DOUBLES = (OPT_THREADS / 32) * NRED + 2 * NRED + STATE_DOUBLES + SP_CACHE_INTS / 2;

template <int R, int DH> static size_t nd_staged_doubles(const KNd &nd) {
  return OPT_SMEM_BASE_DOUBLES + (size_t)nd.max_ytiles * R * DH + (size_t)(nd.max_slots + 1) * nd::PANEL_ROWS * R +
         4 * (size_t)nd.max_gathers + 8;
}

template <int R, int DH> static size_t optimize_smem_doubles(const KParams &kp) {
  if (kp.prm.precond == DPGO_PRECOND_SPARSE_EXACT || kp.prm.precond == DPGO_PRECOND_DENSE_EXACT)
    return nd_staged_doubles<R, DH>(kp.nd) + (size_t)kp.nd.resident_doubles;
  return OPT_SMEM_BASE_DOUBLES + 8;
}

// Everything a CTA may ask for beyond what the plan stages.  No L1 reserve: the step is faster with every resident round
// than with L1 for the block-CSR values and plan records.  sphere2500, 1 agent, H100 80GB HBM3 at 400 W, two alternating
// bench.py runs each: 2023 / 2041 it/s with no reserve, 1987 / 1998 with 32 KB and 1988 / 2009 with 64 KB kept for L1,
// against 1920 / 1924 without resident columns.
int64_t nd_resident_budget(int r, int dh, const KNd &nd) {
  int64_t staged = 0;
  DPGO_DISPATCH(r, dh, staged = (int64_t)nd_staged_doubles<R, DH>(nd) * (int64_t)sizeof(double));
  return std::max<int64_t>(0, (int64_t)OPT_SMEM_LIMIT - staged);
}

// The kernel with the phase clock or the lean one (everything else).
template <int R, int DH> static void *optimize_kernel(bool clock) {
  return clock ? (void *)k_optimize<R, DH, true> : (void *)k_optimize<R, DH, false>;
}

template <int R, int DH> static cudaError_t launch_optimize_t(const KParams &kp_in, cudaStream_t stream) {
  KParams kp = kp_in;
  const bool clock = kp.phase_ns != nullptr;
  const void *kern = optimize_kernel<R, DH>(clock);
  static_assert((OPT_SMEM_BASE_DOUBLES + (size_t)nd_ycap_tiles(R, DH) * R * DH + (size_t)(nd_slot_cap(R) + 1) * nd::PANEL_ROWS * R +
                 4 * (size_t)nd_ycap_tiles(R, DH) + 8) * sizeof(double) <= (size_t)OPT_SMEM_LIMIT,
                "what a plan at the shared-memory capacities stages must fit the kernel's maximum shared memory");
  kp.smem_doubles = (int)optimize_smem_doubles<R, DH>(kp);
  const size_t smem = (size_t)kp.smem_doubles * sizeof(double);
  // per device and kernel variant
  static bool attr_set[2][64] = {};
  int dev = 0;
  cudaGetDevice(&dev);
  if (dev < 0 || dev >= 64 || !attr_set[clock][dev]) {
    cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, OPT_SMEM_LIMIT);
    if (e != cudaSuccess) return e;
    if (dev >= 0 && dev < 64) attr_set[clock][dev] = true;
  }
  {
    // shared-memory carve-out hint: what this launch needs (+ the 1 KB the system reserves), so that L1 gets the rest
    static int last_pct[2][64];
    static bool init = false;
    if (!init) { for (int i = 0; i < 64; ++i) last_pct[0][i] = last_pct[1][i] = -1; init = true; }
    const int pct = std::min(100, (int)((smem + 2048) * 100 / (228 * 1024)) + 1);
    if (dev >= 0 && dev < 64 && last_pct[clock][dev] != pct) {
      cudaFuncSetAttribute(kern, cudaFuncAttributePreferredSharedMemoryCarveout, pct);
      last_pct[clock][dev] = pct;
    }
  }
  if (kp.cluster) {
    // one cluster = the whole grid: an ordinary (non-cooperative) launch, co-scheduling is guaranteed by the cluster
    static bool np_set[2][64] = {};
    if (kp.grid > 8 && (dev < 0 || dev >= 64 || !np_set[clock][dev])) {
      cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeNonPortableClusterSizeAllowed, 1);
      if (e != cudaSuccess) return e;
      if (dev >= 0 && dev < 64) np_set[clock][dev] = true;
    }
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = dim3(kp.grid);
    cfg.blockDim = dim3(OPT_THREADS);
    cfg.dynamicSmemBytes = smem;
    cfg.stream = stream;
    cudaLaunchAttribute at[1];
    at[0].id = cudaLaunchAttributeClusterDimension;
    at[0].val.clusterDim.x = (unsigned)kp.grid;
    at[0].val.clusterDim.y = 1;
    at[0].val.clusterDim.z = 1;
    cfg.attrs = at;
    cfg.numAttrs = 1;
    void *args[] = {(void *)&kp};
    return cudaLaunchKernelExC(&cfg, kern, args);
  }
  void *args[] = {(void *)&kp};
  return cudaLaunchCooperativeKernel(kern, dim3(kp.grid), dim3(OPT_THREADS), args, smem, stream);
}

// Both checks ask for the largest request a launch may make (OPT_SMEM_LIMIT), so that no plan can exceed what they allowed.
template <int R, int DH> static int max_cluster_t(int device) {
  const size_t smem = OPT_SMEM_LIMIT;
  for (int f = 0; f < 2; ++f) {
    cudaFuncSetAttribute(optimize_kernel<R, DH>(f != 0), cudaFuncAttributeNonPortableClusterSizeAllowed, 1);
    cudaFuncSetAttribute(optimize_kernel<R, DH>(f != 0), cudaFuncAttributeMaxDynamicSharedMemorySize, OPT_SMEM_LIMIT);
  }
  for (int cs : {16, 8}) {
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = dim3(cs);
    cfg.blockDim = dim3(OPT_THREADS);
    cfg.dynamicSmemBytes = smem;
    cudaLaunchAttribute at[1];
    at[0].id = cudaLaunchAttributeClusterDimension;
    at[0].val.clusterDim.x = (unsigned)cs;
    at[0].val.clusterDim.y = 1;
    at[0].val.clusterDim.z = 1;
    cfg.attrs = at;
    cfg.numAttrs = 1;
    int n0 = 0, n1 = 0;
    if (cudaOccupancyMaxActiveClusters(&n0, optimize_kernel<R, DH>(false), &cfg) == cudaSuccess && n0 >= 1 &&
        cudaOccupancyMaxActiveClusters(&n1, optimize_kernel<R, DH>(true), &cfg) == cudaSuccess && n1 >= 1)
      return cs;
  }
  cudaGetLastError();
  return 0;
}

template <int R, int DH> static int max_grid_t(int device) {
  const size_t smem = OPT_SMEM_LIMIT;
  int per_sm = 1, sms = 0, optin = 0;
  // the sparse plan's budget assumes the H100's opt-in limit: a device with less cannot run the kernel as planned
  if (cudaDeviceGetAttribute(&optin, cudaDevAttrMaxSharedMemoryPerBlockOptin, device) != cudaSuccess || optin < OPT_SMEM_LIMIT)
    return 0;
  for (int f = 0; f < 2; ++f) {
    const void *kern = optimize_kernel<R, DH>(f != 0);
    cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    int ps = 0;
    if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&ps, kern, OPT_THREADS, smem) != cudaSuccess) return 0;
    per_sm = std::min(per_sm, ps);
  }
  if (cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, device) != cudaSuccess) return 0;
  return per_sm > 0 ? sms : 0;      // one CTA per SM
}

cudaError_t launch_optimize(int r, int dh, const KParams &kp, cudaStream_t stream) {
  cudaError_t e = cudaErrorInvalidValue;
  DPGO_DISPATCH(r, dh, e = (launch_optimize_t<R, DH>(kp, stream)));
  return e;
}

int optimize_max_grid(int r, int dh, int device) {
  int g = 0;
  DPGO_DISPATCH(r, dh, g = (max_grid_t<R, DH>(device)));
  return g;
}

int optimize_max_cluster(int r, int dh, int device) {
  int g = 0;
  DPGO_DISPATCH(r, dh, g = (max_cluster_t<R, DH>(device)));
  return g;
}

cudaError_t launch_spmv(int r, int dh, int n, const int *rowptr, const int *bcol, const double *bval,
                        const double *X, const double *G, double *out, cudaStream_t stream) {
  bool ok = false;
  DPGO_DISPATCH(r, dh, {
    constexpr int SG = SubGroup<R>::SG;
    const int per_block = SPMV_THREADS / SG;
    const int blocks = (n + per_block - 1) / per_block;
    k_spmv<R, DH><<<blocks, SPMV_THREADS, 0, stream>>>(n, rowptr, bcol, bval, X, G, out);
    ok = true;
  });
  if (!ok) return cudaErrorInvalidValue;
  return cudaGetLastError();
}

cudaError_t launch_stiefel_project(int r, int dh, int n, const double *M, double *out, cudaStream_t stream, double c0,
                                   const double *B, double c1, const double *C, double c2) {
  bool ok = false;
  DPGO_DISPATCH(r, dh, {
    k_stiefel_project<R, DH><<<(n + 127) / 128, 128, 0, stream>>>(n, M, out, c0, B, c1, C, c2);
    ok = true;
  });
  if (!ok) return cudaErrorInvalidValue;
  return cudaGetLastError();
}

cudaError_t launch_pack_tiles(int ts, int count, const int *pose, const double *X, double *out, cudaStream_t stream,
                              const unsigned char *gate) {
  if (count <= 0) return cudaSuccess;
  const int total = count * ts;
  k_pack_tiles<<<(total + 255) / 256, 256, 0, stream>>>(ts, count, pose, X, out, gate);
  return cudaGetLastError();
}


cudaError_t launch_build_G(int r, int dh, int nposes, const int *pose_ids, const int *pose_ptr, const int *edge_slot,
                           const int *edge_out, const double *edge_T, const double *edge_om, const double *gathered,
                           double *G, cudaStream_t stream, const unsigned char *gate) {
  if (nposes <= 0) return cudaSuccess;
  bool ok = false;
  DPGO_DISPATCH(r, dh, {
    const int total = nposes * R * DH;
    k_build_G<R, DH><<<(total + 127) / 128, 128, 0, stream>>>(nposes, pose_ids, pose_ptr, edge_slot, edge_out, edge_T,
                                                              edge_om, gathered, G, gate);
    ok = true;
  });
  if (!ok) return cudaErrorInvalidValue;
  return cudaGetLastError();
}

cudaError_t launch_assemble_Q(int64_t nb, const int *cptr, const int2 *contrib, const double *eT, const double *eom, const double *ew,
                              const double *sblk, double *bval, cudaStream_t stream) {
  if (nb > 0) k_assemble_Q<<<(unsigned)((nb * 16 + 255) / 256), 256, 0, stream>>>(nb, cptr, contrib, eT, eom, ew, sblk, bval);
  return cudaGetLastError();
}

cudaError_t launch_edge_weights(int r, int dh, int64_t m, const int *p1, const int *p2, const double *eT, const double *eom,
                                const int *fixed, const double *X, int cost, double mu, double param, double *w, double *resid,
                                unsigned long long *gnc, cudaStream_t stream) {
  if (m <= 0) return cudaSuccess;
  bool ok = false;
  DPGO_DISPATCH(r, dh, {
    k_edge_weights<R, DH><<<(unsigned)((m + 127) / 128), 128, 0, stream>>>(m, p1, p2, eT, eom, fixed, X, cost, mu, param, w, resid,
                                                                            gnc);
    ok = true;
  });
  if (!ok) return cudaErrorInvalidValue;
  return cudaGetLastError();
}


}  // namespace dpgo
