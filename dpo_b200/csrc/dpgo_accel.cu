// dpgo_accel.cu -- Nesterov-accelerated rounds of the device RBCD runners (ref PGOAgent::iterate / updateGamma /
// updateAlpha / updateY / updateV / restart, src/PGOAgent.cpp:685-695,1033-1091).
//
//  k_accel_agents<R,DH>  every local agent of one GPU in one launch, one thread per pose: advances the agent's momentum
//                        record, XPrev = X, Y = proj((1 - alpha) X + alpha V); an idle agent also finishes its
//                        iterate(false): X = Y, V = proj(V + gamma (X - Y)), and on a restart round X = XPrev, V = Y = X.
//                        Each public pose then writes its tiles of X and Y into the agent's send buffers (pose -> public
//                        slot index), so the packing needs no grid-wide synchronisation.  The record is read by every CTA
//                        of the agent and written by its last one (ticket counter), so a replayed round takes no
//                        per-round kernel arguments.
//  k_accel_finish<R,DH>  an active agent after its step: V = proj(V + gamma (X - Y)); on a restart round X = XPrev before
//                        the plain step and V = Y = X after it.  The launch that ends the round (ACCEL_FINISH_V on a
//                        plain round, ACCEL_FINISH_RESTART_END on a restart round) also writes the agent's status record
//                        as the reference's iterate() does (src/PGOAgent.cpp:673,703-716): relative change
//                        sqrt(|X - XPrev|^2 / n) of the whole accelerated iteration, and one optimising call more than at
//                        the round's begin (k_accel_agents snapshots the count), however many steps the round took.
//                        Per-CTA partials, summed in CTA order by the agent's last CTA (ticket counter), as k_agents_status.
// Both reuse stiefel_project_tile with the operand order of k_stiefel_project, so the iterates are bitwise those of the
// per-agent dpgo_agent_accel_* calls.
#include <cuda_runtime.h>

#include "dpgo_device.cuh"
#include "dpgo_kernels.cuh"
#include "dpgo_rotation.cuh"

namespace dpgo {

namespace {

// gamma' = (1 + sqrt(1 + ((4 N) N) (gamma gamma))) / (2 N), alpha = 1 / (gamma' N) in exactly this operation order, with no
// contraction into an FMA: the host's recurrence gives the same bits.
__device__ __forceinline__ double momentum_gamma(double gamma, double N) {
  const double q = __dmul_rn(__dmul_rn(4.0, N), N);
  return __ddiv_rn(__dadd_rn(1.0, __dsqrt_rn(__dadd_rn(1.0, __dmul_rn(q, __dmul_rn(gamma, gamma))))), __dmul_rn(2.0, N));
}
__device__ __forceinline__ double momentum_alpha(double gamma, double N) { return __ddiv_rn(1.0, __dmul_rn(gamma, N)); }

template <int TS> __device__ __forceinline__ void copy_tile(const double *src, double *dst) {
#pragma unroll
  for (int e = 0; e < TS; ++e) dst[e] = src[e];
}

// V = proj(1 V + gamma X + (-gamma) Y), the operands of dpgo_agent_accel_end
template <int R, int DH> __device__ __forceinline__ void update_V(const double *X, const double *Y, double *V, double gamma) {
  const double ng = -gamma;
  stiefel_project_tile<R, DH>(
      [&](int e) {
        double v = 1.0 * V[e];
        v = fma(gamma, X[e], v);
        v = fma(ng, Y[e], v);
        return v;
      },
      [&](int e, double v) { V[e] = v; });
}

template <int R, int DH>
__global__ void __launch_bounds__(ACCEL_THREADS) k_accel_agents(int njobs, const AccelJob *__restrict__ jobs, double N,
                                                               int restart_interval) {
  constexpr int TS = R * DH;
  int lo = 0, hi = njobs;                                   // the job whose CTA range holds this CTA
  while (hi - lo > 1) {
    const int mid = (lo + hi) >> 1;
    if (jobs[mid].cta0 <= (int)blockIdx.x) lo = mid; else hi = mid;
  }
  const AccelJob J = jobs[lo];
  const int cta = (int)blockIdx.x - J.cta0;
  const double gamma = momentum_gamma(__ldcg(J.state), N);
  const double alpha = momentum_alpha(gamma, N);
  const long long it = (long long)__ldcg(J.state + 2) + 1;
  const bool restart = (it + 1) % restart_interval == 0;
  const int j = cta * ACCEL_THREADS + (int)threadIdx.x;
  if (j < J.n) {
    double *X = J.X + (size_t)j * TS, *Y = J.Y + (size_t)j * TS, *V = J.V + (size_t)j * TS, *XP = J.XP + (size_t)j * TS;
    copy_tile<TS>(X, XP);
    const double c0 = 1.0 - alpha;
    stiefel_project_tile<R, DH>(
        [&](int e) {
          double v = c0 * X[e];
          v = fma(alpha, V[e], v);
          return v;
        },
        [&](int e, double v) { Y[e] = v; });
    if (!J.active) {
      copy_tile<TS>(Y, X);
      update_V<R, DH>(X, Y, V, gamma);
      if (restart) {
        copy_tile<TS>(XP, X);
        copy_tile<TS>(X, V);
        copy_tile<TS>(X, Y);
      }
    }
    const int s = J.pub_slot[j];
    if (s >= 0) {
      copy_tile<TS>(X, J.send_x + (size_t)s * TS);
      copy_tile<TS>(Y, J.send_y + (size_t)s * TS);
    }
  }
  __syncthreads();                                          // every thread of the CTA has read the record
  if (threadIdx.x == 0) {
    __threadfence();
    if (atomicAdd(J.ticket, 1u) == (unsigned)(accel_ctas(J.n) - 1)) {
      J.state[0] = restart ? 0.0 : gamma;
      J.state[1] = restart ? 0.0 : alpha;
      J.state[2] = (double)it;
      J.state[3] = gamma;
      J.state[4] = __ldcg(J.opt_record + 1);              // optimising calls at the round's begin
      *J.ticket = 0u;                                       // ready for the next launch on the stream
    }
  }
}

constexpr int ACCEL_WARPS = ACCEL_THREADS / 32;

template <int R, int DH>
__global__ void k_accel_finish(int n, double *X, double *Y, double *V, const double *XP, const double *state, int mode,
                               double *partials, unsigned *ticket, double *opt_record) {
  constexpr int TS = R * DH;
  __shared__ double sm_warp[ACCEL_WARPS];
  __shared__ bool last;
  const int j = blockIdx.x * blockDim.x + threadIdx.x;
  double d2 = 0.0;
  if (j < n) {
    double *Xj = X + (size_t)j * TS, *Yj = Y + (size_t)j * TS, *Vj = V + (size_t)j * TS;
    const double *XPj = XP + (size_t)j * TS;
    if (mode == ACCEL_FINISH_RESTART_END) {
      copy_tile<TS>(Xj, Vj);
      copy_tile<TS>(Xj, Yj);
    } else {
      update_V<R, DH>(Xj, Yj, Vj, __ldg(state + 3));
      if (mode == ACCEL_FINISH_V_RESTART) copy_tile<TS>(XPj, Xj);
    }
    if (mode != ACCEL_FINISH_V_RESTART) {
#pragma unroll
      for (int e = 0; e < TS; ++e) {
        const double t = Xj[e] - XPj[e];
        d2 = fma(t, t, d2);
      }
    }
  }
  if (mode == ACCEL_FINISH_V_RESTART) return;              // the restart's step follows: the round is not over
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  d2 = warp_sum(d2);
  if (lane == 0) sm_warp[warp] = d2;
  __syncthreads();
  const int ncta = accel_ctas(n);
  if (threadIdx.x == 0) {
    double s = 0.0;
    for (int w = 0; w < ACCEL_WARPS; ++w) s += sm_warp[w];
    partials[blockIdx.x] = s;
    __threadfence();                                        // partial visible before the ticket
    last = atomicAdd(ticket, 1u) == (unsigned)(ncta - 1);
  }
  __syncthreads();
  if (!last || warp != 0) return;
  __threadfence();
  double t = 0.0;
  for (int b = lane; b < ncta; b += 32) t += __ldcg(partials + b);   // fixed order: lane-strided, then a fixed shuffle tree
  t = warp_sum(t);
  if (lane == 0) {
    opt_record[0] = sqrt(t / (double)n);
    opt_record[1] = __ldcg(state + 4) + 1.0;
    *ticket = 0u;                                           // ready for the next launch on the stream
  }
}

}  // namespace

cudaError_t launch_accel_agents(int r, int dh, int njobs, int total_ctas, const AccelJob *jobs, double momentum_n,
                                int restart_interval, cudaStream_t stream) {
  if (njobs <= 0 || total_ctas <= 0 || restart_interval < 1) return cudaErrorInvalidValue;
  bool ok = false;
  DPGO_DISPATCH(r, dh, {
    k_accel_agents<R, DH><<<total_ctas, ACCEL_THREADS, 0, stream>>>(njobs, jobs, momentum_n, restart_interval);
    ok = true;
  });
  if (!ok) return cudaErrorInvalidValue;
  return cudaGetLastError();
}

cudaError_t launch_accel_finish(int r, int dh, int n, double *X, double *Y, double *V, const double *XP, const double *state,
                                int mode, double *partials, unsigned *ticket, double *opt_record, cudaStream_t stream) {
  if (n <= 0) return cudaErrorInvalidValue;
  bool ok = false;
  DPGO_DISPATCH(r, dh, {
    k_accel_finish<R, DH><<<accel_ctas(n), ACCEL_THREADS, 0, stream>>>(n, X, Y, V, XP, state, mode, partials, ticket,
                                                                      opt_record);
    ok = true;
  });
  if (!ok) return cudaErrorInvalidValue;
  return cudaGetLastError();
}

}  // namespace dpgo
