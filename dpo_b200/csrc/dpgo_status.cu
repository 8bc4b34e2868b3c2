// dpgo_status.cu -- team status and rounding of the device RBCD runners.
//
//  k_agents_status<R,DH>     every agent of one GPU in one launch: <XQ, X>, <X, G>, |P_X(XQ + G)|^2 of the resident
//                            iterate (the quantities of an evaluation, ref QuadraticProblem::f / RieGrad,
//                            src/QuadraticProblem.cpp:50-66,89-101) and the agent's last relative change (ref
//                            PGOAgentStatus, src/PGOAgent.cpp:703-716).  An agent owns status_ctas(n) CTAs, a number
//                            that depends on its size alone; a CTA owns STATUS_ROWS consecutive rows of the agent's
//                            block-CSR Q, one pose tile per sub-group (the lane mapping of dpgo_device.cuh).  The per-CTA
//                            partials are written out and the agent's last CTA (ticket counter) sums them in CTA order,
//                            so a record is bitwise the same whichever agents share the launch.
//  k_trajectory_global<R,DH> one thread per pose: T_i = [proj_SO(d)(Ya^T Y_i)  Ya^T p_i - Ya^T pa] (ref
//                            getTrajectoryInGlobalFrame, src/PGOAgent.cpp:500-519).
#include <cuda_runtime.h>

#include "dpgo_device.cuh"
#include "dpgo_kernels.cuh"
#include "dpgo_rotation.cuh"

namespace dpgo {

namespace {

constexpr int STATUS_WARPS = STATUS_THREADS / 32;

template <int R, int DH>
__global__ void __launch_bounds__(STATUS_THREADS) k_agents_status(int njobs, const StatusJob *__restrict__ jobs) {
  constexpr int SG = SubGroup<R>::SG;
  constexpr int SGW = 32 / SG;
  constexpr int TS = R * DH;
  __shared__ double sm_warp[STATUS_WARPS][3];
  __shared__ bool last;
  int lo = 0, hi = njobs;                                   // the job whose CTA range holds this CTA
  while (hi - lo > 1) {
    const int mid = (lo + hi) >> 1;
    if (jobs[mid].cta0 <= (int)blockIdx.x) lo = mid; else hi = mid;
  }
  const StatusJob J = jobs[lo];
  const int cta = (int)blockIdx.x - J.cta0, ncta = status_ctas(J.n);
  const int r0 = cta * STATUS_ROWS, r1 = min(J.n, r0 + STATUS_ROWS);
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int l = lane & (SG - 1), a = l >> 2, c = l & 3;
  const bool valid = (a < R) && (c < DH);
  const int e = c * R + a;
  double acc[3] = {0.0, 0.0, 0.0};
  // the loop bound is uniform per warp: every lane takes part in the sub-group shuffles
  for (int jb = r0 + warp * SGW; jb < r1; jb += STATUS_WARPS * SGW) {
    const int j = jb + lane / SG;
    const bool act = j < r1;
    const int js = act ? j : r1 - 1;
    const bool ld = act && valid;
    double xq = gather_tile<R, DH, false, false>(J.rowptr, J.bcol, J.bval, J.X, nullptr, 0.0, js, a, c);
    const size_t idx = (size_t)js * TS + e;
    const double x = ld ? __ldg(J.X + idx) : 0.0;
    const double g = ld ? __ldg(J.G + idx) : 0.0;
    if (!ld) xq = 0.0;
    double ya[3], sym[3];
    const double rg = tangent_project_elem<R, DH>(x, xq + g, a, c, ya, sym);
    acc[0] = fma(xq, x, acc[0]);
    acc[1] = fma(x, g, acc[1]);
    if (ld) acc[2] = fma(rg, rg, acc[2]);
  }
#pragma unroll
  for (int q = 0; q < 3; ++q) {
    const double v = warp_sum(acc[q]);
    if (lane == 0) sm_warp[warp][q] = v;
  }
  __syncthreads();
  if (threadIdx.x == 0) {
#pragma unroll
    for (int q = 0; q < 3; ++q) {
      double s = 0.0;
      for (int w = 0; w < STATUS_WARPS; ++w) s += sm_warp[w][q];
      J.partials[(size_t)cta * 3 + q] = s;
    }
    __threadfence();                                        // partials visible before the ticket
    last = atomicAdd(J.ticket, 1u) == (unsigned)(ncta - 1);
  }
  __syncthreads();
  if (!last || warp != 0) return;
  __threadfence();
  double t[3] = {0.0, 0.0, 0.0};
  for (int b = lane; b < ncta; b += 32)                     // fixed order: lane-strided, then a fixed shuffle tree
#pragma unroll
    for (int q = 0; q < 3; ++q) t[q] += __ldcg(J.partials + (size_t)b * 3 + q);
#pragma unroll
  for (int q = 0; q < 3; ++q) t[q] = warp_sum(t[q]);
  if (lane == 0) {
    J.out[0] = t[0];
    J.out[1] = t[1];
    J.out[2] = t[2];
    J.out[3] = __ldcg(J.opt_record);
    J.out[4] = __ldcg(J.opt_record + 1);
    *J.ticket = 0u;                                         // ready for the next launch on the stream
  }
}

template <int R, int DH>
__global__ void k_trajectory_global(int n, const double *__restrict__ anchor, const double *__restrict__ X, double *__restrict__ T) {
  constexpr int D = DH - 1;
  constexpr int TS = R * DH;
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const double *Xi = X + (size_t)i * TS;                    // column c of the tile: Xi[c * R + a]
  double M[D][D], t[D];
  for (int p = 0; p < D; ++p) {
    for (int c = 0; c < DH; ++c) {
      double s = 0.0;
      for (int a = 0; a < R; ++a) s = fma(anchor[p * R + a], Xi[c * R + a], s);
      if (c < D) M[p][c] = s; else t[p] = s;
    }
    double t0 = 0.0;
    for (int a = 0; a < R; ++a) t0 = fma(anchor[p * R + a], anchor[D * R + a], t0);
    t[p] -= t0;
  }
  double Rm[D][D];
  project_to_rotation<D>(M, Rm);
  double *Ti = T + (size_t)i * D * DH;                      // d x (d+1) column-major
  for (int c = 0; c < D; ++c)
    for (int p = 0; p < D; ++p) Ti[c * D + p] = Rm[p][c];
  for (int p = 0; p < D; ++p) Ti[D * D + p] = t[p];
}

}  // namespace

cudaError_t launch_agents_status(int r, int dh, int njobs, int total_ctas, const StatusJob *jobs, cudaStream_t stream) {
  if (njobs <= 0 || total_ctas <= 0) return cudaErrorInvalidValue;
  bool ok = false;
  DPGO_DISPATCH(r, dh, {
    k_agents_status<R, DH><<<total_ctas, STATUS_THREADS, 0, stream>>>(njobs, jobs);
    ok = true;
  });
  if (!ok) return cudaErrorInvalidValue;
  return cudaGetLastError();
}

cudaError_t launch_trajectory_global(int r, int dh, int n, const double *anchor, const double *X, double *T, cudaStream_t stream) {
  bool ok = false;
  DPGO_DISPATCH(r, dh, {
    k_trajectory_global<R, DH><<<(n + 127) / 128, 128, 0, stream>>>(n, anchor, X, T);
    ok = true;
  });
  if (!ok) return cudaErrorInvalidValue;
  return cudaGetLastError();
}

}  // namespace dpgo
