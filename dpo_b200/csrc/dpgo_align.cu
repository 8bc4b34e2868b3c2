// dpgo_align.cu -- frame alignment of the distributed initialisation on the GPU.
//
// Every agent starts from the chordal initialisation of its private graph, in its own frame.  An agent joins the global
// frame when a neighbour it shares loop closures with is initialised (ref PGOAgent::updateNeighborPoses ->
// initializeInGlobalFrame, src/PGOAgent.cpp:369-440): every shared public pose of the neighbour gives one candidate frame
// transform (computeNeighborTransform, :250-288), and the robust two-stage average of the candidates
// (computeRobustNeighborTransformTwoStage, :290-331) -- GNC-TLS rotation averaging (robustSingleRotationAveraging,
// src/DPGO_utils.cpp:567-629), then the mean translation of the inliers (singleTranslationAveraging, :518-535) -- moves
// the agent's trajectory into the global frame.
//
//  k_align_candidates<D>          one thread per candidate: T_w2w1 = [YLift^T X_b,j ; 0 1] T_f1f2^-1 T_a,i^-1
//  k_robust_rotation_average<D>   one CTA per aligning agent: the whole GNC loop (fixed-order block reductions, so the
//                                 result does not depend on scheduling), neighbours tried in increasing id until one gives
//                                 a non-empty inlier set
//  k_apply_frame_lift<R,D>        X = YLift (T_align T) for every pose of the agents that aligned
#include <cuda_runtime.h>

#include "dpgo_device.cuh"
#include "dpgo_kernels.cuh"
#include "dpgo_rotation.cuh"

namespace dpgo {

namespace {

constexpr int NWARPS = ALIGN_THREADS / 32;

// inverse of a D x D matrix (adjugate / determinant); A[a][c] = A(a, c)
template <int D> __device__ __forceinline__ void invert_small(const double (&A)[D][D], double (&B)[D][D]) {
  if (D == 2) {
    const double det = A[0][0] * A[1][1] - A[0][1] * A[1][0];
    B[0][0] = A[1][1] / det; B[0][1] = -A[0][1] / det;
    B[1][0] = -A[1][0] / det; B[1][1] = A[0][0] / det;
  } else {
    constexpr int E = D - 1;                 // == 2 (keeps the indices in range when D == 2)
    double C[D][D];
    for (int a = 0; a < D; ++a)
      for (int c = 0; c < D; ++c) {
        const int a1 = (a + 1) % D, a2 = (a + E) % D, c1 = (c + 1) % D, c2 = (c + E) % D;
        C[a][c] = A[a1][c1] * A[a2][c2] - A[a1][c2] * A[a2][c1];     // cofactor (cyclic form carries the sign)
      }
    const double det = A[0][0] * C[0][0] + A[0][1] * C[0][1] + A[0][2 % D] * C[0][2 % D];
    for (int a = 0; a < D; ++a)
      for (int c = 0; c < D; ++c) B[a][c] = C[c][a] / det;
  }
}

// sum over the CTA of NV values per thread, fixed reduction order; every thread receives the totals
template <int NV> __device__ __forceinline__ void block_sum(double (&v)[NV], double (*red)[NV], double *out) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
  for (int k = 0; k < NV; ++k) v[k] = warp_sum(v[k]);
  if (lane == 0)
    for (int k = 0; k < NV; ++k) red[warp][k] = v[k];
  __syncthreads();
  if (warp == 0) {
#pragma unroll
    for (int k = 0; k < NV; ++k) {
      const double s = warp_sum(lane < NWARPS ? red[lane][k] : 0.0);
      if (lane == 0) out[k] = s;
    }
  }
  __syncthreads();
#pragma unroll
  for (int k = 0; k < NV; ++k) v[k] = out[k];
  __syncthreads();
}

__device__ __forceinline__ double block_max(double v, double *red, double *out) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  for (int m = 16; m > 0; m >>= 1) v = fmax(v, shfl_xor(v, m));
  if (lane == 0) red[warp] = v;
  __syncthreads();
  if (warp == 0) {
    double s = lane < NWARPS ? red[lane] : 0.0;
    for (int m = 16; m > 0; m >>= 1) s = fmax(s, shfl_xor(s, m));
    if (lane == 0) *out = s;
  }
  __syncthreads();
  v = *out;
  __syncthreads();
  return v;
}

}  // namespace

// Candidate q of job blockIdx.y (ref computeNeighborTransform, src/PGOAgent.cpp:250-288): world1 is the agent's own frame,
// world2 the global one, frame1 its public pose i, frame2 the neighbour's public pose j.  The neighbour's tile is exactly
// YLift T_b,j at initialisation time, so YLift^T X_b,j is its pose without a further projection.
template <int D>
__global__ void k_align_candidates(const AlignJob *__restrict__ jobs, int r, const double *__restrict__ gathered) {
  constexpr int DH = D + 1;
  const AlignJob J = jobs[blockIdx.y];
  const int q = blockIdx.x * blockDim.x + threadIdx.x;
  if (J.ngroups == 0 || q >= J.grp_ptr[J.ngroups]) return;      // an agent without shared edges has no group table
  const int ts = r * DH;
  const double *Xb = gathered + (size_t)J.cand_slot[q] * ts;
  double Tb[D][DH];                                    // T_world2_frame2 = YLift^T X_b,j
  for (int a = 0; a < D; ++a)
    for (int c = 0; c < DH; ++c) {
      double s = 0.0;
      for (int k = 0; k < r; ++k) s = fma(J.ylift[a * r + k], Xb[c * r + k], s);
      Tb[a][c] = s;
    }
  const double *E = J.cand_T + (size_t)q * DH * DH;   // the shared edge's measurement dT
  double A[D][D], Ai[D][D], Fr[D][D], ft[D];           // F = T_frame1_frame2^-1: dT^-1 (outgoing), dT (incoming)
  for (int a = 0; a < D; ++a)
    for (int c = 0; c < D; ++c) A[a][c] = E[a * DH + c];
  if (J.cand_out[q]) {
    invert_small<D>(A, Ai);
    for (int a = 0; a < D; ++a) {
      double s = 0.0;
      for (int c = 0; c < D; ++c) { Fr[a][c] = Ai[a][c]; s = fma(Ai[a][c], E[c * DH + D], s); }
      ft[a] = -s;
    }
  } else {
    for (int a = 0; a < D; ++a) {
      for (int c = 0; c < D; ++c) Fr[a][c] = A[a][c];
      ft[a] = E[a * DH + D];
    }
  }
  double Rw[D][D], tw[D];                              // T_world2_frame1 = T_world2_frame2 F
  for (int a = 0; a < D; ++a) {
    double s = Tb[a][D];
    for (int k = 0; k < D; ++k) s = fma(Tb[a][k], ft[k], s);
    tw[a] = s;
    for (int c = 0; c < D; ++c) {
      double u = 0.0;
      for (int k = 0; k < D; ++k) u = fma(Tb[a][k], Fr[k][c], u);
      Rw[a][c] = u;
    }
  }
  const double *Ta = J.Tloc + (size_t)J.cand_local[q] * D * DH;    // T_world1_frame1 (rotation exactly orthonormal)
  double *Ro = J.cand_R + (size_t)q * D * D, *to = J.cand_t + (size_t)q * D;
  double R[D][D];                                      // T_world2_world1 = T_world2_frame1 T_world1_frame1^-1
  for (int a = 0; a < D; ++a)
    for (int c = 0; c < D; ++c) {
      double s = 0.0;
      for (int k = 0; k < D; ++k) s = fma(Rw[a][k], Ta[k * D + c], s);      // Rw Ra^T
      R[a][c] = s;
      Ro[a * D + c] = s;
    }
  for (int a = 0; a < D; ++a) {
    double s = tw[a];
    for (int k = 0; k < D; ++k) s = fma(-R[a][k], Ta[D * D + k], s);
    to[a] = s;
  }
}

// One CTA per job (ref robustSingleRotationAveraging, src/DPGO_utils.cpp:567-629 with RobustCost GNC_TLS,
// src/DPGO_robust.cpp:23-103): kappa-weighted chordal mean projected to SO(d); mu0 = min(cbar^2 / (2 max r^2 - cbar^2),
// 1e-5), no GNC when mu0 <= 0; otherwise per iteration the weighted mean, its projection, the TLS-GNC weights, stop when
// every weight is within 1e-8 of 0 or 1, else mu *= 1.4; at most 1000 iterations.  Inliers: w > 1 - 1e-8; the translation
// is the plain mean of the inliers' (ref :318-331).  Groups whose neighbour is not ready are skipped; the first group with
// inliers is the result (ref :395-400: an empty inlier set aborts and waits for another neighbour).
template <int D>
__global__ void __launch_bounds__(ALIGN_THREADS) k_robust_rotation_average(const AlignJob *__restrict__ jobs,
                                                                           const int *__restrict__ ready, double cbar) {
  constexpr int DD = D * D;
  constexpr double W_TOL = 1e-8;
  __shared__ double red[NWARPS][DD];
  __shared__ double out[DD];
  __shared__ double Rsh[DD];
  const AlignJob J = jobs[blockIdx.x];
  const int tid = threadIdx.x;
  const double c2 = cbar * cbar;

  // weighted sum of the candidate rotations of [q0, q1) -> projection -> Rsh (and R in every thread)
  auto estimate = [&](int q0, int q1, double (&R)[D][D]) {
    double v[DD];
    for (int k = 0; k < DD; ++k) v[k] = 0.0;
    for (int q = q0 + tid; q < q1; q += ALIGN_THREADS) {
      const double kw = (J.kappa ? J.kappa[q] : 1.0) * J.w[q];
      const double *Rq = J.cand_R + (size_t)q * DD;
      for (int k = 0; k < DD; ++k) v[k] += kw * Rq[k];
    }
    block_sum<DD>(v, red, out);
    if (tid == 0) {
      double M[D][D], P[D][D];
      for (int a = 0; a < D; ++a)
        for (int c = 0; c < D; ++c) M[a][c] = v[a * D + c];
      project_to_rotation<D>(M, P);
      for (int a = 0; a < D; ++a)
        for (int c = 0; c < D; ++c) Rsh[a * D + c] = P[a][c];
    }
    __syncthreads();
    for (int a = 0; a < D; ++a)
      for (int c = 0; c < D; ++c) R[a][c] = Rsh[a * D + c];
    __syncthreads();
  };
  auto residual2 = [&](int q, const double (&R)[D][D]) {
    const double *Rq = J.cand_R + (size_t)q * DD;
    double s = 0.0;
    for (int a = 0; a < D; ++a)
      for (int c = 0; c < D; ++c) { const double e = R[a][c] - Rq[a * D + c]; s += e * e; }
    return (J.kappa ? J.kappa[q] : 1.0) * s;
  };

  bool attempted = false;
  for (int g = 0; g < J.ngroups; ++g) {
    if (!ready[J.grp_nbr[g]]) continue;
    const int q0 = J.grp_ptr[g], q1 = J.grp_ptr[g + 1];
    for (int q = q0 + tid; q < q1; q += ALIGN_THREADS) J.w[q] = 1.0;
    __syncthreads();
    double R[D][D];
    estimate(q0, q1, R);
    double rmax = 0.0;
    for (int q = q0 + tid; q < q1; q += ALIGN_THREADS) rmax = fmax(rmax, residual2(q, R));
    rmax = block_max(rmax, &red[0][0], out);
    const double mu0 = fmin(c2 / (2.0 * rmax - c2), 1e-5);
    int iters = 0;
    if (mu0 > 0.0) {                                   // small residuals everywhere: no GNC (ref :594-595)
      double mu = mu0;
      for (int it = 0; it < 1000; ++it) {
        estimate(q0, q1, R);
        double nc[1] = {0.0};
        for (int q = q0 + tid; q < q1; q += ALIGN_THREADS) {
          const double rr = sqrt(residual2(q, R));     // the reference passes r = sqrt(r^2) to RobustCost::weight
          const double wq = gnc_tls_weight(rr, mu, cbar);
          J.w[q] = wq;
          if (wq < W_TOL || wq > 1.0 - W_TOL) nc[0] += 1.0;
        }
        block_sum<1>(nc, reinterpret_cast<double (*)[1]>(&red[0][0]), out);
        iters = it + 1;
        if (nc[0] == (double)(q1 - q0)) break;
        mu *= 1.4;                                     // RobustCostParameters::GNCMuStep
      }
    }
    // inliers and their mean translation
    double acc[D + 1];
    for (int k = 0; k <= D; ++k) acc[k] = 0.0;
    for (int q = q0 + tid; q < q1; q += ALIGN_THREADS)
      if (J.w[q] > 1.0 - W_TOL) {
        acc[D] += 1.0;
        if (J.cand_t)
          for (int k = 0; k < D; ++k) acc[k] += J.cand_t[(size_t)q * D + k];
      }
    block_sum<D + 1>(acc, reinterpret_cast<double (*)[D + 1]>(&red[0][0]), out);
    if (tid == 0) {                                    // the last attempt stays reported when no neighbour gives inliers
      for (int a = 0; a < D; ++a) {
        for (int c = 0; c < D; ++c) J.T_align[c * D + a] = R[a][c];
        J.T_align[DD + a] = acc[D] > 0.0 ? acc[a] / acc[D] : 0.0;
      }
      J.info[0] = J.grp_nbr[g]; J.info[1] = q1 - q0; J.info[2] = (int)acc[D]; J.info[3] = iters;
    }
    if (acc[D] > 0.0) return;
    attempted = true;
  }
  if (tid == 0 && !attempted) { J.info[0] = -1; J.info[1] = 0; J.info[2] = 0; J.info[3] = 0; }
}

// X_i = YLift (T_align T_i): one thread per element (a, c) of a pose tile of job blockIdx.y
template <int R, int D> __global__ void k_apply_frame_lift(const AlignJob *__restrict__ jobs) {
  constexpr int DH = D + 1, TS = R * DH;
  const AlignJob J = jobs[blockIdx.y];
  if (J.info && J.info[2] <= 0) return;
  const int e = blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= J.n * TS) return;
  const int i = e / TS, a = (e % TS) % R, c = (e % TS) / R;
  const double *T = J.Tloc + (size_t)i * D * DH;
  double s = 0.0;
  for (int q = 0; q < D; ++q) {
    double u;                                          // (T_align T_i)(q, c)
    if (J.T_align) {
      u = (c == D) ? J.T_align[D * D + q] : 0.0;
      for (int p = 0; p < D; ++p) u = fma(J.T_align[p * D + q], T[c * D + p], u);
    } else {
      u = T[c * D + q];
    }
    s = fma(J.ylift[q * R + a], u, s);
  }
  J.X[(size_t)i * TS + c * R + a] = s;
}

cudaError_t launch_align_candidates(int d, int r, int njobs, int max_cands, const AlignJob *jobs, const double *gathered,
                                    cudaStream_t stream) {
  if (njobs <= 0 || max_cands <= 0) return cudaSuccess;
  const dim3 grid((max_cands + 127) / 128, njobs);
  if (d == 3) k_align_candidates<3><<<grid, 128, 0, stream>>>(jobs, r, gathered);
  else if (d == 2) k_align_candidates<2><<<grid, 128, 0, stream>>>(jobs, r, gathered);
  else return cudaErrorInvalidValue;
  return cudaGetLastError();
}

cudaError_t launch_robust_rotation_average(int d, int njobs, const AlignJob *jobs, const int *ready, double cbar,
                                           cudaStream_t stream) {
  if (njobs <= 0) return cudaSuccess;
  if (d == 3) k_robust_rotation_average<3><<<njobs, ALIGN_THREADS, 0, stream>>>(jobs, ready, cbar);
  else if (d == 2) k_robust_rotation_average<2><<<njobs, ALIGN_THREADS, 0, stream>>>(jobs, ready, cbar);
  else return cudaErrorInvalidValue;
  return cudaGetLastError();
}

cudaError_t launch_frame_lift(int d, int r, int njobs, int max_poses, const AlignJob *jobs, cudaStream_t stream) {
  if (njobs <= 0 || max_poses <= 0) return cudaSuccess;
  const int elems = max_poses * r * (d + 1);
  const dim3 grid((elems + 255) / 256, njobs);
  bool ok = false;
  DPGO_DISPATCH(r, d + 1, {
    k_apply_frame_lift<R, DH - 1><<<grid, 256, 0, stream>>>(jobs);
    ok = true;
  });
  if (!ok) return cudaErrorInvalidValue;
  return cudaGetLastError();
}

}  // namespace dpgo
