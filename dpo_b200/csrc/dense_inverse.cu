// dense_inverse.cu -- blocked Gauss-Jordan sweeps of dense SPD matrices in HBM (fp64).
//
// Used by the device refactorisation of the exact preconditioners (nd_refactor.cu) for the fronts of their
// macro nodes: the reference obtains (Q + 0.1 I)^-1 through a CHOLMOD factorisation (ref:
// src/QuadraticProblem.cpp:31-42).
// SPD input, so no pivoting is needed.  Per block step kb (block size B) over the pivots [0, s) of an
// M x M matrix:
//   Pinv = inv(A_kk);  Rw = Pinv * A_k,:  ;  C = A_:,k
//   A_ij -= C_i Rw_j (i,j != k);  A_ik = -C_i Pinv;  A_kj = Rw_j;  A_kk = Pinv
// After all steps, with S = [0, s) and T = [s, M):  A_SS = A_SS^-1, A_ST = A_SS^-1 A_ST, A_TS = -A_TS A_SS^-1 and
// A_TT = A_TT - A_TS A_SS^-1 A_ST (s = M: the inverse).  2 s M^2 flops in s/B rank-B updates; each update streams A once
// (M^2 * 16 B of traffic).  A batch sweeps one matrix per blockIdx (z for the update, y otherwise).
#include <cuda_runtime.h>
#include "dpgo_kernels.cuh"

namespace dpgo {

constexpr int GJB = 32;     // pivot block
constexpr int GJT = 64;     // update tile
static_assert(GJB == nd::REFACTOR_PIVOT_BLOCK, "the refactorisation sizes its workspaces by the pivot block");

__device__ __forceinline__ GjJob gj_job(const GjJob &one, const GjJob *jobs, int z) { return jobs ? jobs[z] : one; }

// invert the bs x bs pivot block (identity padded to GJB) -- one CTA of GJB x GJB threads per matrix.  A pivot that is not
// positive (the matrix is not SPD) sets *fail (when given) and the sweep goes on with garbage, never a trap.
__global__ void k_gj_pivot(GjJob one, const GjJob *jobs, int k0, int *fail) {
  const GjJob J = gj_job(one, jobs, blockIdx.y);
  if (k0 >= J.s) return;
  const int bs = (J.s - k0 < GJB) ? (J.s - k0) : GJB;
  const double *A = J.A;
  const int N = J.M;
  __shared__ double P[GJB][GJB + 1];
  const int i = threadIdx.y, j = threadIdx.x;
  double v = (i == j) ? 1.0 : 0.0;
  if (i < bs && j < bs) v = A[(size_t)(k0 + i) + (size_t)N * (k0 + j)];
  P[i][j] = v;
  __syncthreads();
  for (int k = 0; k < GJB; ++k) {
    const double pkk = P[k][k];
    const double pik = P[i][k], pkj = P[k][j];
    __syncthreads();
    if (fail && i == k && j == k && !(pkk > 0.0)) atomicExch(fail, 1);
    const double inv = 1.0 / pkk;
    double nv;
    if (i == k && j == k) nv = inv;
    else if (i == k) nv = pkj * inv;
    else if (j == k) nv = -pik * inv;
    else nv = P[i][j] - pik * pkj * inv;
    P[i][j] = nv;
    __syncthreads();
  }
  J.piv[i + GJB * j] = P[i][j];
}

// Rw[q, j] = sum_p Pinv[q,p] A[k0+p, j]  (GJB x M, stored q + GJB*j);  C[i, q] = A[i, k0+q] (i + M*q)
__global__ void k_gj_panels(GjJob one, const GjJob *jobs, int k0) {
  const GjJob J = gj_job(one, jobs, blockIdx.y);
  if (k0 >= J.s) return;
  const int bs = (J.s - k0 < GJB) ? (J.s - k0) : GJB;
  const double *A = J.A;
  const int N = J.M;
  __shared__ double P[GJB][GJB + 1];
  const int t = threadIdx.x;                 // 256 threads
  if (blockIdx.x * blockDim.x >= (unsigned)N) return;
  for (int e = t; e < GJB * GJB; e += blockDim.x) P[e % GJB][e / GJB] = J.piv[e];
  __syncthreads();
  const int j = blockIdx.x * blockDim.x + t;
  if (j < N) {
    double a[GJB];
#pragma unroll
    for (int p = 0; p < GJB; ++p) a[p] = (p < bs) ? A[(size_t)(k0 + p) + (size_t)N * j] : 0.0;
#pragma unroll 4
    for (int q = 0; q < GJB; ++q) {
      double s = 0.0;
#pragma unroll
      for (int p = 0; p < GJB; ++p) s = fma(P[q][p], a[p], s);
      J.Rw[q + (size_t)GJB * j] = s;
    }
    // column panel: A symmetric at every step?  No -- Gauss-Jordan intermediates are not symmetric,
    // so read the true column entries.
    for (int q = 0; q < GJB; ++q) J.C[(size_t)j + (size_t)N * q] = (q < bs) ? A[(size_t)j + (size_t)N * (k0 + q)] : 0.0;
  }
}

// rank-GJB update of one GJT x GJT tile
__global__ void __launch_bounds__(256) k_gj_update(GjJob one, const GjJob *jobs, int k0) {
  const GjJob J = gj_job(one, jobs, blockIdx.z);
  if (k0 >= J.s) return;
  const int bs = (J.s - k0 < GJB) ? (J.s - k0) : GJB;
  double *__restrict__ A = J.A;
  const double *__restrict__ piv = J.piv;
  const double *__restrict__ Rw = J.Rw;
  const double *__restrict__ C = J.C;
  const int N = J.M;
  const int i0 = blockIdx.y * GJT, j0 = blockIdx.x * GJT;
  if (i0 >= N || j0 >= N) return;
  __shared__ double sC[GJB][GJT + 1];   // sC[q][i]
  __shared__ double sR[GJB][GJT + 1];   // sR[q][j]
  const int t = threadIdx.x;
  for (int e = t; e < GJB * GJT; e += 256) {
    const int q = e / GJT, ii = e % GJT;
    sC[q][ii] = (i0 + ii < N) ? C[(size_t)(i0 + ii) + (size_t)N * q] : 0.0;
  }
  for (int e = t; e < GJB * GJT; e += 256) {
    const int jj = e / GJB, q = e % GJB;
    sR[q][jj] = (j0 + jj < N) ? Rw[q + (size_t)GJB * (j0 + jj)] : 0.0;
  }
  __syncthreads();
  const int ti = (t % 16) * 4, tj = (t / 16) * 4;
  double acc[4][4];
#pragma unroll
  for (int x = 0; x < 4; ++x)
#pragma unroll
    for (int y = 0; y < 4; ++y) acc[x][y] = 0.0;
#pragma unroll 8
  for (int q = 0; q < GJB; ++q) {
    double c[4], r[4];
#pragma unroll
    for (int x = 0; x < 4; ++x) { c[x] = sC[q][ti + x]; r[x] = sR[q][tj + x]; }
#pragma unroll
    for (int x = 0; x < 4; ++x)
#pragma unroll
      for (int y = 0; y < 4; ++y) acc[x][y] = fma(c[x], r[y], acc[x][y]);
  }
#pragma unroll
  for (int y = 0; y < 4; ++y) {
    const int j = j0 + tj + y;
    if (j >= N) continue;
    const bool jin = (j >= k0 && j < k0 + bs);
#pragma unroll
    for (int x = 0; x < 4; ++x) {
      const int i = i0 + ti + x;
      if (i >= N) continue;
      const bool iin = (i >= k0 && i < k0 + bs);
      double *p = A + (size_t)i + (size_t)N * j;
      if (!iin && !jin) {
        *p = *p - acc[x][y];
      } else if (iin && !jin) {
        *p = sR[i - k0][tj + y];
      } else if (!iin && jin) {
        // -C_i * Pinv[:, j-k0]
        double s = 0.0;
        for (int q = 0; q < bs; ++q) s = fma(sC[q][ti + x], piv[q + GJB * (j - k0)], s);
        *p = -s;
      } else {
        *p = piv[(i - k0) + GJB * (j - k0)];
      }
    }
  }
}

cudaError_t gj_sweep_batch(const GjJob *jobs_dev, int njobs, int max_M, int max_s, int *fail, cudaStream_t stream) {
  if (njobs <= 0 || max_s <= 0) return cudaSuccess;
  const GjJob none = {};
  const int tiles = (max_M + GJT - 1) / GJT;
  for (int j0 = 0; j0 < njobs; j0 += MAX_GRID_YZ) {          // the jobs are independent: slices run one after another
    const GjJob *jobs = jobs_dev + j0;
    const unsigned nj = (unsigned)(njobs - j0 < MAX_GRID_YZ ? njobs - j0 : MAX_GRID_YZ);
    for (int k0 = 0; k0 < max_s; k0 += GJB) {
      k_gj_pivot<<<dim3(1, nj), dim3(GJB, GJB), 0, stream>>>(none, jobs, k0, fail);
      k_gj_panels<<<dim3((max_M + 255) / 256, nj), 256, 0, stream>>>(none, jobs, k0);
      k_gj_update<<<dim3(tiles, tiles, nj), 256, 0, stream>>>(none, jobs, k0);
    }
  }
  return cudaGetLastError();
}

}  // namespace dpgo
