// dpgo_covariance.cu -- pose marginal covariances on the device: the Gauss-Newton information of a trajectory
// (k_assemble_pose_info), factored by the exact preconditioner's device refactorisation (nd_refactor.cu, shift 0), then
// selectively inverted over the same fronts, root stage first (k_nd_selinv_*).  The model is in dpgo_covariance.cuh.
//
// Per stage of the selected inversion, one CTA set per node of the stage (blockIdx.y / z):
//   k_nd_selinv_gather  the front gets W (own x own) and Fm^T (bnd x own) from the node's panels and Sigma_bb from the
//                       parent's front inverse, read through the parent positions of the boundary poses (the Schur
//                       scatter's map in reverse) and from the parent's upper triangle;
//   k_nd_selinv_gemm<0> Sigma_ob = -Fm Sigma_bb;
//   k_nd_selinv_gemm<1> Sigma_oo = W - Sigma_ob Fm^T, upper triangle tiles only;
//   k_nd_selinv_extract the requested 3 x 3 blocks of this stage's fronts.
// Every sum runs in a fixed order (fp64 FMA chains over k ascending), no atomics: two calls are bitwise equal.  Front
// inverses of stage st live where the refactorisation kept its fronts (arena halves by stage parity), so a node's parent
// front (stage st + 1) is intact while the node's is written.
#include <cuda_runtime.h>
#include "dpgo_covariance.cuh"
#include "dpgo_kernels.cuh"

namespace dpgo {

constexpr int COV_DH = 3;           // scalars per node of the embedded information matrix
constexpr int SEL_THREADS = 256;
constexpr int SEL_T = 64;           // output tile of the products
constexpr int SEL_K = 32;           // inner chunk staged in shared memory

template <int D>
__global__ void __launch_bounds__(256) k_assemble_pose_info(KPoseInfo k) {
  const int64_t tid = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (tid >= k.nb * 16) return;
  const int64_t b = tid >> 4;
  const int x = (int)((tid >> 2) & 3), y = (int)(tid & 3);
  if (x >= COV_DH || y >= COV_DH) { k.bval[tid] = 0.0; return; }
  const int2 bn = k.bnode[b];
  const int pa = D == 3 ? bn.x >> 1 : bn.x;
  const int qa = D == 3 ? 3 * (bn.x & 1) + x : x, qc = D == 3 ? 3 * (bn.y & 1) + y : y;
  if (pa == k.anchor) { k.bval[tid] = (bn.x == bn.y && x == y) ? 1.0 : 0.0; return; }
  double v = 0.0;
  for (int q = k.cptr[b]; q < k.cptr[b + 1]; ++q) {
    const int2 cc = k.contrib[q];
    const int e = cc.x;
    const double *Ri = k.T + (size_t)k.p1[e] * D * (D + 1), *Rj = k.T + (size_t)k.p2[e] * D * (D + 1);
    v += cov::edge_info<D>(cc.y & 1, qa, cc.y >> 1, qc, Ri, Rj, k.R + (size_t)e * D * D, k.t + (size_t)e * D, k.kappa[e], k.tau[e],
                           k.w ? k.w[e] : 1.0);
  }
  k.bval[tid] = v;
}

cudaError_t launch_assemble_pose_info(const KPoseInfo &k, cudaStream_t stream) {
  if (k.nb <= 0) return cudaSuccess;
  const unsigned g = (unsigned)((k.nb * 16 + 255) / 256);
  if (k.d == 3) k_assemble_pose_info<3><<<g, 256, 0, stream>>>(k);
  else k_assemble_pose_info<2><<<g, 256, 0, stream>>>(k);
  return cudaGetLastError();
}

// upper-triangle read of a front inverse
__device__ __forceinline__ double sym_at(const double *F, int64_t M, int64_t r, int64_t c) {
  return r <= c ? F[r + M * c] : F[c + M * r];
}

__global__ void __launch_bounds__(SEL_THREADS) k_nd_selinv_gather(KSelinv k, int n0) {
  const int q = n0 + blockIdx.y;
  const nd::RefactorNode rn = k.nodes[q];
  const int64_t s = (int64_t)COV_DH * rn.no, b = (int64_t)COV_DH * rn.nb, M = s + b;
  const int64_t e = (int64_t)blockIdx.x * SEL_THREADS + threadIdx.x;
  if (e >= M * M) return;
  const int64_t r = e % M, c = e / M;
  if (r < s && c >= s) return;                                   // Sigma_ob: written by the first product
  double *F = k.arena + rn.front;
  double v;
  if (c < s && r < s) {                                          // W (symmetrised panels)
    const int64_t fr = r / COV_DH;
    v = k.blob[rn.gf + (fr / 2) * nd::PANEL_ROWS * s + c * nd::PANEL_ROWS + (fr % 2) * COV_DH + r % COV_DH];
  } else if (c < s) {                                            // Fm^T[r - s][c] = Fm[c][r - s]
    const int64_t fc = c / COV_DH;
    v = k.blob[rn.gb + (fc / 2) * nd::PANEL_ROWS * b + (r - s) * nd::PANEL_ROWS + (fc % 2) * COV_DH + c % COV_DH];
  } else {                                                       // Sigma_bb from the parent's front inverse
    const nd::RefactorNode pn = k.nodes[k.parent[q]];
    const int *pm = k.pmap + k.pmap0[q];
    const int64_t rr = r - s, cc = c - s;
    v = sym_at(k.arena + pn.front, (int64_t)COV_DH * (pn.no + pn.nb), pm[rr / COV_DH] * COV_DH + rr % COV_DH,
               pm[cc / COV_DH] * COV_DH + cc % COV_DH);
  }
  F[r + M * c] = v;
}

// MODE 0: Sigma_ob[i][j] = -sum_k Fm[i][k] Sigma_bb[k][j]     (i < s, j < b)
// MODE 1: Sigma_oo[i][j] = W[i][j] - sum_k Sigma_ob[i][k] Fm[j][k]   (i <= j < s: tiles on or above the diagonal)
// Fm[i][k] sits transposed in the front's lower-left block: F[(s + k) + M i].
template <int MODE>
__global__ void __launch_bounds__(SEL_THREADS) k_nd_selinv_gemm(KSelinv k, int n0) {
  const nd::RefactorNode rn = k.nodes[n0 + blockIdx.z];
  const int64_t s = (int64_t)COV_DH * rn.no, b = (int64_t)COV_DH * rn.nb, M = s + b;
  const int64_t ncol = MODE == 0 ? b : s;
  const int64_t i0 = (int64_t)blockIdx.y * SEL_T, j0 = (int64_t)blockIdx.x * SEL_T;
  if (b == 0 || i0 >= s || j0 >= ncol) return;
  if (MODE == 1 && i0 > j0) return;
  double *F = k.arena + rn.front;
  __shared__ double sA[SEL_K][SEL_T + 1];     // sA[kk][i]
  __shared__ double sB[SEL_K][SEL_T + 1];     // sB[kk][j]
  const int t = threadIdx.x;
  const int ti = (t % 16) * 4, tj = (t / 16) * 4;
  double acc[4][4];
#pragma unroll
  for (int x = 0; x < 4; ++x)
#pragma unroll
    for (int y = 0; y < 4; ++y) acc[x][y] = 0.0;
  for (int64_t k0 = 0; k0 < b; k0 += SEL_K) {
    // consecutive threads read consecutive doubles: along k where the operand is stored k-contiguous (Fm^T, Sigma_bb),
    // along i for MODE 1's Sigma_ob (column-major, i-contiguous)
    for (int e = t; e < SEL_K * SEL_T; e += SEL_THREADS) {
      const int kk = MODE == 0 ? e % SEL_K : e / SEL_T, ii = MODE == 0 ? e / SEL_K : e % SEL_T;
      const int64_t kg = k0 + kk, i = i0 + ii;
      sA[kk][ii] = (kg < b && i < s) ? (MODE == 0 ? F[(s + kg) + M * i] : F[i + M * (s + kg)]) : 0.0;
    }
    for (int e = t; e < SEL_K * SEL_T; e += SEL_THREADS) {
      const int kk = e % SEL_K, jj = e / SEL_K;
      const int64_t kg = k0 + kk, j = j0 + jj;
      sB[kk][jj] = (kg < b && j < ncol) ? (MODE == 0 ? F[(s + kg) + M * (s + j)] : F[(s + kg) + M * j]) : 0.0;
    }
    __syncthreads();
#pragma unroll 8
    for (int kk = 0; kk < SEL_K; ++kk) {
      double a[4], bb[4];
#pragma unroll
      for (int x = 0; x < 4; ++x) { a[x] = sA[kk][ti + x]; bb[x] = sB[kk][tj + x]; }
#pragma unroll
      for (int x = 0; x < 4; ++x)
#pragma unroll
        for (int y = 0; y < 4; ++y) acc[x][y] = fma(a[x], bb[y], acc[x][y]);
    }
    __syncthreads();
  }
#pragma unroll
  for (int y = 0; y < 4; ++y) {
    const int64_t j = j0 + tj + y;
    if (j >= ncol) continue;
#pragma unroll
    for (int x = 0; x < 4; ++x) {
      const int64_t i = i0 + ti + x;
      if (i >= s) continue;
      if (MODE == 0) F[i + M * (s + j)] = -acc[x][y];
      else if (i <= j) F[i + M * j] -= acc[x][y];
    }
  }
}

__global__ void k_nd_selinv_extract(KSelinv k, int i0, int i1) {
  const int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= (int64_t)(i1 - i0) * 9) return;
  const CovItem it = k.items[i0 + e / 9];
  const int x = (int)(e % 9) / 3, y = (int)(e % 9) % 3;
  const nd::RefactorNode rn = k.nodes[it.node];
  k.out[it.out + (int64_t)x * k.ld + y] = sym_at(k.arena + rn.front, (int64_t)COV_DH * (rn.no + rn.nb), it.ra + x, it.rc + y);
}

cudaError_t launch_nd_selinv(const KSelinv &k, const nd::Refactor &R, const nd::Selinv &S, const std::vector<int> &item0,
                             cudaStream_t stream) {
  const int ns = (int)R.stage0.size() - 1;
  for (int st = ns - 1; st >= 0; --st) {
    const int n0 = R.stage0[(size_t)st], nn = R.stage0[(size_t)st + 1] - n0;
    if (nn <= 0 || R.max_nfr[(size_t)st] == 0) continue;     // no node of the stage holds a pose (an empty separator)
    const int64_t Mx = (int64_t)COV_DH * R.max_nfr[(size_t)st];
    const int64_t smax = R.max_s[(size_t)st], bmax = S.max_b[(size_t)st];
    const unsigned ts = (unsigned)((smax + SEL_T - 1) / SEL_T), tb = (unsigned)((bmax + SEL_T - 1) / SEL_T);
    // the nodes of one stage are independent: a stage of more than MAX_GRID_YZ nodes runs in consecutive slices
    for (int c0 = n0; c0 < n0 + nn; c0 += MAX_GRID_YZ) {
      const unsigned nc = (unsigned)(n0 + nn - c0 < MAX_GRID_YZ ? n0 + nn - c0 : MAX_GRID_YZ);
      k_nd_selinv_gather<<<dim3((unsigned)((Mx * Mx + SEL_THREADS - 1) / SEL_THREADS), nc), SEL_THREADS, 0, stream>>>(k, c0);
      if (bmax > 0) {
        k_nd_selinv_gemm<0><<<dim3(tb, ts, nc), SEL_THREADS, 0, stream>>>(k, c0);
        k_nd_selinv_gemm<1><<<dim3(ts, ts, nc), SEL_THREADS, 0, stream>>>(k, c0);
      }
    }
    const int a = item0[(size_t)st], z = item0[(size_t)st + 1];
    if (z > a) k_nd_selinv_extract<<<(unsigned)(((int64_t)(z - a) * 9 + 255) / 256), 256, 0, stream>>>(k, a, z);
  }
  return cudaGetLastError();
}

}  // namespace dpgo
