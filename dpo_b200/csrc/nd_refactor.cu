// nd_refactor.cu -- numeric refactorisation of the sparse exact preconditioner (Q + 0.1 I)^-1 on the device, for a Q whose
// block pattern is unchanged (a robust re-weighting): the multifrontal algorithm of nd::build_numeric over the macro nodes,
// stage by stage (deepest first), written into the panel blob in place.  ref: the CHOLMOD refactorisation in
// QuadraticProblem::setQ (src/QuadraticProblem.cpp:31-42) that PGOAgent::updateLoopClosuresWeights triggers through
// constructQMatrix / setQ (src/PGOAgent.cpp:653-667, 1109-1112).
//
// Per stage, three batched steps (one CTA set per node of the stage in blockIdx.y / z):
//   k_nd_front   every front entry gathers its value in a fixed order: the Q block (binary search in the block-CSR row),
//                the +shift of the own diagonal, then the children's Schur updates U_c in mn.children order -- the order
//                build_numeric adds them in, so the front is bitwise repeatable;
//   gj_sweep_batch (dense_inverse.cu) the blocked Gauss-Jordan sweep over the own pivots: W = Foo^-1, Fm = W Fob,
//                U = Fbb - Fob^T Fm in place (fp64; Foo is SPD so no pivoting; a non-positive pivot sets the fail flag);
//   k_nd_pack    [W ; Fm^T] and Fm into the 8-row panels, W symmetrised as host_factor does.
// U stays in the arena until the parent's stage; fronts of consecutive stages live in the two halves of the arena.
#include <cuda_runtime.h>
#include "dpgo_kernels.cuh"

namespace dpgo {

constexpr int REF_THREADS = 256;

__global__ void __launch_bounds__(REF_THREADS) k_nd_front(KRefactor k, int n0) {
  const nd::RefactorNode rn = k.nodes[n0 + blockIdx.y];
  const int nfr = rn.no + rn.nb, dh = k.dh;
  const int64_t e = (int64_t)blockIdx.x * REF_THREADS + threadIdx.x;
  if (e >= (int64_t)nfr * nfr) return;
  const int P = (int)(e % nfr), Qp = (int)(e / nfr);          // front block (P, Qp)
  double v[16];
#pragma unroll
  for (int q = 0; q < 16; ++q) v[q] = 0.0;
  if (P < rn.no || Qp < rn.no) {
    // bval[b][k][c] = Q[dh bcol[b] + k, dh j + c] for b in row j: the block of an own row j against the front pose i
    const bool own_row = P < rn.no;
    const int j = k.poses[rn.pose0 + (own_row ? P : Qp)], i = k.poses[rn.pose0 + (own_row ? Qp : P)];
    int lo = k.rowptr[j], hi = k.rowptr[j + 1];
    while (lo < hi) {
      const int mid = (lo + hi) >> 1;
      if (k.bcol[mid] < i) lo = mid + 1; else hi = mid;
    }
    if (lo < k.rowptr[j + 1] && k.bcol[lo] == i) {
      const double *blk = k.bval + (size_t)lo * 16;
#pragma unroll
      for (int a = 0; a < 4; ++a)
#pragma unroll
        for (int c = 0; c < 4; ++c) v[a * 4 + c] = own_row ? blk[c * 4 + a] : blk[a * 4 + c];   // padding entries are 0
    }
    if (P == Qp)
#pragma unroll
      for (int a = 0; a < 4; ++a) v[a * 4 + a] += k.shift;
  }
  for (int q = 0; q < rn.nch; ++q) {
    const nd::RefactorChild cr = k.child[rn.ch0 + q];
    const int a = k.cmap[cr.map0 + P], b = k.cmap[cr.map0 + Qp];
    if (a < 0 || b < 0) continue;
    const nd::RefactorNode cn = k.nodes[cr.node];
    const int64_t Mc = (int64_t)dh * (cn.no + cn.nb), sc = (int64_t)dh * cn.no;
    const double *U = k.arena + cn.front;
#pragma unroll
    for (int x = 0; x < 4; ++x)
#pragma unroll
      for (int y = 0; y < 4; ++y)
        if (x < dh && y < dh) v[x * 4 + y] += U[(sc + a * dh + x) + Mc * (sc + b * dh + y)];
  }
  double *F = k.arena + rn.front;
  const int64_t M = (int64_t)dh * nfr;
#pragma unroll
  for (int x = 0; x < 4; ++x)
#pragma unroll
    for (int y = 0; y < 4; ++y)
      if (x < dh && y < dh) F[(int64_t)(P * dh + x) + M * (Qp * dh + y)] = v[x * 4 + y];
}

// one thread per panel double of the node; rows a panel does not use (dh = 3, an odd last front pose) keep their zeros
__global__ void __launch_bounds__(REF_THREADS) k_nd_pack(KRefactor k, int n0) {
  const nd::RefactorNode rn = k.nodes[n0 + blockIdx.y];
  const int dh = k.dh, nfr = rn.no + rn.nb;
  const int64_t s = (int64_t)dh * rn.no, b = (int64_t)dh * rn.nb, M = s + b;
  const int64_t nf = (int64_t)((nfr + 1) / 2) * nd::PANEL_ROWS * s, nbk = (int64_t)((rn.no + 1) / 2) * nd::PANEL_ROWS * b;
  int64_t e = (int64_t)blockIdx.x * REF_THREADS + threadIdx.x;
  if (e >= nf + nbk) return;
  const double *F = k.arena + rn.front;
  const bool fwd = e < nf;
  if (!fwd) e -= nf;
  const int64_t cols = fwd ? s : b;
  const int64_t panel = e / (nd::PANEL_ROWS * cols), rem = e % (nd::PANEL_ROWS * cols);
  const int64_t j = rem / nd::PANEL_ROWS;
  const int prow = (int)(rem % nd::PANEL_ROWS), half = prow / dh, c = prow % dh;
  const int64_t fr = 2 * panel + half;
  if (half >= 2 || fr >= (fwd ? nfr : rn.no)) return;
  double val;
  if (!fwd) {
    val = F[(fr * dh + c) + M * (s + j)];                       // Fm row of an own scalar
  } else if (fr < rn.no) {
    const int64_t r = fr * dh + c;                              // W row, symmetrised
    val = (r == j) ? F[r + M * r] : 0.5 * (F[r + M * j] + F[j + M * r]);
  } else {
    val = F[j + M * (s + (fr - rn.no) * dh + c)];               // (F^T)[col][j] = Fm[j][col]
  }
  k.blob[(fwd ? rn.gf : rn.gb) + e] = val;
}

// (Q_jj + shift I)^-1 per pose: Gauss-Jordan on [A | I], exactly the host's jacobi_blocks
__global__ void k_jacobi_blocks(int n, int dh, const int *__restrict__ rowptr, const int *__restrict__ bcol,
                                const double *__restrict__ bval, double shift, double *__restrict__ dinv, int *fail) {
  const int j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= n) return;
  double A[4][8];
#pragma unroll
  for (int k = 0; k < 4; ++k)
#pragma unroll
    for (int c = 0; c < 8; ++c) A[k][c] = (c >= 4 && c - 4 == k) ? 1.0 : 0.0;
#pragma unroll
  for (int k = 0; k < 4; ++k) A[k][k] = (k < dh) ? shift : 1.0;
  for (int b = rowptr[j]; b < rowptr[j + 1]; ++b)
    if (bcol[b] == j)
#pragma unroll
      for (int k = 0; k < 4; ++k)
#pragma unroll
        for (int c = 0; c < 4; ++c)
          if (k < dh && c < dh) A[k][c] += bval[(size_t)b * 16 + k * 4 + c];
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    if (fail && !(A[k][k] > 0.0)) atomicExch(fail, 1);
    const double inv = 1.0 / A[k][k];
#pragma unroll
    for (int c = 0; c < 8; ++c) A[k][c] *= inv;
#pragma unroll
    for (int i = 0; i < 4; ++i)
      if (i != k) {
        const double f = A[i][k];
#pragma unroll
        for (int c = 0; c < 8; ++c) A[i][c] -= f * A[k][c];
      }
  }
#pragma unroll
  for (int k = 0; k < 4; ++k)
#pragma unroll
    for (int c = 0; c < 4; ++c) dinv[(size_t)j * 16 + k * 4 + c] = (k < dh && c < dh) ? A[k][4 + c] : 0.0;
}

cudaError_t launch_nd_refactor(const KRefactor &k, const nd::Refactor &R, cudaStream_t stream) {
  const int ns = (int)R.stage0.size() - 1;
  for (int st = 0; st < ns; ++st) {
    const int n0 = R.stage0[(size_t)st], nn = R.stage0[(size_t)st + 1] - n0;
    if (nn <= 0 || R.max_nfr[(size_t)st] == 0) continue;     // no node of the stage holds a pose: nothing to launch
    // the nodes of one stage are independent: a stage of more than MAX_GRID_YZ nodes runs in consecutive slices
    const int64_t fb = (int64_t)R.max_nfr[(size_t)st] * R.max_nfr[(size_t)st];
    for (int c0 = n0; c0 < n0 + nn; c0 += MAX_GRID_YZ) {
      const unsigned nc = (unsigned)(n0 + nn - c0 < MAX_GRID_YZ ? n0 + nn - c0 : MAX_GRID_YZ);
      k_nd_front<<<dim3((unsigned)((fb + REF_THREADS - 1) / REF_THREADS), nc), REF_THREADS, 0, stream>>>(k, c0);
    }
    const cudaError_t e = gj_sweep_batch(k.jobs + n0, nn, k.dh * R.max_nfr[(size_t)st], R.max_s[(size_t)st], k.fail, stream);
    if (e != cudaSuccess) return e;
    const int64_t pb = R.max_blob[(size_t)st];
    if (pb > 0)
      for (int c0 = n0; c0 < n0 + nn; c0 += MAX_GRID_YZ) {
        const unsigned nc = (unsigned)(n0 + nn - c0 < MAX_GRID_YZ ? n0 + nn - c0 : MAX_GRID_YZ);
        k_nd_pack<<<dim3((unsigned)((pb + REF_THREADS - 1) / REF_THREADS), nc), REF_THREADS, 0, stream>>>(k, c0);
      }
  }
  return cudaGetLastError();
}

cudaError_t launch_jacobi_blocks(int n, int dh, const int *rowptr, const int *bcol, const double *bval, double shift, double *dinv,
                                 int *fail, cudaStream_t stream) {
  if (n > 0) k_jacobi_blocks<<<(n + 127) / 128, 128, 0, stream>>>(n, dh, rowptr, bcol, bval, shift, dinv, fail);
  return cudaGetLastError();
}

}  // namespace dpgo
