// dpgo_chordal.cu -- chordal initialisation on the GPU (SURVEY 8f rank 3).
//
// ref: chordalInitialization / recoverTranslations, src/DPGO_utils.cpp:273-461 -- two sparse linear least-squares
// problems (SPQR there) with the gauge R_0 = I, t_0 = 0:
//   rotations     min sum_e kappa_e |R_j - R_i R_ij|_F^2  over free d x d matrices, then projection onto SO(d) (:463-477)
//   translations  min sum_e tau_e |t_j - t_i - R_i t_ij|^2
// Both normal matrices are connection Laplacians with 3x3 blocks (rotations: -kappa R_ij off the diagonal, kappa I on
// it; translations: the tau-weighted graph Laplacian times I_3), so both are solved by Jacobi-preconditioned conjugate
// gradients whose matrix-vector product is the hot path's own TMA-fed block-CSR kernel (k_spmv_tma, 3 x 3 blocks, r = 3
// rows = the 3 independent right-hand sides).  The CG scalars stay on the device; the host only looks at the residual
// every CHECK iterations.  d = 2 problems are embedded in 3 x 3 blocks (the extra coordinate decouples).
#include <cuda_runtime.h>

#include <algorithm>
#include <cmath>
#include <cstring>
#include <string>
#include <vector>

#include "../../include/dpgo_b200.h"
#include "dpgo_devbuf.cuh"
#include "dpgo_rotation.cuh"

namespace {

constexpr int B3 = 3;                 // block / tile edge of the container problem (d' = 2 -> dh = 3, r = 3)
constexpr int TS9 = 9;                // tile = 3 x 3 doubles, column-major: element (a, k) at k * 3 + a

// scalars on the device: [0] rz, [1] pq, [2] rz_new, [3] rz0
__global__ void k_dot(int len, const double *__restrict__ a, const double *__restrict__ b, double *out) {
  __shared__ double sm[32];
  double s = 0.0;
  for (int i = threadIdx.x; i < len; i += blockDim.x) s = fma(a[i], b[i], s);
  for (int m = 16; m > 0; m >>= 1) s += __shfl_xor_sync(0xffffffffu, s, m);
  if ((threadIdx.x & 31) == 0) sm[threadIdx.x >> 5] = s;
  __syncthreads();
  if (threadIdx.x < 32) {
    double t = (threadIdx.x < (blockDim.x >> 5)) ? sm[threadIdx.x] : 0.0;
    for (int m = 16; m > 0; m >>= 1) t += __shfl_xor_sync(0xffffffffu, t, m);
    if (threadIdx.x == 0) *out = t;
  }
}
// q <- q with the anchored tile zeroed (the product was taken with the full matrix)
__global__ void k_mask_anchor(double *q) {
  if (threadIdx.x < TS9) q[threadIdx.x] = 0.0;
}
// x += alpha p; r -= alpha q; z = r / diag      (alpha = rz / pq, 0 unless pq > 0)
// Between two host checks the loop keeps iterating after convergence; once rz reaches exactly 0, p = 0 and pq = 0, and
// alpha = 0 / 0 would put NaN into x.  alpha = 0 (and beta = 0 below) make a converged solve a fixed point instead.
__global__ void k_update_xrz(int len, const double *__restrict__ sc, const double *__restrict__ p, const double *__restrict__ q,
                             const double *__restrict__ dinv, double *x, double *r, double *z) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= len) return;
  const double alpha = (sc[1] > 0.0) ? sc[0] / sc[1] : 0.0;
  x[i] = fma(alpha, p[i], x[i]);
  const double rr = fma(-alpha, q[i], r[i]);
  r[i] = rr;
  z[i] = rr * dinv[i / 3];            // element (a, k) of tile t sits at 9 t + 3 k + a: column index = i / 3
}
// p = z + beta p  (beta = rz_new / rz, 0 unless rz > 0)
__global__ void k_update_p(int len, double *sc, const double *__restrict__ z, double *p) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  const double beta = (sc[0] > 0.0) ? sc[2] / sc[0] : 0.0;
  if (i < len) p[i] = fma(beta, p[i], z[i]);
}
__global__ void k_rotate_scalars(double *sc) { sc[0] = sc[2]; }
__global__ void k_scale_neg_mask(int len, const double *__restrict__ y, double *b) {   // b = -y, anchored tile zero
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < len) b[i] = (i < TS9) ? 0.0 : -y[i];
}
__global__ void k_jacobi(int len, const double *__restrict__ r, const double *__restrict__ dinv, double *z, double *p) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < len) { const double v = r[i] * dinv[i / 3]; z[i] = v; p[i] = v; }
}

// projection of the leading D x D part of every 3 x 3 tile onto SO(D) (dpgo::project_to_rotation)
template <int D> __global__ void k_project_rotations(int n, const double *__restrict__ tiles, double *__restrict__ out) {
  const int j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= n) return;
  double M[D][D], Rm[D][D];
  for (int c = 0; c < D; ++c)
    for (int a = 0; a < D; ++a) M[a][c] = tiles[(size_t)j * TS9 + c * B3 + a];
  dpgo::project_to_rotation<D>(M, Rm);
  for (int c = 0; c < D; ++c)
    for (int a = 0; a < D; ++a) out[(size_t)j * TS9 + c * B3 + a] = Rm[a][c];
}

struct ProblemGuard {
  dpgo_problem_t *h = nullptr;
  ~ProblemGuard() { if (h) dpgo_problem_destroy(h); }
};

#define CH_CUDA(call)                                                                       \
  do {                                                                                      \
    cudaError_t _e = (call);                                                                \
    if (_e != cudaSuccess) { err = std::string(#call) + ": " + cudaGetErrorString(_e); return DPGO_ERR_CUDA; } \
  } while (0)
#define CH_TRY(call)                                                      \
  do {                                                                    \
    int _s = (call);                                                      \
    if (_s != DPGO_OK) { err = std::string(#call) + ": " + dpgo_last_error(); return _s; } \
  } while (0)

// Solve X Q = B on the free tiles (tile 0 anchored to zero in X) by Jacobi-preconditioned CG; B comes in `b` (anchored tile
// already zero), the solution is left in `x`.  Everything runs on `st` (also the problem's stream).  Stops when
// rz = r D^-1 r^T <= tol^2 rz0; DPGO_ERR_CUDA when rz turns NaN or max_iter iterations do not get there.
int pcg(dpgo_problem_t *h, int n, const double *diag_host, double *x, const double *b, double tol, int max_iter, int *iters,
        cudaStream_t st, std::string &err) {
  const int len = TS9 * n;
  dpgo::DevBuf<double> r, z, p, q, dinv, sc;
  CH_CUDA(r.alloc(len)); CH_CUDA(z.alloc(len)); CH_CUDA(p.alloc(len)); CH_CUDA(q.alloc(len)); CH_CUDA(dinv.alloc(3 * (size_t)n)); CH_CUDA(sc.alloc(8));
  std::vector<double> dh((size_t)3 * n);
  for (int i = 0; i < 3 * n; ++i) dh[(size_t)i] = (diag_host[i] > 0.0) ? 1.0 / diag_host[i] : 0.0;
  for (int k = 0; k < 3; ++k) dh[(size_t)k] = 0.0;                         // anchored tile
  CH_CUDA(cudaMemcpyAsync(dinv.get(), dh.data(), sizeof(double) * dh.size(), cudaMemcpyHostToDevice, st));
  CH_CUDA(cudaMemsetAsync(x, 0, sizeof(double) * len, st));
  CH_CUDA(cudaMemcpyAsync(r.get(), b, sizeof(double) * len, cudaMemcpyDeviceToDevice, st));
  const int TB = 256, GB = (len + TB - 1) / TB;
  k_jacobi<<<GB, TB, 0, st>>>(len, r.get(), dinv.get(), z.get(), p.get());
  k_dot<<<1, 1024, 0, st>>>(len, r.get(), z.get(), sc.get() + 0);
  double rz0 = 0.0;
  CH_CUDA(cudaMemcpyAsync(&rz0, sc.get(), sizeof(double), cudaMemcpyDeviceToHost, st));
  CH_CUDA(cudaStreamSynchronize(st));
  *iters = 0;
  if (!(rz0 > 0.0)) return DPGO_OK;
  const int CHECK = 25;
  bool converged = false;
  for (int it = 0; it < max_iter; ++it) {
    CH_TRY(dpgo_spmv_device(h, p.get(), q.get(), 0));                           // q = p Q  (k_spmv_tma)
    k_mask_anchor<<<1, 32, 0, st>>>(q.get());
    k_dot<<<1, 1024, 0, st>>>(len, p.get(), q.get(), sc.get() + 1);
    k_update_xrz<<<GB, TB, 0, st>>>(len, sc.get(), p.get(), q.get(), dinv.get(), x, r.get(), z.get());
    k_dot<<<1, 1024, 0, st>>>(len, r.get(), z.get(), sc.get() + 2);
    k_update_p<<<GB, TB, 0, st>>>(len, sc.get(), z.get(), p.get());
    k_rotate_scalars<<<1, 1, 0, st>>>(sc.get());
    *iters = it + 1;
    if ((it + 1) % CHECK == 0) {
      double rz = 0.0;
      CH_CUDA(cudaMemcpyAsync(&rz, sc.get(), sizeof(double), cudaMemcpyDeviceToHost, st));
      CH_CUDA(cudaStreamSynchronize(st));
      if (!(rz == rz)) { err = "chordal initialisation: conjugate gradients broke down"; return DPGO_ERR_CUDA; }
      if (rz <= tol * tol * rz0) { converged = true; break; }
    }
  }
  if (!converged) {                                  // the last check was not on convergence (or max_iter % CHECK != 0)
    double rz = 0.0;
    CH_CUDA(cudaMemcpyAsync(&rz, sc.get(), sizeof(double), cudaMemcpyDeviceToHost, st));
    CH_CUDA(cudaStreamSynchronize(st));
    if (!(rz == rz)) { err = "chordal initialisation: conjugate gradients broke down"; return DPGO_ERR_CUDA; }
    if (rz > tol * tol * rz0) {
      err = "chordal initialisation: conjugate gradients did not reach tol in max_iter iterations (" + std::to_string(max_iter) + ")";
      return DPGO_ERR_CUDA;
    }
  }
  CH_CUDA(cudaStreamSynchronize(st));
  return DPGO_OK;
}

thread_local std::string g_chordal_error;

}  // namespace

extern "C" {

const char *dpgo_chordal_last_error(void) { return g_chordal_error.c_str(); }

int dpgo_chordal_initialization(int n, int d, int64_t m, const int32_t *p1, const int32_t *p2, const double *R, const double *t,
                                const double *kappa, const double *tau, int device, double tol, int max_iter, double *T_host,
                                int32_t *iterations2) {
  std::string &err = g_chordal_error;
  err.clear();
  if (n < 1 || (d != 2 && d != 3) || m < 0 || !T_host || (m > 0 && (!p1 || !p2 || !R || !t || !kappa || !tau))) {
    err = "bad arguments";
    return DPGO_ERR_INVALID_ARG;
  }
  if (tol <= 0) tol = 1e-11;
  if (max_iter <= 0) max_iter = 50000;
  const int dh = d + 1;
  if (iterations2) iterations2[0] = iterations2[1] = 0;
  if (n == 1) {
    std::fill(T_host, T_host + (size_t)d * dh, 0.0);
    for (int k = 0; k < d; ++k) T_host[(size_t)k * d + k] = 1.0;
    return DPGO_OK;
  }
  for (int64_t e = 0; e < m; ++e)
    if (p1[e] < 0 || p1[e] >= n || p2[e] < 0 || p2[e] >= n) { err = "edge endpoint out of range"; return DPGO_ERR_INVALID_ARG; }
  CH_CUDA(cudaSetDevice(device));
  const int len = TS9 * n;
  // ---- rotation Laplacian: Q_ii += k I, Q_jj += k I, Q_ij = -k Rt, Q_ji = -k Rt^T  (Rt = R_ij embedded in 3 x 3) ----
  std::vector<int32_t> brow, bcol;
  std::vector<double> blocks, diag((size_t)3 * n, 0.0);
  brow.reserve((size_t)4 * m); bcol.reserve((size_t)4 * m); blocks.reserve((size_t)36 * m);
  auto push = [&](int i, int j, const double *b9) { brow.push_back(i); bcol.push_back(j); blocks.insert(blocks.end(), b9, b9 + 9); };
  for (int64_t e = 0; e < m; ++e) {
    const int i = p1[e], j = p2[e];
    const double k = kappa[e];
    double Rt[9] = {0, 0, 0, 0, 0, 0, 0, 0, 0}, RtT[9], kI[9] = {k, 0, 0, 0, k, 0, 0, 0, k}, kAAt[9] = {0, 0, 0, 0, 0, 0, 0, 0, 0};
    const double *Re = R + (size_t)e * d * d;
    for (int a = 0; a < d; ++a)
      for (int b = 0; b < d; ++b) Rt[a * 3 + b] = -k * Re[a * d + b];
    for (int a = d; a < 3; ++a) Rt[a * 3 + a] = -k;
    for (int a = 0; a < 3; ++a)
      for (int b = 0; b < 3; ++b) RtT[a * 3 + b] = Rt[b * 3 + a];
    // the measured R_ij need not be exactly orthogonal (unnormalised quaternions): the i-block is kappa R_ij R_ij^T (ref :327-331)
    for (int a = 0; a < d; ++a)
      for (int b = 0; b < d; ++b) {
        double s2 = 0.0;
        for (int c = 0; c < d; ++c) s2 += Re[a * d + c] * Re[b * d + c];
        kAAt[a * 3 + b] = k * s2;
      }
    for (int a = d; a < 3; ++a) kAAt[a * 3 + a] = k;
    push(i, i, kAAt); push(j, j, kI); push(i, j, Rt); push(j, i, RtT);
    for (int c = 0; c < 3; ++c) { diag[(size_t)3 * i + c] += kAAt[c * 3 + c]; diag[(size_t)3 * j + c] += k; }
  }
  cudaStream_t st = nullptr;
  CH_CUDA(cudaStreamCreateWithFlags(&st, cudaStreamNonBlocking));
  const dpgo::Stream own(st);
  dpgo::DevBuf<double> x, b, y;
  CH_CUDA(x.alloc(len)); CH_CUDA(b.alloc(len)); CH_CUDA(y.alloc(len));
  std::vector<double> tiles((size_t)len);                   // projected rotations, 3 x 3 tiles (column-major)
  {
    ProblemGuard pr;
    CH_TRY(dpgo_problem_create(n, 2, 3, device, &pr.h));
    CH_TRY(dpgo_problem_set_stream(pr.h, (void *)st));
    CH_TRY(dpgo_problem_set_Q_blocks(pr.h, (int64_t)brow.size(), brow.data(), bcol.data(), blocks.data(), 0u));
    // right-hand side: X0 = [I, 0, ...];  b = -(X0 Q) on the free tiles
    std::vector<double> x0((size_t)len, 0.0);
    for (int k = 0; k < 3; ++k) x0[(size_t)k * 3 + k] = 1.0;
    CH_CUDA(cudaMemcpyAsync(y.get(), x0.data(), sizeof(double) * len, cudaMemcpyHostToDevice, st));
    CH_TRY(dpgo_spmv_device(pr.h, y.get(), x.get(), 0));
    k_scale_neg_mask<<<(len + 255) / 256, 256, 0, st>>>(len, x.get(), b.get());
    int it = 0;
    const int rc = pcg(pr.h, n, diag.data(), x.get(), b.get(), tol, max_iter, &it, st, err);
    if (rc != DPGO_OK) return rc;
    if (iterations2) iterations2[0] = it;
    // anchored tile = identity, then the projection onto SO(d) (pose 0 stays I)
    CH_CUDA(cudaMemcpyAsync(x.get(), x0.data(), sizeof(double) * TS9, cudaMemcpyHostToDevice, st));
    if (d == 3) k_project_rotations<3><<<(n + 127) / 128, 128, 0, st>>>(n, x.get(), y.get());
    else k_project_rotations<2><<<(n + 127) / 128, 128, 0, st>>>(n, x.get(), y.get());
    CH_CUDA(cudaMemcpyAsync(tiles.data(), y.get(), sizeof(double) * len, cudaMemcpyDeviceToHost, st));
    CH_CUDA(cudaStreamSynchronize(st));
  }
  // ---- translations: tau-weighted graph Laplacian (x I_3), right-hand side from the rotations:  gradient of
  //      sum tau |t_j - t_i - R_i t_ij|^2  ->  (T L)_j += tau v, (T L)_i -= tau v  with v = R_i t_ij; row 0 of the 3-row
  //      container carries t^T (poses x 3 coordinates), rows 1, 2 stay zero ----
  brow.clear(); bcol.clear(); blocks.clear();
  std::fill(diag.begin(), diag.end(), 0.0);
  std::vector<double> rhs((size_t)len, 0.0);
  for (int64_t e = 0; e < m; ++e) {
    const int i = p1[e], j = p2[e];
    const double w = tau[e];
    const double wI[9] = {w, 0, 0, 0, w, 0, 0, 0, w}, mI[9] = {-w, 0, 0, 0, -w, 0, 0, 0, -w};
    push(i, i, wI); push(j, j, wI); push(i, j, mI); push(j, i, mI);
    for (int c = 0; c < 3; ++c) { diag[(size_t)3 * i + c] += w; diag[(size_t)3 * j + c] += w; }
    for (int a = 0; a < d; ++a) {
      double v = 0.0;
      for (int c = 0; c < d; ++c) v += tiles[(size_t)i * TS9 + c * 3 + a] * t[(size_t)e * d + c];     // (R_i t_ij)[a]
      rhs[(size_t)j * TS9 + a * 3 + 0] += w * v;            // row 0, column a of tile j
      rhs[(size_t)i * TS9 + a * 3 + 0] -= w * v;
    }
  }
  for (int q = 0; q < TS9; ++q) rhs[(size_t)q] = 0.0;       // t_0 = 0
  std::vector<double> tsol((size_t)len, 0.0);
  {
    ProblemGuard pr;
    CH_TRY(dpgo_problem_create(n, 2, 3, device, &pr.h));
    CH_TRY(dpgo_problem_set_stream(pr.h, (void *)st));
    CH_TRY(dpgo_problem_set_Q_blocks(pr.h, (int64_t)brow.size(), brow.data(), bcol.data(), blocks.data(), 0u));
    CH_CUDA(cudaMemcpyAsync(b.get(), rhs.data(), sizeof(double) * len, cudaMemcpyHostToDevice, st));
    int it = 0;
    const int rc = pcg(pr.h, n, diag.data(), x.get(), b.get(), tol, max_iter, &it, st, err);
    if (rc != DPGO_OK) return rc;
    if (iterations2) iterations2[1] = it;
    CH_CUDA(cudaMemcpyAsync(tsol.data(), x.get(), sizeof(double) * len, cudaMemcpyDeviceToHost, st));
    CH_CUDA(cudaStreamSynchronize(st));
  }
  // ---- T = [R_0 t_0 | R_1 t_1 | ...], d x (d+1) n column-major ----
  for (int p = 0; p < n; ++p) {
    double *Tp = T_host + (size_t)p * dh * d;
    for (int c = 0; c < d; ++c)
      for (int a = 0; a < d; ++a) Tp[(size_t)c * d + a] = tiles[(size_t)p * TS9 + c * 3 + a];
    for (int a = 0; a < d; ++a) Tp[(size_t)d * d + a] = tsol[(size_t)p * TS9 + a * 3 + 0];
  }
  return DPGO_OK;
}

}  // extern "C"
