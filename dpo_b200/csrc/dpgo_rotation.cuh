// dpgo_rotation.cuh -- per-thread SO(d) projection and GNC-TLS weight, shared by the chordal initialisation
// (dpgo_chordal.cu), the robust re-weighting of private edges (dpgo_kernels.cu) and the frame alignment of the distributed
// initialisation (dpgo_align.cu).
#pragma once
#include <cuda_runtime.h>

namespace dpgo {

// Projection of a D x D matrix onto SO(D), M[a][c] = M(a, c): one-sided (Hestenes) Jacobi SVD, U V^T, and a sign flip of the
// direction of the smallest singular value when det < 0 (ref projectToRotationGroup, src/DPGO_utils.cpp:463-477).
template <int D> __device__ __forceinline__ void project_to_rotation(const double (&M)[D][D], double (&Rm)[D][D]) {
  double y[D][D], V[D][D];               // y[c] = column c of M (rows a), V[c] = column c of V
  for (int c = 0; c < D; ++c)
    for (int a = 0; a < D; ++a) { y[c][a] = M[a][c]; V[c][a] = (c == a) ? 1.0 : 0.0; }
  for (int sweep = 0; sweep < 40; ++sweep) {
    bool rotated = false;
    for (int p = 0; p < D; ++p)
      for (int q = p + 1; q < D; ++q) {
        double al = 0, be = 0, ga = 0;
        for (int a = 0; a < D; ++a) { al = fma(y[p][a], y[p][a], al); be = fma(y[q][a], y[q][a], be); ga = fma(y[p][a], y[q][a], ga); }
        if (ga == 0.0 || fabs(ga) <= 1e-17 * sqrt(al * be)) continue;
        rotated = true;
        const double zeta = (be - al) / (2.0 * ga);
        const double tt = (zeta >= 0 ? 1.0 : -1.0) / (fabs(zeta) + sqrt(1.0 + zeta * zeta));
        const double cs = 1.0 / sqrt(1.0 + tt * tt), sn = cs * tt;
        for (int a = 0; a < D; ++a) {
          const double yp = y[p][a], yq = y[q][a];
          y[p][a] = cs * yp - sn * yq; y[q][a] = sn * yp + cs * yq;
          const double vp = V[p][a], vq = V[q][a];
          V[p][a] = cs * vp - sn * vq; V[q][a] = sn * vp + cs * vq;
        }
      }
    if (!rotated) break;
  }
  double sig[D];
  int imin = 0;
  for (int c = 0; c < D; ++c) {
    double s = 0;
    for (int a = 0; a < D; ++a) s = fma(y[c][a], y[c][a], s);
    sig[c] = sqrt(s);
    const double inv = (s > 0.0) ? 1.0 / sig[c] : 0.0;
    for (int a = 0; a < D; ++a) y[c][a] *= inv;        // U columns
    if (sig[c] < sig[imin]) imin = c;
  }
  // R = U V^T : R[a][c] = sum_k U[a,k] V[c,k] = sum_k y[k][a] V[k][c]
  for (int a = 0; a < D; ++a)
    for (int c = 0; c < D; ++c) { double s = 0; for (int k = 0; k < D; ++k) s = fma(y[k][a], V[k][c], s); Rm[a][c] = s; }
  double det;
  if (D == 2) det = Rm[0][0] * Rm[1][1] - Rm[0][1] * Rm[1][0];
  else det = Rm[0][0] * (Rm[1][1] * Rm[2 % D][2 % D] - Rm[1][2 % D] * Rm[2 % D][1]) - Rm[0][1] * (Rm[1][0] * Rm[2 % D][2 % D] - Rm[1][2 % D] * Rm[2 % D][0]) +
             Rm[0][2 % D] * (Rm[1][0] * Rm[2 % D][1] - Rm[1][1] * Rm[2 % D][0]);
  if (det < 0.0)                          // flip the left singular vector of the smallest singular value
    for (int a = 0; a < D; ++a)
      for (int c = 0; c < D; ++c) Rm[a][c] -= 2.0 * y[imin][a] * V[imin][c];
}

// Stiefel (polar-factor) projection of one pose tile, ref: LiftedSEManifold::project, src/manifold/LiftedSEManifold.cpp:34-45 +
// projectToStiefelManifold, src/DPGO_utils.cpp:479-485 (U V^T of the thin SVD = polar factor): one-sided (Hestenes) Jacobi
// SVD of the r x d block -- columns are rotated until mutually orthogonal (Y V = U Sigma), which keeps high relative accuracy
// for ill-conditioned blocks -- then U V^T; the translation column passes through.  in(e) gives element e = c R + a of the
// input tile, out(e, v) stores element e of the result.  Every rotation element is read before the first store and the
// translation is read after the rotation stores, so `out` may write the buffer `in` reads.
template <int R, int DH, class In, class Out> __device__ __forceinline__ void stiefel_project_tile(const In &in, const Out &out) {
  constexpr int D = DH - 1;
  double y[D][R];
  double V[D][D];
#pragma unroll
  for (int c = 0; c < D; ++c) {
#pragma unroll
    for (int a = 0; a < R; ++a) y[c][a] = in(c * R + a);
#pragma unroll
    for (int q = 0; q < D; ++q) V[c][q] = (c == q) ? 1.0 : 0.0;     // V[c] = column c of V
  }
  for (int sweep = 0; sweep < 30; ++sweep) {
    bool rotated = false;
#pragma unroll
    for (int p = 0; p < D; ++p)
#pragma unroll
      for (int q = p + 1; q < D; ++q) {
        double alpha = 0, beta = 0, gamma = 0;
#pragma unroll
        for (int a = 0; a < R; ++a) {
          alpha = fma(y[p][a], y[p][a], alpha);
          beta = fma(y[q][a], y[q][a], beta);
          gamma = fma(y[p][a], y[q][a], gamma);
        }
        if (fabs(gamma) <= 1e-17 * sqrt(alpha * beta) || gamma == 0.0) continue;
        rotated = true;
        const double zeta = (beta - alpha) / (2.0 * gamma);
        const double t = (zeta >= 0 ? 1.0 : -1.0) / (fabs(zeta) + sqrt(1.0 + zeta * zeta));
        const double cs = 1.0 / sqrt(1.0 + t * t), sn = cs * t;
#pragma unroll
        for (int a = 0; a < R; ++a) {
          const double yp = y[p][a], yq = y[q][a];
          y[p][a] = cs * yp - sn * yq;
          y[q][a] = sn * yp + cs * yq;
        }
#pragma unroll
        for (int k = 0; k < D; ++k) {
          const double vp = V[p][k], vq = V[q][k];
          V[p][k] = cs * vp - sn * vq;
          V[q][k] = sn * vp + cs * vq;
        }
      }
    if (!rotated) break;
  }
  // normalise the rotated columns: U = (Y V) Sigma^-1
#pragma unroll
  for (int c = 0; c < D; ++c) {
    double s = 0;
#pragma unroll
    for (int a = 0; a < R; ++a) s = fma(y[c][a], y[c][a], s);
    const double inv = (s > 0.0) ? 1.0 / sqrt(s) : 0.0;
#pragma unroll
    for (int a = 0; a < R; ++a) y[c][a] *= inv;
  }
  // out = U V^T : out[a, c] = sum_k U[a,k] V[c,k]   (V[k][c'] holds entry c' of column k)
#pragma unroll
  for (int c = 0; c < D; ++c)
#pragma unroll
    for (int a = 0; a < R; ++a) {
      double s = 0;
#pragma unroll
      for (int k = 0; k < D; ++k) s = fma(y[k][a], V[k][c], s);
      out(c * R + a, s);
    }
#pragma unroll
  for (int a = 0; a < R; ++a) out(D * R + a, in(D * R + a));
}

// GNC-TLS weight of a squared residual r2 at control parameter mu and threshold cbar (Yang et al., eq. 14; ref
// RobustCost::weight, src/DPGO_robust.cpp:49-61): 0 above (mu+1)/mu cbar^2, 1 below mu/(mu+1) cbar^2, in between
// cbar sqrt(mu (mu+1)) / r - mu.
__device__ __forceinline__ double gnc_tls_weight(double r2, double mu, double cbar) {
  const double c2 = cbar * cbar;
  if (r2 >= c2 * (mu + 1.0) / mu) return 0.0;
  if (r2 <= c2 * mu / (mu + 1.0)) return 1.0;
  return sqrt(c2 * mu * (mu + 1.0) / r2) - mu;
}

}  // namespace dpgo
