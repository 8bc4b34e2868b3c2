// dpgo_rotation.cuh -- per-thread SO(d) projection and GNC-TLS weight, shared by the chordal initialisation
// (dpgo_chordal.cu), the robust re-weighting of private edges (dpgo_kernels.cu) and the frame alignment of the distributed
// initialisation (dpgo_align.cu).
#pragma once
#include <cuda_runtime.h>

namespace dpgo {

// sqrt(alpha * beta) of the Jacobi convergence test.  For tiles scaled beyond about 1e+-77 the product leaves the normal
// double range (inf: every rotation would be skipped; 0: none would ever be), so it is then taken as sqrt(alpha) sqrt(beta);
// inside the range the test is the plain product's, bit for bit.
__device__ __forceinline__ double jacobi_norm_product(double alpha, double beta) {
  const double ab = alpha * beta;
  return (ab < 0x1p-1022 || ab > 0x1p1023) ? sqrt(alpha) * sqrt(beta) : sqrt(ab);
}

// Columns y[c] of length L with nul[c] (zero after the Jacobi sweeps: exactly rank-deficient input) are replaced by an
// orthonormal completion of the others, as JacobiSVD's U always is orthonormal (ref src/DPGO_utils.cpp:463-485): the unit
// vector with the least weight in the span of the columns so far, Gram-Schmidt'ed twice against them and normalised.
// Columns that are not nul are left alone, so full-rank results do not change.
template <int D, int L> __device__ __forceinline__ void complete_null_columns(double (&y)[D][L], const bool (&nul)[D]) {
  bool have[D];
#pragma unroll
  for (int c = 0; c < D; ++c) have[c] = !nul[c];
#pragma unroll
  for (int c = 0; c < D; ++c) {
    if (!nul[c]) continue;
    int kbest = 0;
    double wbest = 2.0;
#pragma unroll
    for (int k = 0; k < L; ++k) {
      double w = 0.0;
#pragma unroll
      for (int j = 0; j < D; ++j)
        if (have[j]) w = fma(y[j][k], y[j][k], w);
      if (w < wbest) { wbest = w; kbest = k; }
    }
#pragma unroll
    for (int a = 0; a < L; ++a) y[c][a] = (a == kbest) ? 1.0 : 0.0;
#pragma unroll
    for (int pass = 0; pass < 2; ++pass)
#pragma unroll
      for (int j = 0; j < D; ++j) {
        if (!have[j]) continue;
        double h = 0.0;
#pragma unroll
        for (int a = 0; a < L; ++a) h = fma(y[j][a], y[c][a], h);
#pragma unroll
        for (int a = 0; a < L; ++a) y[c][a] = fma(-h, y[j][a], y[c][a]);
      }
    double s = 0.0;
#pragma unroll
    for (int a = 0; a < L; ++a) s = fma(y[c][a], y[c][a], s);
    const double inv = 1.0 / sqrt(s);
#pragma unroll
    for (int a = 0; a < L; ++a) y[c][a] *= inv;
    have[c] = true;
  }
}

// Projection of a D x D matrix onto SO(D), M[a][c] = M(a, c): one-sided (Hestenes) Jacobi SVD, U V^T, and a sign flip of the
// direction of the smallest singular value when det < 0 (ref projectToRotationGroup, src/DPGO_utils.cpp:463-477).  For a
// rank-deficient M the zero columns of U are completed first, and the flip falls on a completed column.
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
        if (ga == 0.0 || fabs(ga) <= 1e-17 * jacobi_norm_product(al, be)) continue;
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
  bool nul[D], any_nul = false;
  int imin = 0;
  for (int c = 0; c < D; ++c) {
    double s = 0;
    for (int a = 0; a < D; ++a) s = fma(y[c][a], y[c][a], s);
    sig[c] = sqrt(s);
    nul[c] = !(s > 0.0);
    any_nul |= nul[c];
    const double inv = nul[c] ? 0.0 : 1.0 / sig[c];
    for (int a = 0; a < D; ++a) y[c][a] *= inv;        // U columns
    if (sig[c] < sig[imin]) imin = c;
  }
  if (any_nul) complete_null_columns<D, D>(y, nul);
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
        if (fabs(gamma) <= 1e-17 * jacobi_norm_product(alpha, beta) || gamma == 0.0) continue;
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
  // normalise the rotated columns: U = (Y V) Sigma^-1; zero columns (rank-deficient input) get an orthonormal completion
  bool nul[D], any_nul = false;
#pragma unroll
  for (int c = 0; c < D; ++c) {
    double s = 0;
#pragma unroll
    for (int a = 0; a < R; ++a) s = fma(y[c][a], y[c][a], s);
    nul[c] = !(s > 0.0);
    any_nul |= nul[c];
    const double inv = nul[c] ? 0.0 : 1.0 / sqrt(s);
#pragma unroll
    for (int a = 0; a < R; ++a) y[c][a] *= inv;
  }
  if (any_nul) complete_null_columns<D, R>(y, nul);
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

// GNC-TLS weight of a residual r at control parameter mu and threshold cbar (Yang et al., eq. 14; ref
// RobustCost::weight, src/DPGO_robust.cpp:49-61): 0 above (mu+1)/mu cbar^2, 1 below mu/(mu+1) cbar^2, in between
// cbar sqrt(mu (mu+1)) / r - mu.  Every operation in the reference's order, so that the weights that are exactly 0 or 1
// (which the GNC stop counts) are the reference's: r is squared again, and the bounds are (mu+1)/mu c^2 and mu/(mu+1) c^2.
__device__ __forceinline__ double gnc_tls_weight(double r, double mu, double cbar) {
  const double r2 = r * r, c2 = cbar * cbar;
  if (r2 >= (mu + 1.0) / mu * c2) return 0.0;
  if (r2 <= mu / (mu + 1.0) * c2) return 1.0;
  return sqrt(c2 * mu * (mu + 1.0) / r2) - mu;
}

}  // namespace dpgo
