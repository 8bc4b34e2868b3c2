// dpgo_covariance.cuh -- the Gauss-Newton information of a trajectory, per block entry, shared by the device assembly
// (k_assemble_pose_info, dpgo_covariance.cu) and the host emulation of dpgo_pose_covariances_debug_emulate.
//
// Model (include/dpgo_b200.h, dpgo_pose_covariances): right perturbations R_i exp([w_i]x), t_i + R_i v_i, tangent
// x_i = (w_i, v_i) of dimension b = 6 (d = 3) or 3 (d = 2, w_i the angle).  Edge e = i -> j has the residuals
//     r_rot = R_j - R_i Rt  (d x d, weight kappa),   r_tra = t_j - t_i - R_i tt  (d, weight tau),
// so that sum_e 1/2 r^T Om r (Om = weight diag(kappa .., tau ..)) is f = 1/2 <Q, T^T T>.  Their Jacobians at T:
//     d r_rot / d w_j = R_j G_k              d r_tra / d v_j = R_j e_k
//     d r_rot / d w_i = -R_i G_k Rt          d r_tra / d w_i = -R_i G_k tt         d r_tra / d v_i = -R_i e_k
// with G_k = [e_k]x (d = 3) or [[0, -1], [1, 0]] (d = 2), and H = sum_e J^T Om J (Gauss-Newton: positive semidefinite).
#pragma once

namespace dpgo {
namespace cov {

// Column q of the Jacobian of edge e's residual with respect to the tangent of its endpoint `role` (0: p1 = i, 1: p2 = j):
// col[0 .. d*d) the rotation residual (row-major), col[d*d .. d*d + d) the translation residual.
// Ri, Rj: d x d column-major (the trajectory's layout); Rt: d x d row-major, tt: d (the edge's measurement).
template <int D>
__host__ __device__ inline void jac_col(int role, int q, const double *Ri, const double *Rj, const double *Rt, const double *tt,
                                        double *col) {
  for (int k = 0; k < D * D + D; ++k) col[k] = 0.0;
  constexpr int NW = D == 3 ? 3 : 1;
  const double *Rp = role ? Rj : Ri;
  if (q >= NW) {                                           // translation coordinate: +/- R_p e_k
    const int k = q - NW;
    for (int a = 0; a < D; ++a) col[D * D + a] = (role ? 1.0 : -1.0) * Rp[k * D + a];
    return;
  }
  double G[D][D];                                          // generator of rotation coordinate q
  for (int a = 0; a < D; ++a)
    for (int c = 0; c < D; ++c) G[a][c] = 0.0;
  if (D == 2) {
    G[0][D - 1] = -1.0; G[D - 1][0] = 1.0;
  } else {
    const int a = (q + 1) % 3, c = (q + 2) % 3;           // [e_q]x: (a, c) = -1, (c, a) = +1
    G[a][c] = -1.0; G[c][a] = 1.0;
  }
  double RG[D][D];                                         // R_p G
  for (int a = 0; a < D; ++a)
    for (int c = 0; c < D; ++c) {
      double s = 0.0;
      for (int u = 0; u < D; ++u) s += Rp[u * D + a] * G[u][c];
      RG[a][c] = s;
    }
  if (role) {
    for (int a = 0; a < D; ++a)
      for (int c = 0; c < D; ++c) col[a * D + c] = RG[a][c];
    return;
  }
  for (int a = 0; a < D; ++a) {
    for (int c = 0; c < D; ++c) {
      double s = 0.0;
      for (int u = 0; u < D; ++u) s += RG[a][u] * Rt[u * D + c];
      col[a * D + c] = -s;
    }
    double s = 0.0;
    for (int u = 0; u < D; ++u) s += RG[a][u] * tt[u];
    col[D * D + a] = -s;
  }
}

// One edge's contribution to H[x_a, x_c] for tangent coordinates qa of endpoint role ra and qc of role rc.
template <int D>
__host__ __device__ inline double edge_info(int ra, int qa, int rc, int qc, const double *Ri, const double *Rj, const double *Rt,
                                            const double *tt, double kappa, double tau, double w) {
  double ja[D * D + D], jc[D * D + D];
  jac_col<D>(ra, qa, Ri, Rj, Rt, tt, ja);
  jac_col<D>(rc, qc, Ri, Rj, Rt, tt, jc);
  double sr = 0.0, st = 0.0;
  for (int k = 0; k < D * D; ++k) sr += ja[k] * jc[k];
  for (int k = D * D; k < D * D + D; ++k) st += ja[k] * jc[k];
  return w * (kappa * sr + tau * st);
}

}  // namespace cov
}  // namespace dpgo
