// DPGO_utils.cpp -- host utilities of the GPU pose-graph optimiser (reader, Laplacian assembly, initial
// guesses, small dense projections, single-pose averaging).  One-shot setup work: nothing here runs per
// iteration.  Behaviour follows the reference's src/DPGO_utils.cpp (cited per function); the code is
// written against the Eigen-compatible shim, without SuiteSparse / ROPTLIB / Boost.
#include <DPGO/DPGO_robust.h>
#include <DPGO/DPGO_utils.h>

#include "dpgo_b200.h"

#include <algorithm>
#include <cmath>
#include <fstream>
#include <sstream>

#include "sparse_ldl.h"

namespace DPGO {

// ---------------------------------------------------------------------------------------------------
// file output (ref src/DPGO_utils.cpp:21-49)
// ---------------------------------------------------------------------------------------------------
void writeMatrixToFile(const Matrix &M, const std::string &filename) {
  std::ofstream file(filename);
  if (!file.is_open()) {
    printf("Cannot write to specified file: %s\n", filename.c_str());
    return;
  }
  file << std::setprecision(17);
  for (Eigen::Index i = 0; i < M.rows(); ++i) {
    for (Eigen::Index j = 0; j < M.cols(); ++j) file << (j ? ", " : "") << M(i, j);
    file << "\n";
  }
}

void writeSparseMatrixToFile(const SparseMatrix &M, const std::string &filename) {
  std::ofstream file(filename);
  if (!file.is_open()) {
    printf("Cannot write to specified file: %s\n", filename.c_str());
    return;
  }
  for (Eigen::Index k = 0; k < M.outerSize(); ++k)
    for (SparseMatrix::InnerIterator it(M, k); it; ++it) file << it.row() << "," << it.col() << "," << it.value() << "\n";
}

// ---------------------------------------------------------------------------------------------------
// .g2o reader (ref src/DPGO_utils.cpp:64-197)
// ---------------------------------------------------------------------------------------------------
namespace {
// trace of the inverse of a small symmetric matrix given by its upper triangle
double invTrace2(double a, double b, double c) {   // [[a b],[b c]]
  const double det = a * c - b * b;
  return (a + c) / det;
}
double invTrace3(const double s[6]) {               // [[s0 s1 s2],[s1 s3 s4],[s2 s4 s5]]
  const double c00 = s[3] * s[5] - s[4] * s[4], c11 = s[0] * s[5] - s[2] * s[2], c22 = s[0] * s[3] - s[1] * s[1];
  const double det = s[0] * c00 - s[1] * (s[1] * s[5] - s[4] * s[2]) + s[2] * (s[1] * s[4] - s[3] * s[2]);
  return (c00 + c11 + c22) / det;
}
}  // namespace

std::vector<RelativeSEMeasurement> read_g2o_file(const std::string &filename, size_t &num_poses) {
  std::vector<RelativeSEMeasurement> out;
  std::ifstream in(filename);
  std::string line, tag;
  num_poses = 0;
  while (std::getline(in, line)) {
    std::istringstream ss(line);
    if (!(ss >> tag)) continue;
    RelativeSEMeasurement m;
    m.weight = 1.0;
    m.r1 = m.r2 = 0;
    if (tag == "EDGE_SE3:QUAT") {
      size_t i, j;
      double v[28];
      ss >> i >> j;
      for (double &x : v) ss >> x;
      m.p1 = i;
      m.p2 = j;
      m.t = Matrix(3, 1);
      m.t(0) = v[0]; m.t(1) = v[1]; m.t(2) = v[2];
      const double qx = v[3], qy = v[4], qz = v[5], qw = v[6];
      // quaternion -> matrix WITHOUT normalising (ref :160: Eigen::Quaterniond::toRotationMatrix)
      const double tx = 2 * qx, ty = 2 * qy, tz = 2 * qz;
      const double twx = tx * qw, twy = ty * qw, twz = tz * qw, txx = tx * qx, txy = ty * qx, txz = tz * qx;
      const double tyy = ty * qy, tyz = tz * qy, tzz = tz * qz;
      m.R = Matrix(3, 3);
      m.R(0, 0) = 1 - (tyy + tzz); m.R(0, 1) = txy - twz; m.R(0, 2) = txz + twy;
      m.R(1, 0) = txy + twz; m.R(1, 1) = 1 - (txx + tzz); m.R(1, 2) = tyz - twx;
      m.R(2, 0) = txz - twy; m.R(2, 1) = tyz + twx; m.R(2, 2) = 1 - (txx + tyy);
      // information matrix upper triangle: I11..I16, I22..I26, I33.., I44 I45 I46 I55 I56 I66
      const double *I = v + 7;
      const double tran[6] = {I[0], I[1], I[2], I[6], I[7], I[11]};
      const double rot[6] = {I[15], I[16], I[17], I[18], I[19], I[20]};
      m.tau = 3.0 / invTrace3(tran);               // ref :168
      m.kappa = 3.0 / (2.0 * invTrace3(rot));      // ref :175
    } else if (tag == "EDGE_SE2") {
      size_t i, j;
      double dx, dy, dth, I11, I12, I13, I22, I23, I33;
      ss >> i >> j >> dx >> dy >> dth >> I11 >> I12 >> I13 >> I22 >> I23 >> I33;
      m.p1 = i;
      m.p2 = j;
      m.t = Matrix(2, 1);
      m.t(0) = dx; m.t(1) = dy;
      m.R = Matrix(2, 2);
      m.R(0, 0) = std::cos(dth); m.R(0, 1) = -std::sin(dth);
      m.R(1, 0) = std::sin(dth); m.R(1, 1) = std::cos(dth);
      m.tau = 2.0 / invTrace2(I11, I12, I22);      // ref :122-123
      m.kappa = I33;                               // ref :125
      (void)I13; (void)I23;
    } else if (tag == "VERTEX_SE2" || tag == "VERTEX_SE3:QUAT") {
      continue;
    } else {
      std::cout << "Error: unrecognized type: " << tag << "!" << std::endl;
      continue;
    }
    num_poses = std::max(num_poses, std::max(m.p1, m.p2));
    out.push_back(m);
  }
  num_poses++;   // zero-based ids
  return out;
}

// ---------------------------------------------------------------------------------------------------
// connection Laplacian (ref src/DPGO_utils.cpp:199-271)
// ---------------------------------------------------------------------------------------------------
void constructOrientedConnectionIncidenceMatrixSE(const std::vector<RelativeSEMeasurement> &measurements,
                                                  SparseMatrix &AT, DiagonalMatrix &OmegaT) {
  const size_t d = measurements.empty() ? 0 : (size_t)measurements[0].t.size();
  const size_t dh = d + 1, m = measurements.size();
  size_t n = 0;
  for (const auto &e : measurements) n = std::max(n, std::max(e.p1, e.p2));
  n++;
  std::vector<Eigen::Triplet<double>> trip;
  trip.reserve(m * (dh * dh + dh));
  DiagonalMatrix Omega((Eigen::Index)(dh * m));
  for (size_t k = 0; k < m; ++k) {
    const auto &e = measurements[k];
    // block leaving node i: -T ; block entering node j: +I   (ref :232-251)
    for (size_t c = 0; c < d; ++c)
      for (size_t r = 0; r < d; ++r) trip.emplace_back((int)(e.p1 * dh + r), (int)(k * dh + c), -e.R(r, c));
    for (size_t r = 0; r < d; ++r) trip.emplace_back((int)(e.p1 * dh + r), (int)(k * dh + d), -e.t(r));
    trip.emplace_back((int)(e.p1 * dh + d), (int)(k * dh + d), -1.0);
    for (size_t r = 0; r < dh; ++r) trip.emplace_back((int)(e.p2 * dh + r), (int)(k * dh + r), 1.0);
    for (size_t r = 0; r < d; ++r) Omega.diagonal()(k * dh + r) = e.weight * e.kappa;
    Omega.diagonal()(k * dh + d) = e.weight * e.tau;
  }
  SparseMatrix A((Eigen::Index)(dh * n), (Eigen::Index)(dh * m));
  A.setFromTriplets(trip.begin(), trip.end());
  AT = A;
  OmegaT = Omega;
}

SparseMatrix constructConnectionLaplacianSE(const std::vector<RelativeSEMeasurement> &measurements) {
  // Q = A Omega A^T assembled block-wise: per edge i->j with T = [R t; 0 1], Om = diag(w kappa.., w tau):
  //   Q_ii += T Om T^T,  Q_jj += Om,  Q_ij = -T Om,  Q_ji = -Om T^T
  const size_t d = measurements.empty() ? 0 : (size_t)measurements[0].t.size();
  const size_t dh = d + 1;
  size_t n = 0;
  for (const auto &e : measurements) n = std::max(n, std::max(e.p1, e.p2));
  n++;
  std::vector<Eigen::Triplet<double>> trip;
  trip.reserve(measurements.size() * 4 * dh * dh);
  Matrix T(dh, dh), TO(dh, dh);
  for (const auto &e : measurements) {
    T.setZero();
    for (size_t r = 0; r < d; ++r) {
      for (size_t c = 0; c < d; ++c) T(r, c) = e.R(r, c);
      T(r, d) = e.t(r);
    }
    T(d, d) = 1.0;
    std::vector<double> om(dh, e.weight * e.kappa);
    om[d] = e.weight * e.tau;
    for (size_t r = 0; r < dh; ++r)
      for (size_t c = 0; c < dh; ++c) TO(r, c) = T(r, c) * om[c];
    const size_t bi = e.p1 * dh, bj = e.p2 * dh;
    for (size_t r = 0; r < dh; ++r)
      for (size_t c = 0; c < dh; ++c) {
        double w = 0.0;
        for (size_t q = 0; q < dh; ++q) w += TO(r, q) * T(c, q);
        trip.emplace_back((int)(bi + r), (int)(bi + c), w);              // T Om T^T
        trip.emplace_back((int)(bi + r), (int)(bj + c), -TO(r, c));      // -T Om
        trip.emplace_back((int)(bj + c), (int)(bi + r), -TO(r, c));      // -(T Om)^T
      }
    for (size_t r = 0; r < dh; ++r) trip.emplace_back((int)(bj + r), (int)(bj + r), om[r]);
  }
  SparseMatrix Q((Eigen::Index)(dh * n), (Eigen::Index)(dh * n));
  Q.setFromTriplets(trip.begin(), trip.end());
  return Q;
}

// ---------------------------------------------------------------------------------------------------
// small dense factorizations
// ---------------------------------------------------------------------------------------------------
void smallSVD(const Matrix &M, Matrix &U, Vector &s, Matrix &V) {
  // one-sided Jacobi: rotate the columns of W = M until orthogonal; W V^T... M V = U diag(s)
  const Eigen::Index rows = M.rows(), cols = M.cols();
  Matrix W = M;
  V = Matrix::Identity(cols, cols);
  for (int sweep = 0; sweep < 60; ++sweep) {
    bool rotated = false;
    for (Eigen::Index p = 0; p < cols; ++p)
      for (Eigen::Index q = p + 1; q < cols; ++q) {
        double alpha = 0, beta = 0, gamma = 0;
        for (Eigen::Index a = 0; a < rows; ++a) {
          alpha += W(a, p) * W(a, p);
          beta += W(a, q) * W(a, q);
          gamma += W(a, p) * W(a, q);
        }
        if (gamma == 0.0 || std::fabs(gamma) <= 1e-17 * std::sqrt(alpha * beta)) continue;
        rotated = true;
        const double zeta = (beta - alpha) / (2.0 * gamma);
        const double t = (zeta >= 0 ? 1.0 : -1.0) / (std::fabs(zeta) + std::sqrt(1.0 + zeta * zeta));
        const double c = 1.0 / std::sqrt(1.0 + t * t), sn = c * t;
        for (Eigen::Index a = 0; a < rows; ++a) {
          const double wp = W(a, p), wq = W(a, q);
          W(a, p) = c * wp - sn * wq;
          W(a, q) = sn * wp + c * wq;
        }
        for (Eigen::Index a = 0; a < cols; ++a) {
          const double vp = V(a, p), vq = V(a, q);
          V(a, p) = c * vp - sn * vq;
          V(a, q) = sn * vp + c * vq;
        }
      }
    if (!rotated) break;
  }
  s = Vector(cols);
  U = Matrix(rows, cols);
  for (Eigen::Index c = 0; c < cols; ++c) {
    double nrm = 0;
    for (Eigen::Index a = 0; a < rows; ++a) nrm += W(a, c) * W(a, c);
    nrm = std::sqrt(nrm);
    s(c) = nrm;
    for (Eigen::Index a = 0; a < rows; ++a) U(a, c) = nrm > 0 ? W(a, c) / nrm : 0.0;
  }
  // order singular values descending (Eigen's convention)
  for (Eigen::Index a = 0; a < cols; ++a)
    for (Eigen::Index b = a + 1; b < cols; ++b)
      if (s(b) > s(a)) {
        std::swap(s(a), s(b));
        for (Eigen::Index i = 0; i < rows; ++i) std::swap(U(i, a), U(i, b));
        for (Eigen::Index i = 0; i < cols; ++i) std::swap(V(i, a), V(i, b));
      }
}

Matrix projectToRotationGroup(const Matrix &M) {   // ref :463-477
  Matrix U, V;
  Vector s;
  smallSVD(M, U, s, V);
  if (U.determinant() * V.determinant() <= 0) {
    const Eigen::Index last = U.cols() - 1;
    for (Eigen::Index i = 0; i < U.rows(); ++i) U(i, last) = -U(i, last);
  }
  return U * V.transpose();
}

Matrix projectToStiefelManifold(const Matrix &M) {  // ref :479-485
  assert(M.rows() >= M.cols());
  Matrix U, V;
  Vector s;
  smallSVD(M, U, s, V);
  return U * V.transpose();
}

Matrix fixedStiefelVariable(unsigned d, unsigned r) {
  // ref :487-492 draws from ROPTLIB's RandInManifold after srand(1); that value is unpinned (any element of
  // St(d, r) gives the same cost / gradient norm / trajectory up to the lift), so a fixed recurrence is used:
  // orthonormalise a deterministic r x d matrix by modified Gram-Schmidt (positive diagonal).
  Matrix A(r, d);
  unsigned long long state = 0x9E3779B97F4A7C15ULL;
  for (unsigned j = 0; j < d; ++j)
    for (unsigned i = 0; i < r; ++i) {
      state = state * 6364136223846793005ULL + 1442695040888963407ULL;
      A(i, j) = ((double)((state >> 11) & ((1ULL << 53) - 1)) / (double)(1ULL << 53)) * 2.0 - 1.0;
    }
  for (int pass = 0; pass < 2; ++pass)
    for (unsigned j = 0; j < d; ++j) {
      for (unsigned q = 0; q < j; ++q) {
        double dot = 0;
        for (unsigned i = 0; i < r; ++i) dot += A(i, q) * A(i, j);
        for (unsigned i = 0; i < r; ++i) A(i, j) -= dot * A(i, q);
      }
      double nrm = 0;
      for (unsigned i = 0; i < r; ++i) nrm += A(i, j) * A(i, j);
      nrm = std::sqrt(nrm);
      for (unsigned i = 0; i < r; ++i) A(i, j) /= nrm;
    }
  return A;
}

// ---------------------------------------------------------------------------------------------------
// initial guesses (ref src/DPGO_utils.cpp:362-461)
// ---------------------------------------------------------------------------------------------------
Matrix odometryInitialization(size_t dimension, size_t num_poses, const std::vector<RelativeSEMeasurement> &odometry) {
  const size_t d = dimension, n = num_poses, dh = d + 1;
  Matrix T(d, n * dh);
  Matrix R = Matrix::Identity(d, d), t = Matrix::Zero(d, 1);
  T.block(0, 0, d, d) = R;
  for (size_t src = 0; src < odometry.size(); ++src) {
    const RelativeSEMeasurement &m = odometry[src];
    assert(m.p1 == src && m.p2 == src + 1);
    t = t + R * m.t;
    R = R * m.R;
    T.block(0, (src + 1) * dh, d, d) = R;
    T.block(0, (src + 1) * dh + d, d, 1) = t;
  }
  return T;
}

Matrix chordalInitializationGPU(size_t dimension, size_t num_poses, const std::vector<RelativeSEMeasurement> &measurements,
                                int device, double tol) {
  const size_t d = dimension, m = measurements.size();
  std::vector<int32_t> p1(m), p2(m);
  std::vector<double> R(m * d * d), t(m * d), kappa(m), tau(m);
  for (size_t e = 0; e < m; ++e) {
    const RelativeSEMeasurement &ms = measurements[e];
    p1[e] = (int32_t)ms.p1;
    p2[e] = (int32_t)ms.p2;
    for (size_t a = 0; a < d; ++a) {
      for (size_t b = 0; b < d; ++b) R[e * d * d + a * d + b] = ms.R(a, b);
      t[e * d + a] = ms.t(a);
    }
    kappa[e] = ms.weight * ms.kappa;
    tau[e] = ms.weight * ms.tau;
  }
  if (device < 0) { const char *ev = std::getenv("DPGO_DEVICE"); device = ev ? std::atoi(ev) : 0; }
  Matrix T((Eigen::Index)d, (Eigen::Index)((d + 1) * num_poses));
  if (dpgo_chordal_initialization((int)num_poses, (int)d, (int64_t)m, p1.data(), p2.data(), R.data(), t.data(), kappa.data(), tau.data(),
                                  device, tol, 0, T.data(), nullptr) != DPGO_OK)
    throw std::runtime_error(std::string("dpgo_chordal_initialization: ") + dpgo_chordal_last_error());
  return T;
}

PoseCovariances poseCovariancesGPU(size_t dimension, size_t num_poses, const std::vector<RelativeSEMeasurement> &measurements,
                                   const Matrix &T, size_t anchor, const std::vector<std::pair<size_t, size_t>> &pairs,
                                   int device) {
  const size_t d = dimension, m = measurements.size(), n = num_poses, b = d == 3 ? 6 : 3;
  if ((size_t)T.rows() != d || (size_t)T.cols() != (d + 1) * n)
    throw std::runtime_error("poseCovariancesGPU: the trajectory must be d x (d+1)n");
  std::vector<int32_t> p1(m), p2(m), pr(2 * pairs.size());
  std::vector<double> R(m * d * d), t(m * d), kappa(m), tau(m), weight(m);
  for (size_t e = 0; e < m; ++e) {
    const RelativeSEMeasurement &ms = measurements[e];
    p1[e] = (int32_t)ms.p1;
    p2[e] = (int32_t)ms.p2;
    for (size_t a = 0; a < d; ++a) {
      for (size_t c = 0; c < d; ++c) R[e * d * d + a * d + c] = ms.R(a, c);
      t[e * d + a] = ms.t(a);
    }
    kappa[e] = ms.kappa;
    tau[e] = ms.tau;
    weight[e] = ms.weight;
  }
  for (size_t q = 0; q < pairs.size(); ++q) { pr[2 * q] = (int32_t)pairs[q].first; pr[2 * q + 1] = (int32_t)pairs[q].second; }
  if (device < 0) { const char *ev = std::getenv("DPGO_DEVICE"); device = ev ? std::atoi(ev) : 0; }
  std::vector<double> cov(n * b * b), pcov(std::max<size_t>(pairs.size(), 1) * b * b);
  if (dpgo_pose_covariances((int)n, (int)d, (int64_t)m, p1.data(), p2.data(), R.data(), t.data(), kappa.data(), tau.data(),
                            weight.data(), T.data(), (int)anchor, device, (int64_t)pairs.size(), pr.data(), cov.data(),
                            pcov.data(), nullptr) != DPGO_OK)
    throw std::runtime_error(std::string("dpgo_pose_covariances: ") + dpgo_last_error());
  auto block = [&](const double *src) {                  // row-major b x b
    Matrix M((Eigen::Index)b, (Eigen::Index)b);
    for (size_t a = 0; a < b; ++a)
      for (size_t c = 0; c < b; ++c) M((Eigen::Index)a, (Eigen::Index)c) = src[a * b + c];
    return M;
  };
  PoseCovariances out;
  for (size_t p = 0; p < n; ++p) out.pose.push_back(block(cov.data() + p * b * b));
  for (size_t q = 0; q < pairs.size(); ++q) out.pair.push_back(block(pcov.data() + q * b * b));
  return out;
}

Matrix chordalInitialization(size_t dimension, size_t num_poses, const std::vector<RelativeSEMeasurement> &measurements) {
  // Chordal relaxation with the gauge R_0 = I, t_0 = 0 (ref :362-409 rotations, :434-461 translations).
  // Rotations: min sum_e kappa_e |R_j - R_i Rij|_F^2 over free d x d matrices.  The d rows of the unknowns
  // decouple and share one normal matrix of order (n-1) d, so it is factored once and solved for d right-hand
  // sides; likewise the translations share the (n-1) x (n-1) tau-weighted graph Laplacian.
  const size_t d = dimension, n = num_poses, dh = d + 1;
  assert(measurements.empty() || (size_t)measurements[0].t.size() == d);
  if (n == 1) {
    Matrix T = Matrix::Zero(d, dh);
    T.block(0, 0, d, d) = Matrix::Identity(d, d);
    return T;
  }
  using dpgo_host::Triplet;
  const int NR = (int)((n - 1) * d);
  std::vector<Triplet> ent;
  std::vector<std::vector<double>> rhs(d, std::vector<double>((size_t)NR, 0.0));   // one per row l of R
  auto idx = [&](size_t pose, size_t c) { return (int)((pose - 1) * d + c); };
  for (const auto &e : measurements) {
    const size_t i = e.p1, j = e.p2;
    const double k = e.kappa;
    // x_p = (row l of R_p)^T;  residual x_j - A^T x_i with A = Rij;  normal blocks: ii: k A A^T, jj: k I, ij: -k A
    Matrix AAt = e.R * e.R.transpose();
    if (i > 0)
      for (size_t a = 0; a < d; ++a)
        for (size_t b = a; b < d; ++b) ent.push_back({idx(i, a), idx(i, b), k * AAt(a, b)});
    if (j > 0)
      for (size_t a = 0; a < d; ++a) ent.push_back({idx(j, a), idx(j, a), k});
    if (i > 0 && j > 0) {
      for (size_t a = 0; a < d; ++a)
        for (size_t b = 0; b < d; ++b) {
          const int r = idx(i, a), c = idx(j, b);
          ent.push_back({std::min(r, c), std::max(r, c), -k * e.R(a, b)});
        }
    } else if (i == 0 && j > 0) {
      // x_0 = e_l is known: rhs_j += k A^T e_l = k * (row l of A)^T
      for (size_t l = 0; l < d; ++l)
        for (size_t b = 0; b < d; ++b) rhs[l][(size_t)idx(j, b)] += k * e.R(l, b);
    } else if (j == 0 && i > 0) {
      // x_j = e_l known: rhs_i += k A e_l = k * column l of A
      for (size_t l = 0; l < d; ++l)
        for (size_t a = 0; a < d; ++a) rhs[l][(size_t)idx(i, a)] += k * e.R(a, l);
    }
  }
  dpgo_host::SparseLDL ldlR;
  ldlR.factor(NR, ent);
  std::vector<Matrix> Rs(n, Matrix::Identity(d, d));
  for (size_t l = 0; l < d; ++l) {
    ldlR.solve(rhs[l].data());
    for (size_t p = 1; p < n; ++p)
      for (size_t c = 0; c < d; ++c) Rs[p](l, c) = rhs[l][(size_t)idx(p, c)];
  }
  for (size_t p = 1; p < n; ++p) Rs[p] = projectToRotationGroup(Rs[p]);

  // translations: min sum_e tau_e |t_j - t_i - R_i tij|^2
  const int NT = (int)(n - 1);
  std::vector<Triplet> entT;
  std::vector<std::vector<double>> rhsT(d, std::vector<double>((size_t)NT, 0.0));
  for (const auto &e : measurements) {
    const size_t i = e.p1, j = e.p2;
    const double w = e.tau;
    Matrix v = Rs[i] * e.t;   // d x 1
    if (i > 0) entT.push_back({(int)i - 1, (int)i - 1, w});
    if (j > 0) entT.push_back({(int)j - 1, (int)j - 1, w});
    if (i > 0 && j > 0) entT.push_back({(int)std::min(i, j) - 1, (int)std::max(i, j) - 1, -w});
    for (size_t c = 0; c < d; ++c) {
      if (j > 0) rhsT[c][j - 1] += w * v(c);
      if (i > 0) rhsT[c][i - 1] -= w * v(c);
    }
  }
  dpgo_host::SparseLDL ldlT;
  ldlT.factor(NT, entT);
  Matrix T(d, n * dh);
  for (size_t c = 0; c < d; ++c) ldlT.solve(rhsT[c].data());
  for (size_t p = 0; p < n; ++p) {
    T.block(0, p * dh, d, d) = Rs[p];
    for (size_t c = 0; c < d; ++c) T(c, p * dh + d) = (p == 0) ? 0.0 : rhsT[c][p - 1];
  }
  return T;
}

// ---------------------------------------------------------------------------------------------------
// scalar helpers
// ---------------------------------------------------------------------------------------------------
double computeMeasurementError(const RelativeSEMeasurement &m, const Matrix &R1, const Matrix &t1, const Matrix &R2,
                               const Matrix &t2) {
  const double rotSq = (R1 * m.R - R2).squaredNorm();
  const double tranSq = (t2 - t1 - R1 * m.t).squaredNorm();
  return m.kappa * rotSq + m.tau * tranSq;
}

namespace {
// regularised lower incomplete gamma P(a, x)
double gammaP(double a, double x) {
  if (x <= 0) return 0.0;
  const double lg = std::lgamma(a);
  if (x < a + 1.0) {
    double sum = 1.0 / a, term = sum;
    for (int k = 1; k < 1000; ++k) {
      term *= x / (a + k);
      sum += term;
      if (std::fabs(term) < std::fabs(sum) * 1e-16) break;
    }
    return sum * std::exp(-x + a * std::log(x) - lg);
  }
  double b = x + 1.0 - a, c = 1e300, dd = 1.0 / b, h = dd;
  for (int k = 1; k < 1000; ++k) {
    const double an = -k * (k - a);
    b += 2.0;
    dd = an * dd + b;
    if (std::fabs(dd) < 1e-300) dd = 1e-300;
    c = b + an / c;
    if (std::fabs(c) < 1e-300) c = 1e-300;
    dd = 1.0 / dd;
    const double del = dd * c;
    h *= del;
    if (std::fabs(del - 1.0) < 1e-16) break;
  }
  return 1.0 - std::exp(-x + a * std::log(x) - lg) * h;
}
}  // namespace

double chi2inv(double quantile, size_t dof) {
  double lo = 0.0, hi = std::max(10.0, 10.0 * (double)dof);
  while (gammaP(0.5 * dof, 0.5 * hi) < quantile) hi *= 2.0;
  for (int it = 0; it < 200; ++it) {
    const double mid = 0.5 * (lo + hi);
    if (gammaP(0.5 * dof, 0.5 * mid) < quantile) lo = mid; else hi = mid;
  }
  return 0.5 * (lo + hi);
}

double angular2ChordalSO3(double rad) { return 2 * std::sqrt(2.0) * std::sin(rad / 2); }

void checkRotationMatrix(const Matrix &R) {
  const auto d = R.rows();
  assert(R.cols() == d);
  assert(std::fabs(R.determinant() - 1.0) < 1e-8);
  assert((R.transpose() * R - Matrix::Identity(d, d)).norm() < 1e-8);
  (void)d;
}

// ---------------------------------------------------------------------------------------------------
// single pose averaging (ref src/DPGO_utils.cpp:518-711)
// ---------------------------------------------------------------------------------------------------
void singleTranslationAveraging(Vector &tOpt, const std::vector<Vector> &tVec, const Vector &tau) {
  const int n = (int)tVec.size();
  assert(n > 0);
  Vector w = (tau.rows() == n) ? tau : Vector::Ones(n);
  Matrix s = Matrix::Zero(tVec[0].rows(), 1);
  double tot = 0;
  for (int i = 0; i < n; ++i) {
    s += w(i) * tVec[(size_t)i];
    tot += w(i);
  }
  tOpt = Vector(s / tot);
}

void singleRotationAveraging(Matrix &ROpt, const std::vector<Matrix> &RVec, const Vector &kappa) {
  const int n = (int)RVec.size();
  assert(n > 0);
  Vector w = (kappa.rows() == n) ? kappa : Vector::Ones(n);
  Matrix M = Matrix::Zero(RVec[0].rows(), RVec[0].rows());
  for (int i = 0; i < n; ++i) M += w(i) * RVec[(size_t)i];
  ROpt = projectToRotationGroup(M);
}

void singlePoseAveraging(Matrix &ROpt, Vector &tOpt, const std::vector<Matrix> &RVec, const std::vector<Vector> &tVec,
                         const Vector &kappa, const Vector &tau) {
  assert(!RVec.empty() && RVec.size() == tVec.size());
  singleTranslationAveraging(tOpt, tVec, tau);
  singleRotationAveraging(ROpt, RVec, kappa);
}

namespace {
// shared GNC loop: residual(i) gives the squared weighted residual of sample i at the current estimate
template <class Update, class Residual>
void gncAverage(int n, double errorThreshold, unsigned maxIters, Vector &weights, Update update, Residual residual) {
  const double w_tol = 1e-8;
  update(weights);
  double maxR = 0;
  for (int i = 0; i < n; ++i) maxR = std::max(maxR, residual(i));
  const double barcSq = errorThreshold * errorThreshold;
  double muInit = std::min(barcSq / (2 * maxR - barcSq), 1e-5);
  if (muInit <= 0) return;          // all residuals already small: skip GNC (ref :590-591)
  RobustCostParameters params;
  params.GNCBarc = errorThreshold;
  params.GNCMaxNumIters = maxIters;
  params.GNCInitMu = muInit;
  RobustCost cost(RobustCostType::GNC_TLS, params);
  for (unsigned iter = 0; iter < maxIters; ++iter) {
    update(weights);
    int converged = 0;
    for (int i = 0; i < n; ++i) {
      const double wi = cost.weight(std::sqrt(residual(i)));
      if (wi < w_tol || wi > 1 - w_tol) converged++;
      weights(i) = wi;
    }
    if (converged == n) break;
    cost.update();
  }
}
}  // namespace

void robustSingleRotationAveraging(Matrix &ROpt, std::vector<size_t> &inlierIndices, const std::vector<Matrix> &RVec,
                                   const Vector &kappa, double errorThreshold) {
  const int n = (int)RVec.size();
  assert(n > 0);
  Vector k = (kappa.rows() == n) ? kappa : Vector::Ones(n);
  Vector w = Vector::Ones(n);
  for (const auto &Ri : RVec) checkRotationMatrix(Ri);
  gncAverage(
      n, errorThreshold, 1000, w, [&](const Vector &wt) { singleRotationAveraging(ROpt, RVec, Vector(k.cwiseProduct(wt))); },
      [&](int i) { return k(i) * (ROpt - RVec[(size_t)i]).squaredNorm(); });
  inlierIndices.clear();
  for (int i = 0; i < n; ++i)
    if (w(i) > 1 - 1e-8) inlierIndices.push_back((size_t)i);
}

void robustSinglePoseAveraging(Matrix &ROpt, Vector &tOpt, std::vector<size_t> &inlierIndices,
                               const std::vector<Matrix> &RVec, const std::vector<Vector> &tVec, const Vector &kappa,
                               const Vector &tau, double errorThreshold) {
  const int n = (int)RVec.size();
  assert(n > 0 && (int)tVec.size() == n);
  Vector k = (kappa.rows() == n) ? kappa : Vector::Constant(n, 10000.0);
  Vector t = (tau.rows() == n) ? tau : Vector::Constant(n, 100.0);
  Vector w = Vector::Ones(n);
  for (const auto &Ri : RVec) checkRotationMatrix(Ri);
  gncAverage(
      n, errorThreshold, 10000, w,
      [&](const Vector &wt) { singlePoseAveraging(ROpt, tOpt, RVec, tVec, Vector(k.cwiseProduct(wt)), Vector(t.cwiseProduct(wt))); },
      [&](int i) {
        return k(i) * (ROpt - RVec[(size_t)i]).squaredNorm() + t(i) * (tOpt - tVec[(size_t)i]).squaredNorm();
      });
  inlierIndices.clear();
  for (int i = 0; i < n; ++i)
    if (w(i) > 1 - 1e-8) inlierIndices.push_back((size_t)i);
}

}  // namespace DPGO
