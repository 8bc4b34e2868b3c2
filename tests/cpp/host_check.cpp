// Host-side checks of libDPGO that need no GPU: g2o reader, connection Laplacian, chordal initialisation, small
// manifold utilities, robust-cost weights.  Prints `key value...` lines; tests/test_host_cpp.py compares them with the
// NumPy oracle and closed forms.  (Everything that touches QuadraticProblem / PGOAgent needs a device and lives in the
// gpu-marked tests.)
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <string>
#include <vector>

#include "DPGO/DPGO_robust.h"
#include "DPGO/DPGO_types.h"
#include "DPGO/DPGO_utils.h"

using namespace DPGO;

static void print_matrix(const char *key, const Matrix &M) {
  std::printf("%s %d %d", key, (int)M.rows(), (int)M.cols());
  for (int j = 0; j < M.cols(); ++j)
    for (int i = 0; i < M.rows(); ++i) std::printf(" %.17g", M(i, j));   // column-major
  std::printf("\n");
}

// `host_check --weights <file>`: one line `cost r mu c` per probe (cost as in RobustCostNames, the numbers in any strtod
// form, hex floats included), RobustCost::weight(r) printed as `weight %a` per line, exactly.  mu and c enter through
// RobustCostParameters (GNCInitMu, GNCBarc, Huber and TLS thresholds), as a caller sets them.
static int robust_weights(const char *path) {
  FILE *f = std::fopen(path, "r");
  if (!f) { std::fprintf(stderr, "cannot open %s\n", path); return 2; }
  char name[32], rs[64], mus[64], cs[64];
  while (std::fscanf(f, "%31s %63s %63s %63s", name, rs, mus, cs) == 4) {
    const double r = std::strtod(rs, nullptr), mu = std::strtod(mus, nullptr), c = std::strtod(cs, nullptr);
    int t = 0;
    while (t < (int)RobustCostNames.size() && RobustCostNames[t] != name) ++t;
    if (t == (int)RobustCostNames.size()) { std::fprintf(stderr, "unknown cost %s\n", name); return 2; }
    RobustCost cost((RobustCostType)t, RobustCostParameters(100, c, 1.4, mu, c, c));
    std::printf("weight %a\n", cost.weight(r));
  }
  std::fclose(f);
  return 0;
}

int main(int argc, char **argv) {
  if (argc == 3 && std::string(argv[1]) == "--weights") return robust_weights(argv[2]);
  if (argc < 3) {
    std::fprintf(stderr, "usage: host_check <file.g2o> <chordal_out.txt> | host_check --weights <probes.txt>\n");
    return 2;
  }
  size_t n = 0;
  std::vector<RelativeSEMeasurement> ms = read_g2o_file(argv[1], n);
  const size_t d = ms[0].t.size();
  std::printf("poses %zu\nedges %zu\ndim %zu\n", n, ms.size(), d);
  double sk = 0, st = 0;
  for (const auto &m : ms) { sk += m.kappa; st += m.tau; }
  std::printf("kappa_sum %.17g\ntau_sum %.17g\n", sk, st);
  std::printf("edge0 %zu %zu %.17g %.17g\n", ms[0].p1, ms[0].p2, ms[0].kappa, ms[0].tau);
  print_matrix("edge0_R", ms[0].R);
  print_matrix("edge0_t", ms[0].t);

  // connection Laplacian: dimension, nnz, trace, squared Frobenius norm, symmetry defect, row sums of the
  // translation rows/cols are not zero in general, so compare plain invariants with the oracle's Q
  SparseMatrix Q = constructConnectionLaplacianSE(ms);
  double tr = 0, fro = 0, asym = 0;
  size_t nnz = 0;
  for (int k = 0; k < Q.outerSize(); ++k)
    for (SparseMatrix::InnerIterator it(Q, k); it; ++it) {
      ++nnz;
      fro += it.value() * it.value();
      if (it.row() == it.col()) tr += it.value();
      asym = std::fmax(asym, std::fabs(it.value() - Q.coeff(it.col(), it.row())));
    }
  std::printf("Q_dim %d\nQ_nnz %zu\nQ_trace %.17g\nQ_fro2 %.17g\nQ_asym %.17g\n", (int)Q.rows(), nnz, tr, fro, asym);

  // chordal initialisation d x (d+1)n, written for the Python side (cost / gradient norm against the pinned constants)
  Matrix T = chordalInitialization(d, n, ms);
  writeMatrixToFile(T, argv[2]);
  std::printf("chordal %d %d\n", (int)T.rows(), (int)T.cols());

  // small utilities
  Matrix Y = fixedStiefelVariable((unsigned)d, 5);
  print_matrix("YLift_gram", Y.transpose() * Y);
  Matrix A(5, 3);
  for (int i = 0; i < 5; ++i)
    for (int j = 0; j < 3; ++j) A(i, j) = std::sin(1.0 + 3 * i + 7 * j) + 0.1 * i;
  print_matrix("stiefel_in", A);
  print_matrix("stiefel_out", projectToStiefelManifold(A));
  Matrix B(3, 3);
  for (int i = 0; i < 3; ++i)
    for (int j = 0; j < 3; ++j) B(i, j) = std::cos(2.0 + i - 2 * j) - 0.3 * (i == j);
  print_matrix("rot_in", B);
  print_matrix("rot_out", projectToRotationGroup(B));
  std::printf("chi2inv %.17g %.17g %.17g\n", chi2inv(0.9, 3), chi2inv(0.5, 6), chi2inv(0.99, 2));
  std::printf("ang2chord %.17g\n", angular2ChordalSO3(0.7));
  std::printf("meas_err %.17g\n", computeMeasurementError(ms[0], Matrix::Identity(d, d), Matrix::Zero(d, 1), ms[0].R, ms[0].t));

  // robust-cost weights (ref src/DPGO_robust.cpp:23-66) at fixed residuals, GNC schedule advanced 0 / 5 / 20 times
  const double rs[6] = {0.1, 1.0, 2.9, 3.1, 9.0, 30.0};
  const RobustCostType types[6] = {L2, L1, TLS, Huber, GM, GNC_TLS};
  for (int t = 0; t < 6; ++t) {
    RobustCost c(types[t], RobustCostParameters());
    for (int upd : {0, 5, 20}) {
      c.reset();
      for (int u = 0; u < upd; ++u) c.update();
      std::printf("robust %s %d", RobustCostNames[t].c_str(), upd);
      for (double r : rs) std::printf(" %.17g", c.weight(r));
      std::printf("\n");
    }
  }
  std::printf("quantile_threshold %.17g\n", RobustCost::computeErrorThresholdAtQuantile(0.9, 3));
  return 0;
}
