// DeviceRBCD::poseCovariances on one GPU, for tests/test_gpu_covariance.py to compare with the Python function.
//   covariance_check <file.g2o> <agents> <rounds> <out_dir> [i j]...
// Runs the coloured schedule for <rounds> rounds, then writes out_dir/trajectory.txt (d x (d+1)n, one row per line),
// out_dir/cov.txt (the n b x b pose blocks, one block row per line) and out_dir/pairs.txt (the requested cross blocks),
// full precision.
#include <cstdio>
#include <cstdlib>
#include <string>
#include <utility>
#include <vector>

#include "DPGO/DPGO_utils.h"
#include "DPGO/DeviceRBCD.h"

using namespace DPGO;

static bool write(const std::string &path, const std::vector<Matrix> &blocks) {
  std::FILE *f = std::fopen(path.c_str(), "w");
  if (!f) return false;
  for (const Matrix &M : blocks)
    for (long i = 0; i < (long)M.rows(); ++i) {
      for (long j = 0; j < (long)M.cols(); ++j) std::fprintf(f, "%.17g ", M(i, j));
      std::fprintf(f, "\n");
    }
  std::fclose(f);
  return true;
}

int main(int argc, char **argv) {
  if (argc < 5 || (argc - 5) % 2 != 0) {
    std::fprintf(stderr, "usage: covariance_check <file.g2o> <agents> <rounds> <out_dir> [i j]...\n");
    return 2;
  }
  size_t n = 0;
  const std::vector<RelativeSEMeasurement> graph = read_g2o_file(argv[1], n);
  if (graph.empty()) return 2;
  const unsigned d = (unsigned)graph[0].t.size(), r = 5, K = (unsigned)std::atoi(argv[2]);
  const std::string out = argv[4];
  std::vector<std::pair<size_t, size_t>> pairs;
  for (int a = 5; a + 1 < argc; a += 2) pairs.push_back({(size_t)std::atol(argv[a]), (size_t)std::atol(argv[a + 1])});
  try {
    DeviceRBCDOptions ro;
    ro.r = r;
    ro.schedule = "coloured";
    DeviceRBCD run(graph, n, K, Matrix(fixedStiefelVariable(d, r) * chordalInitialization(d, n, graph)), ro);
    run.runRounds((unsigned)std::atoi(argv[3]));
    run.sync();
    const PoseCovariances cov = run.poseCovariances(-1, pairs);
    if (!write(out + "/trajectory.txt", {run.trajectory()}) || !write(out + "/cov.txt", cov.pose) ||
        !write(out + "/pairs.txt", cov.pair))
      return 2;
  } catch (const std::exception &e) {
    std::fprintf(stderr, "%s\n", e.what());
    return 1;
  }
  return 0;
}
