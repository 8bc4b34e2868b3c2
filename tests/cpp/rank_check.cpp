// DeviceRBCD at a chosen relaxation rank, for tests/test_gpu_ranks.py to compare with the Python runner.
//   rank_check <file.g2o> <agents> <schedule> <r> <rounds> <out_dir>
// Runs <rounds> rounds through solve (stop rule off), prints "rounds <n> reason <r> cost <2f> gradnorm <g>" and writes
// out_dir/status.txt (one record per agent) and out_dir/trajectory.txt (d x (d+1)n, one row per line), full precision.
// A rank the library refuses ends with the library's message on stderr and exit code 3.
#include <cstdio>
#include <cstdlib>
#include <string>

#include "DPGO/DPGO_utils.h"
#include "DPGO/DeviceRBCD.h"

using namespace DPGO;

int main(int argc, char **argv) {
  if (argc < 7) {
    std::fprintf(stderr, "usage: rank_check <file.g2o> <agents> <schedule> <r> <rounds> <out_dir>\n");
    return 2;
  }
  size_t n = 0;
  const std::vector<RelativeSEMeasurement> graph = read_g2o_file(argv[1], n);
  if (graph.empty()) return 2;
  const unsigned d = (unsigned)graph[0].t.size(), K = (unsigned)std::atoi(argv[2]), r = (unsigned)std::atoi(argv[4]);
  DeviceRBCDOptions ro;
  ro.r = r;
  ro.schedule = argv[3];
  DeviceRBCDSolveOptions so;
  so.maxRounds = (unsigned)std::atoi(argv[5]);
  so.gradnormTol = 0.0;
  so.relChangeTol = 0.0;
  const std::string out = argv[6];
  try {
    DeviceRBCD run(graph, n, K, Matrix(fixedStiefelVariable(d, r) * chordalInitialization(d, n, graph)), ro);
    const DeviceRBCDSolveReport rep = run.solve(so);
    std::printf("rounds %u reason %s cost %.17g gradnorm %.17g\n", rep.rounds, rep.reason.c_str(), rep.cost, rep.gradnorm);
    const DeviceRBCDStatus st = run.status();
    std::FILE *f = std::fopen((out + "/status.txt").c_str(), "w");
    if (!f) return 2;
    for (unsigned a = 0; a < K; ++a) {
      for (unsigned q = 0; q < 5; ++q) std::fprintf(f, "%.17g ", st.at(a, q));
      std::fprintf(f, "\n");
    }
    std::fclose(f);
    const Matrix T = run.trajectory();
    f = std::fopen((out + "/trajectory.txt").c_str(), "w");
    if (!f) return 2;
    for (long i = 0; i < (long)T.rows(); ++i) {
      for (long j = 0; j < (long)T.cols(); ++j) std::fprintf(f, "%.17g ", T(i, j));
      std::fprintf(f, "\n");
    }
    std::fclose(f);
  } catch (const std::exception &e) {
    std::fprintf(stderr, "%s\n", e.what());
    return 3;
  }
  return 0;
}
