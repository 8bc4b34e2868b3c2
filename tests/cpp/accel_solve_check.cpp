// DeviceRBCD::solve with accelerated coloured rounds on one GPU, for tests/test_gpu_accel_solve.py to compare with the
// Python runner.
//   accel_solve_check <file.g2o> <agents> <momentumBlocks> <maxRounds> <gradnormTol> <relChangeTol> <checkEvery> <out_dir>
// Prints "rounds <n> reason <r> cost <2f> gradnorm <g>" and writes out_dir/status.txt (one record per agent, the final
// status), full precision.  A configuration solve() rejects prints the exception and exits with 1.
#include <cstdio>
#include <cstdlib>
#include <string>

#include "DPGO/DPGO_utils.h"
#include "DPGO/DeviceRBCD.h"

using namespace DPGO;

int main(int argc, char **argv) {
  if (argc < 9) {
    std::fprintf(stderr, "usage: accel_solve_check <file.g2o> <agents> <momentumBlocks> <maxRounds> <gradnormTol> "
                         "<relChangeTol> <checkEvery> <out_dir>\n");
    return 2;
  }
  size_t n = 0;
  const std::vector<RelativeSEMeasurement> graph = read_g2o_file(argv[1], n);
  if (graph.empty()) return 2;
  const unsigned d = (unsigned)graph[0].t.size(), r = 5, K = (unsigned)std::atoi(argv[2]);
  DeviceRBCDOptions ro;
  ro.r = r;
  ro.schedule = "coloured";
  ro.acceleration = true;
  ro.momentumBlocks = argv[3];
  DeviceRBCDSolveOptions so;
  so.maxRounds = (unsigned)std::atoi(argv[4]);
  so.gradnormTol = std::atof(argv[5]);
  so.relChangeTol = std::atof(argv[6]);
  so.checkEvery = (unsigned)std::atoi(argv[7]);
  const std::string out = argv[8];
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
  } catch (const std::exception &e) {
    std::fprintf(stderr, "%s\n", e.what());
    return 1;
  }
  return 0;
}
