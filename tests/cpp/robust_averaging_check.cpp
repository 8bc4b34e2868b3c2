// Host restatement of robustSingleRotationAveraging (libDPGO, no GPU needed) on fixtures written by
// tests/test_dist_init_cpu.py.  Input file: "d m cbar" then m rotations, d x d row-major, one per line.  Prints
// "R v..." (row-major) and "inliers i...".
#include <cstdio>
#include <vector>

#include "DPGO/DPGO_types.h"
#include "DPGO/DPGO_utils.h"

using namespace DPGO;

int main(int argc, char **argv) {
  if (argc < 2) {
    std::fprintf(stderr, "usage: robust_averaging_check <fixture.txt>\n");
    return 2;
  }
  std::FILE *f = std::fopen(argv[1], "r");
  if (!f) return 2;
  int d = 0, m = 0;
  double cbar = 0;
  if (std::fscanf(f, "%d %d %lf", &d, &m, &cbar) != 3) return 2;
  std::vector<Matrix> RVec;
  for (int q = 0; q < m; ++q) {
    Matrix R(d, d);
    for (int a = 0; a < d; ++a)
      for (int c = 0; c < d; ++c)
        if (std::fscanf(f, "%lf", &R(a, c)) != 1) return 2;
    RVec.push_back(R);
  }
  std::fclose(f);
  Matrix ROpt;
  std::vector<size_t> inliers;
  robustSingleRotationAveraging(ROpt, inliers, RVec, Vector::Ones(m), cbar);
  std::printf("R");
  for (int a = 0; a < d; ++a)
    for (int c = 0; c < d; ++c) std::printf(" %.17g", ROpt(a, c));
  std::printf("\ninliers");
  for (size_t i : inliers) std::printf(" %zu", i);
  std::printf("\n");
  return 0;
}
