// DeviceRBCD's resources over its whole life, for tests/test_gpu_handle_lifetime.py: this program defines the C calls the
// runner creates and releases its streams, device buffers, pinned buffer and NCCL communicators with, counts every call
// libDPGO.so makes to them and forwards it to the library that defines it (the executable's definitions take
// precedence).  Three runners on <file.g2o> (smallGrid3D), 4 agents over <gpus> GPUs:
//   a  initialization "distributed" with the last agent's shared edges removed: the constructor throws
//   b  schedule "coloured", acceleration with momentumBlocks "colours": solve() for a few rounds, status()
//   c  schedule "greedy_set": a few step() calls, selectionLog()
//   runner_lifetime_check <file.g2o> <gpus>
// Prints "error a <message>" for the constructor's exception and, after each runner is gone,
// "counts <case> <call> <count> ..." (releases counted for non-null handles only).
#include <dlfcn.h>
#include <nccl.h>

#include <algorithm>
#include <cstdio>
#include <cstdlib>
#include <string>

#include "DPGO/DPGO_utils.h"
#include "DPGO/DeviceRBCD.h"
#include "dpgo_b200.h"

using namespace DPGO;

namespace {
enum Call { StreamCreate, StreamDestroy, DeviceMalloc, DeviceFree, HostAllocPinned, HostFreePinned, CommInit, CommDestroy, Calls };
const char *const kName[Calls] = {"dpgo_stream_create", "dpgo_stream_destroy", "dpgo_device_malloc", "dpgo_device_free",
                                  "dpgo_host_alloc_pinned", "dpgo_host_free_pinned", "ncclCommInitAll", "ncclCommDestroy"};
long counts[Calls];

template <class F> F next(const char *name) {
  void *f = dlsym(RTLD_NEXT, name);
  if (!f) {
    std::fprintf(stderr, "dlsym(RTLD_NEXT, %s) found nothing\n", name);
    std::abort();
  }
  return reinterpret_cast<F>(f);
}

void report(const char *which) {
  std::printf("counts %s", which);
  for (int c = 0; c < Calls; ++c) std::printf(" %s %ld", kName[c], counts[c]);
  std::printf("\n");
  for (long &c : counts) c = 0;
}
}  // namespace

extern "C" {
int dpgo_stream_create(int device, void **stream) {
  static const auto f = next<int (*)(int, void **)>("dpgo_stream_create");
  const int rc = f(device, stream);
  if (rc == DPGO_OK) ++counts[StreamCreate];
  return rc;
}
int dpgo_stream_destroy(int device, void *stream) {
  static const auto f = next<int (*)(int, void *)>("dpgo_stream_destroy");
  if (stream) ++counts[StreamDestroy];
  return f(device, stream);
}
int dpgo_device_malloc(int device, size_t bytes, void **ptr) {
  static const auto f = next<int (*)(int, size_t, void **)>("dpgo_device_malloc");
  const int rc = f(device, bytes, ptr);
  if (rc == DPGO_OK) ++counts[DeviceMalloc];
  return rc;
}
int dpgo_device_free(int device, void *ptr) {
  static const auto f = next<int (*)(int, void *)>("dpgo_device_free");
  if (ptr) ++counts[DeviceFree];
  return f(device, ptr);
}
int dpgo_host_alloc_pinned(size_t bytes, void **ptr) {
  static const auto f = next<int (*)(size_t, void **)>("dpgo_host_alloc_pinned");
  const int rc = f(bytes, ptr);
  if (rc == DPGO_OK) ++counts[HostAllocPinned];
  return rc;
}
int dpgo_host_free_pinned(void *ptr) {
  static const auto f = next<int (*)(void *)>("dpgo_host_free_pinned");
  if (ptr) ++counts[HostFreePinned];
  return f(ptr);
}
ncclResult_t ncclCommInitAll(ncclComm_t *comm, int ndev, const int *devlist) {
  static const auto f = next<ncclResult_t (*)(ncclComm_t *, int, const int *)>("ncclCommInitAll");
  const ncclResult_t rc = f(comm, ndev, devlist);
  if (rc == ncclSuccess) counts[CommInit] += ndev;
  return rc;
}
ncclResult_t ncclCommDestroy(ncclComm_t comm) {
  static const auto f = next<ncclResult_t (*)(ncclComm_t)>("ncclCommDestroy");
  if (comm) ++counts[CommDestroy];
  return f(comm);
}
}

int main(int argc, char **argv) {
  if (argc < 3) {
    std::fprintf(stderr, "usage: runner_lifetime_check <file.g2o> <gpus>\n");
    return 2;
  }
  size_t n = 0;
  const std::vector<RelativeSEMeasurement> graph = read_g2o_file(argv[1], n);
  if (graph.empty()) return 2;
  const unsigned d = (unsigned)graph[0].t.size(), r = 5, K = 4;
  const Matrix X0 = fixedStiefelVariable(d, r) * chordalInitialization(d, n, graph);
  DeviceRBCDOptions base;
  base.r = r;
  base.gpus = (unsigned)std::atoi(argv[2]);

  // a: the constructor fails in the alignment waves, after the streams, buffers and communicators exist
  std::vector<RelativeSEMeasurement> cut;
  const size_t per = n / K;
  for (const auto &m : graph) {
    const size_t a1 = std::min<size_t>(m.p1 / per, K - 1), a2 = std::min<size_t>(m.p2 / per, K - 1);
    if (a1 == a2 || (a1 != K - 1 && a2 != K - 1)) cut.push_back(m);
  }
  DeviceRBCDOptions oa = base;
  oa.schedule = "coloured";
  oa.initialization = "distributed";
  try {
    DeviceRBCD run(cut, n, K, Matrix(), oa);
  } catch (const std::exception &e) {
    std::printf("error a %s\n", e.what());
  }
  report("a");

  try {
    DeviceRBCDOptions ob = base;
    ob.schedule = "coloured";
    ob.acceleration = true;
    ob.momentumBlocks = "colours";
    {
      DeviceRBCD run(graph, n, K, X0, ob);
      DeviceRBCDSolveOptions so;
      so.maxRounds = 6;
      so.gradnormTol = 0;
      so.relChangeTol = 0;
      run.solve(so);
      run.status();
    }
    report("b");

    DeviceRBCDOptions oc = base;
    oc.schedule = "greedy_set";
    {
      DeviceRBCD run(graph, n, K, X0, oc);
      for (int it = 0; it < 4; ++it) run.step(it % 2 == 1);
      run.selectionLog();
    }
    report("c");
  } catch (const std::exception &e) {
    std::fprintf(stderr, "%s\n", e.what());
    return 1;
  }
  return 0;
}
