// DeviceRBCD.cpp -- device-resident multi-GPU RBCD runner of the C++ host API: iterates stay in HBM, the agents'
// public poses travel by ONE ncclAllGather per round (see include/DPGO/DeviceRBCD.h).
// ref: examples/MultiRobotExample.cpp:63-151 (partition), :229-334 (synchronous driver, greedy selection),
//      src/PGOAgent.cpp:95-105,434-458 (public-pose exchange), :783-859 (G), :1131-1137 (updateX constants).
#include <DPGO/DeviceRBCD.h>
#include <DPGO/QuadraticProblem.h>

#include <nccl.h>

#include <algorithm>
#include <cmath>
#include <map>
#include <memory>
#include <stdexcept>
#include <type_traits>

#include "dpgo_b200.h"

namespace DPGO {

namespace {
void check(int code, const char *what) {
  if (code != DPGO_OK) throw std::runtime_error(std::string(what) + ": " + dpgo_last_error());
}
void checkNccl(ncclResult_t r, const char *what) {
  if (r != ncclSuccess) throw std::runtime_error(std::string(what) + ": " + ncclGetErrorString(r));
}
// the next agent of the greedy schedule (ref examples/MultiRobotExample.cpp:308-325): the largest block gradient norm,
// except that an agent without neighbours stays selected
unsigned greedySelection(unsigned selected, const DeviceRBCDStatus &st, unsigned K, bool hasNeighbours) {
  if (!hasNeighbours) return selected;
  unsigned arg = 0;
  for (unsigned a = 1; a < K; ++a)
    if (std::sqrt(st.at(a, 2)) > std::sqrt(st.at(arg, 2))) arg = a;
  return arg;
}

// Owners of the runner's resources, as in dpo_b200/csrc/dpgo_devbuf.cuh but over the C ABI (this library does not link
// the CUDA runtime).  Dropping one releases what it holds, so a constructor that throws half way leaks nothing.
struct DeviceFree {
  int device = 0;
  void operator()(double *p) const { dpgo_device_free(device, p); }
};
struct StreamDestroy {
  int device = 0;
  void operator()(void *s) const { dpgo_stream_destroy(device, s); }
};
struct PinnedFree { void operator()(double *p) const { dpgo_host_free_pinned(p); } };
struct CommDestroy { void operator()(ncclComm_t c) const { ncclCommDestroy(c); } };
using DeviceBuffer = std::unique_ptr<double, DeviceFree>;
using Stream = std::unique_ptr<void, StreamDestroy>;
using PinnedBuffer = std::unique_ptr<double, PinnedFree>;
using Comm = std::unique_ptr<std::remove_pointer_t<ncclComm_t>, CommDestroy>;

DeviceBuffer deviceBuffer(int device, size_t count) {   // zero-initialised
  void *p = nullptr;
  check(dpgo_device_malloc(device, sizeof(double) * count, &p), "dpgo_device_malloc");
  return DeviceBuffer(static_cast<double *>(p), DeviceFree{device});
}

// An array of `part` doubles per agent that every GPU holds for all K agents (`all`), each GPU writing the parts of its
// own agents into `own()` and one all-gather filling every `all` from them.  One GPU writes straight into `all`.
struct Gathered {
  DeviceBuffer all, ownParts;      // ownParts: more than one GPU only
  double *own() const { return ownParts ? ownParts.get() : all.get(); }
};
Gathered gathered(int device, size_t part, unsigned K, unsigned perGpu) {
  Gathered b;
  b.all = deviceBuffer(device, K * part);
  if (perGpu < K) b.ownParts = deviceBuffer(device, perGpu * part);
  return b;
}

// One GPU: its stream, buffers and communicator (released in reverse order: communicator, buffers, stream), and the
// fixed arguments of the calls that take every agent of its contiguous block first .. first + perGpu - 1.
struct Gpu {
  Stream stream;
  Gathered tiles;                  // the agents' padded public tiles of X (slotElems doubles each)
  Gathered auxTiles;               // accelerated rounds: the public tiles of Y
  Gathered records;                // status records, DPGO_STATUS_DOUBLES each
  Comm comm;                       // more than one GPU only
  unsigned first = 0;
  std::vector<dpgo_problem *> handles;
  std::vector<int32_t> ids;        // first, first + 1, ...
  std::vector<double *> tileDst, auxTileDst;   // each agent's slot in tiles.own() / auxTiles.own()
};
}  // namespace

struct DeviceRBCD::Impl {
  unsigned d = 3, r = 5, dh = 4, ts = 20, K = 1, N = 1, perGpu = 1, pmax = 1;
  size_t n = 0;
  std::vector<RelativeSEMeasurement> graph;       // the global pose graph (poseCovariances)
  size_t slotElems = 0;            // one agent's padded public tiles: pmax * ts doubles
  int64_t numSlots = 0;            // the slots of a gathered tile buffer: K * pmax
  std::string schedule;
  std::vector<std::unique_ptr<PGOAgent>> agents;
  std::vector<size_t> count;
  std::vector<std::vector<size_t>> globalOf;      // agent -> global pose ids in local order
  std::vector<dpgo_problem *> h;
  std::vector<Gpu> gpu;
  std::vector<int32_t> slots;      // 0 .. perGpu - 1: a GPU's agents' places in its status records
  PinnedBuffer statusHost;         // all agents' records in agent order
  bool acceleration = false;
  unsigned restartInterval = 30;
  double momentumN = 1;
  bool colourMomentum = false;     // momentumBlocks == "colours"
  std::vector<std::vector<unsigned>> neighbors;
  dpgo_opt_params_t prm;
  unsigned selected = 0;
  bool concurrent = false;         // active agents of a GPU side by side (cluster launches, own streams)
  bool gatheredCurrent = false;    // the gathered buffers hold every agent's current public tiles
  bool recordsCurrent = false;     // records.all holds the records of the current iterates

  // also when the constructor throws: the agents' problems run on the GPU streams, so they go before the members
  ~Impl() {
    for (unsigned g = 0; g < gpu.size(); ++g)
      if (gpu[g].stream) dpgo_stream_synchronize((int)g, gpu[g].stream.get());   // errors ignored
    agents.clear();
  }

  double *tileDst(unsigned a) const {
    const Gpu &G = gpu[a / perGpu];
    return G.tileDst[a - G.first];
  }
  // one ncclAllGather group: every GPU's own parts of `buf` (`part` doubles per agent) into every GPU's copy of all
  void allGather(Gathered Gpu::*buf, size_t part) {
    if (N == 1) return;
    checkNccl(ncclGroupStart(), "ncclGroupStart");
    for (unsigned g = 0; g < N; ++g) {
      check(dpgo_device_set((int)g), "dpgo_device_set");
      const Gathered &b = gpu[g].*buf;
      checkNccl(ncclAllGather(b.own(), b.all.get(), (size_t)perGpu * part, ncclDouble, gpu[g].comm.get(),
                              (cudaStream_t)gpu[g].stream.get()),
                "ncclAllGather");
    }
    checkNccl(ncclGroupEnd(), "ncclGroupEnd");
  }
  void buildG() {                  // every agent's G from the gathered tiles
    for (unsigned a = 0; a < K; ++a)
      check(dpgo_agent_build_G(h[a], gpu[a / perGpu].tiles.all.get(), numSlots), "dpgo_agent_build_G");
  }
};

DeviceRBCD::DeviceRBCD(const std::vector<RelativeSEMeasurement> &graph, size_t n, unsigned numAgents, const Matrix &XInit,
                       const DeviceRBCDOptions &opt)
    : impl(new Impl()) {
  Impl &I = *impl;
  if (graph.empty()) throw std::runtime_error("DeviceRBCD: empty pose graph");
  I.d = (unsigned)graph[0].t.size();
  I.graph = graph;
  I.r = opt.r;
  I.dh = I.d + 1;
  I.ts = I.r * I.dh;
  I.K = numAgents;
  I.N = std::max(1u, opt.gpus);
  I.n = n;
  I.schedule = opt.schedule;
  if (I.schedule != "greedy" && I.schedule != "coloured" && I.schedule != "parallel" && I.schedule != "greedy_set")
    throw std::runtime_error("DeviceRBCD: schedule must be greedy, coloured, parallel or greedy_set");
  if (I.schedule == "greedy_set" && opt.acceleration)
    throw std::invalid_argument("DeviceRBCD: acceleration is not supported with the greedy_set schedule: the Nesterov momentum "
                                "assumes a fixed block set per round");
  if (I.K == 0 || n / I.K == 0) throw std::runtime_error("DeviceRBCD: more agents than poses");
  const bool distributed = (opt.initialization == "distributed");
  if (!distributed && opt.initialization != "central")
    throw std::runtime_error("DeviceRBCD: initialization must be central or distributed");
  if (distributed && XInit.size() != 0)
    throw std::runtime_error("DeviceRBCD: the distributed initialisation computes the start itself: XInit must be empty");
  if (!distributed && ((size_t)XInit.rows() != opt.r || (size_t)XInit.cols() != (graph[0].t.size() + 1) * n))
    throw std::runtime_error("DeviceRBCD: XInit must be r x (d+1)n");
  if (I.K % I.N != 0) throw std::runtime_error("DeviceRBCD: the agents must divide evenly over the GPUs");
  if (opt.momentumBlocks != "agents" && opt.momentumBlocks != "colours")
    throw std::invalid_argument("DeviceRBCD: momentumBlocks must be agents or colours");
  if (opt.momentumBlocks == "colours" && I.schedule != "coloured")
    throw std::invalid_argument("DeviceRBCD: momentumBlocks = colours counts the colour classes of the coloured schedule");
  if (opt.acceleration && opt.restartInterval < 1) throw std::invalid_argument("DeviceRBCD: restartInterval must be >= 1");
  I.acceleration = opt.acceleration;
  I.colourMomentum = opt.momentumBlocks == "colours";
  I.restartInterval = opt.restartInterval;
  int ndev = 0;
  check(dpgo_device_count(&ndev), "dpgo_device_count");
  if ((int)I.N > ndev) throw std::runtime_error("DeviceRBCD: fewer CUDA devices than requested GPUs");
  I.perGpu = I.K / I.N;
  const unsigned K = I.K, d = I.d, dh = I.dh, r = I.r;

  // ---- ownership: partition file or contiguous ranges (ref examples/MultiRobotExample.cpp:76-151) ----
  const size_t per = n / K;
  std::vector<unsigned> owner(n), local(n);
  if (!opt.owner.empty() && opt.owner.size() != n) throw std::runtime_error("DeviceRBCD: owner map must have one entry per pose");
  I.count.assign(K, 0);
  for (size_t g = 0; g < n; ++g) {
    owner[g] = opt.owner.empty() ? (unsigned)std::min<size_t>(g / per, K - 1) : opt.owner[g];
    if (owner[g] >= K) throw std::runtime_error("DeviceRBCD: agent id out of range in the owner map");
    local[g] = (unsigned)I.count[owner[g]]++;
  }
  I.globalOf.assign(K, {});
  for (size_t g = 0; g < n; ++g) I.globalOf[owner[g]].push_back(g);
  std::vector<std::vector<RelativeSEMeasurement>> odo(K), priv(K), shared(K);
  for (const auto &e : graph) {
    const unsigned a1 = owner[e.p1], a2 = owner[e.p2];
    RelativeSEMeasurement m(a1, a2, local[e.p1], local[e.p2], e.R, e.t, e.kappa, e.tau);
    m.weight = e.weight;
    if (a1 != a2) { shared[a1].push_back(m); shared[a2].push_back(m); }
    else if (e.p1 + 1 == e.p2) odo[a1].push_back(m);
    else priv[a1].push_back(m);
  }

  // ---- agent graph and its greedy colouring in agent order (needed before the agents exist: it decides the launch mode) ----
  I.neighbors.assign(K, {});
  for (unsigned a = 0; a < K; ++a) {
    for (const auto &m : shared[a]) I.neighbors[a].push_back((unsigned)(m.r1 == a ? m.r2 : m.r1));
    std::sort(I.neighbors[a].begin(), I.neighbors[a].end());
    I.neighbors[a].erase(std::unique(I.neighbors[a].begin(), I.neighbors[a].end()), I.neighbors[a].end());
  }
  mColour.assign(K, 0);
  {
    std::vector<int> col(K, -1);
    for (unsigned a = 0; a < K; ++a) {
      int c = 0;
      for (bool clash = true; clash; ) {
        clash = false;
        for (unsigned b : I.neighbors[a])
          if (col[b] == c) { clash = true; ++c; break; }
      }
      col[a] = c;
      mColour[a] = (unsigned)c;
      mNumColours = std::max(mNumColours, (unsigned)c + 1);
    }
  }
  {
    unsigned most = 1;
    if (I.schedule == "coloured")
      for (unsigned g = 0; g < I.N; ++g)
        for (unsigned c = 0; c < mNumColours; ++c) {
          unsigned cnt = 0;
          for (unsigned a = g * I.perGpu; a < (g + 1) * I.perGpu; ++a) cnt += (mColour[a] == c);
          most = std::max(most, cnt);
        }
    if (I.schedule == "greedy_set")                      // some GPU hosts two agents that are not neighbours
      for (unsigned g = 0; g < I.N; ++g)
        for (unsigned a = g * I.perGpu; a < (g + 1) * I.perGpu; ++a)
          for (unsigned b = a + 1; b < (g + 1) * I.perGpu; ++b)
            if (!std::binary_search(I.neighbors[a].begin(), I.neighbors[a].end(), b)) most = 2;
    const bool agentMomentum = opt.acceleration && opt.momentumBlocks == "agents";
    I.concurrent = opt.concurrent < 0 ? (most >= 2 && !agentMomentum) : (opt.concurrent != 0);
    if (I.concurrent && I.schedule == "parallel")
      throw std::runtime_error("DeviceRBCD: concurrent rounds are implemented for the greedy and coloured schedules");
  }

  // ---- distributed initialisation: every private graph must be connected, or its chordal initialisation is singular ----
  if (distributed)
    for (unsigned a = 0; a < K; ++a) {
      std::vector<size_t> root(I.count[a]);
      for (size_t q = 0; q < root.size(); ++q) root[q] = q;
      auto find = [&](size_t q) { while (root[q] != q) q = root[q] = root[root[q]]; return q; };
      size_t pieces = root.size();
      for (const auto *set : {&odo[a], &priv[a]})
        for (const auto &m : *set) {
          const size_t x = find(m.p1), y = find(m.p2);
          if (x != y) { root[x] = y; --pieces; }
        }
      if (pieces > 1)
        throw std::runtime_error("DeviceRBCD: agent " + std::to_string(a) + ": the private pose graph (odometry + private loop "
                                 "closures) has " + std::to_string(pieces) + " connected components, so its local chordal "
                                 "initialisation is singular");
    }

  // ---- streams, agents (Q on the agent's GPU), resident iterates ----
  I.gpu.resize(I.N);
  for (unsigned g = 0; g < I.N; ++g) {
    void *s = nullptr;
    check(dpgo_stream_create((int)g, &s), "dpgo_stream_create");
    I.gpu[g].stream = Stream(s, StreamDestroy{(int)g});
    I.gpu[g].first = g * I.perGpu;
  }
  I.h.assign(K, nullptr);
  Matrix lift;
  for (unsigned a = 0; a < K; ++a) {
    Gpu &G = I.gpu[a / I.perGpu];
    PGOAgentParameters prm(d, r, K);
    prm.algorithm = opt.algorithm;
    prm.preconditioner = opt.preconditioner;
    prm.device = (int)(a / I.perGpu);
    prm.cluster = I.concurrent;
    I.agents.emplace_back(new PGOAgent(a, prm));
    if (a == 0) I.agents[0]->getLiftingMatrix(lift);
    else I.agents[a]->setLiftingMatrix(lift);
    // a zero trajectory of the right shape skips the agent's own host chordal initialisation: X comes from XInit, or from
    // the GPU chordal initialisation and the alignment waves
    I.agents[a]->setPoseGraph(odo[a], priv[a], shared[a], Matrix::Zero(d, dh * I.count[a]));
    I.h[a] = I.agents[a]->problem()->handle();
    if (!I.h[a]) throw std::runtime_error("DeviceRBCD: agent without a device problem");
    check(dpgo_problem_set_stream(I.h[a], G.stream.get()), "dpgo_problem_set_stream");
    G.handles.push_back(I.h[a]);
    G.ids.push_back((int32_t)a);
    if (!distributed) {
      Matrix Xa0(r, dh * I.count[a]);
      for (size_t q = 0; q < I.count[a]; ++q) Xa0.block(0, q * dh, r, dh) = Matrix(XInit).block(0, I.globalOf[a][q] * dh, r, dh);
      I.agents[a]->setX(Xa0);
      Matrix Xa;
      I.agents[a]->getX(Xa);
      check(dpgo_problem_upload_X(I.h[a], Xa.data()), "dpgo_problem_upload_X");
      continue;
    }
    // ref localInitialization, src/PGOAgent.cpp:947-962: chordal initialisation of the private graph on the agent's GPU
    const size_t na = I.count[a];
    Matrix T = Matrix::Zero(d, dh * na);
    for (unsigned k = 0; k < d; ++k) T(k, k) = 1.0;
    if (na > 1) {
      std::vector<int32_t> p1, p2;
      std::vector<double> R, t, kap, tau;
      for (const auto *set : {&odo[a], &priv[a]})
        for (const auto &m : *set) {
          p1.push_back((int32_t)m.p1); p2.push_back((int32_t)m.p2);
          for (unsigned i = 0; i < d; ++i) {
            for (unsigned j = 0; j < d; ++j) R.push_back(m.R(i, j));
            t.push_back(m.t(i));
          }
          kap.push_back(m.weight * m.kappa); tau.push_back(m.weight * m.tau);
        }
      if (dpgo_chordal_initialization((int)na, (int)d, (int64_t)p1.size(), p1.data(), p2.data(), R.data(), t.data(), kap.data(),
                                      tau.data(), prm.device, 0.0, 0, T.data(), nullptr) != DPGO_OK)
        throw std::runtime_error(std::string("dpgo_chordal_initialization: ") + dpgo_chordal_last_error());
    }
    check(dpgo_agent_set_local_trajectory(I.h[a], T.data(), lift.data()), "dpgo_agent_set_local_trajectory");
  }

  // ---- exchange plan: public poses, padded slots, per-agent edge tables ----
  std::vector<std::vector<int32_t>> pub(K);
  for (unsigned a = 0; a < K; ++a) {
    for (const auto &m : shared[a]) pub[a].push_back((int32_t)(m.r1 == a ? m.p1 : m.p2));
    std::sort(pub[a].begin(), pub[a].end());
    pub[a].erase(std::unique(pub[a].begin(), pub[a].end()), pub[a].end());
    I.pmax = std::max<unsigned>(I.pmax, (unsigned)pub[a].size());
  }
  for (unsigned a = 0; a < K; ++a) {
    const size_t m = shared[a].size();
    std::vector<int32_t> loc(m), slot(m), outg(m);
    std::vector<double> T(m * dh * dh, 0.0), om(m * dh, 0.0);
    for (size_t e = 0; e < m; ++e) {
      const RelativeSEMeasurement &s = shared[a][e];
      const bool out = (s.r1 == a);
      const unsigned b = (unsigned)(out ? s.r2 : s.r1);
      const int32_t q = (int32_t)(out ? s.p2 : s.p1);
      loc[e] = (int32_t)(out ? s.p1 : s.p2);
      const auto it = std::lower_bound(pub[b].begin(), pub[b].end(), q);
      slot[e] = (int32_t)(b * I.pmax + (unsigned)(it - pub[b].begin()));
      outg[e] = out ? 1 : 0;
      for (unsigned i = 0; i < d; ++i) {
        for (unsigned j = 0; j < d; ++j) T[e * dh * dh + i * dh + j] = s.R(i, j);
        T[e * dh * dh + i * dh + d] = s.t(i);
        om[e * dh + i] = s.weight * s.kappa;
      }
      T[e * dh * dh + d * dh + d] = 1.0;
      om[e * dh + d] = s.weight * s.tau;
    }
    check(dpgo_agent_set_public_poses(I.h[a], (int)pub[a].size(), pub[a].data()), "dpgo_agent_set_public_poses");
    check(dpgo_agent_set_shared_edges(I.h[a], (int)m, loc.data(), slot.data(), outg.data(), T.data(), om.data()),
          "dpgo_agent_set_shared_edges");
  }
  // ---- exchange and status buffers, communicators ----
  constexpr unsigned S = DPGO_STATUS_DOUBLES;
  I.slotElems = (size_t)I.pmax * I.ts;
  I.numSlots = (int64_t)K * I.pmax;
  for (unsigned g = 0; g < I.N; ++g) {
    Gpu &G = I.gpu[g];
    G.tiles = gathered((int)g, I.slotElems, K, I.perGpu);
    if (I.acceleration) G.auxTiles = gathered((int)g, I.slotElems, K, I.perGpu);
    G.records = gathered((int)g, S, K, I.perGpu);
    for (unsigned i = 0; i < I.perGpu; ++i) {
      G.tileDst.push_back(G.tiles.own() + i * I.slotElems);
      if (I.acceleration) G.auxTileDst.push_back(G.auxTiles.own() + i * I.slotElems);
    }
  }
  for (unsigned i = 0; i < I.perGpu; ++i) I.slots.push_back((int32_t)i);
  void *hp = nullptr;
  check(dpgo_host_alloc_pinned(sizeof(double) * S * K, &hp), "dpgo_host_alloc_pinned");
  I.statusHost.reset(static_cast<double *>(hp));
  if (I.N > 1) {
    std::vector<int> devs(I.N);
    std::vector<ncclComm_t> comm(I.N, nullptr);
    for (unsigned g = 0; g < I.N; ++g) devs[g] = (int)g;
    checkNccl(ncclCommInitAll(comm.data(), (int)I.N, devs.data()), "ncclCommInitAll");
    for (unsigned g = 0; g < I.N; ++g) I.gpu[g].comm.reset(comm[g]);
  }
  if (distributed) {
    // candidate tables (ref computeNeighborTransform / findSharedLoopClosureWithNeighbor, src/PGOAgent.cpp:250-288,922-934):
    // one candidate per public pose (b, j) of a neighbour the agent shares an edge with, through the FIRST such edge,
    // grouped per neighbour in increasing id, j increasing (std::map order)
    for (unsigned a = 0; a < K; ++a) {
      std::map<std::pair<unsigned, int32_t>, size_t> first;
      for (size_t e = 0; e < shared[a].size(); ++e) {
        const RelativeSEMeasurement &s = shared[a][e];
        const bool out = (s.r1 == a);
        first.emplace(std::make_pair((unsigned)(out ? s.r2 : s.r1), (int32_t)(out ? s.p2 : s.p1)), e);
      }
      std::vector<int32_t> grp, ptr, loc, slot, outg;
      std::vector<double> T;
      for (const auto &kv : first) {
        const unsigned b = kv.first.first;
        if (grp.empty() || grp.back() != (int32_t)b) { grp.push_back((int32_t)b); ptr.push_back((int32_t)loc.size()); }
        const RelativeSEMeasurement &s = shared[a][kv.second];
        const bool out = (s.r1 == a);
        loc.push_back((int32_t)(out ? s.p1 : s.p2));
        const auto it = std::lower_bound(pub[b].begin(), pub[b].end(), kv.first.second);
        slot.push_back((int32_t)(b * I.pmax + (unsigned)(it - pub[b].begin())));
        outg.push_back(out ? 1 : 0);
        for (unsigned i = 0; i <= d; ++i)
          for (unsigned j = 0; j <= d; ++j)
            T.push_back(i < d ? (j < d ? s.R(i, j) : s.t(i)) : (j == d ? 1.0 : 0.0));
      }
      ptr.push_back((int32_t)loc.size());
      check(dpgo_agent_set_align_candidates(I.h[a], (int)grp.size(), grp.data(), ptr.data(), loc.data(), slot.data(), outg.data(),
                                            T.data()),
            "dpgo_agent_set_align_candidates");
    }
    alignWaves();
  }
  if (I.acceleration) {
    I.momentumN = opt.momentumBlocks == "colours" ? (double)mNumColours : (double)K;
    for (unsigned a = 0; a < K; ++a) check(dpgo_agent_accel_init(I.h[a]), "dpgo_agent_accel_init");
  }
  if (I.schedule == "greedy_set") {                     // the agent graph in CSR form, with each GPU's first agent
    std::vector<int32_t> ptr{0}, adj;
    for (unsigned a = 0; a < K; ++a) {
      for (unsigned b : I.neighbors[a]) adj.push_back((int32_t)b);
      ptr.push_back((int32_t)adj.size());
    }
    for (const Gpu &G : I.gpu)
      check(dpgo_agents_set_agent_graph(G.handles[0], (int)K, ptr.data(), adj.data()), "dpgo_agents_set_agent_graph");
  }
  dpgo_opt_params_default(&I.prm);
  I.prm.algorithm = (opt.algorithm == ROPTALG::RTR) ? DPGO_ALG_RTR : DPGO_ALG_RGD;
  I.prm.precond = (int)opt.preconditioner;
  I.prm.tr_tolerance = 1e-2;          // ref src/PGOAgent.cpp:1134-1137
  I.prm.tr_iterations = 1;
  I.prm.tr_max_inner = 10;
  I.prm.tr_initial_radius = 100;
}

DeviceRBCD::~DeviceRBCD() = default;

// Wave w >= 1 (ref src/PGOAgent.cpp:369-440, examples/MultiRobotExample.cpp:245-256): one exchange of the public tiles;
// every agent that is not initialised and has a neighbour initialised before the wave tries those neighbours in increasing
// id, all such agents of a GPU in one dpgo_agents_align_async call; the first neighbour with inliers wins.  At most K - 1
// waves: a wave that initialises nobody is an error.
void DeviceRBCD::alignWaves() {
  Impl &I = *impl;
  std::vector<int32_t> ready(I.K, 0);
  ready[0] = 1;
  mInitReport.assign(I.K, DeviceRBCDInitRecord());
  mInitReport[0].wave = 0;
  for (int wave = 1; std::find(ready.begin(), ready.end(), 0) != ready.end(); ++wave) {
    exchange();
    std::vector<unsigned> todo;
    for (unsigned a = 0; a < I.K; ++a) {
      if (ready[a]) continue;
      for (unsigned b : I.neighbors[a])
        if (ready[b]) { todo.push_back(a); break; }
    }
    for (unsigned g = 0; g < I.N; ++g) {
      std::vector<dpgo_problem *> hs;
      for (unsigned a : todo)
        if (a / I.perGpu == g) hs.push_back(I.h[a]);
      if (!hs.empty())
        check(dpgo_agents_align_async(hs.data(), (int)hs.size(), I.gpu[g].tiles.all.get(), I.numSlots, ready.data(), (int)I.K,
                                      I.gpu[g].stream.get()),
              "dpgo_agents_align_async");
    }
    std::vector<unsigned> newly;
    for (unsigned a : todo) {
      int32_t info[4];
      check(dpgo_agent_align_result(I.h[a], nullptr, info), "dpgo_agent_align_result");
      DeviceRBCDInitRecord &rec = mInitReport[a];
      rec.neighbor = info[0]; rec.candidates = info[1]; rec.inliers = info[2]; rec.iterations = info[3];
      if (info[2] > 0) { rec.wave = wave; newly.push_back(a); }
    }
    if (newly.empty()) {
      std::string rest;
      for (unsigned a = 0; a < I.K; ++a)
        if (!ready[a]) rest += (rest.empty() ? "" : ", ") + std::to_string(a);
      throw std::runtime_error("DeviceRBCD: distributed initialisation: agents [" + rest + "] cannot join the global frame "
                               "(no initialised neighbour gives a non-empty inlier set; is the agent graph connected?)");
    }
    for (unsigned a : newly) ready[a] = 1;
  }
  for (unsigned a = 0; a < I.K; ++a) {                 // the host copy of every agent's iterate, as setX leaves it
    Matrix Xa(I.r, I.dh * I.count[a]);
    check(dpgo_problem_download_X(I.h[a], Xa.data()), "dpgo_problem_download_X");
    I.agents[a]->setX(Xa);
  }
}

size_t DeviceRBCD::allGatherBytesPerGpu() const { return sizeof(double) * impl->perGpu * impl->slotElems; }

void DeviceRBCD::exchange() {
  Impl &I = *impl;
  for (unsigned a = 0; a < I.K; ++a) check(dpgo_agent_pack_public(I.h[a], I.tileDst(a)), "dpgo_agent_pack_public");
  I.allGather(&Gpu::tiles, I.slotElems);
  I.buildG();
}

void DeviceRBCD::sync() {
  Impl &I = *impl;
  for (unsigned g = 0; g < I.N; ++g) check(dpgo_stream_synchronize((int)g, I.gpu[g].stream.get()), "dpgo_stream_synchronize");
}

static std::vector<unsigned> activeSet(const std::string &schedule, unsigned K, unsigned selected, unsigned round,
                                       const std::vector<unsigned> &colour, unsigned ncolours) {
  std::vector<unsigned> act;
  if (schedule == "greedy") act.push_back(selected);
  else
    for (unsigned a = 0; a < K; ++a)
      if (schedule == "parallel" || colour[a] == round % ncolours) act.push_back(a);
  return act;
}

bool DeviceRBCD::concurrent() const { return impl->concurrent; }

// one accelerated round: per GPU one begin call (momentum, Y, the idle agents' iterate(false), packs of the X and Y tiles),
// one all-gather group per buffer, per GPU one call for the active agents (G from the Y tiles, step from Y, V, restart)
void DeviceRBCD::roundAccelerated(const std::vector<unsigned> &active) {
  Impl &I = *impl;
  for (Gpu &G : I.gpu) {
    std::vector<int32_t> flags;
    for (int32_t a : G.ids) flags.push_back(std::find(active.begin(), active.end(), (unsigned)a) != active.end() ? 1 : 0);
    check(dpgo_agents_accel_begin_async(G.handles.data(), (int)G.handles.size(), flags.data(), I.momentumN,
                                        (int)I.restartInterval, G.tileDst.data(), G.auxTileDst.data(), G.stream.get()),
          "dpgo_agents_accel_begin_async");
  }
  I.allGather(&Gpu::tiles, I.slotElems);
  I.allGather(&Gpu::auxTiles, I.slotElems);
  for (unsigned g = 0; g < I.N; ++g) {
    std::vector<dpgo_problem *> hs;
    for (unsigned a : active)
      if (a / I.perGpu == g) hs.push_back(I.h[a]);
    if (hs.empty()) continue;
    check(dpgo_agents_accel_round_async(hs.data(), (int)hs.size(), &I.prm, I.gpu[g].tiles.all.get(), I.gpu[g].auxTiles.all.get(),
                                        I.numSlots, I.gpu[g].stream.get()),
          "dpgo_agents_accel_round_async");
  }
  I.gatheredCurrent = false;                           // the gathered X tiles predate the active agents' steps
}

// one round of the schedule's active agents, asynchronous on the GPU streams.  A plain round starts from the current
// gathered tiles (one exchange first when they are not) and keeps them current: per GPU ONE dpgo_agents_round_async call
// (G rebuild -> RTR step -> pack per active agent), then the all-gather that publishes the new public tiles.
std::vector<unsigned> DeviceRBCD::issueRound() {
  Impl &I = *impl;
  if (I.schedule == "greedy_set") {
    selectRound();
    return {};
  }
  I.recordsCurrent = false;
  const std::vector<unsigned> active = activeSet(I.schedule, I.K, I.selected, mRound, mColour, mNumColours);
  if (I.acceleration) {
    roundAccelerated(active);
  } else {
    if (!I.gatheredCurrent) { exchange(); I.gatheredCurrent = true; }
    for (unsigned g = 0; g < I.N; ++g) {
      std::vector<dpgo_problem *> hs;
      std::vector<double *> dst;
      for (unsigned a : active)
        if (a / I.perGpu == g) {
          hs.push_back(I.h[a]);
          dst.push_back(I.tileDst(a));
        }
      if (hs.empty()) continue;
      check(dpgo_agents_round_async(hs.data(), (int)hs.size(), &I.prm, I.gpu[g].tiles.all.get(), I.numSlots, dst.data(),
                                    I.gpu[g].stream.get(), I.schedule == "parallel"),
            "dpgo_agents_round_async");
    }
    I.allGather(&Gpu::tiles, I.slotElems);
  }
  ++mRound;
  return active;
}

// one greedy_set round: the status records of the current iterates on every GPU (skipped when current; N > 1: one
// all-gather group of the records), per GPU ONE dpgo_agents_select_round_async call (selection on the device, then the
// gated G rebuild -> step -> pack of every agent of the GPU), then the all-gather of the new public tiles.  No host
// synchronisation: the round's agents are in the selection log.
void DeviceRBCD::selectRound() {
  Impl &I = *impl;
  if (!I.gatheredCurrent) { exchange(); I.gatheredCurrent = true; }
  if (!I.recordsCurrent) statusDevice();
  for (Gpu &G : I.gpu)
    check(dpgo_agents_select_round_async(G.handles.data(), (int)G.handles.size(), G.ids.data(), &I.prm, G.records.all.get(),
                                         G.tiles.all.get(), I.numSlots, G.tileDst.data(), G.stream.get()),
          "dpgo_agents_select_round_async");
  I.allGather(&Gpu::tiles, I.slotElems);
  I.recordsCurrent = false;
  ++mRound;
}

std::vector<std::vector<unsigned>> DeviceRBCD::selectionLog(unsigned first, unsigned count) {
  Impl &I = *impl;
  if (I.schedule != "greedy_set") throw std::invalid_argument("DeviceRBCD::selectionLog: needs the greedy_set schedule");
  int64_t total = 0;
  check(dpgo_agents_selection_log(I.h[0], 0, 0, nullptr, &total), "dpgo_agents_selection_log");
  const int64_t rows = std::max<int64_t>(0, std::min<int64_t>(count, total - (int64_t)first));
  std::vector<uint8_t> buf((size_t)std::max<int64_t>(rows, 1) * I.K);
  if (rows > 0) check(dpgo_agents_selection_log(I.h[0], first, rows, buf.data(), &total), "dpgo_agents_selection_log");
  std::vector<std::vector<unsigned>> out((size_t)rows);
  for (int64_t q = 0; q < rows; ++q)
    for (unsigned a = 0; a < I.K; ++a)
      if (buf[(size_t)q * I.K + a]) out[(size_t)q].push_back(a);
  return out;
}

void DeviceRBCD::runRounds(unsigned rounds) {
  for (unsigned it = 0; it < rounds; ++it) issueRound();
}

DeviceRBCDStats DeviceRBCD::step(bool evaluate) {
  Impl &I = *impl;
  DeviceRBCDStats st;
  st.active = issueRound();
  if (!evaluate) return st;
  const DeviceRBCDStatus s = status();
  st.cost = s.cost;
  st.gradnorm = s.gradnorm;
  if (I.schedule == "greedy_set") st.active = selectionLog(mRound - 1, 1)[0];
  if (I.schedule == "greedy") I.selected = greedySelection(I.selected, s, I.K, !I.neighbors[I.selected].empty());
  return st;
}

Matrix DeviceRBCD::assemble() {
  Impl &I = *impl;
  Matrix X(I.r, I.dh * I.n);
  for (unsigned a = 0; a < I.K; ++a) {
    Matrix Xa(I.r, I.dh * I.count[a]);
    check(dpgo_problem_download_X(I.h[a], Xa.data()), "dpgo_problem_download_X");
    for (size_t q = 0; q < I.count[a]; ++q) X.block(0, I.globalOf[a][q] * I.dh, I.r, I.dh) = Xa.block(0, q * I.dh, I.r, I.dh);
  }
  return X;
}

// ---- running to convergence -------------------------------------------------------------------------------------------
DeviceRBCDStatus DeviceRBCD::status() {
  Impl &I = *impl;
  constexpr unsigned S = DPGO_STATUS_DOUBLES;
  statusDevice();
  for (unsigned g = 0; g < I.N; ++g)
    check(dpgo_copy_to_host_async((int)g, I.statusHost.get() + (size_t)g * I.perGpu * S, I.gpu[g].records.own(),
                                  sizeof(double) * S * I.perGpu, I.gpu[g].stream.get()),
          "dpgo_copy_to_host_async");
  sync();
  DeviceRBCDStatus st;
  st.records.assign(I.statusHost.get(), I.statusHost.get() + (size_t)S * I.K);
  double gn2 = 0;
  for (unsigned a = 0; a < I.K; ++a) {
    st.cost += st.at(a, 0) + st.at(a, 1);
    gn2 += st.at(a, 2);
  }
  st.gradnorm = std::sqrt(gn2);
  return st;
}

// every agent's status record on the device (G first, from the current tiles), N > 1: all-gathered; no synchronisation
void DeviceRBCD::statusDevice() {
  Impl &I = *impl;
  if (I.gatheredCurrent) {
    I.buildG();
  } else {
    exchange();
    I.gatheredCurrent = true;
  }
  for (Gpu &G : I.gpu)
    check(dpgo_agents_status_async(G.handles.data(), (int)G.handles.size(), I.slots.data(), G.records.own(), G.stream.get()),
          "dpgo_agents_status_async");
  I.allGather(&Gpu::records, DPGO_STATUS_DOUBLES);
  I.recordsCurrent = true;
}

DeviceRBCDSolveReport DeviceRBCD::solve(const DeviceRBCDSolveOptions &o) {
  Impl &I = *impl;
  if (I.acceleration && !I.colourMomentum)
    throw std::invalid_argument("DeviceRBCD::solve: acceleration is supported only with the coloured schedule and "
                                "momentumBlocks = colours; drive other accelerated runs with step()");
  if (o.maxRounds < 1 || o.checkEvery < 1) throw std::invalid_argument("DeviceRBCD::solve: maxRounds and checkEvery must be >= 1");
  if (I.schedule == "greedy" && o.checkEvery != 1)
    throw std::invalid_argument("DeviceRBCD::solve: the greedy schedule selects the next agent from every round's status: "
                                "checkEvery must be 1");
  const DeviceRBCDStatus st0 = status();
  std::vector<double> callsAtStart(I.K);
  for (unsigned a = 0; a < I.K; ++a) callsAtStart[a] = st0.at(a, 4);
  DeviceRBCDSolveReport rep;
  while (true) {
    issueRound();
    ++rep.rounds;
    if (rep.rounds % o.checkEvery != 0 && rep.rounds < o.maxRounds) continue;
    const DeviceRBCDStatus st = status();
    if (o.callback) o.callback(rep.rounds, st.cost, st.gradnorm);
    if (I.schedule == "greedy") I.selected = greedySelection(I.selected, st, I.K, !I.neighbors[I.selected].empty());
    bool team = o.relChangeTol > 0;
    for (unsigned a = 0; a < I.K && team; ++a) team = st.at(a, 4) > callsAtStart[a] && st.at(a, 3) <= o.relChangeTol;
    if (o.gradnormTol > 0 && st.gradnorm < o.gradnormTol) rep.reason = "gradnorm";
    else if (team) rep.reason = "team";
    else if (rep.rounds >= o.maxRounds) rep.reason = "max_rounds";
    if (!rep.reason.empty()) {
      rep.cost = st.cost;
      rep.gradnorm = st.gradnorm;
      rep.relativeChange.resize(I.K);
      for (unsigned a = 0; a < I.K; ++a) rep.relativeChange[a] = st.at(a, 3);
      return rep;
    }
  }
}

Matrix DeviceRBCD::trajectory() {
  Impl &I = *impl;
  Matrix X0(I.r, I.dh * I.count[0]);
  check(dpgo_problem_download_X(I.h[0], X0.data()), "dpgo_problem_download_X");
  std::vector<double> anchor(X0.data(), X0.data() + (size_t)I.r * I.dh);    // agent 0's pose 0, r x (d+1) column-major
  Matrix T(I.d, I.dh * I.n);
  for (unsigned a = 0; a < I.K; ++a) {
    Matrix Ta(I.d, I.dh * I.count[a]);
    check(dpgo_agent_trajectory_global(I.h[a], anchor.data(), Ta.data()), "dpgo_agent_trajectory_global");
    for (size_t q = 0; q < I.count[a]; ++q) T.block(0, I.globalOf[a][q] * I.dh, I.d, I.dh) = Ta.block(0, q * I.dh, I.d, I.dh);
  }
  return T;
}

PoseCovariances DeviceRBCD::poseCovariances(long anchor, const std::vector<std::pair<size_t, size_t>> &pairs) {
  Impl &I = *impl;
  const Matrix T = trajectory();
  const size_t a = anchor < 0 ? I.globalOf[0][0] : (size_t)anchor;
  return poseCovariancesGPU(I.d, I.n, I.graph, T, a, pairs, 0);
}

}  // namespace DPGO
