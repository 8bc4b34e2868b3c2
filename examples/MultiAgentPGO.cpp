// MultiAgentPGO -- command-line driver of the GPU distributed pose-graph optimiser (C++ host API).
//
//   MultiAgentPGO <file.g2o> [--robots K] [--iters N] [--stop GRADNORM] [--accel] [--rgd] [--jacobi]
//                 [--rank R] [--trace out.csv] [--resident [--gpus N] [--schedule greedy|coloured|parallel|greedy_set] [--bench ROUNDS]
//                                                           [--partition FILE] [--init central|distributed]]
//
// --resident runs the device-resident multi-GPU runner (DPGO::DeviceRBCD): iterates stay in HBM, K agents over N GPUs
// of this node, ONE ncclAllGather of the public poses per round; --bench times ROUNDS rounds without the central
// evaluation.  --init distributed starts it from the reference's multi-robot initialisation (per-agent chordal
// initialisation on the GPUs, then frame-alignment waves) instead of the centralised chordal relaxation, and prints one
// "init <agent> <wave> <neighbour> <candidates> <inliers> <GNC iterations>" line per agent.
//
// Splits the pose graph into K contiguous agents, initialises every agent from the centralised chordal
// relaxation lifted to rank R, then runs synchronous Riemannian block-coordinate descent with greedy agent
// selection (largest block of the centralised Riemannian gradient), optionally Nesterov-accelerated.  Each line of
// the trace is "iteration,agent,2f,gradnorm".  Same protocol as the reference's examples/MultiRobotExample.cpp
// (which is hard-wired to 5 robots on torus3D), written against the public PGOAgent interface only.
#include <DPGO/DPGO_utils.h>
#include <DPGO/DeviceRBCD.h>
#include <DPGO/PGOAgent.h>
#include <DPGO/QuadraticProblem.h>

#include <chrono>
#include <cstring>
#include <memory>

using namespace DPGO;

struct Options {
  std::string file, trace;
  unsigned robots = 5, iters = 1000, rank = 5;
  double stop = 0.1;
  bool accel = false, rgd = false, jacobi = false, resident = false;
  unsigned gpus = 1, bench = 0;
  std::string schedule = "greedy", partition, init = "central", momentum = "agents";
};

static Options parse(int argc, char **argv) {
  Options o;
  for (int i = 1; i < argc; ++i) {
    const std::string a = argv[i];
    auto next = [&]() -> std::string { return (i + 1 < argc) ? argv[++i] : ""; };
    if (a == "--robots") o.robots = (unsigned)std::stoul(next());
    else if (a == "--iters") o.iters = (unsigned)std::stoul(next());
    else if (a == "--rank") o.rank = (unsigned)std::stoul(next());
    else if (a == "--stop") o.stop = std::stod(next());
    else if (a == "--trace") o.trace = next();
    else if (a == "--accel") o.accel = true;
    else if (a == "--rgd") o.rgd = true;
    else if (a == "--jacobi") o.jacobi = true;
    else if (a == "--resident") o.resident = true;
    else if (a == "--gpus") o.gpus = (unsigned)std::stoul(next());
    else if (a == "--schedule") o.schedule = next();
    else if (a == "--bench") o.bench = (unsigned)std::stoul(next());
    else if (a == "--partition") o.partition = next();
    else if (a == "--init") o.init = next();
    else if (a == "--momentum") o.momentum = next();
    else if (a.rfind("--", 0) == 0) { std::cerr << "unknown option " << a << std::endl; std::exit(2); }
    else o.file = a;
  }
  if (o.file.empty()) {
    std::cerr << "usage: MultiAgentPGO <file.g2o> [--robots K] [--iters N] [--stop G] [--accel] [--rgd] [--jacobi] "
                 "[--rank R] [--trace out.csv] [--resident [--gpus N] [--schedule greedy|coloured|parallel|greedy_set] [--momentum agents|colours]]"
              << std::endl;
    std::exit(2);
  }
  return o;
}

int main(int argc, char **argv) {
  const Options opt = parse(argc, argv);
  size_t n = 0;
  const std::vector<RelativeSEMeasurement> graph = read_g2o_file(opt.file, n);
  if (graph.empty()) { std::cerr << "no measurements in " << opt.file << std::endl; return 1; }
  const unsigned d = (unsigned)graph[0].t.size(), r = opt.rank, K = opt.robots, dh = d + 1;
  if (n / K == 0) { std::cerr << "more robots than poses" << std::endl; return 1; }

  if (opt.resident) {
    // ---- device-resident runner: K agents over --gpus GPUs, one ncclAllGather per round ----
    DeviceRBCDOptions ro;
    ro.r = r;
    ro.gpus = opt.gpus;
    ro.schedule = opt.schedule;
    ro.algorithm = opt.rgd ? ROPTALG::RGD : ROPTALG::RTR;
    ro.preconditioner = opt.jacobi ? Preconditioner::BlockJacobi : Preconditioner::SparseExact;
    if (!opt.partition.empty()) {                        // one agent id per line, pose order (ref examples/MultiRobotExample.cpp:76-91)
      std::ifstream pf(opt.partition);
      std::string line;
      while (std::getline(pf, line))
        if (!line.empty()) ro.owner.push_back((unsigned)std::stoul(line));
      if (ro.owner.size() != n) { std::cerr << "partition file: " << ro.owner.size() << " lines for " << n << " poses" << std::endl; return 1; }
    }
    ro.initialization = opt.init;
    ro.acceleration = opt.accel;
    ro.momentumBlocks = opt.momentum;
    const Matrix lifted0 = (opt.init == "distributed") ? Matrix() : Matrix(fixedStiefelVariable(d, r) * chordalInitialization(d, n, graph));
    DeviceRBCD run(graph, n, K, lifted0, ro);
    for (size_t a = 0; a < run.initReport().size(); ++a) {
      const DeviceRBCDInitRecord &rec = run.initReport()[a];
      std::cout << "init " << a << " " << rec.wave << " " << rec.neighbor << " " << rec.candidates << " " << rec.inliers << " "
                << rec.iterations << std::endl;
    }
    std::ofstream tr;
    if (!opt.trace.empty()) tr.open(opt.trace);
    const auto t0 = std::chrono::steady_clock::now();
    unsigned it = 0;
    DeviceRBCDStats st;
    for (; it < opt.iters; ++it) {
      st = run.step(true);
      if (tr.is_open()) tr << std::setprecision(12) << it << "," << (st.active.empty() ? 0u : st.active[0]) << "," << st.cost << "," << st.gradnorm << "\n";
      if (st.gradnorm < opt.stop) { ++it; break; }
    }
    const double sec = std::chrono::duration<double>(std::chrono::steady_clock::now() - t0).count();
    std::cout << std::setprecision(10) << "resident: agents = " << K << ", gpus = " << opt.gpus << ", schedule = " << opt.schedule << " ("
              << run.numColours() << " colours), rounds = " << it << ", cost = " << st.cost << ", gradnorm = " << st.gradnorm
              << ", seconds = " << sec << std::endl;
    if (opt.bench > 0) {
      run.runRounds(std::min(opt.bench, 20u));            // warm-up
      run.sync();
      const auto b0 = std::chrono::steady_clock::now();
      run.runRounds(opt.bench);
      run.sync();
      const double bs = std::chrono::duration<double>(std::chrono::steady_clock::now() - b0).count();
      std::cout << "bench: rounds = " << opt.bench << ", rounds/s = " << opt.bench / bs << ", us/round = " << 1e6 * bs / opt.bench
                << ", all-gather bytes per GPU = " << run.allGatherBytesPerGpu()
                << ", agents of a round " << (run.concurrent() ? "side by side (clusters)" : "one at a time (full grid)") << std::endl;
    }
    return 0;
  }

  // contiguous ownership: agent a owns [a * (n/K), (a+1) * (n/K)), the last agent takes the remainder
  const size_t per = n / K;
  std::vector<unsigned> owner(n), local(n), count(K, 0);
  for (size_t g = 0; g < n; ++g) {
    owner[g] = (unsigned)std::min<size_t>(g / per, K - 1);
    local[g] = count[owner[g]]++;
  }
  std::vector<size_t> first(K, 0);
  for (unsigned a = 1; a < K; ++a) first[a] = first[a - 1] + count[a - 1];

  std::vector<std::vector<RelativeSEMeasurement>> odo(K), priv(K), shared(K);
  for (const auto &e : graph) {
    const unsigned a1 = owner[e.p1], a2 = owner[e.p2];
    RelativeSEMeasurement m(a1, a2, local[e.p1], local[e.p2], e.R, e.t, e.kappa, e.tau);
    if (a1 != a2) { shared[a1].push_back(m); shared[a2].push_back(m); }
    else if (e.p1 + 1 == e.p2) odo[a1].push_back(m);
    else priv[a1].push_back(m);
  }

  // centralised problem: evaluation only (cost and gradient of the assembled iterate)
  QuadraticProblem central(n, d, r);
  central.setPreconditioners(false, false);
  central.setQ(constructConnectionLaplacianSE(graph));

  std::vector<std::unique_ptr<PGOAgent>> agents;
  for (unsigned a = 0; a < K; ++a) {
    PGOAgentParameters prm(d, r, K);
    prm.acceleration = opt.accel;
    prm.algorithm = opt.rgd ? ROPTALG::RGD : ROPTALG::RTR;
    prm.preconditioner = opt.jacobi ? Preconditioner::BlockJacobi : Preconditioner::SparseExact;
    agents.emplace_back(new PGOAgent(a, prm));
    if (a > 0) {
      Matrix lift;
      agents[0]->getLiftingMatrix(lift);
      agents[a]->setLiftingMatrix(lift);
    }
    agents[a]->setPoseGraph(odo[a], priv[a], shared[a]);
  }
  const Matrix lifted = fixedStiefelVariable(d, r) * chordalInitialization(d, n, graph);
  for (unsigned a = 0; a < K; ++a) agents[a]->setX(Matrix(lifted).block(0, first[a] * dh, r, count[a] * dh));

  std::ofstream trace;
  if (!opt.trace.empty()) trace.open(opt.trace);
  Matrix X(r, n * dh);
  unsigned selected = 0;
  const auto t0 = std::chrono::steady_clock::now();
  unsigned it = 0;
  double cost = 0, gn = 0;
  for (; it < opt.iters; ++it) {
    PGOAgent &sel = *agents[selected];
    for (auto &ag : agents)
      if (ag->getID() != selected) ag->iterate(false);
    for (auto &ag : agents) {
      if (ag->getID() == selected) continue;
      PoseDict poses;
      if (!ag->getSharedPoseDict(poses)) continue;
      sel.setNeighborStatus(ag->getStatus());
      sel.updateNeighborPoses(ag->getID(), poses);
      if (opt.accel) {
        PoseDict aux;
        if (ag->getAuxSharedPoseDict(aux)) sel.updateAuxNeighborPoses(ag->getID(), aux);
      }
    }
    sel.iterate(true);
    for (unsigned a = 0; a < K; ++a) {
      Matrix Xa;
      agents[a]->getX(Xa);
      X.block(0, first[a] * dh, r, count[a] * dh) = Xa;
    }
    const Matrix grad = central.RieGrad(X);
    gn = grad.norm();
    cost = 2 * central.f(X);
    if (trace.is_open()) trace << std::setprecision(12) << it << "," << selected << "," << cost << "," << gn << "\n";
    if (gn < opt.stop) { ++it; break; }
    if (!sel.getNeighbors().empty()) {
      double best = -1;
      for (unsigned a = 0; a < K; ++a) {
        const double g = grad.block(0, first[a] * dh, r, count[a] * dh).norm();
        if (g > best) { best = g; selected = a; }
      }
    }
  }
  const double sec = std::chrono::duration<double>(std::chrono::steady_clock::now() - t0).count();
  std::cout << std::setprecision(10) << "iterations = " << it << ", cost = " << cost << ", gradnorm = " << gn
            << ", seconds = " << sec << ", iterations/s = " << it / sec << std::endl;
  return 0;
}
