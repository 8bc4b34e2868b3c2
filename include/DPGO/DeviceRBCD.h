// DeviceRBCD.h -- GPU extension of the C++ host API: the device-resident multi-GPU RBCD runner.
//
// The reference's drivers keep every agent's iterate in host Eigen matrices and exchange public poses through
// std::map "PoseDict"s (examples/MultiRobotExample.cpp:229-334, src/PGOAgent.cpp:95-105,434-458).  This runner keeps
// the iterates in HBM and replaces that "network" by ONE ncclAllGather per round over NVLink:
//
//   per round, on every GPU's stream:   dpgo_agents_round_async  per active agent: dpgo_agent_build_G (linear term from
//                                                                the gathered tiles, ref :783-859) -> RTR step ->
//                                                                pack of its public tiles into the send buffer
//                                       ncclAllGather            (padded public-pose slots of all agents)
//
// so the gathered tiles stay current from round to round; an evaluation (step(true), status()) only rebuilds G from them.
// K agents are spread over N GPUs of one node (K % N == 0, contiguous blocks), one process, one stream and one NCCL
// communicator per GPU (ncclCommInitAll).  Schedules: "greedy" (the reference's: one agent per round, argmax of the block
// gradient norms -- reproduces the shipped traces), "coloured" (all agents of one colour class of the agent graph per
// round: same RBCD semantics, concurrent), "parallel" (all agents on the previous round's poses), "greedy_set" (the greedy
// rule applied to as many agents as RBCD allows: each round a maximal set of agents that share no edge, taken in decreasing
// block gradient norm, chosen on the GPU from the status taken before the round; no host synchronisation per round).
// When a GPU hosts several agents of one colour class, their steps run side by side (one thread-block cluster and one
// stream per agent, the whole round of a GPU replayed as a CUDA graph): DeviceRBCDOptions::concurrent.
#ifndef DPGO_DEVICE_RBCD_H
#define DPGO_DEVICE_RBCD_H

#include <DPGO/DPGO_types.h>
#include <DPGO/DPGO_utils.h>
#include <DPGO/PGOAgent.h>
#include <DPGO/RelativeSEMeasurement.h>

#include <functional>
#include <memory>
#include <string>
#include <vector>

namespace DPGO {

struct DeviceRBCDOptions {
  unsigned r = 5;
  unsigned gpus = 1;
  std::string schedule = "greedy";
  ROPTALG algorithm = ROPTALG::RTR;
  Preconditioner preconditioner = Preconditioner::SparseExact;
  // pose -> agent (one entry per pose, e.g. from a graph-partition file, ref examples/MultiRobotExample.cpp:76-91);
  // empty: contiguous ranges, the last agent takes the remainder (ref :95-109)
  std::vector<unsigned> owner;
  // the active agents of a round that share a GPU step side by side, each as one thread-block cluster on its own stream
  // (dpgo_agents_round_async; greedy / coloured / greedy_set schedules): -1 = when some GPU hosts >= 2 agents of one
  // colour class (coloured) or >= 2 agents that are not neighbours (greedy_set)
  int concurrent = -1;
  // "central": the caller's XInit (r x (d+1)n); "distributed": the reference's multi-robot initialisation
  // (PGOAgentParameters::multirobot_initialization, ref include/DPGO/PGOAgent.h:129) on the GPUs -- every agent's chordal
  // initialisation of its private graph in its own frame, then frame-alignment waves (robust average of the frame
  // transforms its shared loop closures give with an initialised neighbour, ref src/PGOAgent.cpp:369-440); XInit empty
  std::string initialization = "central";
  // Nesterov-accelerated rounds (ref src/PGOAgent.cpp:685-695,1033-1091) in the reference driver's order: the idle agents
  // finish iterate(false), the X and Y tiles are exchanged (one ncclAllGather group per buffer), the active agents step
  // from Y.  momentumBlocks is the N of the recurrence: "agents" = the number of agents (the reference's), "colours" = the
  // number of colour classes (schedule "coloured" only: a coloured round is one exact block update).  With "agents" the
  // automatic launch mode is one agent at a time.  solve() takes acceleration with "colours" only: there each accelerated
  // round leaves every active agent's status record as the reference's iterate() does (relative change against XPrev,
  // one optimising call per round, restart or not).
  bool acceleration = false;
  unsigned restartInterval = 30;
  std::string momentumBlocks = "agents";
};

// per agent: the wave it joined the global frame in (agent 0: 0), the neighbour it aligned to (-1 for agent 0), the
// candidate and inlier counts and the GNC iterations of that alignment
struct DeviceRBCDInitRecord {
  int wave = -1, neighbor = -1, candidates = 0, inliers = 0, iterations = 0;
};

struct DeviceRBCDStats {
  double cost = 0;        // 2 f of the assembled iterate (centralised cost)
  double gradnorm = 0;    // norm of the centralised Riemannian gradient
  std::vector<unsigned> active;
};

// Every agent's status record (DPGO_STATUS_DOUBLES = 5 doubles each, agent-major): <XQ, X>, <X, G>, |rgrad|^2, the
// relative change of its last optimising call, its optimising calls so far (dpgo_agents_status_async)
struct DeviceRBCDStatus {
  std::vector<double> records;
  double cost = 0;        // 2 f_central = sum of <XQ, X> + <X, G>
  double gradnorm = 0;    // |grad_central|
  double at(unsigned agent, unsigned field) const { return records[(size_t)agent * 5 + field]; }
};

// Stop rules of DeviceRBCD::solve (a tolerance of 0 disables its rule): the central gradient norm below gradnormTol
// (ref examples/MultiRobotExample.cpp:302-305); every agent optimised since the solve began with its last relative change
// <= relChangeTol (ref PGOAgent::shouldTerminate, src/PGOAgent.cpp:703-716,1007-1031); maxRounds rounds.  The status is
// taken after every checkEvery-th round and after the last; the greedy schedule needs checkEvery == 1 (greedy_set takes
// any: it selects on the GPU).
struct DeviceRBCDSolveOptions {
  unsigned maxRounds = 500;
  double gradnormTol = 0.1;
  double relChangeTol = 5e-3;
  unsigned checkEvery = 1;
  std::function<void(unsigned round, double cost, double gradnorm)> callback;   // every check
};

struct DeviceRBCDSolveReport {
  unsigned rounds = 0;
  std::string reason;                 // "gradnorm", "team" or "max_rounds"
  double cost = 0, gradnorm = 0;
  std::vector<double> relativeChange; // per agent, of its last optimising call
};

class DeviceRBCD {
 public:
  // graph: the global pose graph (global pose ids); XInit: r x (d+1)n lifted initial iterate (empty with
  // options.initialization == "distributed")
  DeviceRBCD(const std::vector<RelativeSEMeasurement> &graph, size_t n, unsigned numAgents, const Matrix &XInit,
             const DeviceRBCDOptions &options);
  ~DeviceRBCD();
  DeviceRBCD(const DeviceRBCD &) = delete;
  DeviceRBCD &operator=(const DeviceRBCD &) = delete;

  void exchange();                              // pack -> all-gather -> G rebuild, asynchronous on the GPU streams
  DeviceRBCDStats step(bool evaluate = true);   // one round (+ status(): central cost / gradient norm / greedy selection)
  void runRounds(unsigned rounds);              // rounds without evaluation (throughput), asynchronous; call sync()
  void sync();
  Matrix assemble();                            // r x (d+1)n iterate on the host
  bool concurrent() const;
  unsigned numColours() const { return mNumColours; }
  const std::vector<unsigned> &colours() const { return mColour; }
  unsigned round() const { return mRound; }
  size_t allGatherBytesPerGpu() const;
  const std::vector<DeviceRBCDInitRecord> &initReport() const { return mInitReport; }   // empty for "central"
  // one exchange (none when the gathered tiles are current), one status launch per GPU, one copy per GPU into pinned
  // host memory, one synchronisation per GPU
  DeviceRBCDStatus status();
  DeviceRBCDSolveReport solve(const DeviceRBCDSolveOptions &options = DeviceRBCDSolveOptions());
  // d x (d+1)n trajectory in global pose order, rounded on the device against agent 0's pose 0
  // (ref getTrajectoryInGlobalFrame, src/PGOAgent.cpp:500-519)
  Matrix trajectory();
  // marginal covariances of trajectory() (poseCovariancesGPU on GPU 0), anchored at agent 0's pose 0 -- the gauge of
  // trajectory() -- unless `anchor` names another global pose.  The runner holds the whole pose graph in this process
  // (its GPUs are one process's), which is what the call needs.
  PoseCovariances poseCovariances(long anchor = -1, const std::vector<std::pair<size_t, size_t>> &pairs = {});
  // greedy_set: the agents of rounds first .. first + count - 1 (those issued so far), each sorted; synchronises the GPUs
  std::vector<std::vector<unsigned>> selectionLog(unsigned first = 0, unsigned count = ~0u);

 private:
  struct Impl;
  std::vector<unsigned> issueRound();           // one round of the schedule's active agents; returns them (greedy_set: none)
  void selectRound();
  void statusDevice();
  void roundAccelerated(const std::vector<unsigned> &active);
  void alignWaves();
  std::vector<DeviceRBCDInitRecord> mInitReport;
  std::unique_ptr<Impl> impl;
  unsigned mNumColours = 1, mRound = 0;
  std::vector<unsigned> mColour;
};

}  // namespace DPGO
#endif
