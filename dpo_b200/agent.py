"""PGOAgent mirror + the multi-GPU runner (one agent per GPU, boundary poses over one all-gather).

`PGOAgent` keeps the reference's public interface for the parts on / next to the hot path
(ref include/DPGO/PGOAgent.h:209-490, src/PGOAgent.cpp): setPoseGraph, setX/getX, getSharedPoseDict,
updateNeighborPoses, iterate, getNeighbors, getTrajectoryInLocalFrame, localPoseGraphOptimization.
Host bookkeeping stays on the host, every numeric step runs in libdpgo_b200.so.

`ExchangePlan` + `DistributedPGO` are the GPU-native replacement of the reference's in-process
"network" (examples/MultiRobotExample.cpp:245-256): public poses are packed on the device,
exchanged with ONE all-gather per round (NCCL over NVLink when the tensors are CUDA), and G is
rebuilt on the device from the gathered tiles (ref PGOAgent::constructGMatrix, src/PGOAgent.cpp:783-859).
"""
from __future__ import annotations

import ctypes as C
import time
from dataclasses import dataclass, field
from typing import Dict, List, Optional, Sequence, Tuple

import numpy as np

from . import _capi as capi
from . import posegraph as pg
from .posegraph import EdgeSet
from .problem import QuadraticOptimizer, QuadraticProblem, ROPTALG

PoseID = Tuple[int, int]


@dataclass
class PGOAgentParameters:
    """ref: include/DPGO/PGOAgent.h:59-136 (fields on the hot path; robust-cost knobs are out of scope)."""
    d: int
    r: int
    numRobots: int = 1
    algorithm: int = ROPTALG.RTR
    acceleration: bool = False
    restartInterval: int = 30
    maxNumIters: int = 500
    relChangeTol: float = 5e-3
    verbose: bool = False
    preconditioner: int = capi.PRECOND_SPARSE_EXACT     # GPU extension (reference operator by default)
    device: int = 0
    cluster: bool = False          # GPU extension: step kernel as one thread-block cluster (several agents per GPU)


class PGOAgentState:
    WAIT_FOR_DATA, WAIT_FOR_INITIALIZATION, INITIALIZED = 0, 1, 2


# ---------------------------------------------------------------------------------------------------
# partitioning (ref examples/MultiRobotExample.cpp:63-151)
# ---------------------------------------------------------------------------------------------------
def contiguous_owner(n: int, k: int) -> np.ndarray:
    """Pose -> agent, contiguous ranges, last agent takes the remainder (ref :95-109)."""
    per = n // k
    if per <= 0:
        raise ValueError("More robots than total number of poses! Decrease the number of robots")
    return np.minimum(np.arange(n) // per, k - 1).astype(np.int64)


def partition_edges(edges: EdgeSet, owner: np.ndarray, k: int):
    """Split a global edge list into per-agent (odometry, private, shared) sets with local pose ids
    (ref :115-151).  Returns (parts, counts, global_index_of[a])."""
    n = owner.shape[0]
    counts = np.bincount(owner, minlength=k).astype(np.int64)
    local = np.empty(n, dtype=np.int64)
    glob = []
    for a in range(k):
        idx = np.flatnonzero(owner == a)
        local[idx] = np.arange(idx.shape[0])
        glob.append(idx)
    a1, a2 = owner[edges.p1], owner[edges.p2]
    re = EdgeSet(edges.d, a1, a2, local[edges.p1], local[edges.p2], edges.R, edges.t, edges.kappa, edges.tau,
                 edges.weight)
    same = a1 == a2
    odo = edges.p1 + 1 == edges.p2                     # ref :134 tests GLOBAL ids
    parts = []
    for a in range(k):
        mine = same & (a1 == a)
        parts.append((re.take(np.flatnonzero(mine & odo)), re.take(np.flatnonzero(mine & ~odo)),
                      re.take(np.flatnonzero(~same & ((a1 == a) | (a2 == a))))))
    return parts, counts, glob


# ---------------------------------------------------------------------------------------------------
# exchange plan: who publishes what, where it lands in the gathered buffer
# ---------------------------------------------------------------------------------------------------
class ExchangePlan:
    """Static tables of the boundary-pose exchange for k agents.

    public[a]   sorted local ids of agent a's public poses (ref localSharedPoseIDs, src/PGOAgent.cpp:236-245)
    pmax        padded slot count per agent (all-gather needs equal counts)
    slot(b, q)  = b * pmax + position of q in public[b]
    edge tables for agent a: local pose, neighbour slot, outgoing flag, T (row-major), omega
    """

    def __init__(self, shared: Sequence[EdgeSet], k: int):
        self.k = k
        self.public: List[np.ndarray] = []
        for a in range(k):
            s = shared[a]
            mine = np.where(s.r1 == a, s.p1, s.p2)
            self.public.append(np.unique(mine).astype(np.int32))
        self.pmax = max(1, max(len(p) for p in self.public))
        self._pos = [{int(q): i for i, q in enumerate(p)} for p in self.public]
        self.tables = []
        for a in range(k):
            s = shared[a]
            out = (s.r1 == a)
            local = np.where(out, s.p1, s.p2).astype(np.int32)
            nbr_agent = np.where(out, s.r2, s.r1)
            nbr_pose = np.where(out, s.p2, s.p1)
            slot = np.array([int(b) * self.pmax + self._pos[int(b)][int(q)] for b, q in zip(nbr_agent, nbr_pose)],
                            dtype=np.int32)
            self.tables.append(dict(local=local, slot=slot, outgoing=out.astype(np.int32),
                                    T=np.ascontiguousarray(s.homogeneous()), omega=np.ascontiguousarray(s.omega()),
                                    neighbors=sorted(set(int(b) for b in nbr_agent))))

    def slot(self, agent: int, local_pose: int) -> int:
        return agent * self.pmax + self._pos[agent][int(local_pose)]

    def colouring(self) -> List[int]:
        """Greedy colouring of the agent graph: agents of one colour share no edge, so they may update
        concurrently with exactly the sequential RBCD semantics (SURVEY section 7, hard part 4)."""
        colour = [-1] * self.k
        for a in range(self.k):
            used = {colour[b] for b in self.tables[a]["neighbors"] if colour[b] >= 0}
            c = 0
            while c in used:
                c += 1
            colour[a] = c
        return colour


# ---------------------------------------------------------------------------------------------------
# distributed initialisation: host tables
# ---------------------------------------------------------------------------------------------------
def check_private_graph_connected(agent: int, n: int, private: EdgeSet) -> None:
    """The chordal initialisation of a private graph (odometry + private loop closures) is singular unless the graph is
    connected; some partitions leave an agent with several pieces."""
    if n <= 1:
        return
    import scipy.sparse as sp
    from scipy.sparse.csgraph import connected_components
    A = sp.coo_matrix((np.ones(len(private)), (private.p1, private.p2)), shape=(n, n))
    pieces = connected_components(A, directed=False)[0]
    if pieces != 1:
        raise ValueError(f"agent {agent}: the private pose graph (odometry + private loop closures) has {pieces} connected "
                         f"components, so its local chordal initialisation is singular")


def alignment_candidates(agent: int, shared: EdgeSet, plan: ExchangePlan):
    """Candidate table of dpgo_agent_set_align_candidates: one candidate per public pose j of a neighbour b that the agent
    shares an edge with, grouped per neighbour in increasing id, j increasing (std::map<PoseID> order), each through the
    FIRST shared edge touching (b, j) (ref findSharedLoopClosureWithNeighbor, src/PGOAgent.cpp:922-934)."""
    out = shared.r1 == agent
    nbr = np.where(out, shared.r2, shared.r1)
    nq = np.where(out, shared.p2, shared.p1)
    first: Dict[PoseID, int] = {}
    for e in range(len(shared)):
        first.setdefault((int(nbr[e]), int(nq[e])), e)
    keys = sorted(first)
    idx = np.array([first[key] for key in keys], dtype=np.int64)
    groups = sorted({b for b, _ in keys})
    ptr = np.searchsorted([b for b, _ in keys], groups + [groups[-1] + 1 if groups else 0]).astype(np.int32)
    return dict(neighbor=np.array(groups, dtype=np.int32), ptr=ptr,
                local=np.where(out, shared.p1, shared.p2)[idx].astype(np.int32),
                slot=np.array([plan.slot(b, j) for b, j in keys], dtype=np.int32),
                outgoing=out[idx].astype(np.int32),
                T=np.ascontiguousarray(shared.homogeneous()[idx]))


# ---------------------------------------------------------------------------------------------------
# PGOAgent
# ---------------------------------------------------------------------------------------------------
def _rbcd_step_optimizer(problem: QuadraticProblem, algorithm: int, preconditioner: int) -> QuadraticOptimizer:
    """The optimiser of one RBCD step: the algorithm, one trust-region iteration of at most 10 inner iterations from radius
    100 with tolerance 1e-2 (ref src/PGOAgent.cpp:1134-1137), and the preconditioner."""
    opt = QuadraticOptimizer(problem)
    opt.setAlgorithm(algorithm)
    opt.setTrustRegionTolerance(1e-2)
    opt.setTrustRegionIterations(1)
    opt.setTrustRegionMaxInnerIterations(10)
    opt.setTrustRegionInitialRadius(100)
    opt.setPreconditioner(preconditioner)
    return opt


class PGOAgent:
    def __init__(self, ID: int, params: PGOAgentParameters):
        self.mID = int(ID)
        self.mParams = params
        self.d, self.r, self.n = params.d, params.r, 1
        self.mState = PGOAgentState.WAIT_FOR_DATA
        self.mIterationNumber = 0
        self.mInstanceNumber = 0
        self.X = np.zeros((self.r, self.d + 1))
        self.X[:self.d, :self.d] = np.eye(self.d)
        self.YLift: Optional[np.ndarray] = pg.fixedStiefelVariable(self.d, self.r) if ID == 0 else None
        self.globalAnchor: Optional[np.ndarray] = None
        self.mProblem: Optional[QuadraticProblem] = None
        self.neighborPoseDict: Dict[PoseID, np.ndarray] = {}
        self.localSharedPoseIDs: List[PoseID] = []
        self.neighborSharedPoseIDs: set = set()
        self.neighborRobotIDs: List[int] = []
        self.relativeChange = 0.0
        self.readyToTerminate = False
        self.lastResult = None
        self.TLocalInit: Optional[np.ndarray] = None
        # Nesterov acceleration (ref src/PGOAgent.cpp:1040-1091)
        self.gamma = 0.0
        self.alpha = 0.0
        self.Y: Optional[np.ndarray] = None
        self.V: Optional[np.ndarray] = None
        self.XPrev: Optional[np.ndarray] = None
        self.neighborAuxPoseDict: Dict[PoseID, np.ndarray] = {}

    # -- getters (ref .h:237-262) --
    def getID(self): return self.mID
    def num_poses(self): return self.n
    def dimension(self): return self.d
    def relaxation_rank(self): return self.r
    def iteration_number(self): return self.mIterationNumber
    def instance_number(self): return self.mInstanceNumber
    def getNeighbors(self): return list(self.neighborRobotIDs)

    def getLiftingMatrix(self):
        assert self.mID == 0
        return self.YLift

    def setLiftingMatrix(self, M):
        M = np.asarray(M, dtype=float)
        assert M.shape == (self.r, self.d)
        self.YLift = M

    def setGlobalAnchor(self, M):
        self.globalAnchor = np.asarray(M, dtype=float)

    # -- pose graph (ref src/PGOAgent.cpp:126-195) --
    def setPoseGraph(self, odometry: EdgeSet, privateLoopClosures: EdgeSet, sharedLoopClosures: EdgeSet,
                     TInit: Optional[np.ndarray] = None, n: Optional[int] = None) -> None:
        assert self.mState == PGOAgentState.WAIT_FOR_DATA and self.n == 1
        if len(odometry) == 0 and n is None:
            return
        self.odometry, self.privateLoopClosures, self.sharedLoopClosures = odometry, privateLoopClosures, sharedLoopClosures
        nn = 1
        for s in (odometry, privateLoopClosures):
            if len(s):
                nn = max(nn, int(max(s.p1.max(), s.p2.max())) + 1)
        sh = sharedLoopClosures
        if len(sh):
            mine = np.where(sh.r1 == self.mID, sh.p1, sh.p2)
            nn = max(nn, int(mine.max()) + 1)
            other_r = np.where(sh.r1 == self.mID, sh.r2, sh.r1)
            other_p = np.where(sh.r1 == self.mID, sh.p2, sh.p1)
            self.localSharedPoseIDs = [(self.mID, int(q)) for q in np.unique(mine)]
            self.neighborSharedPoseIDs = {(int(a), int(q)) for a, q in zip(other_r, other_p)}
            self.neighborRobotIDs = sorted({int(a) for a in other_r})
        self.n = nn if n is None else int(n)
        self.mProblem = QuadraticProblem(self.n, self.d, self.r, device=self.mParams.device,
                                         preconditioners=self._precond_set(), cluster=self.mParams.cluster)
        self.constructQMatrix()
        if TInit is not None and np.shape(TInit) == (self.d, (self.d + 1) * self.n):
            self.TLocalInit = np.array(TInit, dtype=float)
        else:
            self.localInitialization()
        self.mState = PGOAgentState.WAIT_FOR_INITIALIZATION
        if self.mID == 0 and self.YLift is not None:
            self.X = self.YLift @ self.TLocalInit
            self.mState = PGOAgentState.INITIALIZED

    def _precond_set(self):
        s = {capi.PRECOND_BLOCK_JACOBI}
        s.add(self.mParams.preconditioner)
        s.discard(capi.PRECOND_NONE)
        return tuple(sorted(s))

    def localInitialization(self) -> None:
        """ref src/PGOAgent.cpp:945-962 (L2 cost -> chordal initialisation on the private edges)."""
        priv = EdgeSet.join([self.odometry, self.privateLoopClosures])
        self.TLocalInit = pg.chordalInitialization(self.d, self.n, priv)

    def constructQMatrix(self) -> None:
        """Private edges' Laplacian + diagonal terms of the shared edges (ref src/PGOAgent.cpp:720-781)."""
        priv = EdgeSet.join([self.odometry, self.privateLoopClosures])
        sh = self.sharedLoopClosures
        idx, W = None, None
        if len(sh):
            T, om = sh.homogeneous(), sh.omega()
            out = sh.r1 == self.mID
            W = np.zeros_like(T)
            ar = np.arange(self.d + 1)
            W[:, ar, ar] = om                                              # incoming: Omega at p2
            Wout = (T * om[:, None, :]) @ np.transpose(T, (0, 2, 1))       # outgoing: T Omega T^T at p1
            W[out] = Wout[out]
            idx = np.where(out, sh.p1, sh.p2).astype(np.int32)
        # the private edges' Laplacian is assembled on the device from the edge records (k_assemble_Q); the shared edges'
        # diagonal terms enter as static blocks; odometry edges keep their weights under robust re-weighting
        fixed = np.concatenate([np.ones(len(self.odometry), dtype=np.int32), np.zeros(len(self.privateLoopClosures), dtype=np.int32)])
        self.mProblem.setEdges(priv, idx, W, fixed=fixed)

    def constructGMatrix(self, poseDict: Dict[PoseID, np.ndarray]) -> bool:
        """Host form (dictionary of neighbour poses), as the reference does it (src/PGOAgent.cpp:783-859)."""
        sh = self.sharedLoopClosures
        dh = self.d + 1
        G = np.zeros((self.r, dh * self.n))
        T, om = sh.homogeneous(), sh.omega()
        for k in range(len(sh)):
            if sh.r1[k] == self.mID:
                nid = (int(sh.r2[k]), int(sh.p2[k]))
                if nid not in poseDict:
                    return False
                G[:, int(sh.p1[k]) * dh:(int(sh.p1[k]) + 1) * dh] -= (poseDict[nid] * om[k][None, :]) @ T[k].T
            else:
                nid = (int(sh.r1[k]), int(sh.p1[k]))
                if nid not in poseDict:
                    return False
                G[:, int(sh.p2[k]) * dh:(int(sh.p2[k]) + 1) * dh] -= (poseDict[nid] @ T[k]) * om[k][None, :]
        self.mProblem.setG(G)
        return True

    # -- iterate exchange (ref src/PGOAgent.cpp:55-118, 434-458) --
    def setX(self, Xin) -> None:
        Xin = np.asarray(Xin, dtype=float)
        assert self.mState != PGOAgentState.WAIT_FOR_DATA
        assert Xin.shape == (self.r, (self.d + 1) * self.n)
        self.X = Xin.copy()
        self.mState = PGOAgentState.INITIALIZED
        if self.mParams.acceleration:
            self.initializeAcceleration()                  # ref :60-62

    def getX(self) -> np.ndarray:
        return self.X.copy()

    def getSharedPose(self, index: int):
        if self.mState != PGOAgentState.INITIALIZED or index >= self.n:
            return None
        dh = self.d + 1
        return self.X[:, index * dh:(index + 1) * dh].copy()

    def getSharedPoseDict(self) -> Optional[Dict[PoseID, np.ndarray]]:
        if self.mState != PGOAgentState.INITIALIZED:
            return None
        dh = self.d + 1
        return {pid: self.X[:, pid[1] * dh:(pid[1] + 1) * dh].copy() for pid in self.localSharedPoseIDs}

    def updateNeighborPoses(self, neighborID: int, poseDict: Dict[PoseID, np.ndarray]) -> None:
        assert neighborID != self.mID
        for nid, var in poseDict.items():
            assert nid[0] == neighborID and var.shape == (self.r, self.d + 1)
            if nid in self.neighborSharedPoseIDs and self.mState == PGOAgentState.INITIALIZED:
                self.neighborPoseDict[nid] = np.array(var)

    # -- Nesterov acceleration (ref src/PGOAgent.cpp:60-62, 107-118, 460-479, 1040-1091) --
    def initializeAcceleration(self) -> None:
        self.XPrev, self.V, self.Y = self.X.copy(), self.X.copy(), self.X.copy()
        self.gamma = self.alpha = 0.0

    def getAuxSharedPoseDict(self) -> Optional[Dict[PoseID, np.ndarray]]:
        if self.mState != PGOAgentState.INITIALIZED or self.Y is None:
            return None
        dh = self.d + 1
        return {pid: self.Y[:, pid[1] * dh:(pid[1] + 1) * dh].copy() for pid in self.localSharedPoseIDs}

    def updateAuxNeighborPoses(self, neighborID: int, poseDict: Dict[PoseID, np.ndarray]) -> None:
        assert neighborID != self.mID
        for nid, var in poseDict.items():
            if nid in self.neighborSharedPoseIDs and self.mState == PGOAgentState.INITIALIZED:
                self.neighborAuxPoseDict[nid] = np.array(var)

    # -- one RBCD step (ref src/PGOAgent.cpp:642-718, updateX :1093-1165) --
    def iterate(self, doOptimization: bool = True) -> bool:
        self.mIterationNumber += 1
        if self.mState != PGOAgentState.INITIALIZED:
            return True
        if not self.mParams.acceleration:
            return self._updateX(doOptimization, False)
        if self.Y is None:
            self.initializeAcceleration()
        self.XPrev = self.X.copy()
        N = float(self.mParams.numRobots)
        self.gamma = (1 + np.sqrt(1 + 4 * N * N * self.gamma * self.gamma)) / (2 * N)        # ref :1065-1069
        self.alpha = 1.0 / (self.gamma * N)                                                    # ref :1071-1075
        self.Y = self.mProblem.project((1 - self.alpha) * self.X + self.alpha * self.V)       # ref :1077-1083
        ok = self._updateX(doOptimization, True)
        self.V = self.mProblem.project(self.V + self.gamma * (self.X - self.Y))               # ref :1085-1091
        if (self.mIterationNumber + 1) % self.mParams.restartInterval == 0:                    # ref :1033-1052
            self.X = self.XPrev
            self._updateX(doOptimization, False)
            self.V, self.Y = self.X.copy(), self.X.copy()
            self.gamma = self.alpha = 0.0
        return ok

    def _updateX(self, doOptimization: bool, acceleration: bool) -> bool:
        if not doOptimization:
            if acceleration:
                self.X = self.Y.copy()
            return True
        XPrev = self.X
        if not self.constructGMatrix(self.neighborAuxPoseDict if acceleration else self.neighborPoseDict):
            if self.mParams.verbose:
                print(f"Robot {self.mID} could not construct G matrix. Skip update...")
            self.readyToTerminate = False
            return False
        opt = _rbcd_step_optimizer(self.mProblem, self.mParams.algorithm, self.mParams.preconditioner)
        opt.setVerbose(self.mParams.verbose)
        self.X = np.array(opt.optimize(self.Y if acceleration else self.X))
        self.lastResult = opt.getOptResult()
        self.relativeChange = float(np.sqrt(np.sum((self.X - XPrev) ** 2) / self.n))
        self.readyToTerminate = self.relativeChange <= self.mParams.relChangeTol
        return True

    def localPoseGraphOptimization(self) -> np.ndarray:
        """ref src/PGOAgent.cpp:964-990: r = d problem on the private edges, RTR 10 outer / 50 inner."""
        if self.TLocalInit is None:
            self.localInitialization()
        priv = EdgeSet.join([self.odometry, self.privateLoopClosures])
        prob = QuadraticProblem(self.n, self.d, self.d, device=self.mParams.device, preconditioners=self._precond_set())
        prob.setQ_blocks(*pg.connection_laplacian_blocks(priv))
        opt = QuadraticOptimizer(prob)
        opt.setVerbose(self.mParams.verbose)
        opt.setTrustRegionInitialRadius(10)
        opt.setTrustRegionIterations(10)
        opt.setTrustRegionTolerance(1e-1)
        opt.setTrustRegionMaxInnerIterations(50)
        opt.setPreconditioner(self.mParams.preconditioner)
        Topt = np.array(opt.optimize(self.TLocalInit))
        self.lastResult = opt.getOptResult()
        prob.close()
        return Topt

    def getTrajectoryInLocalFrame(self) -> Optional[np.ndarray]:
        """ref src/PGOAgent.cpp:481-498."""
        if self.mState != PGOAgentState.INITIALIZED:
            return None
        d, dh = self.d, self.d + 1
        T = self.X[:, :d].T @ self.X
        t0 = T[:, d].copy()
        for i in range(self.n):
            T[:, i * dh:i * dh + d] = pg.projectToRotationGroup(T[:, i * dh:i * dh + d])
            T[:, i * dh + d] -= t0
        return T

    # -- device-resident exchange path -----------------------------------------------------------------
    def attach_exchange(self, plan: ExchangePlan) -> None:
        lib, h = self.mProblem._lib, self.mProblem._h
        pub = np.ascontiguousarray(plan.public[self.mID], dtype=np.int32)
        capi.check(lib.dpgo_agent_set_public_poses(h, len(pub), capi.iptr(pub)))
        tb = plan.tables[self.mID]
        capi.check(lib.dpgo_agent_set_shared_edges(h, len(tb["local"]), capi.iptr(tb["local"]), capi.iptr(tb["slot"]),
                                                   capi.iptr(tb["outgoing"]), capi.dptr(tb["T"]), capi.dptr(tb["omega"])))

    def pack_public(self, send_ptr: int) -> None:
        capi.check(self.mProblem._lib.dpgo_agent_pack_public(self.mProblem._h, C.c_void_p(send_ptr)))

    def build_G(self, gathered_ptr: int, num_slots: int) -> None:
        capi.check(self.mProblem._lib.dpgo_agent_build_G(self.mProblem._h, C.c_void_p(gathered_ptr), num_slots))


# ---------------------------------------------------------------------------------------------------
# multi-agent runner
# ---------------------------------------------------------------------------------------------------
@dataclass
class RoundStats:
    cost: float            # 2 f_central
    gradnorm: float        # |grad_central|
    selected: List[int]


@dataclass
class TeamStatus:
    records: np.ndarray    # (k, capi.STATUS_DOUBLES): <XQ,X>, <X,G>, |rgrad|^2, last relative change, optimising calls
    cost: float            # 2 f_central = sum(<XQ,X> + <X,G>)
    gradnorm: float        # |grad_central|


@dataclass
class SolveReport:
    rounds: int
    reason: str            # "gradnorm", "team" or "max_rounds"
    cost: float
    gradnorm: float
    relative_change: np.ndarray    # per agent, of its last optimising call


def team_status(records: np.ndarray) -> TeamStatus:
    records = np.asarray(records, dtype=np.float64)
    return TeamStatus(records, float(np.sum(records[:, 0] + records[:, 1])), float(np.sqrt(np.sum(records[:, 2]))))


def stop_reason(records: np.ndarray, calls_at_start: np.ndarray, rounds: int, max_rounds: int, gradnorm_tol: float,
                rel_change_tol: float) -> Optional[str]:
    """Stop rule of DistributedPGO.solve / DeviceRBCD::solve as a function of the team's status records: the central
    gradient norm below gradnorm_tol (ref examples/MultiRobotExample.cpp:302-305); every agent ready to terminate, i.e.
    optimised since the solve began with its last relative change <= rel_change_tol (ref PGOAgent::shouldTerminate,
    src/PGOAgent.cpp:703-716,1007-1031); the round cap.  A tolerance of 0 disables its rule."""
    st = team_status(records)
    if gradnorm_tol > 0 and st.gradnorm < gradnorm_tol:
        return "gradnorm"
    if rel_change_tol > 0 and np.all(st.records[:, 4] > np.asarray(calls_at_start)) and \
            np.all(st.records[:, 3] <= rel_change_tol):
        return "team"
    if rounds >= max_rounds:
        return "max_rounds"
    return None


def greedy_selection(selected: int, agent_gradnorms: np.ndarray, has_neighbours: bool) -> int:
    """The next agent of the greedy schedule (ref examples/MultiRobotExample.cpp:308-325): the largest per-agent gradient
    norm, except that an agent without neighbours stays selected."""
    return int(np.argmax(agent_gradnorms)) if has_neighbours else int(selected)


def greedy_independent_set(gradnorm2: np.ndarray, neighbours: Sequence[Sequence[int]]) -> List[int]:
    """The agents of one round of the greedy_set schedule, sorted: walk the agents in decreasing squared block gradient norm
    (ties to the lower id, as std::max_element), taking an agent unless one of its neighbours is already taken.  The result
    is a maximal independent set of the agent graph; on a complete agent graph it is {argmax}, the reference's greedy choice
    (ref examples/MultiRobotExample.cpp:308-325).  A NaN norm ranks last.  k_select_independent computes the same set."""
    g = np.nan_to_num(np.asarray(gradnorm2, dtype=np.float64), nan=-1.0)
    taken = np.zeros(g.shape[0], dtype=bool)
    for a in sorted(range(g.shape[0]), key=lambda a: (-g[a], a)):
        taken[a] = not any(taken[b] for b in neighbours[a])
    return [int(a) for a in np.flatnonzero(taken)]


def check_solve_arguments(schedule: str, acceleration: bool, max_rounds: int, check_every: int,
                          momentum_blocks: str = "agents") -> None:
    """solve() runs accelerated rounds only with the momentum over colour classes: there an accelerated round ends with
    every active agent's status record as the reference's iterate() leaves it (relative change against XPrev, one
    optimising call per round)."""
    if acceleration and (schedule != "coloured" or momentum_blocks != "colours"):
        raise ValueError("solve() supports acceleration=True only with schedule='coloured' and momentum_blocks='colours'; "
                         "drive other accelerated runs with step()")
    if max_rounds < 1 or check_every < 1:
        raise ValueError("max_rounds and check_every must be >= 1")
    if schedule == "greedy" and check_every != 1:
        raise ValueError("the greedy schedule selects the next agent from every round's status: check_every must be 1")


def check_accel_arguments(schedule: str, momentum_blocks: str) -> None:
    if momentum_blocks not in ("agents", "colours"):
        raise ValueError("momentum_blocks must be 'agents' or 'colours'")
    if momentum_blocks == "colours" and schedule != "coloured":
        raise ValueError("momentum_blocks='colours' counts the colour classes of the coloured schedule: it needs "
                         "schedule='coloured'")


def auto_concurrent(colour: Sequence[int], k: int, world: int, schedule: str, acceleration: bool,
                    neighbours: Optional[Sequence[Sequence[int]]] = None) -> bool:
    """Default launch mode of a k-agent run over `world` ranks (contiguous blocks of k/world agents per rank): the agents of
    a round step side by side (thread-block clusters, dpgo_agents_round_async) when some rank hosts >= 2 agents of one
    colour class under the coloured schedule, or >= 2 agents that are not neighbours under the greedy_set schedule.  A pure
    function of the global plan, so every rank decides alike."""
    per_rank = k // max(world, 1)
    if schedule == "greedy_set" and neighbours is not None:
        return any(b not in neighbours[a] for q in range(max(world, 1))
                   for a in range(q * per_rank, (q + 1) * per_rank) for b in range(a + 1, (q + 1) * per_rank))
    if schedule != "coloured" or acceleration:
        return False
    ncol = max(colour) + 1
    most = max(sum(1 for a in range(q * per_rank, (q + 1) * per_rank) if colour[a] == c)
               for q in range(max(world, 1)) for c in range(ncol))
    return most >= 2


def _ptrs(values) -> C.Array:
    """A C array of pointers: handles, device or pinned host addresses."""
    values = list(values)
    return (C.c_void_p * len(values))(*values)


def _i32(values) -> C.Array:
    values = list(values)
    return (C.c_int32 * len(values))(*values)


class _Gathered:
    """`part` doubles per agent that every rank holds for all k agents, in agent order (`all`).  Each local agent writes its
    part, `part[a]`, into this rank's parts (`own`), and one all-gather fills every rank's `all` from them: a rank's agents
    are a contiguous run, so rank-major all-gather order is agent order.  With one rank `own` is `all` and nothing moves."""

    def __init__(self, torch, dev, k: int, local_ids: Sequence[int], part: int, distributed: bool):
        self.distributed = distributed
        self.all = torch.zeros(k * part, dtype=torch.float64, device=dev)
        self.own = torch.zeros(len(local_ids) * part, dtype=torch.float64, device=dev) if distributed else self.all
        base = local_ids[0] if distributed else 0
        self.part = {a: self.own[(a - base) * part:(a - base + 1) * part] for a in local_ids}

    def gather(self, dist) -> None:
        if self.distributed:
            dist.all_gather_into_tensor(self.all, self.own)


class _Calls:
    """The arguments of the batched C calls for one active set, on this rank: the set's local agents in local order
    (`agents`, `ids`), their handles, the destinations of their X and Y tiles, the 0/1 active flags over every local agent,
    and, once step_host has made its pinned buffers, their host iterates (`host`)."""

    def __init__(self, run: "DistributedPGO", active: Sequence[int]):
        self.agents = [a for a in run.local_ids if a in active]
        self.ids = _i32(self.agents)
        self.flags = _i32(int(a in active) for a in run.local_ids)
        self.handles = _ptrs(run.agents[a].mProblem._h for a in self.agents)
        self.x_dst = _ptrs(run.tiles.part[a].data_ptr() for a in self.agents)
        self.y_dst = _ptrs(run.aux_tiles.part[a].data_ptr() for a in self.agents) if run.acceleration else None
        self.host: Optional[C.Array] = None


@dataclass
class _HostBuffers:
    """The pinned host memory of step_host and step_host_dict."""
    X: Dict[int, np.ndarray]   # each local agent's iterate, an (r, (d+1)n) Fortran-ordered view of its pinned buffer
    send: object               # torch tensors: this rank's public tiles, and every agent's
    gathered: object


class DistributedPGO:
    """One agent per rank (torch.distributed) or all agents in one process (single-GPU simulation).

    schedule = "greedy"   : the reference's synchronous driver (one agent per round, argmax of the per-agent
                            gradient norm; examples/MultiRobotExample.cpp:229-334) -- parity mode;
             = "coloured" : all agents of one colour class per round (concurrent, same RBCD semantics);
             = "parallel" : every agent every round on the neighbours' previous poses;
             = "greedy_set": the greedy rule applied to as many agents as RBCD allows: each round a maximal set of agents
                            that share no edge, taken in decreasing block gradient norm (greedy_independent_set), chosen on
                            the device from the team status taken before the round, so rounds need no host synchronisation.
    Per round: G rebuild from the gathered public poses -> local optimise -> pack -> ONE all-gather; with evaluation, the
    team status (one status launch per GPU, one all-gather of the records) gives the central cost / gradient norm /
    selection.
    """

    def __init__(self, edges: EdgeSet, n: int, k: int, r: int = 5, algorithm: int = ROPTALG.RTR,
                 preconditioner: int = capi.PRECOND_SPARSE_EXACT, schedule: str = "greedy",
                 owner: Optional[np.ndarray] = None, X_init: Optional[np.ndarray] = None,
                 rank: Optional[int] = None, world: Optional[int] = None, device: int = 0, dist=None,
                 acceleration: bool = False, restart_interval: int = 30, concurrent: Optional[bool] = None,
                 initialization: str = "central", momentum_blocks: str = "agents"):
        """initialization: "central" -- every rank computes one chordal initialisation of the whole graph (or takes
        X_init); "distributed" -- the reference's multi-robot protocol (ref PGOAgentParameters::multirobot_initialization,
        include/DPGO/PGOAgent.h:129): each rank solves only its own agents' private graphs, in their own frames, on its
        GPU; agent 0 defines the global frame and the others join it wave by wave through a robust average (GNC-TLS
        rotation averaging, inlier translation mean) of the frame transforms their shared loop closures give with an
        initialised neighbour (ref src/PGOAgent.cpp:369-440).  Needs X_init None; init_report / init_times describe it.

        concurrent: the active agents of a round that share a GPU step side by side (each as one thread-block cluster on
        its own stream, one C call per round: dpgo_agents_round_async) instead of one after the other as full-grid kernels.
        None = automatic: on when some round has >= 2 active agents on a rank (coloured schedule; with acceleration only
        for momentum_blocks="colours").  The iterates of the two modes agree to rounding, not bitwise (different reduction trees), so
        comparisons across world sizes must pin the mode.

        momentum_blocks: the N of the Nesterov recurrence gamma' = (1 + sqrt(1 + 4 N^2 gamma^2)) / (2 N), alpha = 1 / (gamma N)
        (ref src/PGOAgent.cpp:1065-1075), which assumes one block update per iteration.  "agents": N = k, the reference's
        choice.  "colours": N = the number of colour classes; the agents of one class share no edge, so a coloured round is
        one exact block update and the momentum follows the rounds (schedule="coloured" only)."""
        import torch
        check_accel_arguments(schedule, momentum_blocks)
        if schedule not in ("greedy", "coloured", "parallel", "greedy_set"):
            raise ValueError("schedule must be 'greedy', 'coloured', 'parallel' or 'greedy_set'")
        if schedule == "greedy_set" and acceleration:
            raise ValueError("acceleration=True is not supported with schedule='greedy_set': the Nesterov momentum assumes a "
                             "fixed block set per round")
        self.momentum_blocks = momentum_blocks
        self.acceleration, self.restart_interval = bool(acceleration), int(restart_interval)
        self.torch = torch
        self.dist = dist
        self.k, self.n, self.r, self.d = k, n, r, edges.d
        self.edges = edges
        self.rank = rank
        self.distributed = dist is not None and world is not None and world > 1
        self.world = world if self.distributed else 1
        if self.distributed:
            assert k % world == 0, "agents must divide evenly over the ranks (contiguous blocks of k/world agents)"
        self.owner = contiguous_owner(n, k) if owner is None else np.asarray(owner, dtype=np.int64)
        parts, counts, glob = partition_edges(edges, self.owner, k)
        self.counts, self.glob = counts, glob
        self.plan = ExchangePlan([p[2] for p in parts], k)
        self.colour = self.plan.colouring()
        self.ncolours = max(self.colour) + 1
        self.schedule = schedule
        if initialization not in ("central", "distributed"):
            raise ValueError("initialization must be 'central' or 'distributed'")
        if initialization == "distributed" and X_init is not None:
            raise ValueError("initialization='distributed' computes the start itself: X_init must be None")
        self.initialization = initialization
        if X_init is None and initialization == "central":
            X_init = pg.fixedStiefelVariable(self.d, r) @ pg.chordalInitialization(self.d, n, edges)
        per_rank = k // self.world
        self.local_ids = list(range(rank * per_rank, (rank + 1) * per_rank)) if self.distributed else list(range(k))
        if concurrent is None:
            concurrent = auto_concurrent(self.colour, k, self.world, schedule, self.acceleration and momentum_blocks == "agents",
                                         [t["neighbors"] for t in self.plan.tables])
        if concurrent and schedule == "parallel":
            raise ValueError("concurrent rounds are implemented for the greedy and coloured schedules")
        self.concurrent = bool(concurrent)
        self.agents: Dict[int, PGOAgent] = {}
        dh = self.d + 1
        self.dev = torch.device("cuda", device)
        stream = torch.cuda.current_stream(self.dev).cuda_stream
        self._main_stream = stream if stream else 1          # 0 = torch's legacy default stream = cudaStreamLegacy (handle 1)
        # the torch stream the runner's work is issued on (the current stream when it was built)
        self._stream = torch.cuda.default_stream(self.dev) if self._main_stream == 1 else \
            torch.cuda.ExternalStream(self._main_stream, device=self.dev)
        self._lib = capi.load_library()
        YLift = np.asfortranarray(pg.fixedStiefelVariable(self.d, r))
        self.init_times = {}
        if initialization == "distributed":
            for a in range(k):                             # every rank checks every agent, so all ranks raise alike
                check_private_graph_connected(a, int(counts[a]), EdgeSet.join([parts[a][0], parts[a][1]]))
            self.init_times["local_chordal_s"] = 0.0
        for a in self.local_ids:
            prm = PGOAgentParameters(self.d, r, k, algorithm=algorithm, preconditioner=preconditioner, device=device,
                                     cluster=self.concurrent)
            ag = PGOAgent(a, prm)
            ag.mState = PGOAgentState.WAIT_FOR_DATA
            ag.YLift = None
            ag.setPoseGraph(*parts[a], TInit=np.zeros((self.d, dh * int(counts[a]))), n=int(counts[a]))
            ag.mProblem.set_stream(stream)
            if X_init is not None:
                cols = (glob[a][:, None] * dh + np.arange(dh)[None, :]).ravel()
                ag.setX(X_init[:, cols])
                ag.mProblem.upload_X(ag.X)
            else:                                          # ref localInitialization, src/PGOAgent.cpp:947-962
                t_local = time.perf_counter()
                priv = EdgeSet.join([parts[a][0], parts[a][1]])
                T = pg.chordalInitializationGPU(self.d, int(counts[a]), priv, device=device) if counts[a] > 1 else \
                    np.hstack([np.eye(self.d), np.zeros((self.d, 1))])
                capi.check(self._lib.dpgo_agent_set_local_trajectory(ag.mProblem._h, capi.dptr(np.asfortranarray(T)),
                                                                     capi.dptr(YLift)))          # synchronous
                self.init_times["local_chordal_s"] += time.perf_counter() - t_local
            ag.opt = _rbcd_step_optimizer(ag.mProblem, algorithm, preconditioner)
            self.agents[a] = ag
        # every agent's opt holds the same step parameters; the batched calls read them from here
        self._params = C.byref(self.agents[self.local_ids[0]].opt.params())
        self.momentum_N = float(self.ncolours if momentum_blocks == "colours" else k)
        self.slot_elems = self.plan.pmax * r * dh
        self._num_slots = k * self.plan.pmax
        self.tiles = _Gathered(torch, self.dev, k, self.local_ids, self.slot_elems, self.distributed)   # public tiles of X
        # Nesterov-accelerated RBCD (ref src/PGOAgent.cpp:685-695,1040-1091): auxiliary iterates resident per agent,
        # their public tiles in a second gathered buffer (ref getAuxSharedPoseDict / updateAuxNeighborPoses)
        self.aux_tiles = _Gathered(torch, self.dev, k, self.local_ids, self.slot_elems, self.distributed) \
            if self.acceleration else None
        self.records = _Gathered(torch, self.dev, k, self.local_ids, capi.STATUS_DOUBLES, self.distributed)
        self._status_slots = _i32(range(len(self.local_ids)))              # agent order within the rank
        # the active sets of the schedule, and all agents: the parallel and greedy_set rounds, and the calls over every
        # local agent
        sets = [list(range(k))]
        if schedule == "coloured":
            sets += [[a for a in range(k) if self.colour[a] == c] for c in range(self.ncolours)]
        elif schedule == "greedy":
            sets += [[a] for a in range(k)]
        self._calls = {tuple(s): _Calls(self, s) for s in sets}
        self._local = self._calls[tuple(range(k))]
        self._host: Optional[_HostBuffers] = None         # step_host / step_host_dict only, made on first use
        self.selected = [0]
        self.round = 0
        self._gathered_current = False       # `tiles.all` holds every agent's current public tiles
        self._records_current = False        # `records.all` holds every agent's record of the current iterates
        self.init_report = None
        self._setup_agents(candidates=initialization == "distributed")

    def _setup_agents(self, candidates: bool) -> None:
        """The per-agent device setup of the rounds, each call replacing what it set before on the live handles: every local
        agent's public poses and shared edges; with `candidates` its alignment candidates, and under the distributed start
        the alignment waves; with acceleration the auxiliary iterates, from the current X; under greedy_set the agent
        graph."""
        for a in self.local_ids:
            ag = self.agents[a]
            ag.attach_exchange(self.plan)
            if candidates:
                ct = alignment_candidates(a, ag.sharedLoopClosures, self.plan)
                capi.check(self._lib.dpgo_agent_set_align_candidates(ag.mProblem._h, len(ct["neighbor"]),
                                                                     capi.iptr(ct["neighbor"]), capi.iptr(ct["ptr"]),
                                                                     capi.iptr(ct["local"]), capi.iptr(ct["slot"]),
                                                                     capi.iptr(ct["outgoing"]), capi.dptr(ct["T"])))
        if self.initialization == "distributed":
            self._align_waves()
        if self.acceleration:
            for a in self.local_ids:
                capi.check(self._lib.dpgo_agent_accel_init(self.agents[a].mProblem._h))
        if self.schedule == "greedy_set":
            nb = [t["neighbors"] for t in self.plan.tables]
            ptr = np.concatenate([[0], np.cumsum([len(x) for x in nb])]).astype(np.int32)
            adj = np.array([b for x in nb for b in x] or [0], dtype=np.int32)
            capi.check(self._lib.dpgo_agents_set_agent_graph(self._local.handles[0], self.k, capi.iptr(ptr), capi.iptr(adj)))

    # -- distributed initialisation: alignment waves (ref src/PGOAgent.cpp:369-440, examples/MultiRobotExample.cpp:245-256) --
    def _align_waves(self) -> None:
        """Wave w >= 1: one exchange of the public tiles; every agent that is not initialised and has a neighbour
        initialised before the wave tries those neighbours in increasing id on the device (one call per GPU); the first
        with a non-empty inlier set moves the agent into the global frame.  The outcome travels by one small all-gather
        per wave.  At most k - 1 waves: a wave that initialises nobody is an error.  Sets init_report, init_times["waves_s"]
        and every local agent's X."""
        torch, k = self.torch, self.k
        torch.cuda.synchronize(self.dev)
        t_waves = time.perf_counter()
        ready = np.zeros(k, dtype=np.int32)
        ready[0] = 1
        report = [dict(wave=-1, neighbor=-1, candidates=0, inliers=0, iterations=0) for _ in range(k)]
        report[0]["wave"] = 0
        base = self.local_ids[0]
        if self.distributed:
            rec_local = torch.zeros(5 * len(self.local_ids), dtype=torch.float64, device=self.dev)
            rec_all = torch.zeros(5 * k, dtype=torch.float64, device=self.dev)
        wave = 0
        while not ready.all():
            wave += 1
            self.exchange(build=False)
            todo = [a for a in self.local_ids if not ready[a] and any(ready[b] for b in self.plan.tables[a]["neighbors"])]
            rec = np.zeros((len(self.local_ids), 5))        # aligned, neighbour, candidates, inliers, GNC iterations
            if todo:
                hs = _ptrs(self.agents[a].mProblem._h for a in todo)
                capi.check(self._lib.dpgo_agents_align_async(hs, len(todo), self.tiles.all.data_ptr(), self._num_slots,
                                                             capi.iptr(ready), k, self._main_stream))
                info = np.zeros(4, dtype=np.int32)
                for a in todo:
                    capi.check(self._lib.dpgo_agent_align_result(self.agents[a].mProblem._h, None, capi.iptr(info)))
                    rec[a - base] = (1.0 if info[2] > 0 else 0.0, info[0], info[1], info[2], info[3])
            if self.distributed:
                rec_local.copy_(torch.from_numpy(rec.ravel()))
                self.dist.all_gather_into_tensor(rec_all, rec_local)
                rec = rec_all.cpu().numpy().reshape(k, 5)
            newly = []
            for a in range(k):
                if rec[a, 2] > 0:
                    report[a].update(neighbor=int(rec[a, 1]), candidates=int(rec[a, 2]), inliers=int(rec[a, 3]),
                                     iterations=int(rec[a, 4]))
                if rec[a, 0] > 0:
                    report[a]["wave"] = wave
                    newly.append(a)
            if not newly:
                rest = [a for a in range(k) if not ready[a]]
                raise RuntimeError(f"distributed initialisation: agents {rest} cannot join the global frame (no initialised "
                                   f"neighbour gives a non-empty inlier set; is the agent graph connected?)")
            ready[newly] = 1
        torch.cuda.synchronize(self.dev)
        self.init_times["waves_s"] = time.perf_counter() - t_waves
        for a in self.local_ids:
            self.agents[a].X = self.agents[a].mProblem.download_X()
            self.agents[a].mState = PGOAgentState.INITIALIZED
        self.init_report = report

    # -- the exchange: ONE all-gather of the padded public-pose tiles --------------------------------
    def exchange(self, build: bool = True) -> None:
        for a in self.local_ids:
            self.agents[a].pack_public(self.tiles.part[a].data_ptr())
        self.tiles.gather(self.dist)
        if build:
            for a in self.local_ids:
                self.agents[a].build_G(self.tiles.all.data_ptr(), self._num_slots)

    def _round(self, active: List[int], publish: bool = True) -> None:
        """G rebuild -> RTR step -> pack for every active local agent with one C call (thread-block cluster agents side by
        side on their own streams, full-grid agents one after the other); then, with publish, the all-gather of the new
        public tiles.  The gathered tiles must be current.  Asynchronous (no host synchronisation)."""
        self._records_current = False
        call = self._calls[tuple(active)]
        if call.agents:
            capi.check(self._lib.dpgo_agents_round_async(call.handles, len(call.agents), self._params,
                                                         self.tiles.all.data_ptr(), self._num_slots, call.x_dst,
                                                         self._main_stream, int(self.schedule == "parallel")))
        if publish:
            self.tiles.gather(self.dist)

    _round_concurrent = _round               # bench.py times its rounds through this name

    def _select_round(self) -> None:
        """One greedy_set round: the team status of the current iterates on the device (skipped when it is current; multi-rank:
        one all-gather of the records), then one dpgo_agents_select_round_async call (selection, then the gated G rebuild ->
        step -> pack of every local agent), then the all-gather of the new public tiles.  No host synchronisation."""
        self._publish()
        if not self._records_current:
            self._status_device()
        loc = self._local
        capi.check(self._lib.dpgo_agents_select_round_async(loc.handles, len(loc.agents), loc.ids, self._params,
                                                            self.records.all.data_ptr(), self.tiles.all.data_ptr(),
                                                            self._num_slots, loc.x_dst, self._main_stream))
        self.tiles.gather(self.dist)
        self._records_current = False

    def selection_log(self, first: int = 0, count: Optional[int] = None) -> List[List[int]]:
        """The agents each greedy_set round selected (sorted), rounds first .. first + count - 1 (None: to the last round
        issued).  Synchronises the device."""
        if self.schedule != "greedy_set":
            raise ValueError("selection_log() needs schedule='greedy_set'")
        lead = self._local.handles[0]
        total = C.c_int64(0)
        capi.check(self._lib.dpgo_agents_selection_log(lead, 0, 0, None, C.byref(total)))
        count = max(0, total.value - first) if count is None else max(0, min(count, total.value - first))
        buf = np.zeros(max(count, 1) * self.k, dtype=np.uint8)
        if count:
            capi.check(self._lib.dpgo_agents_selection_log(lead, first, count, buf.ctypes.data_as(C.POINTER(C.c_uint8)),
                                                           C.byref(total)))
        return [[int(a) for a in np.flatnonzero(row)] for row in buf[:count * self.k].reshape(count, self.k)]

    def _active(self) -> List[int]:
        if self.schedule == "greedy_set":
            raise ValueError("the greedy_set schedule selects on the device: drive it with step() or solve()")
        if self.schedule == "greedy":
            return list(self.selected)
        if self.schedule == "coloured":
            c = self.round % self.ncolours
            return [a for a in range(self.k) if self.colour[a] == c]
        return list(range(self.k))

    def _step_accelerated(self) -> List[int]:
        """One round of the accelerated schedule, in the reference driver's order (examples/MultiRobotExample.cpp:236-279):
        every agent advances gamma / alpha / Y and the idle agents finish their iterate(false) (X = Y, V, restart), one
        launch per GPU that also packs the public tiles of X and Y; the two tile sets are exchanged; the active agents step
        from Y with G built from the neighbours' Y tiles, then update V (and restart), with one call per GPU.  No host
        synchronisation."""
        active = self._active()
        call, loc = self._calls[tuple(active)], self._local
        capi.check(self._lib.dpgo_agents_accel_begin_async(loc.handles, len(loc.agents), call.flags, self.momentum_N,
                                                           self.restart_interval, loc.x_dst, loc.y_dst, self._main_stream))
        self.tiles.gather(self.dist)
        self.aux_tiles.gather(self.dist)
        if call.agents:
            capi.check(self._lib.dpgo_agents_accel_round_async(call.handles, len(call.agents), self._params,
                                                               self.tiles.all.data_ptr(), self.aux_tiles.all.data_ptr(),
                                                               self._num_slots, self._main_stream))
        for a in call.agents:
            self.agents[a].mIterationNumber += 1
        self._gathered_current = False       # the gathered X tiles predate the active agents' steps
        self._records_current = False
        return active

    def step(self, evaluate: bool = True) -> Optional[RoundStats]:
        """One round, then (optionally) the team status: central cost, gradient norm and the greedy selection.  Under the
        greedy_set schedule the round's agents are read from the selection log, and only when evaluate is True."""
        if self.schedule == "greedy_set":
            with self.torch.cuda.stream(self._stream):
                self._select_round()
            self.round += 1
            if not evaluate:
                return None
            st = self.status()
            return RoundStats(st.cost, st.gradnorm, self.selection_log(self.round - 1, 1)[0])
        if self.acceleration:
            active = self._step_accelerated()
        else:
            active = self._active()
            self._publish()
            self._round(active)
            for a in self.local_ids:
                if a in active:
                    self.agents[a].mIterationNumber += 1
        self.round += 1
        if not evaluate:
            return None
        st = self.status()
        self._select(st)
        return RoundStats(st.cost, st.gradnorm, active)

    # -- one round with host buffers in and out (the public host-level call of the runner) ---------------------------
    def _host_buffers(self) -> _HostBuffers:
        """The pinned host buffers, made on the first host round (only step_host and step_host_dict need them); they also
        complete the call table's host pointers."""
        if self._host is None:
            def pinned(*shape):
                return self.torch.zeros(shape, dtype=self.torch.float64).pin_memory()
            X = {a: pinned((self.d + 1) * self.agents[a].n, self.r) for a in self.local_ids}
            for call in self._calls.values():
                call.host = _ptrs(X[a].data_ptr() for a in call.agents)
            self._host = _HostBuffers({a: t.numpy().T for a, t in X.items()}, pinned(len(self.local_ids) * self.slot_elems),
                                      pinned(self.k * self.slot_elems))
        return self._host

    def step_host(self) -> None:
        """One round with every iterate crossing the host boundary: one call uploads every local agent's X from pinned host
        memory and packs its public tiles, the all-gather publishes them, one call steps the active agents, one call reads
        their iterates back, then one synchronisation (the calls are replayed as CUDA graphs when they can be).  ag.X (host)
        is the state between rounds."""
        self._records_current = False
        hx = self._host_buffers().X
        for a in self.local_ids:
            if hx[a] is not self.agents[a].X:
                hx[a][...] = self.agents[a].X
        active = self._active()
        call, loc = self._calls[tuple(active)], self._local
        capi.check(self._lib.dpgo_agents_host_io_async(loc.handles, len(loc.agents), loc.host, loc.x_dst, 0,
                                                       self._main_stream))
        self.tiles.gather(self.dist)
        self._round(active, publish=False)               # the next host round re-publishes every agent's tiles
        self._gathered_current = False
        if call.agents:
            capi.check(self._lib.dpgo_agents_host_io_async(call.handles, len(call.agents), call.host, None, 1,
                                                           self._main_stream))
            self.agents[call.agents[0]].mProblem.sync()
        for a in call.agents:
            self.agents[a].X = hx[a]
            self.agents[a].mIterationNumber += 1
        self.round += 1

    # -- the same round through the HOST-level interface (reference protocol: host matrices in and out) -------
    def step_host_dict(self) -> None:
        """One round with every iterate crossing the host boundary, as a user of the reference API would drive it:
        getSharedPoseDict -> (all-gather of the host-packed public poses) -> updateNeighborPoses -> iterate(), i.e.
        per active agent H2D of X and G, one persistent kernel, D2H of X.  Used for the end-to-end number."""
        self._records_current = False
        dh, ts = self.d + 1, self.r * (self.d + 1)
        host = self._host_buffers()
        hs = host.send.numpy()
        for li, a in enumerate(self.local_ids):
            ag = self.agents[a]
            base = li * self.slot_elems
            for s, q in enumerate(self.plan.public[a]):
                hs[base + s * ts: base + (s + 1) * ts] = ag.X[:, q * dh:(q + 1) * dh].ravel(order="F")
        if self.distributed:
            self.tiles.own.copy_(host.send, non_blocking=True)
            self.tiles.gather(self.dist)
            host.gathered.copy_(self.tiles.all, non_blocking=False)
            hg = host.gathered.numpy()
        else:
            hg = hs
        active = self._active()
        for a in self.local_ids:
            if a not in active:
                continue
            ag = self.agents[a]
            for b in self.plan.tables[a]["neighbors"]:
                poses = {}
                for s, q in enumerate(self.plan.public[b]):
                    off = (b * self.plan.pmax + s) * ts
                    poses[(b, int(q))] = hg[off:off + ts].reshape(self.r, dh, order="F")
                ag.updateNeighborPoses(b, poses)
            ag.iterate(True)
        self._gathered_current = False       # iterate() replaced the resident iterates behind the gathered tiles
        self.round += 1

    def host_bytes_per_step(self):
        """(h2d, d2h) bytes this rank moves per step_host round: every local agent's X in, the active agents' X out."""
        vb = [self.r * (self.d + 1) * int(self.counts[a]) * 8 for a in self.local_ids]
        nact = max(1, len(self.local_ids) // max(self.ncolours, 1)) if self.schedule == "coloured" else len(self.local_ids)
        return int(sum(vb)), int(sum(sorted(vb)[-nact:]))

    def assemble(self) -> np.ndarray:
        """Gather the full iterate on the host (all local agents; distributed: rank-local block only)."""
        dh = self.d + 1
        X = np.zeros((self.r, dh * self.n))
        for a in self.local_ids:
            cols = (self.glob[a][:, None] * dh + np.arange(dh)[None, :]).ravel()
            X[:, cols] = self.agents[a].mProblem.download_X()
        return X

    # -- running to convergence: team status, stop rule, trajectory -------------------------------------------------
    def status(self) -> TeamStatus:
        """Every agent's status record (capi.STATUS_DOUBLES each) with the central 2f and |grad|: one exchange (skipped
        when the gathered tiles are already current), one status launch for the agents of this GPU, one copy to the host
        (distributed: one all-gather of the records first).  All of it is ordered on the runner's stream, whichever torch
        stream is current."""
        with self.torch.cuda.stream(self._stream):
            return self._status()

    def _publish(self) -> None:
        """Every agent's current public tiles into tiles.all: one exchange, none when they are there already (plain rounds
        keep them so)."""
        if not self._gathered_current:
            self.exchange(build=False)
            self._gathered_current = True

    def _refresh_G(self) -> None:
        """Every local agent's G from the current public tiles."""
        self._publish()
        for a in self.local_ids:
            self.agents[a].build_G(self.tiles.all.data_ptr(), self._num_slots)

    def _status(self) -> TeamStatus:
        self._status_device()
        return team_status(self.records.all.cpu().numpy().reshape(self.k, capi.STATUS_DOUBLES))

    def _status_device(self) -> None:
        """Every agent's status record into records.all on the device (multi-rank: one all-gather of the records), on the
        runner's stream, without a host synchronisation."""
        self._refresh_G()
        loc = self._local
        capi.check(self._lib.dpgo_agents_status_async(loc.handles, len(loc.agents), self._status_slots,
                                                      self.records.own.data_ptr(), self._main_stream))
        self.records.gather(self.dist)
        self._records_current = True

    def _select(self, st: TeamStatus) -> None:
        if self.schedule == "greedy":
            cur = self.selected[0]
            self.selected = [greedy_selection(cur, np.sqrt(st.records[:, 2]), bool(self.plan.tables[cur]["neighbors"]))]

    def solve(self, max_rounds: int = 500, gradnorm_tol: float = 0.1, rel_change_tol: float = 5e-3, check_every: int = 1,
              callback=None) -> SolveReport:
        """Run rounds until the stop rule holds (see stop_reason): the status is taken after every check_every-th round
        and after the last one; the rounds in between are issued without a host synchronisation.  callback(round, cost,
        gradnorm) sees every check.  The greedy schedule selects the next agent from each round's status, as step() does,
        so it needs check_every = 1.  Accelerated runs need schedule="coloured" with momentum_blocks="colours"."""
        check_solve_arguments(self.schedule, self.acceleration, max_rounds, check_every, self.momentum_blocks)
        with self.torch.cuda.stream(self._stream):
            return self._solve(max_rounds, gradnorm_tol, rel_change_tol, check_every, callback)

    def _solve(self, max_rounds, gradnorm_tol, rel_change_tol, check_every, callback) -> SolveReport:
        calls_at_start = self.status().records[:, 4].copy()
        rounds = 0
        while True:
            self.step(evaluate=False)
            rounds += 1
            if rounds % check_every != 0 and rounds < max_rounds:
                continue
            st = self.status()
            if callback is not None:
                callback(rounds, st.cost, st.gradnorm)
            self._select(st)
            reason = stop_reason(st.records, calls_at_start, rounds, max_rounds, gradnorm_tol, rel_change_tol)
            if reason is not None:
                return SolveReport(rounds, reason, st.cost, st.gradnorm, st.records[:, 3].copy())

    def trajectory(self) -> np.ndarray:
        """The d x (d+1)n trajectory in global pose order, rounded on the device (ref getTrajectoryInGlobalFrame,
        src/PGOAgent.cpp:500-519) against agent 0's local pose 0 (ref examples/MultiRobotExample.cpp:328-333).
        Distributed: the anchor is broadcast from agent 0's rank and only this rank's columns are filled."""
        d, dh, r = self.d, self.d + 1, self.r
        anchor = np.zeros((r, dh), order="F")
        if 0 in self.agents:
            anchor[...] = self.agents[0].mProblem.download_X()[:, :dh]
        if self.distributed:
            torch = self.torch
            with torch.cuda.stream(self._stream):
                buf = torch.from_numpy(anchor.ravel(order="F")).to(self.dev)
                self.dist.broadcast(buf, src=0)
                anchor = np.asfortranarray(buf.cpu().numpy().reshape(r, dh, order="F"))
        T = np.zeros((d, dh * self.n))
        for a in self.local_ids:
            ag = self.agents[a]
            out = np.zeros((d, dh * ag.n), order="F")
            capi.check(self._lib.dpgo_agent_trajectory_global(ag.mProblem._h, capi.dptr(anchor), capi.dptr(out)))
            cols = (self.glob[a][:, None] * dh + np.arange(dh)[None, :]).ravel()
            T[:, cols] = out
        return T

    def pose_covariances(self, anchor: Optional[int] = None, pairs=None):
        """Marginal covariances of the rounded trajectory() (pg.poseCovariancesGPU on this process's GPU), anchored at
        agent 0's pose 0, the gauge of trajectory(), unless `anchor` names another global pose.  Single-process runs only:
        the whole graph and trajectory must be on this process."""
        if self.distributed:
            raise ValueError("pose_covariances() needs the whole pose graph in one process: a multi-rank run holds only its "
                             "own agents' poses (call pg.poseCovariancesGPU on a gathered trajectory instead)")
        a = int(self.glob[0][0]) if anchor is None else int(anchor)
        return pg.poseCovariancesGPU(self.edges, self.n, self.trajectory(), anchor=a, pairs=pairs, device=self.dev.index or 0)
