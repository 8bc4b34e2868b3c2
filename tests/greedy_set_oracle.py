"""CPU restatement of the greedy_set round of the device runners: each round, every agent's block of the central Riemannian
gradient selects the round's agents with the shared host rule (dpo_b200.agent.greedy_independent_set); those agents see
their neighbours' poses as they were at the start of the round and step, the others stay put (ref
examples/MultiRobotExample.cpp:229-334, with the single greedy choice replaced by a maximal set of agents that share no
edge)."""
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from oracle import dpgo_oracle as orc  # noqa: E402
from dpo_b200.agent import greedy_independent_set  # noqa: E402


class GreedySetDriver(orc.MultiRobotDriver):
    def __init__(self, meas, n, k, r=5, **kw):
        super().__init__(meas, n, k, r=r, schedule="coloured", **kw)
        self.schedule = "greedy_set"
        self.sets = []               # the agents of every round
        self.norms2 = []             # the squared block gradient norms each round selected from
        self._g2 = self.block_gradnorm2(self.central.rie_grad(self.assemble()))

    def block_gradnorm2(self, RG):
        dh = self.d + 1
        out = np.zeros(self.k)
        for a in range(self.k):
            cols = (self.glob[a][:, None] * dh + np.arange(dh)[None, :]).ravel()
            out[a] = float(np.sum(RG[:, cols] ** 2))
        return out

    def step(self):
        active = greedy_independent_set(self._g2, [ag.neighbors for ag in self.agents])
        self.sets.append(active)
        self.norms2.append(self._g2)
        shared = [ag.get_shared_pose_dict() for ag in self.agents]
        for a in active:
            for b in self.agents[a].neighbors:
                self.agents[a].update_neighbor_poses(b, shared[b])
        for a in active:
            self.agents[a].iterate(True)
        self.round += 1
        X = self.assemble()
        RG = self.central.rie_grad(X)
        self._g2 = self.block_gradnorm2(RG)
        gn = float(np.linalg.norm(RG))
        cost = 2.0 * self.central.f(X)
        self.trace.cost.append(cost)
        self.trace.gradnorm.append(gn)
        self.trace.selected.append(active[0])
        return cost, gn
