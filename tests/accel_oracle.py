"""CPU restatement of the accelerated coloured round of the device runners: the reference driver's order
(examples/MultiRobotExample.cpp:236-279) -- every idle agent finishes iterate(false), the X and Y tiles are exchanged, the
active agents step -- with the momentum recurrence's N selectable (the number of agents, as the reference, or the number of
colour classes: a coloured round is one exact block update)."""
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from oracle import dpgo_oracle as orc  # noqa: E402


class AcceleratedColouredDriver(orc.MultiRobotDriver):
    def __init__(self, meas, n, k, r=5, momentum_blocks="agents", restart_interval=30, **kw):
        super().__init__(meas, n, k, r=r, acceleration=True, schedule="coloured", **kw)
        N = self.ncolours if momentum_blocks == "colours" else k
        for ag in self.agents:
            ag.num_robots = N
            ag.restart_interval = restart_interval

    def _step_concurrent(self):
        active = [a for a in range(self.k) if self.colour[a] == self.round % self.ncolours]
        for a, ag in enumerate(self.agents):
            if a not in active:
                ag.iterate(False)
        shared = [ag.get_shared_pose_dict() for ag in self.agents]
        aux = [ag.get_aux_shared_pose_dict() for ag in self.agents]
        for a in active:
            for b in self.agents[a].neighbors:
                self.agents[a].update_neighbor_poses(b, shared[b])
                self.agents[a].update_aux_neighbor_poses(b, aux[b])
        for a in active:
            self.agents[a].iterate(True)
        self.round += 1
        X = self.assemble()
        gn = float(orc.np.linalg.norm(self.central.rie_grad(X)))
        cost = 2.0 * self.central.f(X)
        self.trace.cost.append(cost)
        self.trace.gradnorm.append(gn)
        self.trace.selected.append(active[0] if active else -1)
        return cost, gn


def momentum_trace(N: float, rounds: int, restart_interval: int = 30):
    """The device record {gamma, alpha, iterations} after each round, by the host recurrence in the device's operation order:
    gamma' = (1 + sqrt(1 + ((4 N) N) (gamma gamma))) / (2 N), alpha = 1 / (gamma' N), cleared on a restart round."""
    import math
    gamma, out = 0.0, []
    for it in range(1, rounds + 1):
        gamma = (1.0 + math.sqrt(1.0 + ((4.0 * N) * N) * (gamma * gamma))) / (2.0 * N)
        alpha = 1.0 / (gamma * N)
        if (it + 1) % restart_interval == 0:
            gamma = alpha = 0.0
        out.append((gamma, alpha, float(it)))
    return out
