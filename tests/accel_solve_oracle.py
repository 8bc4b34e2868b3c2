"""The reference's status fields on the CPU restatement of accelerated coloured rounds (tests/accel_oracle.py): every
agent keeps the relative change sqrt(|X - XPrev|^2 / n) of its last optimising iterate(), XPrev the iterate at that call's
start, and its optimising-call count (src/PGOAgent.cpp:673,703-716), so stop_reason applies round by round."""
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import accel_oracle as ao  # noqa: E402


class StatusRecordingDriver(ao.AcceleratedColouredDriver):
    def __init__(self, meas, n, k, **kw):
        super().__init__(meas, n, k, **kw)
        self.relative_change = np.zeros(k)
        self.calls = np.zeros(k)

    def _step_concurrent(self):
        out = super()._step_concurrent()
        active = [a for a in range(self.k) if self.colour[a] == (self.round - 1) % self.ncolours]
        for a in active:
            ag = self.agents[a]                  # iterate() keeps XPrev = the iterate at its start, restart or not
            self.relative_change[a] = np.sqrt(float(np.sum((ag.X - ag.XPrev) ** 2)) / ag.n)
            self.calls[a] += 1
        return out


def records(drv):
    """The team's status records (capi.STATUS_DOUBLES per agent) of the restatement's current iterates, as stop_reason
    reads them: [0] the central 2f split evenly over the agents, [1] 0, [2] the agent's block of |grad_central|^2,
    [3] relative change, [4] optimising calls."""
    X = drv.assemble()
    RG = drv.central.rie_grad(X)
    dh = drv.d + 1
    rec = np.zeros((drv.k, 5))
    rec[:, 0] = 2.0 * drv.central.f(X) / drv.k
    for a in range(drv.k):
        cols = (drv.glob[a][:, None] * dh + np.arange(dh)[None, :]).ravel()
        rec[a, 2] = float(np.sum(RG[:, cols] ** 2))
    rec[:, 3] = drv.relative_change
    rec[:, 4] = drv.calls
    return rec


# Workloads of the team rule with the colour momentum, and a relative-change tolerance that no agent's relative change
# comes within 1e-6 (relative) of at the stop round or the round before it, so rounding cannot move the stop: the
# restatement stops at the given round (smallGrid3D past its first restart round, torus3D on its first round after one).
TEAM_STOPS = {("smallGrid3D", 5): (5e-4, 31), ("torus3D", 8): (2e-3, 30)}


def team_stop(drv, tol, cap=200):
    """Rounds of the restatement until stop_reason's team rule holds (gradient-norm rule off); returns the stop round and
    every round's relative changes."""
    from dpo_b200.agent import stop_reason
    rcs = []
    for rounds in range(1, cap + 1):
        drv.step()
        rcs.append(drv.relative_change.copy())
        if stop_reason(records(drv), np.zeros(drv.k), rounds, cap, 0.0, tol) == "team":
            return rounds, np.array(rcs)
    return None, np.array(rcs)
