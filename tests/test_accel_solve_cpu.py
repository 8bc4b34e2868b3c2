"""solve() with colour-momentum accelerated rounds, the parts that need no GPU: the argument rules, the restatement's
status fields against the reference's formula (src/PGOAgent.cpp:673,703-716) on a hand-built two-agent graph with a
restart every other iteration, and the team rule's stop round on the restatement."""
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import accel_solve_oracle as aso  # noqa: E402
from oracle import dpgo_oracle as orc  # noqa: E402


def test_solve_arguments_with_acceleration():
    from dpo_b200.agent import check_solve_arguments
    check_solve_arguments("coloured", True, 500, 1, "colours")
    check_solve_arguments("coloured", True, 500, 5, "colours")
    with pytest.raises(ValueError, match="acceleration"):
        check_solve_arguments("coloured", True, 500, 1)                  # the reference's momentum over agents
    for schedule in ("greedy", "parallel", "greedy_set"):
        with pytest.raises(ValueError, match="acceleration"):
            check_solve_arguments(schedule, True, 500, 1, "colours")
    with pytest.raises(ValueError, match="max_rounds"):
        check_solve_arguments("coloured", True, 0, 1, "colours")
    check_solve_arguments("coloured", False, 500, 5, "agents")


def two_agent_loop(path):
    """A noisy square loop of 8 planar poses, split 4 + 4, with two loop closures across the split."""
    rng = np.random.default_rng(7)
    lines = []
    def edge(i, j, dx, dy, dth):
        dx, dy, dth = dx + 0.05 * rng.standard_normal(), dy + 0.05 * rng.standard_normal(), dth + 0.05 * rng.standard_normal()
        lines.append(f"EDGE_SE2 {i} {j} {dx} {dy} {dth} 100 0 0 100 0 400")
    for i in range(7):
        edge(i, i + 1, 1.0, 0.0, np.pi / 4)
    edge(7, 0, 1.0, 0.0, np.pi / 4)
    edge(1, 5, -1.0 - np.sqrt(2.0), 0.0, np.pi)
    edge(2, 6, -1.0 - np.sqrt(2.0), 0.0, np.pi)
    with open(path, "w") as fh:
        fh.write("\n".join(lines) + "\n")


@pytest.mark.parametrize("restart_interval", [2, 30])
def test_restatement_records_follow_the_reference(restart_interval, tmp_path):
    """Per round and active agent: relative change = sqrt(|X_end - XPrev|^2 / n) against the iterate at the round's start,
    one call more; idle agents keep both.  With restart_interval=2 agent 0 restarts on every one of its rounds (iterations
    1, 3, ...) and agent 1 never does (2, 4, ...).  On a restart round the final step starts from XPrev, so its own relative
    change is the reference's.  A plain round's step starts from Y; with restart_interval=30 Y moves away from X after the
    first rounds and the step's own relative change differs."""
    path = str(tmp_path / "loop.g2o")
    two_agent_loop(path)
    meas, n = orc.read_g2o(path)
    drv = aso.StatusRecordingDriver(meas, n, 2, r=3, momentum_blocks="colours", restart_interval=restart_interval)
    assert drv.colour == [0, 1]
    restarts, differs = {0: 0, 1: 0}, 0
    for rnd in range(12):
        before = [ag.X.copy() for ag in drv.agents]
        rel0, calls0 = drv.relative_change.copy(), drv.calls.copy()
        drv.step()
        a, b = rnd % 2, 1 - rnd % 2
        ag = drv.agents[a]
        expect = np.sqrt(np.sum((ag.X - before[a]) ** 2) / ag.n)
        assert drv.relative_change[a] == expect and expect > 0
        assert drv.calls[a] == calls0[a] + 1
        assert drv.relative_change[b] == rel0[b] and drv.calls[b] == calls0[b]
        if (ag.iteration + 1) % restart_interval == 0:
            assert abs(ag.last_result.relativeChange - expect) <= 1e-12 * expect
            restarts[a] += 1
        elif abs(ag.last_result.relativeChange - expect) > 1e-6 * expect:
            differs += 1
    assert restarts == ({0: 6, 1: 0} if restart_interval == 2 else {0: 0, 1: 0})
    assert restart_interval == 2 or differs > 0
    rec = aso.records(drv)
    assert np.array_equal(rec[:, 4], [6, 6]) and np.array_equal(rec[:, 3], drv.relative_change)


@pytest.mark.parametrize("ds,k", sorted(aso.TEAM_STOPS))
def test_team_rule_stops_at_a_definite_round(ds, k, data_dir):
    tol, expect = aso.TEAM_STOPS[(ds, k)]
    meas, n = orc.read_g2o(os.path.join(data_dir, ds + ".g2o"))
    drv = aso.StatusRecordingDriver(meas, n, k, r=5, momentum_blocks="colours")
    stop, rcs = aso.team_stop(drv, tol, cap=expect + 5)
    assert stop == expect
    assert np.all(rcs[stop - 1] <= tol) and np.any(rcs[stop - 2] > tol)
    for row in rcs[stop - 2:stop]:
        assert np.all(np.abs(row - tol) >= 1e-6 * tol), row
