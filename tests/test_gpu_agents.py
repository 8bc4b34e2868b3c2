"""Multi-agent path on the GPU: device-side public-pose packing + G assembly + the greedy RBCD schedule
must reproduce the reference's shipped traces; the coloured schedule must reach the same optimum."""
import os

import numpy as np
import pytest

from oracle import dpgo_oracle as orc

pytestmark = pytest.mark.gpu


def load(ds, data_dir):
    from dpo_b200 import posegraph as pg
    return pg.read_g2o_file(os.path.join(data_dir, ds + ".g2o"))


@pytest.mark.parametrize("ds,iters", [("smallGrid3D", 120), ("sphere2500", 50), ("torus3D", 30), ("CSAIL", 40), ("grid3D", 25),
                                      ("parking-garage", 25), ("rim", 20), ("ais2klinik", 20), ("city10000", 12), ("cubicle", 12),
                                      ("input_INTEL_g2o", 20), ("input_M3500_g2o", 20), ("input_MITb_g2o", 20),
                                      ("sphere_bignoise_vertex3", 15)])
def test_greedy_schedule_reproduces_golden_trace(ds, iters, data_dir, golden_dir):
    from dpo_b200.agent import DistributedPGO
    edges, n = load(ds, data_dir)
    run = DistributedPGO(edges, n, 5, r=5, schedule="greedy")
    gold = np.loadtxt(os.path.join(golden_dir, f"NP{ds}_head400.txt"), delimiter=",")[:iters]
    cost, gn = [], []
    for _ in range(iters):
        st = run.step()
        cost.append(st.cost)
        gn.append(st.gradnorm)
    # parking-garage is ill-conditioned (kappa ~ 2, tau ~ 1: every tCG solve runs to its 10-iteration cap), so the
    # summation-order differences of the device-side G assembly are amplified above the print precision of the trace
    # (ais2klinik, SE(2), 15115 poses: the oracle itself sits 8e-9 from the printed trace, tests/test_oracle_golden.py)
    ctol, gtol = (5e-8, 5e-6) if ds == "parking-garage" else ((2e-8, 5e-8) if ds == "ais2klinik" else (5e-9, 5e-8))
    assert np.max(np.abs(np.array(cost) - gold[:, 0]) / gold[:, 0]) <= ctol
    assert np.max(np.abs(np.array(gn) - gold[:, 1]) / gold[:, 1]) <= gtol


@pytest.mark.parametrize("strength,ds,iters", [("strong", "CSAIL", 60), ("strong", "sphere2500", 40), ("eco", "sphere2500", 20),
                                               ("fast", "torus3D", 15), ("strong", "torus3D", 15), ("strong", "parking-garage", 12),
                                               ("eco", "CSAIL", 30), ("fast", "rim", 10), ("strong", "city10000", 10)])
def test_partition_file_reproduces_golden_trace(strength, ds, iters, data_dir, golden_dir):
    """Non-contiguous ownership from the reference's partition files (graph/5/<strength>/<dataset>, KaHIP presets) through
    the device runner: agents own scattered poses -- against result/graph/<strength><dataset>.txt."""
    from dpo_b200.agent import DistributedPGO
    from dpo_b200 import posegraph as pg
    edges, n = load(ds, data_dir)
    owner = pg.read_partition_file(os.path.join(golden_dir, f"partition5_{strength}_{ds}.txt"), n)
    run = DistributedPGO(edges, n, 5, r=5, schedule="greedy", owner=owner)
    gold = np.loadtxt(os.path.join(golden_dir, f"{strength}{ds}_head400.txt"), delimiter=",")[:iters]
    cost, gn = [], []
    for _ in range(iters):
        st = run.step()
        cost.append(st.cost)
        gn.append(st.gradnorm)
    ctol, gtol = (5e-8, 5e-6) if ds == "parking-garage" else (5e-9, 5e-8)
    assert np.max(np.abs(np.array(cost) - gold[:, 0]) / gold[:, 0]) <= ctol
    assert np.max(np.abs(np.array(gn) - gold[:, 1]) / gold[:, 1]) <= gtol


@pytest.mark.parametrize("ds,k,rounds,conc", [("torus3D", 8, 10, False), ("parking-garage", 4, 8, False), ("sphere2500", 8, 8, False),
                                              ("torus3D", 8, 10, True), ("parking-garage", 4, 8, True), ("sphere2500", 16, 8, True)])
def test_coloured_schedule_matches_oracle(ds, k, rounds, conc, data_dir):
    """The schedule the multi-GPU benchmark runs (BASELINE configs 3 and 4 and the sphere2500 scaling workload): k
    agents, coloured RBCD, exact preconditioner -- per-round central cost / gradient norm and the iterates against the
    oracle's coloured driver (<= 1e-8 relative).  conc: the agents of a round one after the other as full-grid
    cooperative kernels, or side by side as thread-block clusters on their own streams (dpgo_agents_round_async)."""
    from dpo_b200.agent import DistributedPGO
    edges, n = load(ds, data_dir)
    meas, _ = orc.read_g2o(os.path.join(data_dir, ds + ".g2o"))
    import contextlib
    import torch
    # side by side: on a side stream, so that the repeated rounds are replayed as CUDA graphs (the legacy default stream
    # cannot be captured; there the call falls back to eager launches)
    ctx = torch.cuda.stream(torch.cuda.Stream()) if conc else contextlib.nullcontext()
    with ctx:
        run = DistributedPGO(edges, n, k, r=5, schedule="coloured", concurrent=conc)
        assert run.agents[0].mProblem.launch_info()[1] == conc
        drv = orc.MultiRobotDriver(meas, n, k, r=5, schedule="coloured")
        assert run.colour == drv.colour
        # (parking-garage: ill-conditioned -- kappa ~ 2, tau ~ 1, every tCG solve hits its cap -- rounding differences are amplified)
        ctol, gtol, xtol = (1e-7, 1e-5, 1e-5) if ds == "parking-garage" else (1e-8, 1e-7, 1e-8)
        for _ in range(rounds):
            st = run.step()
            cost, gn = drv.step()
            assert abs(st.cost - cost) <= ctol * abs(cost)
            assert abs(st.gradnorm - gn) <= gtol * gn
        Xg, Xo = run.assemble(), drv.assemble()
    assert np.linalg.norm(Xg - Xo) <= xtol * np.linalg.norm(Xo)


def test_final_trajectory_parking_garage(data_dir, golden_dir):
    """The reference's shipped final trajectory (result/opt_pose/NPparking-garage.csv) through the device-resident
    5-agent greedy runner; tolerance as in tests/test_oracle_golden.py."""
    from dpo_b200.agent import DistributedPGO
    edges, n = load("parking-garage", data_dir)
    run = DistributedPGO(edges, n, 5, r=5, schedule="greedy")
    for _ in range(450):
        run.step()
    X = run.assemble()
    T = X[:, :edges.d].T @ X
    ref = np.loadtxt(os.path.join(golden_dir, "NPparking-garage_opt_pose.csv"), delimiter=",")
    assert np.abs(T - ref).max() <= 5e-4


@pytest.mark.parametrize("schedule,conc", [("coloured", False), ("coloured", True), ("greedy", False), ("parallel", False)])
def test_host_level_round_equals_resident_round(schedule, conc, data_dir):
    """DistributedPGO.step_host (X from / to pinned host memory every round) and the rounds bench.py issues by hand
    (exchange, then every active agent's optimize_resident_async) == the device-resident rounds, bit for bit;
    step_host_dict (the reference's PoseDict protocol on the host) agrees to rounding.  The parallel schedule is the one
    whose round call packs after every agent's step."""
    from dpo_b200.agent import DistributedPGO
    edges, n = load("smallGrid3D", data_dir)
    runs = [DistributedPGO(edges, n, 5, r=5, schedule=schedule, concurrent=conc) for _ in range(4)]
    hand = runs[3]
    for _ in range(6):
        runs[0].step(evaluate=False)
        runs[1].step_host()
        runs[2].step_host_dict()
        active = hand._active()
        hand.exchange()
        for a in hand.local_ids:
            if a in active:
                hand.agents[a].opt.optimize_resident_async()
        hand.round += 1
    X0 = runs[0].assemble()
    assert np.array_equal(hand.assemble(), X0)
    dh = edges.d + 1
    for q, tol in ((1, 0.0), (2, 1e-11)):
        Xh = np.zeros_like(X0)
        for a, ag in runs[q].agents.items():
            cols = (runs[q].glob[a][:, None] * dh + np.arange(dh)[None, :]).ravel()
            Xh[:, cols] = ag.X
        assert np.linalg.norm(Xh - X0) <= tol * np.linalg.norm(X0)


def test_accelerated_rbcd_on_the_device_matches_oracle(data_dir):
    """Nesterov-accelerated RBCD (ref src/PGOAgent.cpp:685-695,1040-1091) with every update on the device -- gamma / alpha
    recurrences on the host, Y and V by the fused combination + Stiefel projection kernel, auxiliary public poses in a
    second gathered buffer, restart every 30 iterations -- against the oracle's accelerated greedy driver."""
    from dpo_b200.agent import DistributedPGO
    edges, n = load("smallGrid3D", data_dir)
    meas, _ = orc.read_g2o(os.path.join(data_dir, "smallGrid3D.g2o"))
    iters = 70                                           # two restarts (iterations 29 and 59)
    run = DistributedPGO(edges, n, 5, r=5, schedule="greedy", acceleration=True)
    drv = orc.MultiRobotDriver(meas, n, 5, r=5, acceleration=True)
    sel = []
    for it in range(iters):
        st = run.step()
        cost, gn = drv.step()
        sel.append(st.selected[0])
        assert abs(st.cost - cost) <= 1e-8 * abs(cost), it
        assert abs(st.gradnorm - gn) <= 1e-6 * gn, it
    assert sel == drv.trace.selected
    assert np.linalg.norm(run.assemble() - drv.assemble()) <= 1e-8 * np.linalg.norm(drv.assemble())


def test_accelerated_coloured_schedule_converges(data_dir):
    """All agents of a colour class step from their auxiliary iterates every round (the concurrent accelerated schedule):
    monotone up to the restarts' safeguards, reaches the optimum of smallGrid3D (f* = 1025.4, vis.ipynb:108745)."""
    from dpo_b200.agent import DistributedPGO
    edges, n = load("smallGrid3D", data_dir)
    run = DistributedPGO(edges, n, 5, r=5, schedule="coloured", acceleration=True)
    last = None
    for it in range(300):
        last = run.step(evaluate=(it % 10 == 9))
        if last is not None and last.gradnorm < 0.05:
            break
    assert last is not None and last.gradnorm < 0.1
    assert abs(last.cost - 1025.398) <= 2e-4 * 1025.398


def test_python_host_agent_acceleration_matches_oracle(data_dir):
    """The Python PGOAgent mirror with acceleration = True through the reference's PoseDict protocol
    (examples/MultiRobotExample.cpp:236-279) against the oracle."""
    from dpo_b200.agent import PGOAgent, PGOAgentParameters, contiguous_owner, partition_edges
    from dpo_b200 import posegraph as pg
    edges, n = load("smallGrid3D", data_dir)
    meas, _ = orc.read_g2o(os.path.join(data_dir, "smallGrid3D.g2o"))
    k, r, d = 4, 5, edges.d
    dh = d + 1
    parts, counts, glob = partition_edges(edges, contiguous_owner(n, k), k)
    X0 = pg.fixedStiefelVariable(d, r) @ pg.chordalInitialization(d, n, edges)
    agents = []
    for a in range(k):
        ag = PGOAgent(a, PGOAgentParameters(d, r, k, acceleration=True))
        ag.YLift = None
        ag.setPoseGraph(*parts[a], TInit=np.zeros((d, dh * int(counts[a]))), n=int(counts[a]))
        cols = (glob[a][:, None] * dh + np.arange(dh)[None, :]).ravel()
        ag.setX(X0[:, cols])
        agents.append(ag)
    drv = orc.MultiRobotDriver(meas, n, k, r=r, acceleration=True)
    selected = 0
    for it in range(35):                                  # crosses the restart at iteration 29
        sel = agents[selected]
        for ag in agents:
            if ag.mID != selected:
                ag.iterate(False)
        for ag in agents:
            if ag.mID != selected:
                sel.updateNeighborPoses(ag.mID, ag.getSharedPoseDict())
                sel.updateAuxNeighborPoses(ag.mID, ag.getAuxSharedPoseDict())
        sel.iterate(True)
        drv.step()
        X = np.zeros_like(X0)
        for a, ag in enumerate(agents):
            cols = (glob[a][:, None] * dh + np.arange(dh)[None, :]).ravel()
            X[:, cols] = ag.X
        assert np.linalg.norm(X - drv.assemble()) <= 1e-8 * np.linalg.norm(X), it
        selected = drv.selected                           # follow the oracle's greedy choice


def test_device_G_matches_host_G(data_dir):
    """dpgo_agent_build_G (device, from gathered slots) == constructGMatrix (host dictionary form)."""
    from dpo_b200.agent import DistributedPGO
    edges, n = load("smallGrid3D", data_dir)
    run = DistributedPGO(edges, n, 4, r=5, schedule="parallel")
    run.exchange()
    for a, ag in run.agents.items():
        poses = {}
        for b, other in run.agents.items():
            if b != a:
                other.X = other.mProblem.download_X()
                poses.update(other.getSharedPoseDict())
        # host reference
        sh = ag.sharedLoopClosures
        m = orc.Measurements(sh.d, sh.r1, sh.r2, sh.p1, sh.p2, sh.R, sh.t, sh.kappa, sh.tau, sh.weight)
        oa = orc.PGOAgent(a, ag.d, ag.r)
        oa.n = ag.n
        oa.shared_lc = m
        oa.problem = orc.QuadraticProblem(ag.n, ag.d, ag.r)
        assert oa.construct_G(poses)
        # device G is observable as the resident Euclidean gradient minus X Q: use f/lin instead:
        X = ag.mProblem.download_X()
        quad, lin, gn2, f = ag.opt.problem_stats()
        assert abs(lin - float(np.sum(X * oa.problem.G))) <= 1e-10 * max(1.0, abs(lin))


@pytest.mark.parametrize("schedule", ["coloured", "parallel"])
def test_concurrent_schedules_converge(schedule, data_dir):
    """Throughput schedules reach the same objective as the greedy one (stated tolerance 1e-6 relative)."""
    from dpo_b200.agent import DistributedPGO
    from dpo_b200 import PRECOND_BLOCK_JACOBI
    edges, n = load("smallGrid3D", data_dir)
    run = DistributedPGO(edges, n, 5, r=5, schedule=schedule, preconditioner=PRECOND_BLOCK_JACOBI)
    last = None
    for it in range(400):
        last = run.step(evaluate=(it % 20 == 19))
        if last is not None and last.gradnorm < 0.05:
            break
    assert last is not None and last.gradnorm < 0.1
    assert abs(last.cost - 1025.398) <= 2e-4 * 1025.398       # f* of smallGrid3D (vis.ipynb:108745: 1025.4)
