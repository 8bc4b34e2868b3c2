"""Running the device runner to convergence on the GPU: the batched team status (dpgo_agents_status_async) against the
per-agent evaluation, the stop rules of DistributedPGO.solve against the golden traces, the step() loop and the oracle's
coloured driver, and the rounded trajectory (dpgo_agent_trajectory_global) against the NumPy restatement."""
import contextlib
import ctypes as C
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import solve_oracle as so  # noqa: E402
from oracle import dpgo_oracle as orc  # noqa: E402

pytestmark = pytest.mark.gpu


def load(ds, data_dir):
    from dpo_b200 import posegraph as pg
    return pg.read_g2o_file(os.path.join(data_dir, ds + ".g2o"))


def side_stream(on):
    import torch
    return torch.cuda.stream(torch.cuda.Stream()) if on else contextlib.nullcontext()


def status_alone(run, a):
    """The record of agent a from a status launch that holds agent a only."""
    import torch
    from dpo_b200 import _capi
    buf = torch.zeros(_capi.STATUS_DOUBLES, dtype=torch.float64, device=run.dev)
    hs = (C.c_void_p * 1)(run.agents[a].mProblem._h)
    slot = np.zeros(1, dtype=np.int32)
    lib = run.agents[a].mProblem._lib
    _capi.check(lib.dpgo_agents_status_async(hs, 1, _capi.iptr(slot), C.c_void_p(buf.data_ptr()), C.c_void_p(run._main_stream)))
    return buf.cpu().numpy()


@pytest.mark.parametrize("ds,k,conc", [("sphere2500", 16, True), ("sphere2500", 16, False), ("torus3D", 8, None),
                                       ("parking-garage", 4, None), ("input_INTEL_g2o", 5, None)])
def test_status_matches_per_agent_evaluation(ds, k, conc, data_dir):
    from dpo_b200.agent import DistributedPGO
    edges, n = load(ds, data_dir)
    with side_stream(conc is not False):
        run = DistributedPGO(edges, n, k, r=5, schedule="coloured", concurrent=conc)
        for _ in range(run.ncolours + 1):
            run.step(evaluate=False)
        rel = np.array([run.agents[a].opt.fetch_result().relative_change for a in range(k)])   # before any evaluation
        st = run.status()
        rec = st.records
        assert np.array_equal(rec[:, 3], rel)
        assert np.all(rec[:, 4] >= 1)
        assert np.array_equal(run.status().records, rec)                  # two calls: bitwise equal
        for a in range(k):                                                 # alone == with the others, bitwise
            assert np.array_equal(status_alone(run, a), rec[a]), a
        for a in range(k):
            quad, lin, gn2, _ = run.agents[a].opt.problem_stats()         # OP_EVAL: the result record is overwritten
            assert abs(rec[a, 0] - quad) <= 1e-12 * abs(quad)
            assert abs(rec[a, 1] - lin) <= 1e-12 * (abs(quad) + abs(lin))
            assert abs(rec[a, 2] - gn2) <= 1e-12 * gn2
        assert np.array_equal(run.status().records[:, 3], rel)            # evaluations leave the relative change alone
        run.step(evaluate=True)
        active = [a for a in range(k) if run.colour[a] == (run.round - 1) % run.ncolours]
        after = run.status().records
        for a in range(k):
            if a in active:
                assert after[a, 4] == rec[a, 4] + 1
            else:
                assert after[a, 3] == rel[a] and after[a, 4] == rec[a, 4]


@pytest.mark.parametrize("ds", ["smallGrid3D", "sphere2500"])
def test_greedy_solve_stops_at_the_golden_gradnorm(ds, data_dir, golden_dir):
    """The reference driver's stop at |g| < 0.1 (examples/MultiRobotExample.cpp:302-305): the first line of the shipped
    trace below 0.1 (SURVEY section 6: 118 and 290 rounds), with the trace's cost and gradient norm at every round."""
    from dpo_b200.agent import DistributedPGO
    edges, n = load(ds, data_dir)
    gold = np.loadtxt(os.path.join(golden_dir, f"NP{ds}_head400.txt"), delimiter=",")
    stop = int(np.flatnonzero(gold[:, 1] < 0.1)[0]) + 1
    run = DistributedPGO(edges, n, 5, r=5, schedule="greedy")
    seen = []
    rep = run.solve(gradnorm_tol=0.1, rel_change_tol=0, callback=lambda it, c, g: seen.append((it, c, g)))
    assert rep.reason == "gradnorm" and rep.rounds == stop
    tr = np.array(seen)
    assert np.array_equal(tr[:, 0], np.arange(1, stop + 1))
    assert np.max(np.abs(tr[:, 1] - gold[:stop, 0]) / gold[:stop, 0]) <= 5e-9
    assert np.max(np.abs(tr[:, 2] - gold[:stop, 1]) / gold[:stop, 1]) <= 5e-8


def test_coloured_solve_matches_step_loop(data_dir):
    """16 agents side by side, a check every 5th round: the same stop round as a step() loop that evaluates every 5th
    round, at the same 2f."""
    from dpo_b200.agent import DistributedPGO
    edges, n = load("sphere2500", data_dir)
    with side_stream(True):
        ref = DistributedPGO(edges, n, 16, r=5, schedule="coloured")
        assert ref.concurrent
        stop, last = None, None
        for it in range(1, 501):
            last = ref.step(evaluate=(it % 5 == 0))
            if last is not None and last.gradnorm < 0.1:
                stop = it
                break
        assert stop is not None
        run = DistributedPGO(edges, n, 16, r=5, schedule="coloured")
        rep = run.solve(gradnorm_tol=0.1, rel_change_tol=0, check_every=5)
    assert rep.reason == "gradnorm" and rep.rounds == stop
    assert abs(rep.cost - last.cost) <= 1e-10 * abs(last.cost)


def test_team_stop_matches_oracle_driver(data_dir):
    """Every agent ready to terminate (ref PGOAgent::shouldTerminate, src/PGOAgent.cpp:703-716,1007-1031): the first round
    at which the oracle's coloured driver has every agent optimised with its last relativeChange <= tol."""
    from dpo_b200.agent import DistributedPGO
    edges, n = load("torus3D", data_dir)
    meas, _ = orc.read_g2o(os.path.join(data_dir, "torus3D.g2o"))
    drv = orc.MultiRobotDriver(meas, n, 8, r=5, schedule="coloured")
    rcs = []
    for _ in range(80):
        drv.step()
        rcs.append([ag.last_result.relativeChange if ag.last_result is not None else np.inf for ag in drv.agents])
    rcs = np.array(rcs)

    def first_round(tol):
        ok = np.flatnonzero(np.all(rcs <= tol, axis=1))
        return int(ok[0]) + 1 if len(ok) else None

    for tol in (5e-3, 4.7e-3, 5.3e-3, 4.4e-3, 5.6e-3):      # a tolerance no relative change sits next to
        stop = first_round(tol)
        finite = rcs[:stop][np.isfinite(rcs[:stop])] if stop else rcs[np.isfinite(rcs)]
        if stop is not None and np.all(np.abs(finite - tol) > 1e-6 * tol):
            break
    else:
        pytest.fail("no tolerance away from the oracle's relative changes")
    with side_stream(True):
        run = DistributedPGO(edges, n, 8, r=5, schedule="coloured")
        assert run.colour == drv.colour
        rep = run.solve(gradnorm_tol=0, rel_change_tol=tol)
    assert rep.reason == "team" and rep.rounds == stop
    assert np.all(rep.relative_change <= tol)
    np.testing.assert_allclose(rep.relative_change, rcs[stop - 1], rtol=1e-6)


def test_round_cap(data_dir):
    from dpo_b200.agent import DistributedPGO
    edges, n = load("smallGrid3D", data_dir)
    run = DistributedPGO(edges, n, 5, r=5, schedule="coloured")
    rep = run.solve(max_rounds=7, check_every=3, gradnorm_tol=1e-12, rel_change_tol=1e-12)
    assert rep.reason == "max_rounds" and rep.rounds == 7 and run.round == 7
    with pytest.raises(ValueError, match="check_every"):
        DistributedPGO(edges, n, 5, r=5, schedule="greedy").solve(check_every=2)
    with pytest.raises(ValueError, match="acceleration"):
        DistributedPGO(edges, n, 5, r=5, schedule="greedy", acceleration=True).solve()


@pytest.mark.parametrize("ds,k", [("sphere2500", 16), ("input_INTEL_g2o", 5)])
def test_trajectory_matches_restatement(ds, k, data_dir):
    from dpo_b200.agent import DistributedPGO
    edges, n = load(ds, data_dir)
    d, dh = edges.d, edges.d + 1
    run = DistributedPGO(edges, n, k, r=5, schedule="coloured")
    for _ in range(6):
        run.step(evaluate=False)
    T = run.trajectory()
    X = run.assemble()
    ref = so.trajectory_in_global_frame(X, X[:, :dh], d)
    scale = np.abs(ref[:, d::dh]).max()
    assert np.abs(T - ref).max() <= 1e-12 * scale
    Rs = np.stack([T[:, i * dh:i * dh + d] for i in range(n)])
    assert np.abs(np.einsum("iba,ibc->iac", Rs, Rs) - np.eye(d)).max() <= 1e-12
    assert np.abs(np.linalg.det(Rs) - 1.0).max() <= 1e-12


def test_trajectory_parking_garage_golden(data_dir, golden_dir):
    """The reference's shipped final trajectory (result/opt_pose/NPparking-garage.csv, X[:, :3]^T X without the anchor's
    translation) after 450 greedy rounds through solve(), which stops at the round cap."""
    from dpo_b200.agent import DistributedPGO
    edges, n = load("parking-garage", data_dir)
    run = DistributedPGO(edges, n, 5, r=5, schedule="greedy")
    rep = run.solve(max_rounds=450, gradnorm_tol=0, rel_change_tol=0)
    assert rep.reason == "max_rounds" and rep.rounds == 450
    T = run.trajectory()
    gold = np.loadtxt(os.path.join(golden_dir, "NPparking-garage_opt_pose.csv"), delimiter=",")
    gold[:, 3::4] -= gold[:, 3:4]
    assert np.abs(T - gold).max() <= 5e-4


def test_status_is_ordered_on_the_runner_stream(data_dir):
    """status() / solve() issue their work, the all-gather and the copy on the runner's stream, whichever torch stream is
    current when they are called."""
    import torch
    from dpo_b200.agent import DistributedPGO
    edges, n = load("torus3D", data_dir)
    with side_stream(True):
        run = DistributedPGO(edges, n, 8, r=5, schedule="coloured")
        for _ in range(3):
            run.step(evaluate=False)
        ref = run.status().records
    other = torch.cuda.Stream()
    with torch.cuda.stream(other):
        for _ in range(3):
            assert np.array_equal(run.status().records, ref)
        rep = run.solve(max_rounds=4, gradnorm_tol=0, rel_change_tol=0)
    assert rep.reason == "max_rounds"


@pytest.fixture(scope="module")
def solve_check():
    from dpo_b200 import build
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    return build.build_cpp_program([os.path.join(root, "tests", "cpp", "solve_check.cpp")],
                                   os.path.join(root, "build", "tests", "solve_check"))


@pytest.mark.parametrize("ds,k,schedule,max_rounds,gtol,rtol,every", [("smallGrid3D", 5, "greedy", 500, 0.1, 0.0, 1),
                                                                       ("torus3D", 8, "coloured", 500, 0.1, 0.0, 5),
                                                                       ("smallGrid3D", 5, "coloured", 7, 1e-12, 1e-12, 3)])
def test_cpp_solve_matches_python(ds, k, schedule, max_rounds, gtol, rtol, every, solve_check, tmp_path, data_dir):
    """DeviceRBCD::solve / status / trajectory (C++) against DistributedPGO (Python) on one GPU: the same stop round and
    reason; status records and trajectory to 1e-9 relative (the runners use different fixed lifts, which these
    quantities do not depend on), the optimising-call counts exactly."""
    import subprocess
    from dpo_b200.agent import DistributedPGO
    res = subprocess.run([solve_check, os.path.join(data_dir, ds + ".g2o"), str(k), schedule, str(max_rounds), repr(gtol),
                          repr(rtol), str(every), str(tmp_path)], capture_output=True, text=True, timeout=600)
    assert res.returncode == 0, res.stderr[-2000:]
    words = res.stdout.split()
    rounds, reason = int(words[words.index("rounds") + 1]), words[words.index("reason") + 1]
    edges, n = load(ds, data_dir)
    run = DistributedPGO(edges, n, k, r=5, schedule=schedule)
    rep = run.solve(max_rounds=max_rounds, gradnorm_tol=gtol, rel_change_tol=rtol, check_every=every)
    assert (rounds, reason) == (rep.rounds, rep.reason)
    rec_c, rec_p = np.loadtxt(os.path.join(str(tmp_path), "status.txt")), run.status().records
    scale = np.abs(rec_p[:, 0]) + np.abs(rec_p[:, 1])
    assert np.all(np.abs(rec_c[:, 0] - rec_p[:, 0]) <= 1e-9 * scale)
    assert np.all(np.abs(rec_c[:, 1] - rec_p[:, 1]) <= 1e-9 * scale)
    assert np.all(np.abs(rec_c[:, 2] - rec_p[:, 2]) <= 1e-9 * rec_p[:, 2])
    assert np.all(np.abs(rec_c[:, 3] - rec_p[:, 3]) <= 1e-9 * rec_p[:, 3])
    assert np.array_equal(rec_c[:, 4], rec_p[:, 4])
    T_c, T_p = np.loadtxt(os.path.join(str(tmp_path), "trajectory.txt")), run.trajectory()
    d, dh = edges.d, edges.d + 1
    assert np.abs(T_c - T_p).max() <= 1e-9 * max(1.0, np.abs(T_p[:, d::dh]).max())


def _device_count():
    from dpo_b200 import _capi
    c = C.c_int(0)
    _capi.load_library().dpgo_device_count(C.byref(c))
    return c.value


@pytest.mark.parametrize("conc", [0, 1])
def test_two_rank_solve_bit_equal_to_one_process(conc, tmp_path, data_dir):
    """solve() with the 8 torus3D agents over 2 torchrun ranks (status records by one all-gather, the trajectory's anchor
    broadcast from agent 0's rank) against one process, launch mode pinned: bit-equal iterates, records, report and
    trajectory columns.  Needs 2 GPUs (skipped otherwise)."""
    if _device_count() < 2:
        pytest.skip("needs 2 GPUs")
    import subprocess
    from dpo_b200.agent import DistributedPGO
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    k, max_rounds = 8, 40
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2", "--master-addr", "127.0.0.1",
           "--master-port", "29537", os.path.join(root, "tests", "_solve_multirank_worker.py"), "torus3D", str(k), str(conc),
           str(max_rounds), str(tmp_path)]
    res = subprocess.run(cmd, capture_output=True, text=True, timeout=600)
    assert res.returncode == 0, res.stderr[-2000:]
    edges, n = load("torus3D", data_dir)
    run = DistributedPGO(edges, n, k, r=5, schedule="coloured", concurrent=bool(conc))
    rep = run.solve(max_rounds=max_rounds, gradnorm_tol=0.1, rel_change_tol=5e-3, check_every=1)
    out = str(tmp_path)
    assert open(os.path.join(out, "reason.txt")).read() == rep.reason
    assert np.array_equal(np.load(os.path.join(out, "report.npy")), np.array([rep.rounds, rep.cost, rep.gradnorm]))
    assert np.array_equal(np.load(os.path.join(out, "records.npy")), run.status().records)
    for a in range(k):
        assert np.array_equal(np.load(os.path.join(out, f"X_{a}.npy")), run.agents[a].mProblem.download_X()), a
    T = run.trajectory()
    dh = edges.d + 1
    for rank in range(2):
        Tr = np.load(os.path.join(out, f"T_{rank}.npy"))
        for a in range(rank * k // 2, (rank + 1) * k // 2):
            cols = (run.glob[a][:, None] * dh + np.arange(dh)[None, :]).ravel()
            assert np.array_equal(Tr[:, cols], T[:, cols]), a
