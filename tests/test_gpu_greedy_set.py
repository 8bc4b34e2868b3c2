"""The greedy_set schedule on the GPU: the device selection against the host rule, runs against the CPU restatement
(tests/greedy_set_oracle.py), the complete agent graph against the greedy schedule, repeatability and graph replay, the
gate's effect on an idle agent, solve() with checks every 5 rounds, the C++ runner, and two ranks against one process."""
import contextlib
import ctypes as C
import math
import os
import subprocess
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import greedy_set_oracle as gso  # noqa: E402
from oracle import dpgo_oracle as orc  # noqa: E402

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DATA = os.path.join(ROOT, "data")


def load(ds):
    from dpo_b200 import posegraph as pg
    return pg.read_g2o_file(os.path.join(DATA, ds + ".g2o"))


def side_stream(on):
    import torch
    return torch.cuda.stream(torch.cuda.Stream()) if on else contextlib.nullcontext()


def make(ds, k, conc=None, schedule="greedy_set"):
    from dpo_b200.agent import DistributedPGO
    edges, n = load(ds)
    return DistributedPGO(edges, n, k, r=5, schedule=schedule, concurrent=conc)


def neighbours(run):
    return [run.plan.tables[a]["neighbors"] for a in range(run.k)]


def near_tie(g2, tol=1e-9):
    """two squared norms within tol relative of each other: the walk's order between them is not robust to rounding"""
    s = np.sort(np.asarray(g2))
    return bool(np.any(np.diff(s) <= tol * np.maximum(s[1:], 1e-300)))


@pytest.mark.parametrize("conc", [False, True])
@pytest.mark.parametrize("ds,k", [("sphere2500", 16), ("torus3D", 8), ("parking-garage", 4), ("input_INTEL_g2o", 5)])
def test_device_selection_equals_host_rule(ds, k, conc):
    """Every one of 60 rounds: the device mask equals greedy_independent_set on the same status records."""
    from dpo_b200.agent import greedy_independent_set
    with side_stream(conc):
        run = make(ds, k, conc)
        assert run.agents[0].mProblem.launch_info()[1] == conc
        nb = neighbours(run)
        for i in range(60):
            rec = run.status().records
            run.step(evaluate=False)
            assert run.selection_log(i, 1)[0] == greedy_independent_set(rec[:, 2], nb), i


_ORACLE = {}


def oracle_run(ds, k, rounds):
    if (ds, k, rounds) not in _ORACLE:
        meas, n = orc.read_g2o(os.path.join(DATA, ds + ".g2o"))
        drv = gso.GreedySetDriver(meas, n, k, r=5)
        for _ in range(rounds):
            drv.step()
        _ORACLE[(ds, k, rounds)] = drv
    return _ORACLE[(ds, k, rounds)]


@pytest.mark.parametrize("ds,k", [("sphere2500", 16), ("torus3D", 8), ("parking-garage", 4)])
def test_follows_restatement(ds, k):
    """60 rounds: the per-round sets equal the restatement's (rounds whose selection norms hold a near tie are left out of
    the set check, and counted), 2f and |g| to 1e-9 relative; parking-garage to the coloured test's tolerance."""
    rounds = 60
    drv = oracle_run(ds, k, rounds)
    # parking-garage is ill-conditioned (every tCG solve hits its cap): rounding differences are amplified, as in
    # test_gpu_agents.py::test_coloured_schedule_matches_oracle
    ctol, gtol = (1e-7, 1e-5) if ds == "parking-garage" else (1e-9, 1e-9)
    with side_stream(True):
        run = make(ds, k)
        tr = [run.step() for _ in range(rounds)]
    excluded = 0
    for i, st in enumerate(tr):
        if near_tie(drv.norms2[i]):
            excluded += 1
        else:
            assert st.selected == drv.sets[i], (i, st.selected, drv.sets[i])
        assert abs(st.cost - drv.trace.cost[i]) <= ctol * abs(drv.trace.cost[i]), (i, st.cost, drv.trace.cost[i])
        assert abs(st.gradnorm - drv.trace.gradnorm[i]) <= gtol * drv.trace.gradnorm[i], (i, st.gradnorm, drv.trace.gradnorm[i])
    print(f"{ds}x{k}: {excluded} of {rounds} rounds left out of the set check (near ties)")


def test_complete_graph_equals_greedy():
    """parking-garage x 4 has a complete agent graph, so every set is {argmax}: greedy_set steps exactly the greedy schedule's
    agent, bit for bit, full-grid launches pinned.  The greedy run starts from the same argmax (its driver starts at agent 0)."""
    from dpo_b200.agent import greedy_selection
    rs, rg = make("parking-garage", 4, False), make("parking-garage", 4, False, "greedy")
    assert all(len(nb) == 3 for nb in neighbours(rs))
    rg.selected = [greedy_selection(0, np.sqrt(rg.status().records[:, 2]), True)]
    for i in range(30):
        a, b = rs.step(), rg.step()
        assert a.selected == b.selected, i
        assert (a.cost, a.gradnorm) == (b.cost, b.gradnorm), i
    for q in range(4):
        assert np.array_equal(rs.agents[q].mProblem.download_X(), rg.agents[q].mProblem.download_X()), q


_REPLAY = r'''
import os, sys
import numpy as np
sys.path.insert(0, sys.argv[1])
import torch
from dpo_b200 import posegraph as pg
from dpo_b200.agent import DistributedPGO
edges, n = pg.read_g2o_file(os.path.join(sys.argv[1], "data", "torus3D.g2o"))
with torch.cuda.stream(torch.cuda.Stream()):
    run = DistributedPGO(edges, n, 8, r=5, schedule="greedy_set", concurrent=True)
    for _ in range(int(sys.argv[3])):
        run.step(evaluate=False)
    log = np.zeros((int(sys.argv[3]), 8), dtype=np.uint8)
    for i, s in enumerate(run.selection_log()):
        log[i, s] = 1
    np.savez(sys.argv[2], X=run.assemble(), log=log)
'''


def test_repeatable_and_graph_replay_bit_equal(tmp_path):
    """Two runs in one process give the same bits; so do graph replay (default) and eager launches (DPGO_ROUND_GRAPH=0),
    over more rounds than the log's first capacity (64), so a replay across the log's doubling is included."""
    rounds = 80
    outs = []
    for flag in (None, "0"):
        env = dict(os.environ)
        env.pop("DPGO_ROUND_GRAPH", None)
        if flag is not None:
            env["DPGO_ROUND_GRAPH"] = flag
        out = str(tmp_path / f"run_{flag}.npz")
        res = subprocess.run([sys.executable, "-c", _REPLAY, ROOT, out, str(rounds)], env=env, capture_output=True,
                             text=True, timeout=600)
        assert res.returncode == 0, res.stderr[-2000:]
        outs.append(np.load(out))
    assert np.array_equal(outs[0]["X"], outs[1]["X"]) and np.array_equal(outs[0]["log"], outs[1]["log"])
    with side_stream(True):
        a, b = make("torus3D", 8, True), make("torus3D", 8, True)
        for _ in range(rounds):
            a.step(evaluate=False)
            b.step(evaluate=False)
        assert np.array_equal(a.assemble(), b.assemble()) and a.selection_log() == b.selection_log()
    assert np.array_equal(a.assemble(), outs[0]["X"])


@pytest.mark.parametrize("conc", [False, True])
def test_gated_off_agent_is_untouched(conc):
    """An agent left out of a round keeps its iterate, its <XQ, X> and its optimising-call record (fields 3, 4) bit for bit;
    with no selected neighbour its whole status record is unchanged."""
    with side_stream(conc):
        run = make("sphere2500", 16, conc)
        nb = neighbours(run)
        for i in range(12):
            before = run.status().records.copy()
            X0 = {a: run.agents[a].mProblem.download_X() for a in range(16)}
            run.step(evaluate=False)
            sel = run.selection_log(i, 1)[0]
            after = run.status().records
            assert 0 < len(sel) < 16
            for a in range(16):
                if a in sel:
                    assert after[a, 4] == before[a, 4] + 1, (i, a)
                    continue
                assert np.array_equal(run.agents[a].mProblem.download_X(), X0[a]), (i, a)
                assert np.array_equal(after[a, [0, 3, 4]], before[a, [0, 3, 4]]), (i, a)
                if not any(b in sel for b in nb[a]):
                    assert np.array_equal(after[a], before[a]), (i, a)


def test_solve_check_every_5_stops_at_the_next_multiple():
    with side_stream(True):
        ref = make("torus3D", 8)
        costs, stop = [], None
        for i in range(500):
            st = ref.step()
            costs.append(st.cost)
            if stop is None and st.gradnorm < 0.1:
                stop = i + 1
            if stop is not None and i + 1 >= math.ceil(stop / 5) * 5:
                break
        run = make("torus3D", 8)
        rep = run.solve(max_rounds=500, gradnorm_tol=0.1, rel_change_tol=0.0, check_every=5)
    assert stop is not None
    assert (rep.rounds, rep.reason) == (math.ceil(stop / 5) * 5, "gradnorm")
    assert rep.cost == costs[rep.rounds - 1]
    assert run.selection_log() == ref.selection_log()[:rep.rounds]


@pytest.fixture(scope="module")
def greedy_set_check():
    from dpo_b200 import build
    return build.build_cpp_program([os.path.join(ROOT, "tests", "cpp", "greedy_set_check.cpp")],
                                   os.path.join(ROOT, "build", "tests", "greedy_set_check"))


@pytest.mark.parametrize("ds,k", [("smallGrid3D", 5), ("torus3D", 8)])
def test_cpp_solve_matches_python(ds, k, greedy_set_check, tmp_path):
    """DeviceRBCD::solve (greedy_set, checks every 5 rounds) against DistributedPGO.solve: the same stop round, reason and
    selection log; status records to 1e-9 relative (field 2 as the block gradient norm: near convergence |rgrad|^2 is ~1e-8
    and its last bits are rounding), the optimising-call counts exactly."""
    res = subprocess.run([greedy_set_check, os.path.join(DATA, ds + ".g2o"), str(k), "500", "0.1", "5", str(tmp_path)],
                         capture_output=True, text=True, timeout=600)
    assert res.returncode == 0, res.stderr[-2000:]
    words = res.stdout.split()
    rounds, reason = int(words[words.index("rounds") + 1]), words[words.index("reason") + 1]
    run = make(ds, k)
    rep = run.solve(max_rounds=500, gradnorm_tol=0.1, rel_change_tol=0.0, check_every=5)
    assert (rounds, reason) == (rep.rounds, rep.reason)
    log_c = np.loadtxt(os.path.join(str(tmp_path), "selection.txt"), dtype=int).reshape(-1, k)
    assert [list(np.flatnonzero(r)) for r in log_c] == run.selection_log()
    rec_c, rec_p = np.loadtxt(os.path.join(str(tmp_path), "status.txt")), run.status().records
    scale = np.abs(rec_p[:, 0]) + np.abs(rec_p[:, 1])
    assert np.all(np.abs(rec_c[:, 0] - rec_p[:, 0]) <= 1e-9 * scale)
    assert np.all(np.abs(rec_c[:, 1] - rec_p[:, 1]) <= 1e-9 * scale)
    assert np.all(np.abs(np.sqrt(rec_c[:, 2]) - np.sqrt(rec_p[:, 2])) <= 1e-9 * np.sqrt(rec_p[:, 2]))
    assert np.all(np.abs(rec_c[:, 3] - rec_p[:, 3]) <= 1e-9 * rec_p[:, 3])
    assert np.array_equal(rec_c[:, 4], rec_p[:, 4])


def _device_count():
    from dpo_b200 import _capi
    c = C.c_int(0)
    _capi.load_library().dpgo_device_count(C.byref(c))
    return c.value


@pytest.mark.parametrize("conc", [0, 1])
def test_two_ranks_bit_equal_to_one_process(conc, tmp_path):
    if _device_count() < 2:
        pytest.skip("needs 2 GPUs")
    ds, k, rounds = "torus3D", 8, 20
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2", "--master-addr", "127.0.0.1",
           "--master-port", "29541", os.path.join(ROOT, "tests", "_greedy_set_multirank_worker.py"), ds, str(k), str(rounds),
           str(tmp_path), str(conc)]
    res = subprocess.run(cmd, capture_output=True, text=True, timeout=600)
    assert res.returncode == 0, res.stderr[-2000:]
    run = make(ds, k, bool(conc))
    for _ in range(rounds):
        run.step(evaluate=False)
    for a in range(k):
        assert np.array_equal(np.load(os.path.join(str(tmp_path), f"X_{a}.npy")), run.agents[a].mProblem.download_X()), a
    for q in range(2):
        log = np.load(os.path.join(str(tmp_path), f"log_{q}.npy"))
        assert [list(np.flatnonzero(r)) for r in log] == run.selection_log(), q
