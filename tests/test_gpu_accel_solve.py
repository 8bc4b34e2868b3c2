"""solve() with colour-momentum accelerated rounds on the GPU: the status record an accelerated round leaves (relative
change against the round's XPrev, one optimising call per round, restart or not; src/PGOAgent.cpp:673,703-716) against
the host formula on downloaded iterates, repeatability and graph replay, the stop rounds of the gradient-norm and team
rules against the step() loop and the CPU restatement (tests/accel_solve_oracle.py), the C++ runner against Python, and two
ranks against one process."""
import contextlib
import ctypes as C
import os
import subprocess
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import accel_solve_oracle as aso  # noqa: E402
from oracle import dpgo_oracle as orc  # noqa: E402

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def load(ds, data_dir):
    from dpo_b200 import posegraph as pg
    return pg.read_g2o_file(os.path.join(data_dir, ds + ".g2o"))


def side_stream(on):
    import torch
    return torch.cuda.stream(torch.cuda.Stream()) if on else contextlib.nullcontext()


def accelerated(ds, k, data_dir, concurrent=None):
    from dpo_b200.agent import DistributedPGO
    edges, n = load(ds, data_dir)
    return DistributedPGO(edges, n, k, r=5, schedule="coloured", acceleration=True, momentum_blocks="colours",
                          concurrent=concurrent)


@pytest.mark.parametrize("conc", [False, True])
@pytest.mark.parametrize("ds,k", [("sphere2500", 16), ("torus3D", 8)])
def test_accelerated_round_records(ds, k, conc, data_dir):
    """70 rounds (every agent restarts on its iterations 29 and 59): an active agent's field 3 equals
    sqrt(|X_end - XPrev|^2 / n) from the iterates downloaded before and after the round to 1e-13, its field 4 rises by
    exactly 1; an idle agent's fields 3 and 4 are bitwise unchanged."""
    with side_stream(conc):
        run = accelerated(ds, k, data_dir, concurrent=conc)
        assert run.concurrent == conc
        rec = run.status().records
        restarts = 0
        for rnd in range(70):
            active = [a for a in range(k) if run.colour[a] == rnd % run.ncolours]
            before = {a: run.agents[a].mProblem.download_X() for a in active}
            restarts += (rnd + 2) % run.restart_interval == 0
            run.step(evaluate=False)
            after = run.status().records
            for a in range(k):
                if a in active:
                    X = run.agents[a].mProblem.download_X()
                    expect = np.sqrt(np.sum((X - before[a]) ** 2) / run.agents[a].n)
                    assert abs(after[a, 3] - expect) <= 1e-13 * expect, (rnd, a, after[a, 3], expect)
                    assert after[a, 4] == rec[a, 4] + 1, (rnd, a)
                else:
                    assert after[a, 3] == rec[a, 3] and after[a, 4] == rec[a, 4], (rnd, a)
            rec = after
    assert restarts == 2
    assert [rec[a, 4] for a in range(k)] == [sum(r % run.ncolours == run.colour[a] for r in range(70)) for a in range(k)]


_RUN = r'''
import os, sys
import numpy as np
sys.path.insert(0, sys.argv[1])
import torch
from dpo_b200 import posegraph as pg
from dpo_b200.agent import DistributedPGO
edges, n = pg.read_g2o_file(os.path.join(sys.argv[1], "data", "torus3D.g2o"))
with torch.cuda.stream(torch.cuda.Stream()):
    run = DistributedPGO(edges, n, 8, r=5, schedule="coloured", acceleration=True, momentum_blocks="colours", concurrent=True)
    recs = []
    for _ in range(int(sys.argv[3])):
        run.step(evaluate=False)
        recs.append(run.status().records)
    np.save(sys.argv[2] + "_rec.npy", np.array(recs))
    np.save(sys.argv[2] + "_X.npy", run.assemble())
'''


def test_records_repeatable_and_graph_replay_bit_equal(tmp_path):
    """Two runs with the rounds replayed as CUDA graphs and one with eager launches (DPGO_ROUND_GRAPH=0), 64 rounds over
    two restarts: every round's status records and the final iterate, bit for bit."""
    outs = []
    for i, flag in enumerate((None, None, "0")):
        env = dict(os.environ)
        env.pop("DPGO_ROUND_GRAPH", None)
        if flag is not None:
            env["DPGO_ROUND_GRAPH"] = flag
        out = str(tmp_path / f"run{i}")
        res = subprocess.run([sys.executable, "-c", _RUN, ROOT, out, "64"], env=env, capture_output=True, text=True,
                             timeout=600)
        assert res.returncode == 0, res.stderr[-2000:]
        outs.append((np.load(out + "_rec.npy"), np.load(out + "_X.npy")))
    for rec, X in outs[1:]:
        assert np.array_equal(rec, outs[0][0]) and np.array_equal(X, outs[0][1])


@pytest.mark.parametrize("ds,k,stop,expect_cost", [("sphere2500", 16, 135, 1687.0440), ("torus3D", 8, 98, 24227.0479)])
def test_solve_stops_at_the_gradnorm_round(ds, k, stop, expect_cost, data_dir):
    """solve(gradnorm_tol=0.1) with the team rule off stops where the step() + status() loop does (the restatement's
    rounds, tests/test_gpu_accel.py): after every round at 135 and 98; with check_every=5 at the next multiple of 5, with
    the 2f of a step() loop that evaluates every 5th round, bit for bit."""
    with side_stream(True):
        rep = accelerated(ds, k, data_dir).solve(gradnorm_tol=0.1, rel_change_tol=0, check_every=1)
        assert rep.reason == "gradnorm" and rep.rounds == stop
        assert abs(rep.cost - expect_cost) <= 1e-6 * expect_cost
        every5 = -(-stop // 5) * 5
        rep5 = accelerated(ds, k, data_dir).solve(gradnorm_tol=0.1, rel_change_tol=0, check_every=5)
        assert rep5.reason == "gradnorm" and rep5.rounds == every5
        ref = accelerated(ds, k, data_dir)
        for it in range(1, every5 + 1):
            last = ref.step(evaluate=(it % 5 == 0))
        assert last.gradnorm < 0.1
        assert rep5.cost == last.cost and rep5.gradnorm == last.gradnorm


@pytest.mark.parametrize("ds,k", sorted(aso.TEAM_STOPS))
def test_team_rule_stops_at_the_restatement_round(ds, k, data_dir):
    tol, expect = aso.TEAM_STOPS[(ds, k)]
    meas, n = orc.read_g2o(os.path.join(data_dir, ds + ".g2o"))
    drv = aso.StatusRecordingDriver(meas, n, k, r=5, momentum_blocks="colours")
    stop, rcs = aso.team_stop(drv, tol, cap=expect + 5)
    assert stop == expect
    with side_stream(True):
        run = accelerated(ds, k, data_dir)
        assert run.colour == drv.colour
        rep = run.solve(gradnorm_tol=0, rel_change_tol=tol)
    assert rep.reason == "team" and rep.rounds == expect
    np.testing.assert_allclose(rep.relative_change, rcs[expect - 1], rtol=1e-6)


@pytest.fixture(scope="module")
def accel_solve_check():
    from dpo_b200 import build
    return build.build_cpp_program([os.path.join(ROOT, "tests", "cpp", "accel_solve_check.cpp")],
                                   os.path.join(ROOT, "build", "tests", "accel_solve_check"))


@pytest.mark.parametrize("ds,k,gtol,rtol,every", [("torus3D", 8, 0.1, 0.0, 5), ("smallGrid3D", 5, 0.0, 5e-4, 1)])
def test_cpp_accelerated_solve_matches_python(ds, k, gtol, rtol, every, accel_solve_check, tmp_path, data_dir):
    """DeviceRBCD::solve (C++) against DistributedPGO.solve (Python): the same stop round and reason, the final status
    records to 1e-9 relative and the optimising-call counts exactly."""
    res = subprocess.run([accel_solve_check, os.path.join(data_dir, ds + ".g2o"), str(k), "colours", "500", repr(gtol),
                          repr(rtol), str(every), str(tmp_path)], capture_output=True, text=True, timeout=600)
    assert res.returncode == 0, res.stderr[-2000:]
    words = res.stdout.split()
    rounds, reason = int(words[words.index("rounds") + 1]), words[words.index("reason") + 1]
    run = accelerated(ds, k, data_dir)
    rep = run.solve(gradnorm_tol=gtol, rel_change_tol=rtol, check_every=every)
    assert (rounds, reason) == (rep.rounds, rep.reason)
    rec_c, rec_p = np.loadtxt(os.path.join(str(tmp_path), "status.txt")), run.status().records
    scale = np.abs(rec_p[:, 0]) + np.abs(rec_p[:, 1])
    assert np.all(np.abs(rec_c[:, 0] - rec_p[:, 0]) <= 1e-9 * scale)
    assert np.all(np.abs(rec_c[:, 1] - rec_p[:, 1]) <= 1e-9 * scale)
    assert np.all(np.abs(rec_c[:, 2] - rec_p[:, 2]) <= 1e-9 * rec_p[:, 2])
    assert np.all(np.abs(rec_c[:, 3] - rec_p[:, 3]) <= 1e-9 * rec_p[:, 3])
    assert np.array_equal(rec_c[:, 4], rec_p[:, 4])


def test_cpp_solve_rejects_agent_momentum(accel_solve_check, tmp_path, data_dir):
    res = subprocess.run([accel_solve_check, os.path.join(data_dir, "smallGrid3D.g2o"), "5", "agents", "50", "0.1", "0", "1",
                          str(tmp_path)], capture_output=True, text=True, timeout=600)
    assert res.returncode == 1 and "acceleration" in res.stderr, res.stderr[-2000:]


def _device_count():
    from dpo_b200 import _capi
    c = C.c_int(0)
    _capi.load_library().dpgo_device_count(C.byref(c))
    return c.value


def test_two_rank_accelerated_solve_bit_equal_to_one_process(tmp_path, data_dir):
    """solve() with the 8 torus3D agents over 2 torchrun ranks (side by side) against one process: bit-equal iterates,
    records and report.  Needs 2 GPUs (skipped otherwise)."""
    if _device_count() < 2:
        pytest.skip("needs 2 GPUs")
    k = 8
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2", "--master-addr", "127.0.0.1",
           "--master-port", "29539", os.path.join(ROOT, "tests", "_accel_solve_multirank_worker.py"), "torus3D", str(k), "1",
           "1", str(tmp_path)]
    res = subprocess.run(cmd, capture_output=True, text=True, timeout=600)
    assert res.returncode == 0, res.stderr[-2000:]
    with side_stream(True):
        run = accelerated("torus3D", k, data_dir, concurrent=True)
        rep = run.solve(gradnorm_tol=0.1, rel_change_tol=5e-3, check_every=1)
        records = run.status().records
    out = str(tmp_path)
    assert open(os.path.join(out, "reason.txt")).read() == rep.reason
    assert np.array_equal(np.load(os.path.join(out, "report.npy")), np.array([rep.rounds, rep.cost, rep.gradnorm]))
    assert np.array_equal(np.load(os.path.join(out, "records.npy")), records)
    for a in range(k):
        assert np.array_equal(np.load(os.path.join(out, f"X_{a}.npy")), run.agents[a].mProblem.download_X()), a
