"""Accelerated rounds on the GPU: the device momentum record against the host recurrence, the batched begin launch against
the per-agent calls, coloured accelerated runs against the CPU restatement (tests/accel_oracle.py) in both launch modes
and both momenta, repeatability and graph replay, and the rounds to convergence with the momentum over colour classes."""
import contextlib
import ctypes as C
import os
import subprocess
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import accel_oracle as ao  # noqa: E402
from oracle import dpgo_oracle as orc  # noqa: E402

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def load(ds, data_dir):
    from dpo_b200 import posegraph as pg
    return pg.read_g2o_file(os.path.join(data_dir, ds + ".g2o"))


def side_stream(on):
    import torch
    return torch.cuda.stream(torch.cuda.Stream()) if on else contextlib.nullcontext()


def accel_state(run, a):
    out = np.zeros(3)
    ag = run.agents[a]
    from dpo_b200 import _capi
    _capi.check(ag.mProblem._lib.dpgo_agent_accel_state(ag.mProblem._h, _capi.dptr(out)))
    return tuple(out)


@pytest.mark.parametrize("N", [2, 5, 8, 16])
def test_momentum_record_equals_host_recurrence(N, data_dir):
    from dpo_b200.agent import DistributedPGO
    edges, n = load("smallGrid3D", data_dir)
    run = DistributedPGO(edges, n, 5, r=5, schedule="coloured", acceleration=True)
    run.momentum_N = float(N)
    expect = ao.momentum_trace(float(N), 200, 30)
    for i in range(200):
        run.step(evaluate=False)
        for a in (0, 4):
            assert accel_state(run, a) == expect[i], (i, a)


def test_batched_begin_equals_per_agent_calls(data_dir):
    """dpgo_agents_accel_begin_async with every agent idle == dpgo_agent_accel_begin + dpgo_agent_accel_end(optimized = 0)
    + the restart calls + both packs, bit for bit (the same projection arithmetic), over a restart."""
    from dpo_b200.agent import DistributedPGO
    from dpo_b200 import _capi
    edges, n = load("smallGrid3D", data_dir)
    new, old = (DistributedPGO(edges, n, 5, r=5, schedule="coloured", acceleration=True) for _ in range(2))
    lib = new.agents[0].mProblem._lib
    ids = new.local_ids
    hs = (C.c_void_p * 5)(*[new.agents[a].mProblem._h for a in ids])
    sx = (C.c_void_p * 5)(*[C.c_void_p(new.tiles.part[a].data_ptr()) for a in ids])
    sy = (C.c_void_p * 5)(*[C.c_void_p(new.aux_tiles.part[a].data_ptr()) for a in ids])
    flags = np.zeros(5, dtype=np.int32)
    trace = ao.momentum_trace(5.0, 32, 30)
    import torch
    for i in range(32):
        _capi.check(lib.dpgo_agents_accel_begin_async(hs, 5, _capi.iptr(flags), 5.0, 30, sx, sy,
                                                      C.c_void_p(new._main_stream)))
        gamma = trace[i - 1][0] if i else 0.0
        gamma = (1.0 + np.sqrt(1.0 + ((4.0 * 5.0) * 5.0) * (gamma * gamma))) / (2.0 * 5.0)
        alpha = 1.0 / (gamma * 5.0)
        for a in ids:
            h = old.agents[a].mProblem._h
            _capi.check(lib.dpgo_agent_accel_begin(h, alpha))
            _capi.check(lib.dpgo_agent_accel_end(h, gamma, 0))
            if (i + 2) % 30 == 0:
                _capi.check(lib.dpgo_agent_accel_restart_begin(h))
                _capi.check(lib.dpgo_agent_accel_restart_end(h))
            old.agents[a].pack_public(old.tiles.part[a].data_ptr())
            _capi.check(lib.dpgo_agent_pack_public_aux(h, C.c_void_p(old.aux_tiles.part[a].data_ptr())))
        torch.cuda.synchronize()
        assert torch.equal(new.tiles.all, old.tiles.all) and torch.equal(new.aux_tiles.all, old.aux_tiles.all), i
        for a in ids:
            assert np.array_equal(new.agents[a].mProblem.download_X(), old.agents[a].mProblem.download_X()), (i, a)


_ORACLE = {}


def oracle_trace(ds, k, blocks, rounds, data_dir):
    key = (ds, k, blocks, rounds)
    if key not in _ORACLE:
        meas, n = orc.read_g2o(os.path.join(data_dir, ds + ".g2o"))
        drv = ao.AcceleratedColouredDriver(meas, n, k, r=5, momentum_blocks=blocks)
        for _ in range(rounds):
            drv.step()
        _ORACLE[key] = (list(drv.trace.cost), list(drv.trace.gradnorm), drv.assemble(), drv.colour)
    return _ORACLE[key]


def run_rounds(ds, k, blocks, conc, rounds, data_dir):
    from dpo_b200.agent import DistributedPGO
    edges, n = load(ds, data_dir)
    with side_stream(conc):
        run = DistributedPGO(edges, n, k, r=5, schedule="coloured", acceleration=True, momentum_blocks=blocks,
                             concurrent=conc)
        assert run.agents[0].mProblem.launch_info()[1] == conc
        tr = [run.step() for _ in range(rounds)]
        X = run.assemble()
    return run, [(s.cost, s.gradnorm) for s in tr], X


@pytest.mark.parametrize("blocks", ["agents", "colours"])
@pytest.mark.parametrize("ds,k", [("sphere2500", 16), ("torus3D", 8), ("parking-garage", 4)])
def test_coloured_accelerated_follows_restatement(ds, k, blocks, data_dir):
    """70 rounds (restarts at iterations 29 and 59) in both launch modes: per round 2f to 1e-8 and |g| to 1e-6 of the
    restatement; the two modes agree to rounding; the concurrent mode is bitwise repeatable."""
    rounds = 70
    cost, gn, Xo, colour = oracle_trace(ds, k, blocks, rounds, data_dir)
    # parking-garage is ill-conditioned (kappa ~ 2, tau ~ 1, every tCG solve hits its cap): rounding differences are
    # amplified, as in test_gpu_agents.py::test_coloured_schedule_matches_oracle
    ctol, gtol = (1e-7, 1e-5) if ds == "parking-garage" else (1e-8, 1e-6)
    Xs = {}
    for conc in (False, True):
        run, tr, X = run_rounds(ds, k, blocks, conc, rounds, data_dir)
        assert run.colour == colour
        for i, (c, g) in enumerate(tr):
            assert abs(c - cost[i]) <= ctol * abs(cost[i]), (conc, i, c, cost[i])
            assert abs(g - gn[i]) <= gtol * gn[i], (conc, i, g, gn[i])
        Xs[conc] = X
    assert np.linalg.norm(Xs[True] - Xs[False]) <= 1e-9 * np.linalg.norm(Xs[False])
    _, _, again = run_rounds(ds, k, blocks, True, rounds, data_dir)
    assert np.array_equal(again, Xs[True])


_REPLAY = r'''
import os, sys
import numpy as np
sys.path.insert(0, sys.argv[1])
import torch
from dpo_b200 import posegraph as pg
from dpo_b200.agent import DistributedPGO
edges, n = pg.read_g2o_file(os.path.join(sys.argv[1], "data", "torus3D.g2o"))
with torch.cuda.stream(torch.cuda.Stream()):
    run = DistributedPGO(edges, n, 8, r=5, schedule="coloured", acceleration=True, momentum_blocks="colours", concurrent=True)
    for _ in range(int(sys.argv[3])):
        run.step(evaluate=False)
    np.save(sys.argv[2], run.assemble())
'''


def test_graph_replay_is_bit_equal_to_eager(tmp_path):
    """Repeated accelerated rounds are replayed as CUDA graphs (plain and restart variants); DPGO_ROUND_GRAPH=0 keeps
    the eager launches.  Both give the same bits."""
    rounds = 64
    outs = []
    for flag in (None, "0"):
        env = dict(os.environ)
        env.pop("DPGO_ROUND_GRAPH", None)
        if flag is not None:
            env["DPGO_ROUND_GRAPH"] = flag
        out = str(tmp_path / f"X_{flag}.npy")
        res = subprocess.run([sys.executable, "-c", _REPLAY, ROOT, out, str(rounds)], env=env, capture_output=True,
                             text=True, timeout=600)
        assert res.returncode == 0, res.stderr[-2000:]
        outs.append(np.load(out))
    assert np.array_equal(outs[0], outs[1])


@pytest.mark.parametrize("ds,k,expect_rounds,expect_cost", [("sphere2500", 16, 135, 1687.0440), ("torus3D", 8, 98, 24227.0479)])
def test_colour_momentum_stops_at_the_restatement_round(ds, k, expect_rounds, expect_cost, data_dir):
    """Rounds to |g| < 0.1 with status() after every round, against the CPU restatement's count (135 and 98), with its
    final 2f (printed to 4 decimals) to 1e-6."""
    from dpo_b200.agent import DistributedPGO
    edges, n = load(ds, data_dir)
    with side_stream(True):
        run = DistributedPGO(edges, n, k, r=5, schedule="coloured", acceleration=True, momentum_blocks="colours")
        assert run.concurrent
        stop = None
        for i in range(400):
            run.step(evaluate=False)
            st = run.status()
            if st.gradnorm < 0.1:
                stop = i + 1
                break
    assert stop == expect_rounds
    assert abs(st.cost - expect_cost) <= 1e-6 * expect_cost


def _device_count():
    from dpo_b200 import _capi
    c = C.c_int(0)
    _capi.load_library().dpgo_device_count(C.byref(c))
    return c.value


def test_two_ranks_accelerated_concurrent_bit_equal(tmp_path, data_dir):
    if _device_count() < 2:
        pytest.skip("needs 2 GPUs")
    from dpo_b200.agent import DistributedPGO
    ds, k, rounds = "torus3D", 8, 6
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2", "--master-addr", "127.0.0.1",
           "--master-port", "29537", os.path.join(ROOT, "tests", "_multirank_worker.py"), ds, str(k), str(rounds),
           str(tmp_path), "1", "1"]
    res = subprocess.run(cmd, capture_output=True, text=True, timeout=600)
    assert res.returncode == 0, res.stderr[-2000:]
    edges, n = load(ds, data_dir)
    run = DistributedPGO(edges, n, k, r=5, schedule="coloured", acceleration=True, concurrent=True)
    for _ in range(rounds):
        run.step(evaluate=True)
    for a in range(k):
        assert np.array_equal(np.load(os.path.join(str(tmp_path), f"X_{a}.npy")), run.agents[a].mProblem.download_X()), a


@pytest.mark.parametrize("blocks", ["agents", "colours"])
def test_cpp_resident_accelerated_trace_equals_python(blocks, tmp_path, data_dir):
    """MultiAgentPGO --resident --accel --schedule coloured (DPGO::DeviceRBCD) against DistributedPGO, 70 rounds."""
    exe = os.path.join(ROOT, "build", "examples", "MultiAgentPGO")
    if not os.path.exists(exe):
        pytest.skip("build/examples/MultiAgentPGO not built")
    rounds, trace = 70, str(tmp_path / "trace.csv")
    res = subprocess.run([exe, os.path.join(data_dir, "torus3D.g2o"), "--trace", trace, "--robots", "8", "--iters", str(rounds),
                          "--stop", "0", "--resident", "--schedule", "coloured", "--accel", "--momentum", blocks],
                         capture_output=True, text=True, timeout=900)
    assert res.returncode == 0, res.stderr[-2000:]
    tr = np.loadtxt(trace, delimiter=",").reshape(-1, 4)
    from dpo_b200.agent import DistributedPGO
    edges, n = load("torus3D", data_dir)
    run = DistributedPGO(edges, n, 8, r=5, schedule="coloured", acceleration=True, momentum_blocks=blocks)
    py = np.array([(s.cost, s.gradnorm) for s in (run.step() for _ in range(rounds))])
    assert tr.shape[0] == rounds
    assert np.max(np.abs(tr[:, 2] - py[:, 0]) / py[:, 0]) <= 1e-9
    assert np.max(np.abs(tr[:, 3] - py[:, 1]) / py[:, 1]) <= 1e-9
