"""Setup calls repeated on live problem handles.  Every setup path (set_edges with its preconditioners, the public poses,
the shared edges, the alignment candidates, accel_init, the agent graph) replaces the device buffers it owns; a second
pass of the same calls on the same handles must give the same rounds bit for bit.  Handles destroyed and re-created in
one process must keep working.  The C++ runner releases every resource it creates, also when its constructor throws."""
import os

import numpy as np
import pytest

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DATA = os.path.join(ROOT, "data")
K = 4


def make(schedule, acceleration):
    from dpo_b200 import posegraph as pg
    from dpo_b200.agent import DistributedPGO
    edges, n = pg.read_g2o_file(os.path.join(DATA, "smallGrid3D.g2o"))
    return DistributedPGO(edges, n, K, r=5, schedule=schedule, acceleration=acceleration,
                          momentum_blocks="colours" if acceleration else "agents")


def setup_calls(run, X0):
    """The setup sequence of the runner's constructor, issued again on its live handles, with the alignment candidates of
    the distributed start too."""
    for a in run.local_ids:
        run.agents[a].constructQMatrix()            # dpgo_problem_set_edges: build_from_triplets, then reassemble_Q
        run.agents[a].mProblem.upload_X(X0[a])
    run._setup_agents(candidates=True)              # public poses, shared edges, candidates, accel_init, agent graph
    run.round = 0
    run.selected = [0]
    run._gathered_current = False
    run._records_current = False


def one_pass(run, X0, rounds):
    import torch
    setup_calls(run, X0)
    for _ in range(rounds):
        run.step(evaluate=False)
    records = run.status().records
    torch.cuda.synchronize()
    X = {a: run.agents[a].mProblem.download_X() for a in run.local_ids}
    log = run.selection_log() if run.schedule == "greedy_set" else None
    return X, records, log


@pytest.mark.parametrize("schedule,acceleration", [("coloured", True), ("greedy_set", False)])
def test_setup_twice_on_live_handles(schedule, acceleration):
    run = make(schedule, acceleration)
    X0 = {a: run.agents[a].mProblem.download_X() for a in run.local_ids}
    # coloured: whole sweeps over the colour classes; greedy_set: past 64 rounds, so that the selection log grows
    rounds = 10 * run.ncolours if schedule == "coloured" else 70
    X1, rec1, log1 = one_pass(run, X0, rounds)
    X2, rec2, log2 = one_pass(run, X0, rounds)
    assert any(not np.array_equal(X1[a], X0[a]) for a in run.local_ids)
    for a in run.local_ids:
        assert np.array_equal(X1[a], X2[a]), a
    assert np.array_equal(rec1[:, :4], rec2[:, :4])      # column 4 counts the optimising calls: it grows by design
    assert np.all(rec2[:, 4] >= rec1[:, 4]) and np.sum(rec2[:, 4]) > np.sum(rec1[:, 4])
    if log1 is not None:
        assert len(log1) == rounds and log1 == log2


def test_handles_destroyed_and_recreated():
    import gc
    for _ in range(3):
        run = make("greedy_set", False)
        for _ in range(5):
            run.step(evaluate=False)
        st = run.status()
        assert np.isfinite(st.cost) and np.isfinite(st.gradnorm)
        assert len(run.selection_log()) == 5
        for ag in run.agents.values():
            ag.mProblem.close()
        del run
        gc.collect()


@pytest.fixture(scope="module")
def runner_lifetime_check():
    from dpo_b200 import build
    return build.build_cpp_program([os.path.join(ROOT, "tests", "cpp", "runner_lifetime_check.cpp")],
                                   os.path.join(ROOT, "build", "tests", "runner_lifetime_check"))


def _device_count():
    import ctypes
    from dpo_b200 import _capi
    c = ctypes.c_int(0)
    _capi.load_library().dpgo_device_count(ctypes.byref(c))
    return c.value


@pytest.mark.parametrize("gpus", [1, 2])
def test_cpp_runner_releases_its_resources(gpus, runner_lifetime_check):
    """DPGO::DeviceRBCD releases every stream, device buffer, pinned buffer and NCCL communicator it creates: when its
    constructor throws (the distributed initialisation of a disconnected agent graph), and after solve() / status() with
    accelerated coloured rounds and after step() / selectionLog() with greedy_set rounds."""
    import subprocess
    if gpus > _device_count():
        pytest.skip(f"needs {gpus} GPUs")
    res = subprocess.run([runner_lifetime_check, os.path.join(DATA, "smallGrid3D.g2o"), str(gpus)], capture_output=True,
                         text=True, timeout=600)
    assert res.returncode == 0, res.stderr[-2000:]
    lines = res.stdout.splitlines()
    assert any(ln.startswith("error a ") and "agents [3]" in ln for ln in lines), res.stdout
    counts = {}
    for ln in lines:
        w = ln.split()
        if w[0] == "counts":
            counts[w[1]] = dict(zip(w[2::2], map(int, w[3::2])))
    assert sorted(counts) == ["a", "b", "c"], res.stdout
    for case, c in counts.items():
        assert c["dpgo_stream_create"] == gpus and c["dpgo_device_malloc"] > 0, (case, c)
        assert c["ncclCommInitAll"] == (gpus if gpus > 1 else 0), (case, c)
        for create, release in [("dpgo_stream_create", "dpgo_stream_destroy"), ("dpgo_device_malloc", "dpgo_device_free"),
                                ("dpgo_host_alloc_pinned", "dpgo_host_free_pinned"), ("ncclCommInitAll", "ncclCommDestroy")]:
            assert c[create] == c[release], (case, create, c)
