"""The greedy_set schedule, the parts that need no GPU: the shared selection rule on hand cases, the CPU restatement's
convergence, the argument checks of DistributedPGO, and the new C ABI calls failing loudly without a device."""
import ctypes as C
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import greedy_set_oracle as gso  # noqa: E402
from oracle import dpgo_oracle as orc  # noqa: E402
from dpo_b200.agent import greedy_independent_set, greedy_selection, check_solve_arguments, auto_concurrent  # noqa: E402


def is_maximal(taken, g, nbrs):
    """every agent left out has a taken neighbour that the walk reached first"""
    for a in range(len(g)):
        if a in taken:
            assert not any(b in taken for b in nbrs[a]), a
        else:
            assert any(b in taken and (g[b] > g[a] or (g[b] == g[a] and b < a)) for b in nbrs[a]), a


def ring(k):
    return [sorted({(a - 1) % k, (a + 1) % k}) for a in range(k)]


def test_ring_of_eight_by_hand():
    g = np.array([5.0, 9.0, 1.0, 7.0, 3.0, 8.0, 2.0, 6.0])
    # order 1 (9), 5 (8), 3 (7), 7 (6), 0 (5), 4 (3), 6 (2), 2 (1): take 1, 5, 3, 7; 0, 4, 6, 2 each touch a taken agent
    assert greedy_independent_set(g, ring(8)) == [1, 3, 5, 7]
    is_maximal({1, 3, 5, 7}, g, ring(8))
    g2 = np.array([9.0, 1.0, 2.0, 8.0, 3.0, 4.0, 7.0, 5.0])
    # order 0, 3, 6, 7, 5, 4, 2, 1: take 0, 3, 6; then 7 touches 6, 5 touches 6, 4 touches 3, 2 touches 3, 1 touches 0
    assert greedy_independent_set(g2, ring(8)) == [0, 3, 6]
    is_maximal({0, 3, 6}, g2, ring(8))


def test_ties_go_to_the_lower_id():
    assert greedy_independent_set(np.ones(4), ring(4)) == [0, 2]
    assert greedy_independent_set(np.array([1.0, 2.0, 2.0, 1.0]), ring(4)) == [1, 3]
    assert greedy_independent_set(np.array([0.0, -0.0, 0.0]), [[1], [0, 2], [1]]) == [0, 2]


def test_isolated_agents_are_always_taken():
    nbrs = [[1], [0], [], [], [5], [4]]
    g = np.array([1.0, 2.0, 0.0, 0.0, 3.0, 3.0])
    assert greedy_independent_set(g, nbrs) == [1, 2, 3, 4]
    assert greedy_independent_set(np.zeros(1), [[]]) == [0]


def test_nan_norm_ranks_last():
    assert greedy_independent_set(np.array([np.nan, 1.0]), [[1], [0]]) == [1]


@pytest.mark.parametrize("seed", range(5))
def test_complete_graph_gives_the_greedy_choice(seed):
    rng = np.random.default_rng(seed)
    k = 7
    nbrs = [[b for b in range(k) if b != a] for a in range(k)]
    g = rng.random(k)
    if seed == 0:
        g[2] = g[5] = 2.0                  # a tie for the maximum: std::max_element takes the first
    assert greedy_independent_set(g, nbrs) == [greedy_selection(0, np.sqrt(g), True)]


@pytest.mark.parametrize("seed", range(5))
def test_random_graphs_are_maximal_independent(seed):
    rng = np.random.default_rng(100 + seed)
    k = 20
    A = np.triu(rng.random((k, k)) < 0.2, 1)
    A = A | A.T
    nbrs = [list(np.flatnonzero(A[a])) for a in range(k)]
    g = rng.random(k)
    is_maximal(set(greedy_independent_set(g, nbrs)), g, nbrs)


def test_oracle_converges_on_smallgrid(data_dir):
    meas, n = orc.read_g2o(os.path.join(data_dir, "smallGrid3D.g2o"))
    drv = gso.GreedySetDriver(meas, n, 5, r=5)
    for i in range(400):
        _, gn = drv.step()
        if gn < 0.1:
            break
    assert gn < 0.1, gn
    nbrs = [ag.neighbors for ag in drv.agents]
    for s, g in zip(drv.sets, drv.norms2):
        is_maximal(set(s), g, nbrs)


def test_auto_concurrent_greedy_set():
    path = [[1], [0, 2], [1]]
    assert auto_concurrent([0, 1, 0], 3, 1, "greedy_set", False, path)            # agents 0 and 2 are not neighbours
    assert not auto_concurrent([0, 1, 2], 3, 1, "greedy_set", False, [[1, 2], [0, 2], [0, 1]])
    assert not auto_concurrent([0, 1, 0, 1], 4, 2, "greedy_set", False, ring(4))  # each rank hosts one neighbouring pair


def test_arguments(data_dir):
    from dpo_b200 import posegraph as pg
    from dpo_b200.agent import DistributedPGO
    check_solve_arguments("greedy_set", False, 100, 5)                             # any check_every
    with pytest.raises(ValueError, match="check_every must be 1"):
        check_solve_arguments("greedy", False, 100, 5)
    edges, n = pg.read_g2o_file(os.path.join(data_dir, "smallGrid3D.g2o"))
    with pytest.raises(ValueError, match="greedy_set"):
        DistributedPGO(edges, n, 5, r=5, schedule="greedy_set", acceleration=True)
    with pytest.raises(ValueError, match="schedule must be"):
        DistributedPGO(edges, n, 5, r=5, schedule="greedy-set")


def test_select_calls_without_device():
    from dpo_b200 import _capi
    lib = _capi.load_library()
    c = C.c_int(-1)
    if lib.dpgo_device_count(C.byref(c)) == 0 and c.value > 0:
        pytest.skip("a CUDA device is present")
    handles = (C.c_void_p * 1)(None)
    bufs = (C.c_void_p * 1)(None)
    ptr, adj, idx = np.zeros(2, dtype=np.int32), np.zeros(1, dtype=np.int32), np.zeros(1, dtype=np.int32)
    prm = _capi.OptParams()
    lib.dpgo_opt_params_default(C.byref(prm))
    assert lib.dpgo_agents_set_agent_graph(None, 1, _capi.iptr(ptr), _capi.iptr(adj)) == 2
    assert lib.dpgo_agents_select_round_async(handles, 1, _capi.iptr(idx), C.byref(prm), None, None, 1, bufs, None) == 2
    total = C.c_int64(0)
    assert lib.dpgo_agents_selection_log(None, 0, 0, None, C.byref(total)) == 2
    assert lib.dpgo_abi_version() == 1
