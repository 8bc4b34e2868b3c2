"""Running the device runners to convergence, the parts that need no GPU: the new C ABI calls fail loudly without a
device, the NumPy restatement of the rounding into the global frame, and the stop rule as a function of status records."""
import ctypes as C
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import solve_oracle as so  # noqa: E402


def test_status_and_trajectory_calls_without_device():
    from dpo_b200 import _capi
    lib = _capi.load_library()
    assert "dpgo_agents_status_async" in _capi.SIGNATURES and "dpgo_agent_trajectory_global" in _capi.SIGNATURES
    c = C.c_int(-1)
    if lib.dpgo_device_count(C.byref(c)) == 0 and c.value > 0:
        pytest.skip("a CUDA device is present")
    handles = (C.c_void_p * 1)(None)
    slots = np.zeros(1, dtype=np.int32)
    buf = np.zeros(_capi.STATUS_DOUBLES)
    assert lib.dpgo_agents_status_async(handles, 1, _capi.iptr(slots), C.c_void_p(buf.ctypes.data), None) == 2
    anchor, T = np.zeros((5, 4)), np.zeros((3, 4))
    assert lib.dpgo_agent_trajectory_global(None, _capi.dptr(anchor), _capi.dptr(T)) == 2
    assert lib.dpgo_abi_version() == 1


def triangle_truth():
    """ref tests/testTriangleGraph.cpp:15-29: the three poses of the noise-free triangle, d x (d+1)n."""
    return np.array([[1, 0, 0, 0, 0.1436, 0.7406, 0.6564, 1, -0.4069, -0.4150, -0.8138, 2],
                     [0, 1, 0, 0, -0.8179, -0.2845, 0.5000, 1, 0.4049, 0.7166, -0.5679, 2],
                     [0, 0, 1, 0, 0.5571, -0.6087, 0.5649, 1, 0.8188, -0.5606, -0.1236, 2]], dtype=float)


def test_trajectory_restatement_on_the_triangle():
    """A lifted triangle in an arbitrary global frame rounds back to Ttrue: the printed rotations are orthonormal only
    to their 4 decimals, so the truth is their projection onto SO(3); it then comes back to 1e-12."""
    d, r, dh = 3, 5, 4
    Ttrue = triangle_truth()
    for i in range(3):
        Ttrue[:, i * dh:i * dh + d] = so.project_to_rotation(Ttrue[:, i * dh:i * dh + d])
    assert np.abs(Ttrue - triangle_truth()).max() < 1e-3
    rng = np.random.default_rng(3)
    Y = np.linalg.qr(rng.standard_normal((r, d)))[0]                 # lift (Stiefel)
    Rg = so.project_to_rotation(rng.standard_normal((d, d)))         # global frame of the lifted iterate
    tg = rng.standard_normal(d)
    X = np.zeros((r, dh * 3))
    for i in range(3):
        X[:, i * dh:i * dh + d] = Y @ Rg @ Ttrue[:, i * dh:i * dh + d]
        X[:, i * dh + d] = Y @ (Rg @ Ttrue[:, i * dh + d] + tg)
    T = so.trajectory_in_global_frame(X, X[:, :dh], d)
    assert np.abs(T - Ttrue).max() <= 1e-12
    for i in range(3):
        Ri = T[:, i * dh:i * dh + d]
        assert np.abs(Ri.T @ Ri - np.eye(d)).max() <= 1e-12 and abs(np.linalg.det(Ri) - 1.0) <= 1e-12


def records(gn2, rel, calls):
    k = len(gn2)
    rec = np.zeros((k, 5))
    rec[:, 0], rec[:, 1], rec[:, 2], rec[:, 3], rec[:, 4] = 10.0, -4.0, gn2, rel, calls
    return rec


def test_stop_rule_from_status_records():
    from dpo_b200.agent import stop_reason, team_status
    st = team_status(records([0.01, 0.02], [1e-3, 1e-3], [3, 3]))
    assert st.cost == pytest.approx(12.0) and st.gradnorm == pytest.approx(np.sqrt(0.03))
    start = np.array([1, 1])
    # gradient norm first, then the team, then the cap
    assert stop_reason(records([0.001, 0.001], [1.0, 1.0], [3, 3]), start, 5, 500, 0.1, 5e-3) == "gradnorm"
    assert stop_reason(records([1.0, 1.0], [1e-3, 5e-3], [3, 3]), start, 5, 500, 0.1, 5e-3) == "team"
    assert stop_reason(records([1.0, 1.0], [1e-3, 6e-3], [3, 3]), start, 5, 500, 0.1, 5e-3) is None
    assert stop_reason(records([1.0, 1.0], [1e-3, 6e-3], [3, 3]), start, 500, 500, 0.1, 5e-3) == "max_rounds"
    # an agent that has not optimised since the solve began is not ready, whatever its (stale) relative change
    assert stop_reason(records([1.0, 1.0], [1e-3, 1e-3], [3, 1]), start, 5, 500, 0.1, 5e-3) is None
    assert stop_reason(records([1.0, 1.0], [0.0, 0.0], [0, 0]), np.zeros(2), 5, 500, 0.1, 5e-3) is None
    # a tolerance of 0 disables its rule
    assert stop_reason(records([0.0, 0.0], [1.0, 1.0], [3, 3]), start, 5, 500, 0.0, 5e-3) is None
    assert stop_reason(records([1.0, 1.0], [0.0, 0.0], [3, 3]), start, 5, 500, 0.1, 0.0) is None


def test_greedy_selection_and_solve_arguments():
    from dpo_b200.agent import check_solve_arguments, greedy_selection
    gn = np.array([0.5, 2.0, 1.0])
    assert greedy_selection(0, gn, True) == 1
    assert greedy_selection(2, gn, False) == 2                       # no neighbours: the selection stays (ref :308-325)
    assert greedy_selection(0, np.array([1.0, 1.0, 0.0]), True) == 0  # ties: the first, as std::max_element
    check_solve_arguments("greedy", False, 500, 1)
    check_solve_arguments("coloured", False, 500, 5)
    with pytest.raises(ValueError, match="check_every must be 1"):
        check_solve_arguments("greedy", False, 500, 5)
    with pytest.raises(ValueError, match="acceleration"):
        check_solve_arguments("coloured", True, 500, 1)
    with pytest.raises(ValueError):
        check_solve_arguments("coloured", False, 0, 1)
