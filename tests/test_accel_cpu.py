"""Accelerated coloured rounds, the parts that need no GPU: the restatement's rounds to convergence with the momentum over
colour classes, the argument checks of DistributedPGO, and the new C ABI calls failing loudly without a device."""
import ctypes as C
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import accel_oracle as ao  # noqa: E402
from oracle import dpgo_oracle as orc  # noqa: E402


def rounds_to(drv, tol=0.1, cap=400):
    for i in range(cap):
        _, gn = drv.step()
        if gn < tol:
            return i + 1
    return None


def test_colour_momentum_converges_in_fewer_rounds_than_plain_coloured(data_dir):
    meas, n = orc.read_g2o(os.path.join(data_dir, "smallGrid3D.g2o"))
    plain = rounds_to(orc.MultiRobotDriver(meas, n, 5, r=5, schedule="coloured"))
    colours = rounds_to(ao.AcceleratedColouredDriver(meas, n, 5, r=5, momentum_blocks="colours"))
    assert plain is not None and colours is not None
    assert colours < plain, (colours, plain)


def test_momentum_trace_restarts():
    tr = ao.momentum_trace(2.0, 60)
    assert tr[0] == (0.5, 1.0, 1.0)                          # (1 + 1) / (2 N), 1 / (gamma N)
    assert tr[28] == (0.0, 0.0, 29.0) and tr[58] == (0.0, 0.0, 59.0)
    assert tr[29][0] == tr[0][0] and all(g > 0 for g, _, _ in tr[:28])


@pytest.mark.parametrize("schedule,blocks", [("greedy", "colours"), ("parallel", "colours"), ("coloured", "robots")])
def test_momentum_blocks_arguments(schedule, blocks, data_dir):
    from dpo_b200 import posegraph as pg
    from dpo_b200.agent import DistributedPGO
    edges, n = pg.read_g2o_file(os.path.join(data_dir, "smallGrid3D.g2o"))
    with pytest.raises(ValueError, match="momentum_blocks"):
        DistributedPGO(edges, n, 5, r=5, schedule=schedule, acceleration=True, momentum_blocks=blocks)


def test_accel_calls_without_device():
    from dpo_b200 import _capi
    lib = _capi.load_library()
    c = C.c_int(-1)
    if lib.dpgo_device_count(C.byref(c)) == 0 and c.value > 0:
        pytest.skip("a CUDA device is present")
    handles = (C.c_void_p * 1)(None)
    bufs = (C.c_void_p * 1)(None)
    flags = np.zeros(1, dtype=np.int32)
    prm = _capi.OptParams()
    lib.dpgo_opt_params_default(C.byref(prm))
    assert lib.dpgo_agents_accel_begin_async(handles, 1, _capi.iptr(flags), 2.0, 30, bufs, bufs, None) == 2
    assert lib.dpgo_agents_accel_round_async(handles, 1, C.byref(prm), None, None, 1, None) == 2
    assert lib.dpgo_agent_accel_state(None, _capi.dptr(np.zeros(3))) == 2
    assert lib.dpgo_abi_version() == 1
