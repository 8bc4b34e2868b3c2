"""DistributedPGO allocates every device buffer it uses while it is built: its rounds, team status, solve(), host rounds and
greedy_set selection log allocate nothing on the device afterwards."""
import os

import pytest

pytestmark = pytest.mark.gpu

CASES = {
    "coloured": dict(schedule="coloured"),
    "coloured_accelerated": dict(schedule="coloured", acceleration=True, momentum_blocks="colours"),
    "greedy_set": dict(schedule="greedy_set"),
    "distributed_start": dict(schedule="coloured", initialization="distributed"),
}


@pytest.mark.parametrize("case", list(CASES))
def test_no_device_allocation_after_construction(case, data_dir):
    import torch
    from dpo_b200 import posegraph as pg
    from dpo_b200.agent import DistributedPGO
    edges, n = pg.read_g2o_file(os.path.join(data_dir, "smallGrid3D.g2o"))
    run = DistributedPGO(edges, n, 4, r=5, **CASES[case])
    torch.cuda.synchronize(run.dev)
    allocated = torch.cuda.memory_stats(run.dev)["allocation.all.allocated"]
    run.step(True)
    run.step(False)
    run.status()
    run.solve(max_rounds=3)
    if case == "coloured":
        run.step_host()
    if case == "greedy_set":
        run.selection_log()
    torch.cuda.synchronize(run.dev)
    assert torch.cuda.memory_stats(run.dev)["allocation.all.allocated"] == allocated
