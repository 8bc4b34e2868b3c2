"""CPU checks of the block solve's shared-memory residency (nd::assign_residency, dpo_b200/csrc/nd_precond.cpp): the
first nres columns of a job are copied to the CTA's shared-memory region by a launch's first application and read from
there by every later one.  Through the host emulation of the plan (dpgo_nd_debug_emulate, which runs a filling pass and
then a reading pass) at a given per-CTA budget, and the plan's job records (DPGO_ND_DUMP_JOBS):
  - the solve is bitwise the same at every budget;
  - a CTA's region stays within its budget and its jobs' pieces do not overlap;
  - within a (CTA, phase) every warp streams the same number of rounds per step, or all of its own if it has fewer,
    and a warp's resident rounds come first in its job order."""
import os

import numpy as np
import pytest

from dpo_b200 import posegraph as pg
from dpo_b200.agent import contiguous_owner, partition_edges
from dpo_b200.posegraph import EdgeSet

import structure_cases as sc
from test_nd_plan import emulate

ROUND = 32                     # columns per round of the job loop (nd::RES_ROUND)
UNLIMITED = 1 << 40
BUDGETS = (0, 48 * 1024, UNLIMITED)


def rounds(c):
    return (c + ROUND - 1) // ROUND


def region_doubles(nres):
    return (nres + 3) // 4 * 32


def emulate_at(budget, tmp_path, monkeypatch, n, d, r, brow, bcol, blocks, V, grid):
    path = os.path.join(str(tmp_path), f"jobs_{budget}.csv")
    monkeypatch.setenv("DPGO_ND_RESIDENT_BYTES", str(budget))
    monkeypatch.setenv("DPGO_ND_DUMP_JOBS", path)
    Z, _ = emulate(n, d, r, brow, bcol, blocks, V, grid=grid)
    jobs = np.loadtxt(path, delimiter=",", skiprows=1, dtype=np.int64, ndmin=2)
    return Z, jobs


def check_layout(jobs, budget, grid):
    phase, cta, step, warp, ncols, nres, soff = (jobs[:, k] for k in range(7))
    assert np.all((nres == 0) | (nres == ncols) | ((nres % ROUND == 0) & (nres < ncols)))
    if budget == 0:
        assert np.all(nres == 0)
    if budget == UNLIMITED:
        assert np.all(nres == ncols)
    for c in range(grid):
        m = (cta == c) & (nres > 0)
        lo, hi = soff[m], soff[m] + region_doubles(nres[m])
        if lo.size:
            assert hi.max() * 8 <= budget, (c, hi.max() * 8, budget)
            o = np.argsort(lo, kind="stable")
            assert np.all(hi[o][:-1] <= lo[o][1:]), c                 # pieces do not overlap
        for ph in np.unique(phase[cta == c]):
            sel = np.flatnonzero((cta == c) & (phase == ph))
            per = {}                                                   # (step, warp) -> [(ncols, nres)] in job order
            for q in sel:
                per.setdefault((int(step[q]), int(warp[q])), []).append((int(ncols[q]), int(nres[q])))
            streamed = {k: sum(rounds(a) - rounds(b) for a, b in v) for k, v in per.items()}
            total = {k: sum(rounds(a) for a, _ in v) for k, v in per.items()}
            level = max(streamed.values())
            for k, v in per.items():
                assert streamed[k] == min(total[k], level), (c, ph, k, streamed[k], total[k], level)
                # resident rounds first: fully resident jobs, then at most one partly resident job, then streamed ones
                kind = [2 if b == a else (1 if b > 0 else 0) for a, b in v if a > 0]
                assert kind == sorted(kind, reverse=True) and kind.count(1) <= 1, (c, ph, k, v)


def run_budgets(tmp_path, monkeypatch, n, d, r, brow, bcol, blocks, grid, seed=1):
    V = np.random.default_rng(seed).standard_normal((r, (d + 1) * n))
    Z0 = None
    for budget in BUDGETS:
        Z, jobs = emulate_at(budget, tmp_path, monkeypatch, n, d, r, brow, bcol, blocks, V, grid)
        assert np.all(np.isfinite(Z))
        if Z0 is None:
            Z0 = Z
        assert np.array_equal(Z, Z0), budget
        check_layout(jobs, budget, grid)
    return Z0


def agent0(ds, agents, data_dir):
    edges, n = pg.read_g2o_file(os.path.join(data_dir, ds + ".g2o"))
    parts, counts, _ = partition_edges(edges, contiguous_owner(n, agents), agents)
    return EdgeSet.join([parts[0][0], parts[0][1]]), int(counts[0])


@pytest.mark.parametrize("ds,agents,grid", [("sphere2500", 1, 132), ("sphere2500", 16, 16), ("torus3D", 16, 16)])
def test_resident_solve_is_bitwise_the_same(ds, agents, grid, data_dir, tmp_path, monkeypatch):
    if agents == 1:
        edges, n = pg.read_g2o_file(os.path.join(data_dir, ds + ".g2o"))
    else:
        edges, n = agent0(ds, agents, data_dir)
    brow, bcol, blocks = pg.connection_laplacian_blocks(edges)
    run_budgets(tmp_path, monkeypatch, n, edges.d, 5, brow, bcol, blocks, grid)


@pytest.mark.parametrize("name,d", [("hub191", 3), ("tail_isolated", 2), ("components", 3), ("clique700", 3)])
def test_resident_solve_on_structure_cases(name, d, tmp_path, monkeypatch):
    c = sc.make_case(name, d)
    brow, bcol, blocks = c.triplets()
    for grid in (132, 16):
        run_budgets(tmp_path, monkeypatch, c.n, d, 5, brow, bcol, blocks, grid)


def test_launch_budget_partly_resident(data_dir, tmp_path, monkeypatch):
    """Without a budget override the emulator uses the launch's: sphere2500's panels at the H100's full grid are mostly
    but not all resident, and every CTA's region fits next to what the step stages in 227 KB."""
    edges, n = pg.read_g2o_file(os.path.join(data_dir, "sphere2500.g2o"))
    brow, bcol, blocks = pg.connection_laplacian_blocks(edges)
    path = os.path.join(str(tmp_path), "jobs.csv")
    monkeypatch.delenv("DPGO_ND_RESIDENT_BYTES", raising=False)
    monkeypatch.setenv("DPGO_ND_DUMP_JOBS", path)
    V = np.random.default_rng(2).standard_normal((5, 4 * n))
    emulate(n, 3, 5, brow, bcol, blocks, V, grid=132)
    jobs = np.loadtxt(path, delimiter=",", skiprows=1, dtype=np.int64, ndmin=2)
    budget = int(jobs[0, 7])
    assert 64 * 1024 < budget < 227 * 1024
    frac = (jobs[:, 5].sum()) / jobs[:, 4].sum()
    assert 0.5 < frac < 1.0, frac
    check_layout(jobs, budget, 132)
