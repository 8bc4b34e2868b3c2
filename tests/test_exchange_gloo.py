"""N>1 host logic on CPU: world-size-2 gloo run of the boundary-pose exchange plan (dpo_b200.agent.ExchangePlan).

The device kernels (k_pack_tiles, k_build_G) cannot run without a GPU, so each rank emulates them with the SAME
index tables in NumPy: pack public tiles -> ONE all_gather (gloo) -> rebuild G from the gathered slots, and compares
with the oracle's dictionary-based constructGMatrix.  This pins the slot / padding / edge tables across processes."""
import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _worker(rank, world, port, ds, ret, k=None):
    sys.path.insert(0, ROOT)
    import torch
    import torch.distributed as dist
    from dpo_b200 import posegraph as pg
    from dpo_b200.agent import ExchangePlan, contiguous_owner, partition_edges
    from oracle import dpgo_oracle as orc
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        edges, n = pg.read_g2o_file(os.path.join(ROOT, "data", ds + ".g2o"))
        d, r, dh = edges.d, 5, edges.d + 1
        k = world if k is None else k                      # k agents, k/world per rank (contiguous blocks)
        per_rank = k // world
        mine = list(range(rank * per_rank, (rank + 1) * per_rank))
        owner = contiguous_owner(n, k)
        parts, counts, glob = partition_edges(edges, owner, k)
        plan = ExchangePlan([p[2] for p in parts], k)
        rng = np.random.default_rng(7)                     # same on every rank
        Xfull = rng.standard_normal((r, dh * n))
        ts = r * dh
        # --- pack (what k_pack_tiles does): slot s <- tile public[a][s], column-major tiles; a rank's agents are
        #     contiguous in the send buffer so that rank-major all-gather order == agent order
        send = np.zeros(per_rank * plan.pmax * ts)
        for li, a in enumerate(mine):
            cols = (glob[a][:, None] * dh + np.arange(dh)[None, :]).ravel()
            Xloc = Xfull[:, cols]
            for s, q in enumerate(plan.public[a]):
                o = (li * plan.pmax + s) * ts
                send[o:o + ts] = Xloc[:, q * dh:(q + 1) * dh].ravel(order="F")
        gathered = torch.zeros(k * plan.pmax * ts, dtype=torch.float64)
        dist.all_gather_into_tensor(gathered, torch.from_numpy(send))
        gathered = gathered.numpy()
        worst, nedges_total = 0.0, 0
        for a in mine:
            worst = max(worst, _check_agent(a, k, plan, parts, counts, glob, gathered, Xfull, d, r, dh, ts, orc))
            nedges_total += len(plan.tables[a]["local"])
        ret[rank] = (worst, int(plan.pmax), nedges_total)
    finally:
        dist.destroy_process_group()


def _check_agent(agent, k, plan, parts, counts, glob, gathered, Xfull, d, r, dh, ts, orc):
    """Rebuild agent `agent`'s G from the gathered slots with the plan tables (what k_build_G does) and compare it
    with the oracle's dictionary-based constructGMatrix fed with the true neighbour poses."""
    # --- rebuild G (what k_build_G does) from the tables
    tb = plan.tables[agent]
    G = np.zeros((r, dh * int(counts[agent])))
    for e in range(len(tb["local"])):
        Xn = gathered[tb["slot"][e] * ts:(tb["slot"][e] + 1) * ts].reshape(r, dh, order="F")
        T, om = tb["T"][e], tb["omega"][e]
        L = (Xn * om[None, :]) @ T.T if tb["outgoing"][e] else (Xn @ T) * om[None, :]
        p = tb["local"][e]
        G[:, p * dh:(p + 1) * dh] -= L
    # --- oracle: dictionary form with the true neighbour poses
    sh = parts[agent][2]
    m = orc.Measurements(d, sh.r1, sh.r2, sh.p1, sh.p2, sh.R, sh.t, sh.kappa, sh.tau, sh.weight)
    oa = orc.PGOAgent(agent, d, r)
    oa.n = int(counts[agent])
    oa.shared_lc = m
    oa.problem = orc.QuadraticProblem(oa.n, d, r)
    poses = {}
    for b in range(k):
        if b == agent:
            continue
        cb = (glob[b][:, None] * dh + np.arange(dh)[None, :]).ravel()
        Xb = Xfull[:, cb]
        for q in plan.public[b]:
            poses[(b, int(q))] = Xb[:, q * dh:(q + 1) * dh]
    assert oa.construct_G(poses)
    return float(np.abs(G - oa.problem.G).max())


@pytest.mark.parametrize("ds", ["smallGrid3D", "CSAIL"])
def test_exchange_plan_world2_gloo(ds):
    import torch.multiprocessing as mp
    port = 29600 + (os.getpid() % 300)
    mgr = mp.Manager()
    ret = mgr.dict()
    procs = [mp.get_context("spawn").Process(target=_worker, args=(rk, 2, port, ds, ret)) for rk in range(2)]
    for p in procs:
        p.start()
    for p in procs:
        p.join(180)
        assert p.exitcode == 0
    assert len(ret) == 2
    for rk in range(2):
        err, pmax, nedges = ret[rk]
        assert err <= 1e-12, (rk, err)
        assert pmax >= 1 and nedges >= 1
    assert ret[0][2] == ret[1][2]          # both agents see the same cut edges


def test_exchange_plan_four_agents_on_two_ranks_gloo():
    """k = 4 agents over world = 2 ranks (two agents per rank): the all-gather order must equal agent order."""
    import torch.multiprocessing as mp
    port = 29900 + (os.getpid() % 90)
    mgr = mp.Manager()
    ret = mgr.dict()
    procs = [mp.get_context("spawn").Process(target=_worker, args=(rk, 2, port, "smallGrid3D", ret, 4)) for rk in range(2)]
    for p in procs:
        p.start()
    for p in procs:
        p.join(180)
        assert p.exitcode == 0
    assert len(ret) == 2
    for rk in range(2):
        assert ret[rk][0] <= 1e-12, ret[rk]


def _gathered_worker(rank, world, port, ret):
    sys.path.insert(0, ROOT)
    import torch
    import torch.distributed as dist
    from dpo_b200.agent import _Gathered
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        mine = [2 * rank, 2 * rank + 1]
        g = _Gathered(torch, torch.device("cpu"), 4, mine, 3, True)
        assert g.own.numel() == 2 * 3 and g.own.data_ptr() != g.all.data_ptr()
        for a in mine:
            g.part[a].copy_(10.0 * a + torch.arange(3, dtype=torch.float64))
        g.gather(dist)
        ret[rank] = g.all.tolist()
    finally:
        dist.destroy_process_group()


def test_gathered_buffer_four_agents_on_two_ranks_gloo():
    """The runner's gathered buffers over world = 2 ranks with two agents each: after the all-gather every rank holds agent
    a's part at a * part, in agent order."""
    import torch.multiprocessing as mp
    port = 29500 + (os.getpid() % 90)
    mgr = mp.Manager()
    ret = mgr.dict()
    procs = [mp.get_context("spawn").Process(target=_gathered_worker, args=(rk, 2, port, ret)) for rk in range(2)]
    for p in procs:
        p.start()
    for p in procs:
        p.join(180)
        assert p.exitcode == 0
    expect = [10.0 * a + i for a in range(4) for i in range(3)]
    assert ret[0] == expect and ret[1] == expect


def test_gathered_buffer_one_rank_writes_in_place():
    """With one rank each agent's part is a view of `all` (no copy, nothing to gather)."""
    import torch
    sys.path.insert(0, ROOT)
    from dpo_b200.agent import _Gathered
    g = _Gathered(torch, torch.device("cpu"), 4, [0, 1, 2, 3], 3, False)
    for a in range(4):
        assert g.part[a].untyped_storage().data_ptr() == g.all.untyped_storage().data_ptr()
        assert g.part[a].data_ptr() == g.all.data_ptr() + a * 3 * 8
        g.part[a].fill_(a)
    g.gather(None)
    assert g.all.tolist() == [float(a) for a in range(4) for _ in range(3)]


def test_partition_and_colouring():
    sys.path.insert(0, ROOT)
    from dpo_b200 import posegraph as pg
    from dpo_b200.agent import ExchangePlan, contiguous_owner, partition_edges
    edges, n = pg.read_g2o_file(os.path.join(ROOT, "data", "smallGrid3D.g2o"))
    owner = contiguous_owner(n, 5)
    assert owner[0] == 0 and owner[-1] == 4 and np.all(np.diff(owner) >= 0)       # ref ex:95-109 contiguous blocks
    parts, counts, glob = partition_edges(edges, owner, 5)
    assert counts.sum() == n
    n_private = sum(len(p[0]) + len(p[1]) for p in parts)
    n_shared = sum(len(p[2]) for p in parts)
    assert n_private + n_shared // 2 == len(edges)                                 # shared edges appear in both agents
    plan = ExchangePlan([p[2] for p in parts], 5)
    col = plan.colouring()
    for a in range(5):
        for b in plan.tables[a]["neighbors"]:
            assert col[a] != col[b]


def test_auto_concurrent_launch_mode():
    """The default launch mode of the device runner is a pure function of the global plan (every rank decides alike):
    agents side by side only under the coloured schedule when a rank hosts >= 2 agents of one colour class."""
    sys.path.insert(0, ROOT)
    from dpo_b200.agent import auto_concurrent
    chain16 = [a % 2 for a in range(16)]                     # the bench workload: 16 agents in a chain, 2 colours
    assert auto_concurrent(chain16, 16, 1, "coloured", False)            # 8 per colour on one GPU
    assert auto_concurrent(chain16, 16, 2, "coloured", False)            # 4 per colour and rank
    assert auto_concurrent(chain16, 16, 4, "coloured", False)            # 2 per colour and rank
    assert not auto_concurrent(chain16, 16, 8, "coloured", False)        # one of each colour per rank: full-grid kernels
    assert not auto_concurrent(chain16, 16, 1, "greedy", False)
    assert not auto_concurrent(chain16, 16, 1, "parallel", False)
    assert not auto_concurrent(chain16, 16, 1, "coloured", True)         # accelerated rounds keep the sequential path
    assert not auto_concurrent([0, 1, 2], 3, 1, "coloured", False)       # a triangle of agents: one per colour
