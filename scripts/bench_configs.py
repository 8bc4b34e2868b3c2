#!/usr/bin/env python
"""Secondary benchmark: the multi-agent BASELINE.json configs (torus3D / 8 agents, parking-garage / 4 agents,
synthetic grid / 8 agents) with k agents spread over N = WORLD_SIZE GPUs (k % N == 0; N = 1 without torchrun).

    python scripts/bench_configs.py --dataset torus3D --agents 8 --schedule coloured --precond exact
    python -m torch.distributed.run --nproc-per-node 8 ... scripts/bench_configs.py --dataset torus3D --agents 8

Prints ONE JSON line on rank 0: rounds/s and agent-steps/s over --rounds timed rounds (CUDA events, max over
ranks), then the convergence record of a fresh run to central gradient norm < --stop (rounds, wall time, final
2f against the reference's f* where known).  Parity of the same paths is covered by tests/test_gpu_agents.py.
--init distributed starts from the reference's multi-robot initialisation instead of one central chordal solve (per-agent
chordal solves on each rank, then frame-alignment waves; tests/test_gpu_dist_init.py) and records its wall time, split into
the local chordal solves and the waves (host clock after a device synchronise, rank 0), the waves and the inlier counts.
"""
from __future__ import annotations

import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

FSTAR = {"sphere2500": 1687.01, "torus3D": 24227.0, "parking-garage": 1.26248, "smallGrid3D": 1025.4}   # ref vis.ipynb:108745


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--dataset", default="torus3D")
    ap.add_argument("--agents", type=int, default=8)
    ap.add_argument("--schedule", default="coloured", choices=["greedy", "coloured", "parallel"])
    ap.add_argument("--precond", default="exact", choices=["exact", "jacobi"])
    ap.add_argument("--alg", default="rtr", choices=["rtr", "rgd"])
    ap.add_argument("--rounds", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--stop", type=float, default=0.1)
    ap.add_argument("--max-rounds", type=int, default=3000)
    ap.add_argument("--grid", default="100,100,10", help="synthetic grid dims when --dataset synthetic")
    ap.add_argument("--init", default="central", choices=["central", "distributed"],
                    help="start: one chordal solve of the whole graph (synthetic grid: perturbed ground truth), or the "
                         "distributed initialisation from the measurements alone")
    ap.add_argument("--partition", default="blocks", choices=["blocks", "ranges"],
                    help="synthetic grid: kx*ky*kz lattice blocks (public poses only at the block faces) or the reference's "
                         "contiguous id ranges (1.25-layer slabs: every pose public)")
    args = ap.parse_args()

    import torch
    import dpo_b200 as dp
    from dpo_b200 import posegraph as pg
    from dpo_b200.agent import DistributedPGO

    rank = int(os.environ.get("RANK", "0"))
    world = int(os.environ.get("WORLD_SIZE", "1"))
    local_rank = int(os.environ.get("LOCAL_RANK", "0"))
    dist = None
    torch.cuda.set_device(local_rank)
    if world > 1:
        import torch.distributed as dist
        dist.init_process_group("nccl", device_id=torch.device("cuda", local_rank))
    dev = torch.device("cuda", local_rank)

    if args.dataset == "synthetic":
        dims = tuple(int(v) for v in args.grid.split(","))
        edges, n, Tgt = pg.synthetic_grid_graph(*dims, edges_per_pose=4.0, seed=0)
        # initial guess: ground truth with perturbed translations (a chordal solve of a 100k-pose 3-D lattice is a
        # separate, one-shot host problem; the odometry chain along the boustrophedon path drifts too far)
        rng = np.random.default_rng(1)
        T0 = Tgt.copy()
        T0.reshape(3, n, 4)[:, :, 3] += 0.3 * rng.standard_normal((3, n))
        label = f"synthetic grid {dims} = {n} poses / {len(edges)} edges, partition {args.partition}"
        owner = pg.grid_block_owner(*dims, args.agents) if args.partition == "blocks" else None
    else:
        edges, n = pg.read_g2o_file(os.path.join(ROOT, "data", args.dataset + ".g2o"))
        T0 = pg.chordalInitialization(edges.d, n, edges) if args.init == "central" else None
        label = f"{args.dataset}.g2o = {n} poses / {len(edges)} edges"
        owner = None
    r = 5
    X0 = pg.fixedStiefelVariable(edges.d, r) @ T0 if args.init == "central" else None
    precond = dp.PRECOND_SPARSE_EXACT if args.precond == "exact" else dp.PRECOND_BLOCK_JACOBI
    alg = dp.ROPTALG.RTR if args.alg == "rtr" else dp.ROPTALG.RGD

    def make():
        return DistributedPGO(edges, n, args.agents, r=r, algorithm=alg, preconditioner=precond, schedule=args.schedule,
                              X_init=X0, rank=rank, world=world, device=local_rank, dist=dist, owner=owner,
                              initialization=args.init)

    def barrier():
        if world > 1:
            dist.barrier()
        torch.cuda.synchronize()

    # ---- throughput over a fixed number of rounds (no evaluation inside the timed region) ----
    run = make()
    for _ in range(args.warmup):
        run.step(evaluate=False)
    barrier()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    steps = 0
    e0.record()
    for _ in range(args.rounds):
        steps += len([a for a in run._active() if a in run.local_ids])
        run.step(evaluate=False)
    e1.record()
    barrier()
    t = torch.tensor([e0.elapsed_time(e1), float(steps)], dtype=torch.float64, device=dev)
    tmax, tsum = t.clone(), t.clone()
    if world > 1:
        dist.all_reduce(tmax, op=dist.ReduceOp.MAX)
        dist.all_reduce(tsum, op=dist.ReduceOp.SUM)
    ms = float(tmax[0])
    total_steps = float(tsum[1])
    del run

    # ---- convergence of a fresh run ----
    run = make()
    barrier()
    t0 = time.perf_counter()
    hist = []
    rounds = 0
    every = 1 if args.schedule == "greedy" else 5
    st = None
    while rounds < args.max_rounds:
        rounds += 1
        st = run.step(evaluate=(rounds % every == 0))
        if st is not None:
            hist.append((rounds, st.cost, st.gradnorm))
            if st.gradnorm < args.stop:
                break
    barrier()
    wall = time.perf_counter() - t0
    if rank == 0:
        out = {"workload": label, "agents": args.agents, "n_gpus": world, "schedule": args.schedule, "colours": run.ncolours,
               "precond": args.precond, "algorithm": args.alg, "timed_rounds": args.rounds,
               "rounds_per_sec": args.rounds / (ms * 1e-3), "agent_steps_per_sec": total_steps / (ms * 1e-3),
               "ms_per_round": ms / args.rounds, "public_poses_max": int(run.plan.pmax),
               "allgather_bytes_per_agent": int(run.plan.pmax * r * (edges.d + 1) * 8),
               "convergence": {"stop_gradnorm": args.stop, "rounds": rounds, "wall_s": wall,
                               "final_cost_2f": st.cost if st else None, "final_gradnorm": st.gradnorm if st else None,
                               "fstar_reference": FSTAR.get(args.dataset)},
               "trace_head": hist[:5], "trace_tail": hist[-3:]}
        if args.init == "distributed":
            rep = run.init_report
            out["init"] = {"mode": "distributed", **run.init_times, "waves": max(a["wave"] for a in rep),
                           "per_agent": [[a["wave"], a["neighbor"], a["candidates"], a["inliers"], a["iterations"]]
                                         for a in rep],
                           "per_agent_fields": ["wave", "neighbor", "candidates", "inliers", "gnc_iterations"]}
        print(json.dumps(out))
    if world > 1:
        dist.destroy_process_group()


if __name__ == "__main__":
    main()
