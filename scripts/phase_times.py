#!/usr/bin/env python
"""Phase clock of k_optimize on the bench workload (sphere2500, 1 agent, r = 5, exact preconditioner): where one
RTR step spends its time, per phase kind, as seen by CTA 0 up to each closing grid barrier
(dpgo_debug_phase_times64).  Prints one JSON line; --dataset / --rank / --precond select other workloads."""
import argparse
import ctypes as C
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import numpy as np
import torch
import dpo_b200 as dp
from dpo_b200 import posegraph as pg, _capi

KINDS = ["eval", None, None, "hessian", "tcg_update", "retract", "final"]     # slots 1, 2: unused


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--dataset", default="sphere2500")
    ap.add_argument("--rank", type=int, default=5)
    ap.add_argument("--precond", default="exact", choices=["exact", "dense", "jacobi"])
    ap.add_argument("--steps", type=int, default=30)
    ap.add_argument("--agents", type=int, default=1, help="> 1: the private sub-graph of agent 0 of a contiguous split")
    args = ap.parse_args()
    edges, n = pg.read_g2o_file(os.path.join(ROOT, "data", args.dataset + ".g2o"))
    d = edges.d
    X0 = pg.fixedStiefelVariable(d, args.rank) @ pg.chordalInitialization(d, n, edges)
    if args.agents > 1:
        from dpo_b200.agent import contiguous_owner, partition_edges
        from dpo_b200.posegraph import EdgeSet
        owner = contiguous_owner(n, args.agents)
        parts, counts, glob = partition_edges(edges, owner, args.agents)
        edges = EdgeSet.join([parts[0][0], parts[0][1]])
        n = int(counts[0])
        X0 = X0[:, :(d + 1) * n]
    PRE = {"exact": dp.PRECOND_SPARSE_EXACT, "dense": dp.PRECOND_DENSE_EXACT, "jacobi": dp.PRECOND_BLOCK_JACOBI}[args.precond]
    prob = dp.QuadraticProblem(n, d, args.rank, preconditioners=(dp.PRECOND_BLOCK_JACOBI, PRE))
    prob.setQ_blocks(*pg.connection_laplacian_blocks(edges))
    prob.set_stream(torch.cuda.current_stream().cuda_stream)
    opt = dp.QuadraticOptimizer(prob)
    opt.setTrustRegionTolerance(1e-2)
    opt.setTrustRegionIterations(1)
    opt.setTrustRegionMaxInnerIterations(10)
    opt.setTrustRegionInitialRadius(100)
    opt.setPreconditioner(PRE)
    X0d = torch.from_numpy(np.asfortranarray(X0).ravel(order="F").copy()).cuda()

    def steps(count):
        applies = passes = 0
        for i in range(count):
            if i % 6 == 0:
                prob.copy_X_from_device(X0d.data_ptr())
            opt.optimize_resident_async()
            r = opt.fetch_result()
            applies += r.precond_applies
            passes += r.spmv_passes
        return applies, passes

    steps(6)
    ms = (C.c_double * 64)()
    _capi.check(prob._lib.dpgo_debug_phase_times64(prob._h, 1, ms))
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    e0.record()
    applies, passes = steps(args.steps)
    e1.record()
    torch.cuda.synchronize()
    _capi.check(prob._lib.dpgo_debug_phase_times64(prob._h, 0, ms))
    out = {"workload": f"{args.dataset} agent 0 of {args.agents} ({n} poses) r={args.rank} {args.precond}", "steps": args.steps,
           "ms_per_step_events": e0.elapsed_time(e1) / args.steps, "precond_applies": applies, "q_passes": passes,
           "ms_per_step_by_kind": {k: ms[i] / args.steps for i, k in enumerate(KINDS) if k and ms[i] > 0},
           "us_per_hessian": 1e3 * ms[3] / max(passes - 2 * args.steps, 1)}
    out["hessian_cta0_us"] = {"first_gather": 1e3 * ms[27] / max(passes - 2 * args.steps, 1), "whole_loop": 1e3 * ms[28] / max(passes - 2 * args.steps, 1)}
    if args.precond in ("exact", "dense"):
        nphases = 1                                   # dense: the block solve's single macro level, one phase
        if args.precond == "exact":
            out["nd"] = prob.nd_info()
            nphases = out["nd"]["phases"]
        out["us_per_apply_by_nd_phase"] = [1e3 * ms[8 + k] / max(applies, 1) for k in range(nphases)]
        out["us_per_apply_cta0"] = {"gathers": 1e3 * ms[24] / max(applies, 1), "jobs": 1e3 * ms[25] / max(applies, 1),
                                    "epilogues": 1e3 * ms[26] / max(applies, 1)}
        out["us_per_apply_cta0_by_phase"] = [[round(1e3 * ms[32 + 3 * k + q] / max(applies, 1), 3) for q in range(3)]
                                             for k in range(nphases)]
    print(json.dumps(out))


if __name__ == "__main__":
    main()
