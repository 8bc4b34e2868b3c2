"""Cost of the relaxation rank on one GPU: sphere2500 at r = 3..8.

    python scripts/rank_bench.py [--steps 300] [--rounds 200] [--out result.json]

Prints the card, its power limit and maximum SM clock, then per rank:
  * RTR iterations/s of one agent (the bench.py workload: updateX constants, exact preconditioner, resident iterate reset
    to the chordal start every 6 steps), timed with CUDA events;
  * the Q.X product alone (TMA-fed SpMV): its algorithmic bytes and the bandwidth they give over the kernel time;
and, at r = 5 and r = 8, the rounds/s of 16 coloured agents stepped side by side on the GPU (thread-block clusters on a
side stream, the rounds replayed as CUDA graphs), 2f and |g| not evaluated inside the timed window.
Needs a CUDA device; writes nothing in the tree (--out is optional)."""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def card():
    q = "name,power.limit,clocks.max.sm"
    try:
        out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader", "-i", "0"], capture_output=True,
                             text=True, timeout=60).stdout.strip()
    except (OSError, subprocess.SubprocessError) as e:
        out = f"nvidia-smi unavailable: {e}"
    return out


def main():
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--steps", type=int, default=300)
    ap.add_argument("--rounds", type=int, default=200)
    ap.add_argument("--out", default="")
    args = ap.parse_args()
    import torch
    import dpo_b200 as dp
    from dpo_b200 import posegraph as pg
    from dpo_b200.agent import DistributedPGO
    if not torch.cuda.is_available():
        raise SystemExit("rank_bench.py needs a CUDA device")
    edges, n = pg.read_g2o_file(os.path.join(ROOT, "data", "sphere2500.g2o"))
    d = edges.d
    T0 = pg.chordalInitialization(d, n, edges)
    blocks = pg.connection_laplacian_blocks(edges)
    res = {"card (name, power limit, max SM clock)": card(), "dataset": "sphere2500", "rtr": {}, "spmv": {}, "rounds16": {}}
    print(res["card (name, power limit, max SM clock)"], flush=True)
    dev = torch.device("cuda:0")
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    for r in range(3, 9):
        prob = dp.QuadraticProblem(n, d, r, preconditioners=(dp.PRECOND_BLOCK_JACOBI, dp.PRECOND_SPARSE_EXACT))
        prob.setQ_blocks(*blocks)
        prob.set_stream(torch.cuda.current_stream().cuda_stream)
        opt = dp.QuadraticOptimizer(prob)
        opt.setTrustRegionTolerance(1e-2)
        opt.setTrustRegionIterations(1)
        opt.setTrustRegionMaxInnerIterations(10)
        opt.setTrustRegionInitialRadius(100)
        opt.setPreconditioner(dp.PRECOND_SPARSE_EXACT)
        X0 = pg.fixedStiefelVariable(d, r) @ T0
        X0d = torch.from_numpy(np.asfortranarray(X0).ravel(order="F").copy()).to(dev)

        def steps(count):
            for i in range(count):
                if i % 6 == 0:
                    prob.copy_X_from_device(X0d.data_ptr())
                opt.optimize_resident_async()

        steps(30)
        torch.cuda.synchronize()
        e0.record()
        steps(args.steps)
        e1.record()
        torch.cuda.synchronize()
        res["rtr"][r] = args.steps / (e0.elapsed_time(e1) * 1e-3)
        # the SpMV alone
        x = torch.randn(r * (d + 1) * n, dtype=torch.float64, device=dev)
        y = torch.empty_like(x)
        for _ in range(20):
            prob.spmv_device(x.data_ptr(), y.data_ptr(), False)
        reps = 500
        torch.cuda.synchronize()
        e0.record()
        for _ in range(reps):
            prob.spmv_device(x.data_ptr(), y.data_ptr(), False)
        e1.record()
        torch.cuda.synchronize()
        us = e0.elapsed_time(e1) * 1e3 / reps
        nbytes = prob.spmv_algorithmic_bytes(False)
        res["spmv"][r] = {"bytes": nbytes, "us": us, "GB/s": nbytes / (us * 1e-6) / 1e9}
        prob.close()
        print(f"r={r}: RTR {res['rtr'][r]:.1f} it/s; SpMV {nbytes} B in {us:.2f} us = {res['spmv'][r]['GB/s']:.0f} GB/s",
              flush=True)
    side = torch.cuda.Stream()
    for r in (5, 8):
        with torch.cuda.stream(side):
            run = DistributedPGO(edges, n, 16, r=r, schedule="coloured", concurrent=True)
            for _ in range(20):
                run.step(evaluate=False)
            torch.cuda.synchronize()
            e0.record(side)
            for _ in range(args.rounds):
                run.step(evaluate=False)
            e1.record(side)
            torch.cuda.synchronize()
        res["rounds16"][r] = args.rounds / (e0.elapsed_time(e1) * 1e-3)
        print(f"16 agents side by side, r={r}: {res['rounds16'][r]:.0f} rounds/s", flush=True)
    print(json.dumps(res))
    if args.out:
        with open(args.out, "w") as fh:
            json.dump(res, fh, indent=1)


if __name__ == "__main__":
    main()
