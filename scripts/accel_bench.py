#!/usr/bin/env python
"""Accelerated coloured rounds on the device runner: what a round costs and what the momentum over colour classes buys.
One GPU, one process; the variants alternate and each is run twice.

    python scripts/accel_bench.py [--rounds 200] [--out result.json]

Per workload (sphere2500 / 16 agents, torus3D / 8 agents, coloured schedule, r = 5, exact preconditioner):
  rounds_per_s   step(evaluate=False) rounds per second, host clock over --rounds rounds ending in a device synchronise:
                 "plain_concurrent" (no acceleration, agents side by side), "accel_sequential" (momentum over agents,
                 full-grid steps one after the other), "accel_concurrent" (momentum over agents, side by side),
                 "accel_colours" (momentum over colour classes, side by side)
  to_tol         rounds and wall time to |g| < 0.1 (all side by side, a check after every 5th round): the step() loop with
                 status() for plain coloured rounds ("plain") and for momentum_blocks="colours" ("colours"), and
                 solve(check_every=5, rel_change_tol=0) for momentum_blocks="colours" ("colours_solve")
Prints ONE JSON line with the GPU's name, power limit and maximum SM clock, read in the same run.
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

WORKLOADS = [("sphere2500", 16), ("torus3D", 8)]
RATE_VARIANTS = {"plain_concurrent": dict(acceleration=False, concurrent=True),
                 "accel_sequential": dict(acceleration=True, concurrent=False),
                 "accel_concurrent": dict(acceleration=True, concurrent=True),
                 "accel_colours": dict(acceleration=True, momentum_blocks="colours", concurrent=True)}
COLOURS = dict(acceleration=True, momentum_blocks="colours")
TOL_VARIANTS = {"plain": (dict(acceleration=False), False), "colours": (COLOURS, False), "colours_solve": (COLOURS, True)}


def device_info():
    q = "name,power.limit,clocks.max.sm"
    try:
        out = subprocess.run(["nvidia-smi", "--id=0", f"--query-gpu={q}", "--format=csv,noheader,nounits"],
                             capture_output=True, text=True, timeout=30).stdout.strip().split(",")
        return {"name": out[0].strip(), "power_limit_w": float(out[1]), "sm_max_mhz": float(out[2])}
    except Exception:
        return {"name": None, "power_limit_w": None, "sm_max_mhz": None}


def make(edges, n, k, **kw):
    from dpo_b200.agent import DistributedPGO
    return DistributedPGO(edges, n, k, r=5, schedule="coloured", **kw)


def rate(torch, edges, n, k, rounds, kw):
    run = make(edges, n, k, **kw)
    for _ in range(10):                           # warm-up: first launches, graph capture of both colour classes
        run.step(evaluate=False)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(rounds):
        run.step(evaluate=False)
    torch.cuda.synchronize()
    return rounds / (time.perf_counter() - t0)


def to_tol(torch, edges, n, k, kw, use_solve, check_every=5, cap=1000):
    run = make(edges, n, k, **kw)
    run.status()
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    if use_solve:
        rep = run.solve(max_rounds=cap, gradnorm_tol=0.1, rel_change_tol=0, check_every=check_every)
        i, cost, gradnorm = rep.rounds, rep.cost, rep.gradnorm
    else:
        st = None
        for i in range(1, cap + 1):
            run.step(evaluate=False)
            if i % check_every == 0:
                st = run.status()
                if st.gradnorm < 0.1:
                    break
        cost, gradnorm = st.cost, st.gradnorm
    torch.cuda.synchronize()
    return {"rounds": i, "wall_s": time.perf_counter() - t0, "cost": cost, "gradnorm": gradnorm}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=200)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import torch
    from dpo_b200 import posegraph as pg
    if not torch.cuda.is_available():
        raise SystemExit("accel_bench.py measures on a CUDA device; none is available")
    res = {"device": device_info(), "rounds": args.rounds, "workloads": {}}
    with torch.cuda.stream(torch.cuda.Stream()):     # a capturable stream: repeated rounds replay as CUDA graphs
        for ds, k in WORKLOADS:
            edges, n = pg.read_g2o_file(os.path.join(ROOT, "data", ds + ".g2o"))
            w = {"rounds_per_s": {v: [] for v in RATE_VARIANTS}, "to_tol": {v: [] for v in TOL_VARIANTS}}
            for _ in range(2):
                for v, kw in RATE_VARIANTS.items():
                    w["rounds_per_s"][v].append(round(rate(torch, edges, n, k, args.rounds, kw), 1))
            for _ in range(2):
                for v, (kw, use_solve) in TOL_VARIANTS.items():
                    r = to_tol(torch, edges, n, k, kw, use_solve)
                    w["to_tol"][v].append({"rounds": r["rounds"], "wall_s": round(r["wall_s"], 4),
                                           "cost": round(r["cost"], 4), "gradnorm": round(r["gradnorm"], 5)})
            res["workloads"][f"{ds}x{k}"] = w
    line = json.dumps(res)
    print(line)
    if args.out:
        with open(args.out, "w") as fh:
            fh.write(line + "\n")


if __name__ == "__main__":
    main()
