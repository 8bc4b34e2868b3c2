#!/usr/bin/env python
"""The greedy_set schedule against coloured and greedy rounds on the device runner: rounds, agent-steps and wall time to
|g| < 0.1, and the round rate.  One GPU, one process; the schedules alternate and each is run twice.

    python scripts/greedy_set_bench.py [--rounds 200] [--out result.json]
    python scripts/greedy_set_bench.py --oracle        # the same round counts from the CPU restatement (no GPU)

Workloads (r = 5, exact preconditioner): sphere2500 / 16 agents, torus3D / 8 agents, parking-garage / 4 agents (complete
agent graph), torus3D / 5 agents owned by tests/golden/partition5_strong_torus3D.txt (an irregular agent graph).
  to_tol        solve(gradnorm_tol=0.1, rel_change_tol=0): check_every=5 for coloured and greedy_set, 1 for greedy (it selects
                from every round's status); rounds, agent-steps (agents stepped, summed over the rounds) and wall time
  rounds_per_s  step(evaluate=False) rounds per second over --rounds rounds, host clock ending in a device synchronise;
                greedy has no such loop (it needs every round's status), so its rate is that of step(evaluate=True)
Prints ONE JSON line with the GPU's name, power limit and maximum SM clock, read in the same run.
"""
from __future__ import annotations

import argparse
import json
import math
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

WORKLOADS = [("sphere2500", 16, None), ("torus3D", 8, None), ("parking-garage", 4, None),
             ("torus3D", 5, "partition5_strong_torus3D.txt")]
SCHEDULES = ("coloured", "greedy_set", "greedy")
CAP = 5000


def device_info():
    q = "name,power.limit,clocks.max.sm"
    try:
        out = subprocess.run(["nvidia-smi", "--id=0", f"--query-gpu={q}", "--format=csv,noheader,nounits"],
                             capture_output=True, text=True, timeout=30).stdout.strip().split(",")
        return {"name": out[0].strip(), "power_limit_w": float(out[1]), "sm_max_mhz": float(out[2])}
    except Exception:
        return {"name": None, "power_limit_w": None, "sm_max_mhz": None}


def owner_of(part):
    return None if part is None else np.loadtxt(os.path.join(ROOT, "tests", "golden", part), dtype=np.int64)


def label(ds, k, part):
    return f"{ds}x{k}" + ("" if part is None else f"_{part[:-4]}")


def agent_steps(run, schedule, rounds):
    if schedule == "greedy":
        return rounds
    if schedule == "greedy_set":
        return sum(len(s) for s in run.selection_log())
    size = np.bincount(run.colour, minlength=run.ncolours)
    return int(sum(size[i % run.ncolours] for i in range(rounds)))


def make(edges, n, k, owner, schedule):
    from dpo_b200.agent import DistributedPGO
    return DistributedPGO(edges, n, k, r=5, schedule=schedule, owner=owner)


def to_tol(torch, edges, n, k, owner, schedule):
    run = make(edges, n, k, owner, schedule)
    run.status()
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    rep = run.solve(max_rounds=CAP, gradnorm_tol=0.1, rel_change_tol=0.0, check_every=1 if schedule == "greedy" else 5)
    torch.cuda.synchronize()
    wall = time.perf_counter() - t0
    return {"rounds": rep.rounds, "agent_steps": agent_steps(run, schedule, rep.rounds), "wall_s": round(wall, 4),
            "reason": rep.reason, "cost": round(rep.cost, 4)}


def rate(torch, edges, n, k, owner, schedule, rounds):
    run = make(edges, n, k, owner, schedule)
    evaluate = schedule == "greedy"
    for _ in range(10):                           # warm-up: first launches, graph capture
        run.step(evaluate=evaluate)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(rounds):
        run.step(evaluate=evaluate)
    torch.cuda.synchronize()
    return round(rounds / (time.perf_counter() - t0), 1)


def oracle_counts():
    """Rounds and agent-steps to |g| < 0.1 of the CPU restatement, |g| after every round; "rounds_check5" is the first
    multiple of 5 at or after it (what solve(check_every=5) reports)."""
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    import greedy_set_oracle as gso
    from oracle import dpgo_oracle as orc
    res = {}
    for ds, k, part in WORKLOADS:
        meas, n = orc.read_g2o(os.path.join(ROOT, "data", ds + ".g2o"))
        owner = owner_of(part)
        w = {}
        for schedule in SCHEDULES:
            t0 = time.perf_counter()
            drv = gso.GreedySetDriver(meas, n, k, r=5, owner=owner) if schedule == "greedy_set" else \
                orc.MultiRobotDriver(meas, n, k, r=5, owner=owner, schedule=schedule)
            steps, rounds = 0, None
            for i in range(CAP):
                before = len(drv.sets) if schedule == "greedy_set" else None
                _, gn = drv.step()
                if schedule == "greedy_set":
                    steps += len(drv.sets[before])
                elif schedule == "greedy":
                    steps += 1
                else:
                    steps += sum(1 for c in drv.colour if c == i % drv.ncolours)
                if gn < 0.1:
                    rounds = i + 1
                    break
            w[schedule] = {"rounds": rounds, "agent_steps": steps,
                           "rounds_check5": None if rounds is None or schedule == "greedy" else 5 * math.ceil(rounds / 5),
                           "cpu_s": round(time.perf_counter() - t0, 1)}
            print(label(ds, k, part), schedule, w[schedule], file=sys.stderr, flush=True)
        res[label(ds, k, part)] = w
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=200)
    ap.add_argument("--out", default=None)
    ap.add_argument("--oracle", action="store_true", help="the CPU restatement's round counts instead (no GPU)")
    args = ap.parse_args()
    if args.oracle:
        res = {"oracle": oracle_counts()}
    else:
        import torch
        from dpo_b200 import posegraph as pg
        if not torch.cuda.is_available():
            raise SystemExit("greedy_set_bench.py measures on a CUDA device; none is available (--oracle runs on the CPU)")
        res = {"device": device_info(), "rounds": args.rounds, "workloads": {}}
        with torch.cuda.stream(torch.cuda.Stream()):     # a capturable stream: repeated rounds replay as CUDA graphs
            for ds, k, part in WORKLOADS:
                edges, n = pg.read_g2o_file(os.path.join(ROOT, "data", ds + ".g2o"))
                owner = owner_of(part)
                w = {"to_tol": {s: [] for s in SCHEDULES}, "rounds_per_s": {s: [] for s in SCHEDULES}}
                for _ in range(2):
                    for s in SCHEDULES:
                        w["to_tol"][s].append(to_tol(torch, edges, n, k, owner, s))
                for _ in range(2):
                    for s in SCHEDULES:
                        w["rounds_per_s"][s].append(rate(torch, edges, n, k, owner, s, args.rounds))
                res["workloads"][label(ds, k, part)] = w
    line = json.dumps(res)
    print(line)
    if args.out:
        with open(args.out, "w") as fh:
            fh.write(line + "\n")


if __name__ == "__main__":
    main()
