#!/usr/bin/env python
"""Cost of checking convergence on the device runner, and what it buys: DistributedPGO.solve against the hand-written
step() loop of scripts/bench_configs.py.  One GPU, one process; the variants alternate and each is repeated twice.

    python scripts/solve_bench.py [--reps 50] [--out result.json]

Per workload (sphere2500 / 16 agents coloured side by side, torus3D / 8 agents coloured, sphere2500 / 5 agents greedy):
  eval_us      one evaluated round's check, host clock over --reps calls, each ending in a device synchronise:
               "batched" = DistributedPGO.status() (exchange + one dpgo_agents_status_async + copy + synchronise),
               "per_agent" = the same exchange (or G rebuild, when the gathered tiles are current) + every agent's
               problem_stats() (one OP_EVAL launch and one synchronising fetch per agent)
  solve        rounds to |g| < 0.1 and wall time of solve(check_every = c) and of the step() loop evaluating every c-th round
Prints ONE JSON line with the GPU's name, power limit and maximum SM clock, and the registers / spills ptxas reported for
the status kernel's instantiations (dpo_b200/lib/obj/dpgo_status.cu.ptxas.log, written by the build).
"""
from __future__ import annotations

import argparse
import json
import os
import re
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

WORKLOADS = [("sphere2500", 16, "coloured"), ("torus3D", 8, "coloured"), ("sphere2500", 5, "greedy")]


def device_info():
    q = "name,power.limit,clocks.max.sm"
    try:
        out = subprocess.run(["nvidia-smi", "--id=0", f"--query-gpu={q}", "--format=csv,noheader,nounits"],
                             capture_output=True, text=True, timeout=30).stdout.strip().split(",")
        return {"name": out[0].strip(), "power_limit_w": float(out[1]), "sm_max_mhz": float(out[2])}
    except Exception:
        return {"name": None, "power_limit_w": None, "sm_max_mhz": None}


def status_kernel_registers():
    log = os.path.join(ROOT, "dpo_b200", "lib", "obj", "dpgo_status.cu.ptxas.log")
    if not os.path.exists(log):
        return None
    out, name = {}, None
    for line in open(log):
        m = re.search(r"Compiling entry function '\S*?(k_agents_status|k_trajectory_global)ILi(\d)ELi(\d)E", line)
        if m:
            name = f"{m.group(1)}<{m.group(2)},{m.group(3)}>"
            continue
        if name:
            m = re.search(r"(\d+) bytes spill stores", line)
            if m:
                out.setdefault(name, {})["spill_stores"] = int(m.group(1))
            m = re.search(r"Used (\d+) registers", line)
            if m:
                out.setdefault(name, {})["registers"] = int(m.group(1))
                name = None
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=50)
    ap.add_argument("--max-rounds", type=int, default=500)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("solve_bench.py measures the GPU: no CUDA device")
    from dpo_b200 import posegraph as pg
    from dpo_b200.agent import DistributedPGO
    result = {"gpu": device_info(), "status_kernel": status_kernel_registers(), "workloads": []}
    stream = torch.cuda.Stream()          # a side stream: repeated concurrent rounds are replayed as CUDA graphs
    with torch.cuda.stream(stream):
        for ds, k, schedule in WORKLOADS:
            edges, n = pg.read_g2o_file(os.path.join(ROOT, "data", ds + ".g2o"))
            make = lambda: DistributedPGO(edges, n, k, r=5, schedule=schedule)     # noqa: E731
            run = make()
            for _ in range(5):
                run.step(evaluate=False)
            run.status()
            run._refresh_G()
            for a in run.local_ids:
                run.agents[a].opt.problem_stats()
            ev = {"batched": [], "per_agent": []}
            for _ in range(2):
                for variant in ("batched", "per_agent"):
                    torch.cuda.synchronize()
                    t0 = time.perf_counter()
                    for _ in range(args.reps):
                        if variant == "batched":
                            run.status()
                        else:                            # the same exchange work as status()
                            run._refresh_G()
                            for a in run.local_ids:
                                run.agents[a].opt.problem_stats()
                    ev[variant].append(round((time.perf_counter() - t0) / args.reps * 1e6, 1))
            rec = {"dataset": ds, "agents": k, "schedule": schedule, "concurrent": run.concurrent, "eval_us": ev,
                   "solve": []}
            del run
            for every in ((1,) if schedule == "greedy" else (1, 5)):
                row = {"check_every": every, "solve": [], "step_loop": []}
                for _ in range(2):
                    for variant in ("solve", "step_loop"):
                        r = make()
                        torch.cuda.synchronize()
                        t0 = time.perf_counter()
                        if variant == "solve":
                            rep = r.solve(max_rounds=args.max_rounds, gradnorm_tol=0.1, rel_change_tol=0, check_every=every)
                            rounds, cost = rep.rounds, rep.cost
                        else:
                            rounds, cost = None, None
                            for it in range(1, args.max_rounds + 1):
                                st = r.step(evaluate=(it % every == 0))
                                if st is not None and st.gradnorm < 0.1:
                                    break
                            rounds, cost = it, (st.cost if st is not None else None)
                        torch.cuda.synchronize()
                        row[variant].append({"rounds": rounds, "wall_s": round(time.perf_counter() - t0, 4), "cost": cost})
                        del r
                rec["solve"].append(row)
            result["workloads"].append(rec)
            print(json.dumps(rec), file=sys.stderr)
    line = json.dumps(result)
    print(line)
    if args.out:
        with open(args.out, "w") as fh:
            fh.write(line + "\n")


if __name__ == "__main__":
    main()
