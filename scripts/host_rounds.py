#!/usr/bin/env python
"""Rounds/s of DistributedPGO.step_host (every iterate crosses the host boundary each round) with all agents on one GPU."""
import argparse, json, os, sys, time
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch
from dpo_b200 import posegraph as pg
from dpo_b200.agent import DistributedPGO

ap = argparse.ArgumentParser()
ap.add_argument("--dataset", default="sphere2500")
ap.add_argument("--agents", type=int, default=16)
ap.add_argument("--rounds", type=int, default=100)
ap.add_argument("--concurrent", choices=("auto", "0", "1"), default="auto",
                help="launch mode: agents side by side (1), one after the other as full-grid kernels (0), or the runner's default")
args = ap.parse_args()
edges, n = pg.read_g2o_file(os.path.join(ROOT, "data", args.dataset + ".g2o"))
side = torch.cuda.Stream()
with torch.cuda.stream(side):
    run = DistributedPGO(edges, n, args.agents, r=5, schedule="coloured",
                         concurrent=None if args.concurrent == "auto" else args.concurrent == "1")
    for _ in range(6):
        run.step_host()
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(args.rounds):
        run.step_host()
    torch.cuda.synchronize()
    dt = time.perf_counter() - t0
    st = run.step(evaluate=True)
print(json.dumps({"dataset": args.dataset, "agents": args.agents, "concurrent": run.concurrent, "host_rounds_per_sec": args.rounds / dt,
                  "us_per_round": 1e6 * dt / args.rounds, "host_bytes_per_step": run.host_bytes_per_step(), "cost": st.cost}))
