#!/usr/bin/env python
"""Experiment: the RTR steps of one colour class of small agents on ONE GPU, (a) one after the other as full-grid
cooperative kernels on one stream, (b) concurrently on per-agent streams.  When the runner steps a colour class side by
side, the agents run as single thread-block clusters (non-cooperative launches that can share the GPU)."""
import argparse, json, os, sys, time
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import numpy as np
import torch
import dpo_b200 as dp
from dpo_b200 import posegraph as pg
from dpo_b200.agent import DistributedPGO

ap = argparse.ArgumentParser()
ap.add_argument("--dataset", default="sphere2500")
ap.add_argument("--agents", type=int, default=16)
ap.add_argument("--rounds", type=int, default=40)
args = ap.parse_args()
edges, n = pg.read_g2o_file(os.path.join(ROOT, "data", args.dataset + ".g2o"))
run = DistributedPGO(edges, n, args.agents, r=5, schedule="coloured")
for _ in range(4):
    run.step(evaluate=False)
torch.cuda.synchronize()
out = {"dataset": args.dataset, "agents": args.agents, "colours": run.ncolours, "nd": run.agents[0].mProblem.nd_info()}
main = torch.cuda.current_stream().cuda_stream
for mode in ("one_stream", "own_streams"):
    for a in run.local_ids:
        run.agents[a].mProblem.set_stream(main if mode == "one_stream" else None)
    def rounds(cnt):
        for i in range(cnt):
            act = [a for a in range(run.k) if run.colour[a] == i % run.ncolours]
            for a in act:
                run.agents[a].opt.optimize_resident_async()
            for a in act:
                run.agents[a].mProblem.sync()
    rounds(4)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    rounds(args.rounds)
    torch.cuda.synchronize()
    out[mode + "_us_per_round"] = 1e6 * (time.perf_counter() - t0) / args.rounds
print(json.dumps(out))
