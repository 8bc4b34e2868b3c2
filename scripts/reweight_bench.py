"""Cost of a robust weight update: the synchronous path (k_assemble_Q, host copy, host rebuild of the exact
preconditioner on its next use) against the stream-ordered one (k_assemble_Q and the device refactorisation,
nd_refactor.cu), and the wall time of the reference's single-agent GNC loop with either.

    python scripts/reweight_bench.py [--datasets sphere2500,torus3D,grid3D] [--runs 3] [--updates 10]

Prints one JSON line per workload.  Times per update run from the weight change to a preconditioner that is ready for
the next step: a host clock around setEdgeWeights + the rebuild it triggers (sync), CUDA events around
setEdgeWeightsAsync on the handle's stream (async); the two alternate.  The algorithmic work of one refactorisation
(refactor_work) follows from the macro-node sizes alone.
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

PIVOT_BLOCK = 32          # nd::REFACTOR_PIVOT_BLOCK: pivots per Gauss-Jordan step


def refactor_work(own, bnd, dh):
    """(flops, bytes) one refactorisation needs, from the macro nodes' own / boundary pose counts.
    flops: the Gauss-Jordan sweep of every front over its own pivots, 2 s M^2 (s = dh own, M = dh (own + bnd)).
    bytes: every front written once by the assembly (M^2 doubles) and streamed once (read + write) per 32-pivot step,
    the child updates read by the parents (b^2 doubles), the panels written once (what the apply reads)."""
    s = dh * np.asarray(own, dtype=np.float64)
    b = dh * np.asarray(bnd, dtype=np.float64)
    M = s + b
    flops = float(np.sum(2.0 * s * M * M))
    steps = np.ceil(s / PIVOT_BLOCK)
    panels = np.ceil((own + bnd) / 2.0) * 8 * s + np.ceil(own / 2.0) * 8 * b
    byts = float(np.sum(8.0 * M * M + 16.0 * steps * M * M + 8.0 * b * b + 8.0 * panels))
    return flops, byts


def gpu_info():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        name, power, clock = [x.strip() for x in out.split(",")]
        return {"gpu": name, "power_limit": power, "max_sm_clock": clock}
    except Exception as e:                                   # the measurement itself still needs the GPU
        return {"gpu": "unknown", "error": str(e)}


def setup(ds, seed=3):
    from dpo_b200 import posegraph as pg
    edges, n = pg.read_g2o_file(os.path.join(ROOT, "data", ds + ".g2o"))
    fixed = np.zeros(len(edges), dtype=np.int32)
    seen = set()
    for e in range(len(edges)):
        if edges.p2[e] == edges.p1[e] + 1 and int(edges.p1[e]) not in seen:
            seen.add(int(edges.p1[e]))
            fixed[e] = 1
    # a seeded 10 % of the loop closures replaced with random relative poses
    rng = np.random.default_rng(seed)
    lc = np.flatnonzero(fixed == 0)
    bad = rng.choice(lc, size=max(1, len(lc) // 10), replace=False)
    d = edges.d
    Rr = np.linalg.qr(rng.standard_normal((len(bad), d, d)))[0]
    Rr[np.linalg.det(Rr) < 0, :, 0] *= -1
    edges.R[bad] = Rr
    edges.t[bad] = rng.uniform(-10.0, 10.0, (len(bad), d))
    odo = edges.take(np.flatnonzero(fixed))
    odo = odo.take(np.argsort(odo.p1))
    r = 5 if d == 3 else 3
    X0 = pg.fixedStiefelVariable(d, r) @ pg.odometryInitialization(d, n, odo)
    return edges, n, fixed, X0, r


def problem(edges, n, fixed, r):
    import dpo_b200 as dp
    gp = dp.QuadraticProblem(n, edges.d, r)
    gp.setEdges(edges, fixed=fixed)
    return gp


def gnc_wall(gp, X0, use_async, updates):
    import dpo_b200 as dp
    opt = dp.QuadraticOptimizer(gp)
    opt.setTrustRegionTolerance(1e-2)
    opt.setTrustRegionIterations(1)
    opt.setTrustRegionMaxInnerIterations(10)
    opt.setTrustRegionInitialRadius(100)
    gp.upload_X(X0)
    mu = 1e-4
    t0 = time.perf_counter()
    for _ in range(updates):
        for _ in range(30):
            opt.optimize_resident_async()
        if use_async:
            gp.robustReweightAsync("GNC_TLS", mu, 10.0)
        else:
            gp.robustReweight("GNC_TLS", mu, 10.0)
        mu *= 1.4
    gp.sync()
    return time.perf_counter() - t0


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--datasets", default="sphere2500,torus3D,grid3D")
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--updates", type=int, default=10)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("reweight_bench needs a CUDA device")
    info = gpu_info()
    for ds in args.datasets.split(","):
        edges, n, fixed, X0, r = setup(ds)
        m = len(edges)
        sp_, ap_ = problem(edges, n, fixed, r), problem(edges, n, fixed, r)
        own, bnd, _ = ap_.nd_node_sizes()
        flops, byts = refactor_work(own, bnd, edges.d + 1)
        rng = np.random.default_rng(1)
        ws = [rng.uniform(0.0, 1.0, m) for _ in range(args.runs + 1)]
        s = torch.cuda.Stream()
        ap_.set_stream(s.cuda_stream)
        ap_.setEdgeWeightsAsync(torch.tensor(ws[-1], device="cuda"))       # builds the structure (synchronises)
        ap_.sync()
        sp_.setEdgeWeights(ws[-1])
        sp_.nd_info()
        t_sync, t_async = [], []
        for k in range(args.runs):
            t0 = time.perf_counter()
            sp_.setEdgeWeights(ws[k])
            sp_.nd_info()                                                  # the host rebuild the next step would trigger
            t_sync.append(1e3 * (time.perf_counter() - t0))
            wt = torch.tensor(ws[k], device="cuda")
            torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record(s)
            ap_.setEdgeWeightsAsync(wt)
            e1.record(s)
            e1.synchronize()
            t_async.append(e0.elapsed_time(e1))
        ap_.set_stream(None)
        gnc = {}
        for use_async in (False, True, False, True):
            key = "async" if use_async else "sync"
            gnc.setdefault(key, []).append(gnc_wall(problem(edges, n, fixed, r), X0, use_async, args.updates))
        best = min(t_async) * 1e-3
        rec = dict(info, workload=ds, poses=n, edges=m, macro_nodes=int(len(own)),
                   update_ms_sync=[round(x, 3) for x in t_sync], update_ms_async=[round(x, 3) for x in t_async],
                   gnc_updates=args.updates, gnc_steps_per_update=30,
                   gnc_wall_s_sync=[round(x, 3) for x in gnc["sync"]], gnc_wall_s_async=[round(x, 3) for x in gnc["async"]],
                   refactor_gflop=round(flops / 1e9, 3), refactor_gbytes=round(byts / 1e9, 3),
                   refactor_gflops_per_s=round(flops / best / 1e9, 1), refactor_gbytes_per_s=round(byts / best / 1e9, 1))
        print(json.dumps(rec), flush=True)


if __name__ == "__main__":
    main()
