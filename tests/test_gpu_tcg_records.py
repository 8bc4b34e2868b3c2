"""Bit-exact record of the RTR step with the sparse exact preconditioner (nested-dissection block solve).  Every scalar
reduction of k_optimize has a fixed order, so a change that only reorders or fuses the phases of the tCG loop and the
block solve must reproduce the result records and iterates exactly.  tests/golden/tcg_records.json holds six RTR steps
(updateX constants) of each workload in both launch modes.  The workloads are sphere2500 (3-level plan), smallGrid3D,
and agent 0 of a 16-agent sphere2500 split (1-level plan).  The records were made on an H100 SXM, whose cooperative grid
has 132 CTAs, with

    python tests/test_gpu_tcg_records.py --record

A GPU with another SM count has another grid and other reduction trees, so grid mode is skipped there."""
import hashlib
import json
import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)
GOLDEN = os.path.join(ROOT, "tests", "golden", "tcg_records.json")

# (dataset, agents): agents > 1 = the private sub-graph of agent 0 of a contiguous split
WORKLOADS = [("sphere2500", 1), ("smallGrid3D", 1), ("sphere2500", 16)]
MODES = ["grid", "cluster"]
RECORDED_GRID = 132
STEPS = 6
RANK = 5
FIELDS = ["success", "tcg_status", "tcg_iterations", "outer_iterations", "rejections", "spmv_passes", "precond_applies",
          "f_init", "gradnorm_init", "f_opt", "gradnorm_opt", "relative_change", "quad_init", "lin_init"]
TCG_LCON, TCG_SCON = 2, 3


def run_case(dataset, agents, mode, check_grid=False):
    import dpo_b200 as dp
    from dpo_b200 import posegraph as pg
    edges, n = pg.read_g2o_file(os.path.join(ROOT, "data", dataset + ".g2o"))
    d = edges.d
    X0 = pg.fixedStiefelVariable(d, RANK) @ pg.chordalInitialization(d, n, edges)
    if agents > 1:
        from dpo_b200.agent import contiguous_owner, partition_edges
        from dpo_b200.posegraph import EdgeSet
        parts, counts, _ = partition_edges(edges, contiguous_owner(n, agents), agents)
        edges = EdgeSet.join([parts[0][0], parts[0][1]])
        n = int(counts[0])
        X0 = X0[:, :(d + 1) * n]
    prob = dp.QuadraticProblem(n, d, RANK, preconditioners=(dp.PRECOND_BLOCK_JACOBI, dp.PRECOND_SPARSE_EXACT),
                               cluster=(mode == "cluster"))
    try:
        prob.setQ_blocks(*pg.connection_laplacian_blocks(edges))           # sizes the grid
        if check_grid and mode == "grid" and prob.launch_info()[0] != RECORDED_GRID:
            pytest.skip(f"records made with a {RECORDED_GRID}-CTA grid, this GPU runs {prob.launch_info()[0]}")
        opt = dp.QuadraticOptimizer(prob)
        opt.setTrustRegionTolerance(1e-2)
        opt.setTrustRegionIterations(1)
        opt.setTrustRegionMaxInnerIterations(10)
        opt.setTrustRegionInitialRadius(100)
        opt.setPreconditioner(dp.PRECOND_SPARSE_EXACT)
        X = np.asfortranarray(X0)
        records = []
        for _ in range(STEPS):
            X = np.asfortranarray(opt.optimize(X))
            r = opt.getOptResult()
            records.append({k: (float(getattr(r, k)).hex() if isinstance(getattr(r, k), float) else int(getattr(r, k)))
                            for k in FIELDS})
        return {"records": records, "X_sha256": hashlib.sha256(np.ascontiguousarray(X, dtype=np.float64).tobytes()).hexdigest(),
                "nd_phases": prob.nd_info()["phases"], "cluster": prob.launch_info()[1]}
    finally:
        prob.close()


def case_id(dataset, agents, mode):
    return f"{dataset}/{agents}/{mode}"


@pytest.mark.gpu
@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("dataset,agents", WORKLOADS)
def test_rtr_records_bit_identical(dataset, agents, mode):
    with open(GOLDEN) as fh:
        want = json.load(fh)[case_id(dataset, agents, mode)]
    got = run_case(dataset, agents, mode, check_grid=True)
    assert got["cluster"] == (mode == "cluster")
    assert got["nd_phases"] == want["nd_phases"]
    for step, (g, w) in enumerate(zip(got["records"], want["records"])):
        assert g == w, (step, g, w)
        if g["tcg_status"] in (TCG_LCON, TCG_SCON):
            # z0 = M^-1 g plus one application per tCG iteration that did not stop
            assert g["precond_applies"] == g["tcg_iterations"], (step, g)
    assert got["X_sha256"] == want["X_sha256"]


def test_records_cover_both_plan_depths():
    """The records exercise a multi-phase block solve (sphere2500: 3 levels, 5 phases) and a one-phase one (the
    16-agent split's agent), and residual stops (LCON / SCON) as well as the iteration cap."""
    with open(GOLDEN) as fh:
        g = json.load(fh)
    assert set(g) == {case_id(ds, a, m) for ds, a in WORKLOADS for m in MODES}
    for mode in MODES:
        assert g[case_id("sphere2500", 1, mode)]["nd_phases"] == 5
        assert g[case_id("sphere2500", 16, mode)]["nd_phases"] == 1
    statuses = {r["tcg_status"] for v in g.values() for r in v["records"]}
    assert {TCG_LCON, TCG_SCON} & statuses and 4 in statuses


if __name__ == "__main__" and "--record" in sys.argv:
    out = {case_id(ds, a, m): run_case(ds, a, m) for ds, a in WORKLOADS for m in MODES}
    path = sys.argv[sys.argv.index("--record") + 1] if len(sys.argv) > sys.argv.index("--record") + 1 else GOLDEN
    os.makedirs(os.path.dirname(path), exist_ok=True)
    with open(path, "w") as fh:
        json.dump(out, fh, indent=1, sort_keys=True)
    print(json.dumps({k: (v["nd_phases"], [r["tcg_iterations"] for r in v["records"]]) for k, v in out.items()}))
