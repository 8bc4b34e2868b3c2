"""Relaxation ranks compiled since r = 5 was the largest -- r = 4 in SE(2), r = 6..8 in both dimensions -- on the GPU:
every single-operation entry point and RTR sequences in both launch modes against the oracle, and the device runners
(Python and C++) at r = 8.  Tolerances are those of the r <= 5 tests (tests/test_gpu_ops.py, tests/test_gpu_optimize.py,
tests/test_gpu_agents.py, tests/test_gpu_solve.py)."""
import contextlib
import os
import subprocess
import sys

import numpy as np
import pytest

from oracle import dpgo_oracle as orc

import greedy_set_oracle as gso  # noqa: E402
import solve_oracle as so  # noqa: E402

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NEW = [("CSAIL", 4), ("CSAIL", 6), ("CSAIL", 7), ("CSAIL", 8), ("smallGrid3D", 6), ("smallGrid3D", 7), ("smallGrid3D", 8)]


def relerr(a, b):
    return float(np.linalg.norm(np.asarray(a) - np.asarray(b)) / max(np.linalg.norm(b), 1e-300))


def load(ds, data_dir):
    from dpo_b200 import posegraph as pg
    return pg.read_g2o_file(os.path.join(data_dir, ds + ".g2o"))


def side_stream(on):
    import torch
    return torch.cuda.stream(torch.cuda.Stream()) if on else contextlib.nullcontext()


def problem(ds, r, data_dir, cluster=False, seed=0):
    import dpo_b200 as dp
    meas, n = orc.read_g2o(os.path.join(data_dir, ds + ".g2o"))
    d = meas.d
    Q = orc.construct_connection_laplacian(meas, n)
    rng = np.random.default_rng(seed)
    X = orc.manifold_project(rng.standard_normal((r, (d + 1) * n)), d)
    G = 0.5 * rng.standard_normal((r, (d + 1) * n))
    op = orc.QuadraticProblem(n, d, r)
    op.set_Q(Q)
    op.set_G(G)
    gp = dp.QuadraticProblem(n, d, r, cluster=cluster,
                             preconditioners=(dp.PRECOND_BLOCK_JACOBI, dp.PRECOND_SPARSE_EXACT, dp.PRECOND_DENSE_EXACT))
    gp.setQ(Q)
    gp.setG(G)
    return op, gp, X, rng


# ---- single-agent primitives ------------------------------------------------------------------------------------------
@pytest.mark.parametrize("ds,r", NEW)
def test_primitives(ds, r, data_dir):
    import dpo_b200 as dp
    op, gp, X, rng = problem(ds, r, data_dir)
    d = op.d
    assert abs(gp.f(X) - op.f(X)) <= 1e-12 * max(1.0, abs(op.f(X)))
    assert relerr(gp.EucGrad(X), op.euc_grad(X)) <= 1e-13
    rg = op.rie_grad(X)
    assert relerr(gp.RieGrad(X), rg) <= 1e-13
    V = rng.standard_normal(X.shape)
    assert relerr(gp.EucHessianEta(V), op.euc_hess(V)) <= 1e-13
    Vt = orc.tangent_project(X, V, d)
    assert relerr(gp.RieHessianEta(X, Vt), op.rie_hess(X, op.euc_grad(X), Vt)) <= 1e-12
    # preconditioners
    exact = op.precondition(X, V)
    assert relerr(gp.PreConditioner(X, V, dp.PRECOND_SPARSE_EXACT), exact) <= 1e-11
    assert relerr(gp.PreConditioner(X, V, dp.PRECOND_DENSE_EXACT), exact) <= 1e-9       # one macro level, as r <= 5
    oo = orc.QuadraticOptimizer(op, precond="jacobi")
    assert relerr(gp.PreConditioner(X, V, dp.PRECOND_BLOCK_JACOBI), oo._apply_precond(X, V)) <= 1e-12
    assert relerr(gp.PreConditioner(X, V, dp.PRECOND_NONE), orc.tangent_project(X, V, d)) <= 1e-13
    # projection, retraction, Stiefel projection
    Z = rng.standard_normal(X.shape)
    assert relerr(gp.Projection(X, Z), orc.tangent_project(X, Z, d)) <= 1e-13
    eta = 0.3 * orc.tangent_project(X, Z, d)
    Xr = gp.Retraction(X, eta)
    assert relerr(Xr, orc.retract(X, eta, d)) <= 1e-13
    Yt = Xr.reshape(r, -1, d + 1)[:, :, :d]
    assert np.abs(np.einsum("ani,anj->nij", Yt, Yt) - np.eye(d)[None]).max() <= 1e-13
    M = rng.standard_normal(X.shape)
    assert relerr(gp.project(M), orc.manifold_project(M, d)) <= 1e-12


# ---- RTR sequences ----------------------------------------------------------------------------------------------------
def rtr_sequence(gp, X0, calls):
    import dpo_b200 as dp
    go = dp.QuadraticOptimizer(gp)
    go.setTrustRegionTolerance(1e-2)
    go.setTrustRegionIterations(1)
    go.setTrustRegionMaxInnerIterations(10)
    go.setTrustRegionInitialRadius(100)
    go.setPreconditioner(dp.PRECOND_SPARSE_EXACT)
    X, log = X0, []
    for _ in range(calls):
        X = go.optimize(X)
        res = go.getOptResult()
        log.append((res.success, res.tcg_iterations, res.tcg_status, res.f_init, res.f_opt, res.gradnorm_opt))
    return X, log


@pytest.mark.parametrize("cluster", [False, True])
@pytest.mark.parametrize("ds,r", [("sphere2500", r) for r in (6, 7, 8)] + [("CSAIL", r) for r in (4, 6, 7, 8)])
def test_rtr_sequence_matches_oracle_and_repeats_bitwise(ds, r, cluster, data_dir):
    """updateX constants (tol 1e-2, 1 outer, <= 10 inner, radius 100), exact preconditioner, four calls: the tCG counts and
    exits of the oracle, iterates within 1e-8; a second handle gives the same bits."""
    import dpo_b200 as dp
    meas, n = orc.read_g2o(os.path.join(data_dir, ds + ".g2o"))
    d = meas.d
    Q = orc.construct_connection_laplacian(meas, n)
    X0 = orc.fixed_stiefel_variable(d, r) @ orc.chordal_initialization(meas, n)
    op = orc.QuadraticProblem(n, d, r)
    op.set_Q(Q)
    runs = []
    for _ in range(2):
        gp = dp.QuadraticProblem(n, d, r, cluster=cluster)
        gp.setQ(Q)
        assert gp.launch_info()[1] == cluster
        runs.append(rtr_sequence(gp, X0, 4))
        gp.close()
    Xo = X0
    for it, rec in enumerate(runs[0][1]):
        oo = orc.QuadraticOptimizer(op, precond="exact")
        oo.tr_tolerance, oo.tr_iterations, oo.tr_max_inner, oo.tr_initial_radius = 1e-2, 1, 10, 100.0
        Xo = oo.optimize(Xo)
        assert rec[0] == 1
        assert (rec[1], rec[2]) == (oo.result.tcg_iterations, oo.result.tcg_status), (it, rec, oo.result)
        assert abs(rec[3] - oo.result.fInit) <= 1e-9 * abs(oo.result.fInit)
        assert abs(rec[4] - oo.result.fOpt) <= 1e-9 * abs(oo.result.fOpt)
    assert relerr(runs[0][0], Xo) <= 1e-8
    assert runs[0][1] == runs[1][1] and np.array_equal(runs[0][0], runs[1][0])


# ---- device runners at r = 8 --------------------------------------------------------------------------------------------
@pytest.mark.parametrize("ds,k,rounds,conc,r", [("sphere2500", 16, 8, True, 8), ("sphere2500", 16, 8, False, 8),
                                                ("torus3D", 8, 10, False, 8), ("torus3D", 8, 10, True, 8),
                                                ("input_INTEL_g2o", 5, 10, False, 4), ("input_M3500_g2o", 5, 10, True, 4)])
def test_coloured_rounds_match_oracle(ds, k, rounds, conc, r, data_dir):
    """k agents, coloured RBCD, exact preconditioner: per-round 2f and |g| and the final iterate against the oracle's
    coloured driver.  conc: the agents of a colour class side by side as thread-block clusters on a side stream (the
    repeated rounds replay a CUDA graph), else one after the other as full-grid launches."""
    from dpo_b200.agent import DistributedPGO
    edges, n = load(ds, data_dir)
    meas, _ = orc.read_g2o(os.path.join(data_dir, ds + ".g2o"))
    with side_stream(conc):
        run = DistributedPGO(edges, n, k, r=r, schedule="coloured", concurrent=conc)
        assert run.agents[0].mProblem.launch_info()[1] == conc
        drv = orc.MultiRobotDriver(meas, n, k, r=r, schedule="coloured")
        assert run.colour == drv.colour
        for _ in range(rounds):
            st = run.step()
            cost, gn = drv.step()
            assert abs(st.cost - cost) <= 1e-8 * abs(cost)
            assert abs(st.gradnorm - gn) <= 1e-7 * gn
        Xg, Xo = run.assemble(), drv.assemble()
    assert np.linalg.norm(Xg - Xo) <= 1e-8 * np.linalg.norm(Xo)


@pytest.mark.parametrize("ds,k,r5_cost", [("torus3D", 8, 24227.0479)])
def test_accelerated_solve_at_rank_8(ds, k, r5_cost, data_dir):
    """solve() with colour momentum to the gradient-norm rule: it stops on that rule, at the cost the r = 5 run stops at
    (the relaxation is tight on torus3D, so both reach the same optimum), and twice the same run gives the same bits."""
    from dpo_b200.agent import DistributedPGO
    edges, n = load(ds, data_dir)
    reps = []
    with side_stream(True):
        for _ in range(2):
            run = DistributedPGO(edges, n, k, r=8, schedule="coloured", acceleration=True, momentum_blocks="colours")
            reps.append((run.solve(gradnorm_tol=0.1, rel_change_tol=0, check_every=1), run.assemble()))
    rep = reps[0][0]
    assert rep.reason == "gradnorm" and rep.gradnorm < 0.1
    assert abs(rep.cost - r5_cost) <= 1e-5 * r5_cost
    assert (reps[1][0].rounds, reps[1][0].cost) == (rep.rounds, rep.cost) and np.array_equal(reps[0][1], reps[1][1])


def test_greedy_set_at_rank_8(data_dir):
    """30 greedy independent-set rounds of 16 sphere2500 agents against the restatement: the sets (rounds with a near tie
    in the selection norms left out), 2f and |g| to 1e-9."""
    from dpo_b200.agent import DistributedPGO
    from test_gpu_greedy_set import near_tie
    edges, n = load("sphere2500", data_dir)
    meas, _ = orc.read_g2o(os.path.join(data_dir, "sphere2500.g2o"))
    rounds = 30
    drv = gso.GreedySetDriver(meas, n, 16, r=8)
    for _ in range(rounds):
        drv.step()
    with side_stream(True):
        run = DistributedPGO(edges, n, 16, r=8, schedule="greedy_set", concurrent=True)
        tr = [run.step() for _ in range(rounds)]
    for i, st in enumerate(tr):
        if not near_tie(drv.norms2[i]):
            assert st.selected == drv.sets[i], (i, st.selected, drv.sets[i])
        assert abs(st.cost - drv.trace.cost[i]) <= 1e-9 * abs(drv.trace.cost[i]), i
        assert abs(st.gradnorm - drv.trace.gradnorm[i]) <= 1e-9 * drv.trace.gradnorm[i], i


@pytest.mark.parametrize("ds,k,r", [("sphere2500", 16, 8), ("input_INTEL_g2o", 5, 4)])
def test_trajectory_at_new_ranks(ds, k, r, data_dir):
    """trajectory() rounds to SE(d) on the device: the restatement's rounding of the same iterate, proper rotations."""
    from dpo_b200.agent import DistributedPGO
    edges, n = load(ds, data_dir)
    d, dh = edges.d, edges.d + 1
    run = DistributedPGO(edges, n, k, r=r, schedule="coloured")
    for _ in range(6):
        run.step(evaluate=False)
    T = run.trajectory()
    X = run.assemble()
    ref = so.trajectory_in_global_frame(X, X[:, :dh], d)
    assert np.abs(T - ref).max() <= 1e-12 * np.abs(ref[:, d::dh]).max()
    Rs = np.stack([T[:, i * dh:i * dh + d] for i in range(n)])
    assert np.abs(np.einsum("iba,ibc->iac", Rs, Rs) - np.eye(d)).max() <= 1e-12
    assert np.abs(np.linalg.det(Rs) - 1.0).max() <= 1e-12


def test_rank_9_is_refused_by_the_runners(data_dir):
    import dpo_b200 as dp
    from dpo_b200.agent import DistributedPGO
    edges, n = load("tinyGrid3D", data_dir)
    with pytest.raises(dp.DpgoError) as ei:
        DistributedPGO(edges, n, 2, r=9, schedule="coloured")
    assert ei.value.code == 5 and "<= 8" in str(ei.value)


# ---- the C++ runner ---------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def rank_check():
    from dpo_b200 import build
    return build.build_cpp_program([os.path.join(ROOT, "tests", "cpp", "rank_check.cpp")],
                                   os.path.join(ROOT, "build", "tests", "rank_check"))


def test_cpp_device_rbcd_at_rank_8(rank_check, tmp_path, data_dir):
    """DeviceRBCD (C++) at r = 8 against DistributedPGO (Python): status records and rounded trajectory to 1e-9 relative
    after 20 coloured rounds (the runners use different fixed lifts, which these quantities do not depend on); r = 9 is
    refused with the library's message."""
    from dpo_b200.agent import DistributedPGO
    ds, k, rounds = "torus3D", 8, 20
    res = subprocess.run([rank_check, os.path.join(data_dir, ds + ".g2o"), str(k), "coloured", "8", str(rounds), str(tmp_path)],
                         capture_output=True, text=True, timeout=600)
    assert res.returncode == 0, res.stderr[-2000:]
    edges, n = load(ds, data_dir)
    run = DistributedPGO(edges, n, k, r=8, schedule="coloured")
    rep = run.solve(max_rounds=rounds, gradnorm_tol=0, rel_change_tol=0)
    words = res.stdout.split()
    assert (int(words[words.index("rounds") + 1]), words[words.index("reason") + 1]) == (rep.rounds, rep.reason)
    rec_c, rec_p = np.loadtxt(os.path.join(str(tmp_path), "status.txt")), run.status().records
    scale = np.abs(rec_p[:, 0]) + np.abs(rec_p[:, 1])
    assert np.all(np.abs(rec_c[:, :2] - rec_p[:, :2]) <= 1e-9 * scale[:, None])
    assert np.all(np.abs(rec_c[:, 2:4] - rec_p[:, 2:4]) <= 1e-9 * rec_p[:, 2:4])
    assert np.array_equal(rec_c[:, 4], rec_p[:, 4])
    T_c, T_p = np.loadtxt(os.path.join(str(tmp_path), "trajectory.txt")), run.trajectory()
    d, dh = edges.d, edges.d + 1
    assert np.abs(T_c - T_p).max() <= 1e-9 * max(1.0, np.abs(T_p[:, d::dh]).max())
    bad = subprocess.run([rank_check, os.path.join(data_dir, "tinyGrid3D.g2o"), "2", "coloured", "9", "1", str(tmp_path)],
                         capture_output=True, text=True, timeout=600)
    assert bad.returncode == 3 and "<= 8" in bad.stderr, (bad.returncode, bad.stderr)


# ---- memcheck -----------------------------------------------------------------------------------------------------------
def test_memcheck_of_rank_8_steps():
    """compute-sanitizer memcheck over one r = 8 RTR step in each launch mode (tests/_rank_sanitizer_worker.py)."""
    import shutil
    tool = next((c for c in (shutil.which("compute-sanitizer"), "/usr/local/cuda/bin/compute-sanitizer") if c and os.path.exists(c)),
                None)
    if tool is None:
        pytest.skip("compute-sanitizer is not installed")
    worker = os.path.join(os.path.dirname(os.path.abspath(__file__)), "_rank_sanitizer_worker.py")
    res = subprocess.run([tool, "--tool", "memcheck", "--leak-check", "no", sys.executable, worker], capture_output=True,
                         text=True, timeout=900)
    out = res.stdout + res.stderr
    if "Device not supported" in out or "ERROR SUMMARY" not in out:
        pytest.skip("compute-sanitizer cannot check this device or could not start its target: " + out[:300])
    assert "ERROR SUMMARY: 0 errors" in out and res.returncode == 0, out[-3000:]
    assert "ok" in res.stdout
