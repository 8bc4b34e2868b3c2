"""Every trust-region decision of the RTR step kernel against the oracle, on the cases of rtr_cases.py: boundary and
negative-curvature exits, residual and iteration-cap stops, rejected and abandoned steps, radius growth, cap and shrink,
the tolerance stop and the early exit, with every preconditioner in both launch modes.  The decisions on each case's
path are clear of their thresholds (test_rtr_cases.py), so the kernel must take the oracle's path: the counters are
compared exactly, the iterate within the tolerances of test_rtr_single_step_sequence, and a step that returns its input
bit for bit.  Last, one batched round of three agents against the same steps run one by one."""
import ctypes as C

import numpy as np
import pytest

import rtr_cases as rc

pytestmark = pytest.mark.gpu

DR = [(d, r) for d in (2, 3) for r in rc.RANKS[d]]
MODES = [0, 1]                                   # dpgo_problem_set_launch_mode: cooperative grid, one cluster
ORACLE = {"none": "none", "jacobi": "jacobi", "sparse": "exact", "dense": "exact"}
BITWISE = ("giveup", "early_exit", "stationary")
RECORD = ("success", "tcg_status", "tcg_iterations", "outer_iterations", "rejections", "spmv_passes", "precond_applies",
          "f_init", "gradnorm_init", "f_opt", "gradnorm_opt", "relative_change", "quad_init", "lin_init")


def pid(name):
    import dpo_b200 as dp
    return {"none": dp.PRECOND_NONE, "jacobi": dp.PRECOND_BLOCK_JACOBI, "sparse": dp.PRECOND_SPARSE_EXACT,
            "dense": dp.PRECOND_DENSE_EXACT}[name]


def handle(c, mode, precs):
    import dpo_b200 as dp
    from dpo_b200 import _capi
    gp = dp.QuadraticProblem(c.n, c.d, c.r, preconditioners=precs)
    _capi.check(gp._lib.dpgo_problem_set_launch_mode(gp._h, mode))
    gp.setQ(c.Q)
    if c.G is not None:
        gp.setG(c.G)
    return gp


def optimizer(gp, c, precond):
    import dpo_b200 as dp
    go = dp.QuadraticOptimizer(gp)
    go.setTrustRegionTolerance(c.tol)
    go.setTrustRegionIterations(c.iters)
    go.setTrustRegionMaxInnerIterations(c.inner)
    go.setTrustRegionInitialRadius(c.radius)
    go.setPreconditioner(precond)
    return go


def relerr(a, b):
    return float(np.linalg.norm(np.asarray(a) - np.asarray(b)) / max(np.linalg.norm(b), 1e-300))


def check_step(c, Xg, res, what):
    o = c.result
    att = c.attempts()
    assert res.success == 1, what
    got = (res.tcg_status, res.tcg_iterations, res.outer_iterations, res.rejections)
    assert got == (o.tcg_status, o.tcg_iterations, o.outer_iterations, o.rejections), (what, res.as_dict(), o)
    # initial evaluation, one Hessian product per inner iteration, one candidate evaluation per attempt
    assert res.spmv_passes == 1 + res.tcg_iterations + res.outer_iterations, (what, res.as_dict())
    # z0 per attempt (a reused one included) plus one per inner iteration that did not stop the solve
    stopped = sum(a[0] != rc.MAXITER for a in att)
    assert res.precond_applies == res.outer_iterations + res.tcg_iterations - stopped, (what, res.as_dict())
    if c.name in BITWISE or c.name == "batch_giveup":
        assert np.array_equal(Xg, c.X), what
        assert res.f_opt == res.f_init and res.gradnorm_opt == res.gradnorm_init and res.relative_change == 0.0, what
        assert all(np.isfinite(getattr(res, k)) for k in RECORD), (what, res.as_dict())
        return
    xtol, ftol = rc.tolerances(c.precond)
    assert relerr(Xg, c.X_out) <= xtol, (what, relerr(Xg, c.X_out))
    assert abs(res.f_opt - o.fOpt) <= ftol * abs(o.fOpt), (what, res.f_opt, o.fOpt)
    # near a critical point the gradient is what CG's last residual left, rounding amplified by the solve included, so
    # the kernel's gradient norm is checked at its own iterate, which is checked against the oracle's above
    gn = rc.grad_norm(c, Xg)
    assert abs(res.gradnorm_opt - gn) <= 1e-9 * max(gn, 1e-3), (what, res.gradnorm_opt, gn, o.gradNormOpt)


@pytest.mark.parametrize("mode", MODES, ids=["grid", "cluster"])
@pytest.mark.parametrize("d,r", DR)
@pytest.mark.parametrize("name", rc.CASE_NAMES)
def test_rtr_branch(name, d, r, mode):
    import dpo_b200 as dp
    for precond in ("sparse", "dense", "jacobi", "none"):
        c = rc.case(name, d, r, ORACLE[precond])
        precs = (dp.PRECOND_BLOCK_JACOBI,) + ((pid(precond),) if precond in ("sparse", "dense") else ())
        gp = handle(c, mode, precs)
        try:
            go = optimizer(gp, c, pid(precond))
            Xg = np.array(go.optimize(c.X))
            check_step(c, Xg, go.getOptResult(), (name, d, r, mode, precond))
        finally:
            gp.close()


def tiles_of(X, poses, d):
    dh = d + 1
    return np.concatenate([np.asfortranarray(X[:, p * dh:(p + 1) * dh]).ravel(order="F") for p in poses])


@pytest.mark.parametrize("mode", MODES, ids=["grid", "cluster"])
@pytest.mark.parametrize("d,r", rc.BATCH_DR)
def test_batched_round_matches_single_steps(d, r, mode):
    """dpgo_agents_round_async with three agents (give-up, rejected then accepted, accepted at once): each agent's
    iterate and result record bit for bit those of the same step run alone on its handle; the agent that gives up
    leaves its iterate and its public tiles as they were"""
    import torch
    import dpo_b200 as dp
    from dpo_b200 import _capi
    agents = rc.batch_agents(d, r)
    gps = [handle(a, mode, (dp.PRECOND_BLOCK_JACOBI, dp.PRECOND_SPARSE_EXACT)) for a in agents]
    try:
        lib = gps[0]._lib
        publics = [np.array([0, a.n // 2, a.n - 1], dtype=np.int32) for a in agents]
        for gp, pub in zip(gps, publics):
            _capi.check(lib.dpgo_agent_set_public_poses(gp._h, len(pub), _capi.iptr(pub)))
        prm = optimizer(gps[0], agents[0], dp.PRECOND_SPARSE_EXACT).params()
        alone = []
        for gp, a in zip(gps, agents):
            go = optimizer(gp, a, dp.PRECOND_SPARSE_EXACT)
            gp.upload_X(a.X)
            go.optimize_resident_async()
            gp.sync()
            alone.append((gp.download_X(), go.fetch_result()))
            check_step(a, alone[-1][0], alone[-1][1], (a.name, d, r, mode))
        for gp, a in zip(gps, agents):
            gp.upload_X(a.X)
            gp.sync()
        ts = r * (d + 1)
        send = [torch.full((len(p) * ts,), float("nan"), dtype=torch.float64, device="cuda") for p in publics]
        torch.cuda.synchronize()
        hs = (C.c_void_p * 3)(*[gp._h for gp in gps])
        sp = (C.c_void_p * 3)(*[C.c_void_p(t.data_ptr()) for t in send])
        _capi.check(lib.dpgo_agents_round_async(hs, 3, C.byref(prm), None, 0, sp, None, 0))
        for gp in gps:
            gp.sync()
        torch.cuda.synchronize()
        for gp, a, (X1, r1), s, pub in zip(gps, agents, alone, send, publics):
            res = dp.QuadraticOptimizer(gp).fetch_result()
            X2 = gp.download_X()
            assert np.array_equal(X2, X1), a.name
            assert all(getattr(res, k) == getattr(r1, k) for k in RECORD), (a.name, res.as_dict(), r1.as_dict())
            assert np.array_equal(s.cpu().numpy(), tiles_of(X2, pub, d)), a.name
            if a.name == "batch_giveup":
                assert np.array_equal(X2, a.X) and np.array_equal(s.cpu().numpy(), tiles_of(a.X, pub, d))
    finally:
        for gp in gps:
            gp.close()
