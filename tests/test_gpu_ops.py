"""GPU parity of every single-operation entry point of the C ABI against the CPU oracle.

Bar: fp64 floating point; relative Frobenius error <= 1e-13 for the SpMV / projection / retraction
kernels (SURVEY 8d), <= 1e-9 for the preconditioners (a dense inverse vs a sparse LU solve).
"""
import numpy as np
import pytest

from oracle import dpgo_oracle as orc

pytestmark = pytest.mark.gpu


def relerr(a, b):
    return float(np.linalg.norm(np.asarray(a) - np.asarray(b)) / max(np.linalg.norm(b), 1e-300))


def make_problem(ds, r, data_dir, with_G=True, seed=0):
    import os
    import dpo_b200 as dp
    meas, n = orc.read_g2o(os.path.join(data_dir, ds + ".g2o"))
    d = meas.d
    Q = orc.construct_connection_laplacian(meas, n)
    rng = np.random.default_rng(seed)
    X = orc.manifold_project(rng.standard_normal((r, (d + 1) * n)), d)
    G = 0.5 * rng.standard_normal((r, (d + 1) * n)) if with_G else np.zeros((r, (d + 1) * n))
    op = orc.QuadraticProblem(n, d, r)
    op.set_Q(Q)
    op.set_G(G)
    gp = dp.QuadraticProblem(n, d, r, preconditioners=(dp.PRECOND_BLOCK_JACOBI, dp.PRECOND_SPARSE_EXACT, dp.PRECOND_DENSE_EXACT))
    gp.setQ(Q)
    gp.setG(G)
    return op, gp, X, rng


CASES = [("tinyGrid3D", 3), ("smallGrid3D", 5), ("smallGrid3D", 3), ("smallGrid3D", 4), ("sphere2500", 5),
         ("sphere2500", 3), ("CSAIL", 5), ("CSAIL", 2), ("CSAIL", 3)]


@pytest.mark.parametrize("ds,r", CASES)
def test_f_grad_hess(ds, r, data_dir):
    op, gp, X, rng = make_problem(ds, r, data_dir)
    d = op.d
    assert abs(gp.f(X) - op.f(X)) <= 1e-12 * max(1.0, abs(op.f(X)))
    assert relerr(gp.EucGrad(X), op.euc_grad(X)) <= 1e-13
    rg = op.rie_grad(X)
    assert relerr(gp.RieGrad(X), rg) <= 1e-13
    assert abs(gp.RieGradNorm(X) - np.linalg.norm(rg)) <= 1e-12 * np.linalg.norm(rg)
    V = rng.standard_normal(X.shape)
    assert relerr(gp.EucHessianEta(V), op.euc_hess(V)) <= 1e-13
    Vt = orc.tangent_project(X, V, d)
    EG = op.euc_grad(X)
    assert relerr(gp.RieHessianEta(X, Vt), op.rie_hess(X, EG, Vt)) <= 1e-12


@pytest.mark.parametrize("ds,r", CASES)
def test_manifold_ops(ds, r, data_dir):
    op, gp, X, rng = make_problem(ds, r, data_dir, with_G=False)
    d = op.d
    Z = rng.standard_normal(X.shape)
    assert relerr(gp.Projection(X, Z), orc.tangent_project(X, Z, d)) <= 1e-13
    eta = 0.3 * orc.tangent_project(X, Z, d)
    Xr = gp.Retraction(X, eta)
    assert relerr(Xr, orc.retract(X, eta, d)) <= 1e-13
    # property: retracted rotation blocks are orthonormal
    Yt = Xr.reshape(r, -1, d + 1)[:, :, :d]
    gram = np.einsum("ani,anj->nij", Yt, Yt)
    assert np.abs(gram - np.eye(d)[None]).max() <= 1e-13
    # a large step (trust-region radius 100 can produce these)
    big = 50.0 * Z
    assert relerr(gp.Retraction(X, big), orc.retract(X, big, d)) <= 1e-12
    M = rng.standard_normal(X.shape)
    assert relerr(gp.project(M), orc.manifold_project(M, d)) <= 1e-12


@pytest.mark.parametrize("ds,r", [("tinyGrid3D", 3), ("smallGrid3D", 5), ("sphere2500", 5), ("CSAIL", 5),
                                  ("parking-garage", 3), ("sphere2500", 4)])
def test_preconditioners(ds, r, data_dir):
    import dpo_b200 as dp
    op, gp, X, rng = make_problem(ds, r, data_dir, with_G=False)
    V = rng.standard_normal(X.shape)
    exact = op.precondition(X, V)
    assert relerr(gp.PreConditioner(X, V, dp.PRECOND_SPARSE_EXACT), exact) <= 1e-11      # nested-dissection block solve (default)
    assert relerr(gp.PreConditioner(X, V, dp.PRECOND_DENSE_EXACT), exact) <= 1e-9        # one macro level (A/B)
    oo = orc.QuadraticOptimizer(op, precond="jacobi")
    assert relerr(gp.PreConditioner(X, V, dp.PRECOND_BLOCK_JACOBI), oo._apply_precond(X, V)) <= 1e-12
    assert relerr(gp.PreConditioner(X, V, dp.PRECOND_NONE), orc.tangent_project(X, V, op.d)) <= 1e-13


def test_dense_exact_bytes_and_phase_clock(data_dir):
    """dpgo_precond_algorithmic_bytes reports the bytes of the operator's blocks once it is prepared (the dense inverse
    of the connected sphere2500 graph); dpgo_debug_phase_times64 accumulates per-phase time of the persistent kernel."""
    import ctypes as C
    import dpo_b200 as dp
    from dpo_b200 import _capi
    op, gp, X, rng = make_problem("sphere2500", 5, data_dir, with_G=False)
    n, N, vec = op.n, X.shape[1], X.size * 8
    assert gp.precond_algorithmic_bytes(dp.PRECOND_BLOCK_JACOBI) == n * 128 + 2 * vec
    assert gp.precond_algorithmic_bytes(dp.PRECOND_DENSE_EXACT) == 0                         # nothing prepared yet
    gp.PreConditioner(X, rng.standard_normal(X.shape), dp.PRECOND_DENSE_EXACT)
    assert gp.precond_algorithmic_bytes(dp.PRECOND_DENSE_EXACT) == 8 * N * N + 2 * vec
    ms = (C.c_double * 64)()
    _capi.check(gp._lib.dpgo_debug_phase_times64(gp._h, 1, ms))
    opt = dp.QuadraticOptimizer(gp)
    opt.setTrustRegionIterations(1)
    opt.setTrustRegionMaxInnerIterations(5)
    opt.setPreconditioner(dp.PRECOND_DENSE_EXACT)
    opt.optimize(X)
    res = opt.getOptResult()
    _capi.check(gp._lib.dpgo_debug_phase_times64(gp._h, 0, ms))
    assert ms[0] > 0 and ms[8] > 0 and ms[3] > 0                                              # eval, dense apply, Hessian
    assert ms[1] == 0 and ms[2] == 0 and ms[9] == 0                                           # one phase per application
    assert sum(ms[:24]) <= res.elapsed_ms * 1.5 + 1.0
    _capi.check(gp._lib.dpgo_debug_phase_times64(gp._h, 0, ms))                               # switched off: zeros
    assert all(v == 0.0 for v in ms)


def test_argument_errors(data_dir):
    import dpo_b200 as dp
    with pytest.raises(dp.DpgoError):
        dp.QuadraticProblem(10, 3, 2)        # r < d  (ref: assert(r >= d))
    with pytest.raises(dp.DpgoError):
        dp.QuadraticProblem(10, 4, 5)        # d not in {2,3}
    p = dp.QuadraticProblem(4, 3, 3)
    with pytest.raises(ValueError):
        p.f(np.zeros((3, 15)))               # wrong shape (ref: assert on cols)
    # empty Q, zero G: f == 0, gradient == 0 (ref ctor sets empty Q and G)
    X = orc.manifold_project(np.random.default_rng(0).standard_normal((3, 16)), 3)
    assert p.f(X) == 0.0
    assert np.abs(p.EucGrad(X)).max() == 0.0


@pytest.mark.parametrize("dims,r", [((12, 10, 6), 5), ((30, 30, 20), 5), ((30, 30, 20), 3), ((50, 40, 30), 5)])
def test_spmv_device_synthetic_grid(dims, r):
    """The stand-alone Q.X kernel (TMA-fed row groups) on graphs spanning many groups, against scipy CSR.
    Size-independent property as well: linearity  Q(aX + bY) = a QX + b QY."""
    import torch
    import dpo_b200 as dp
    from dpo_b200 import posegraph as pg
    edges, n, _ = pg.synthetic_grid_graph(*dims, edges_per_pose=4.0, seed=1)
    Q = pg.constructConnectionLaplacianSE(edges, n)
    prob = dp.QuadraticProblem(n, 3, r, preconditioners=(dp.PRECOND_BLOCK_JACOBI,))
    prob.setQ_blocks(*pg.connection_laplacian_blocks(edges))
    prob.set_stream(torch.cuda.current_stream().cuda_stream)
    rng = np.random.default_rng(0)
    X = rng.standard_normal((r, 4 * n))
    Y = rng.standard_normal((r, 4 * n))

    def run(M):
        t = torch.from_numpy(np.asfortranarray(M).ravel(order="F").copy()).cuda()
        o = torch.empty_like(t)
        prob.spmv_device(t.data_ptr(), o.data_ptr(), False)
        torch.cuda.synchronize()
        return o.cpu().numpy().reshape(r, 4 * n, order="F")

    ref = (Q @ X.T).T
    got = run(X)
    assert relerr(got, ref) <= 1e-13
    lin = run(2.0 * X - 3.0 * Y)
    assert relerr(lin, 2.0 * got - 3.0 * run(Y)) <= 1e-13
    # with the linear term
    G = rng.standard_normal((r, 4 * n))
    prob.setG(G)
    t = torch.from_numpy(np.asfortranarray(X).ravel(order="F").copy()).cuda()
    o = torch.empty_like(t)
    prob.spmv_device(t.data_ptr(), o.data_ptr(), True)
    torch.cuda.synchronize()
    assert relerr(o.cpu().numpy().reshape(r, 4 * n, order="F"), ref + G) <= 1e-13
    assert prob.spmv_algorithmic_bytes(False) == 132 * prob.num_blocks() + 4 * (n + 1) + 64 * r * n
