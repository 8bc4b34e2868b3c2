"""Every single-operation kernel on the structure cases of structure_cases.py (hub rows at and past one TMA stage, a
hub row past the shared block-CSR cache, empty row groups, n = 1..3, disconnected graphs, a 700-pose clique, duplicated
and reversed edges, a 5000-pose path), for every compiled (d, r), in both launch modes (full cooperative grid, and one
thread-block cluster), against long-double references with componentwise forward-error bounds."""
import numpy as np
import pytest

import structure_cases as sc
from oracle import dpgo_oracle as orc

pytestmark = pytest.mark.gpu

PARAMS = [(name, d, r) for name in sc.CASE_NAMES for d in (2, 3) for r in sc.RANKS[d]
          if not (name in sc.LARGE + ("clique700",) and r not in sc.large_ranks(d))]
_CASES = {}


def case(name, d):
    if (name, d) not in _CASES:
        c = sc.make_case(name, d)
        _CASES[(name, d)] = (c, c.Q(), sc.pose_K(c, d))
    return _CASES[(name, d)]


def make(c, Q, r, cluster, dense):
    import dpo_b200 as dp
    precs = [dp.PRECOND_BLOCK_JACOBI, dp.PRECOND_SPARSE_EXACT] + ([dp.PRECOND_DENSE_EXACT] if dense else [])
    gp = dp.QuadraticProblem(c.n, c.d, r, preconditioners=precs, cluster=cluster)
    gp.setQ(Q)
    return gp


def spmv(gp, M, add_G):
    import torch
    r, N = M.shape
    t = torch.from_numpy(np.asfortranarray(M).ravel(order="F").copy()).cuda()
    o = torch.full_like(t, float("nan"))
    gp.set_stream(torch.cuda.current_stream().cuda_stream)
    gp.spmv_device(t.data_ptr(), o.data_ptr(), add_G)
    torch.cuda.synchronize()
    gp.set_stream(None)
    return o.cpu().numpy().reshape(r, N, order="F")


@pytest.mark.parametrize("cluster", [False, True], ids=["grid", "cluster"])
@pytest.mark.parametrize("name,d,r", PARAMS)
def test_single_operations(name, d, r, cluster):
    import dpo_b200 as dp
    c, Q, K = case(name, d)
    dense = c.N <= sc.DENSE_MAX_N
    gp = make(c, Q, r, cluster, dense)
    assert gp.launch_info()[1] == cluster
    assert gp.num_blocks() == int(c.row_blocks().sum())
    rng = np.random.default_rng([r, d, sc.CASE_NAMES.index(name)])
    X = orc.manifold_project(rng.standard_normal((r, c.N)), d)
    G = rng.standard_normal((r, c.N))
    V = rng.standard_normal((r, c.N))
    Vt = orc.tangent_project(X, V, d)
    gp.setG(G)
    C = sc.stage_c(K, r, d)

    # products
    sc.check_product(spmv(gp, X, False), Q, X, K, what="spmv_device")
    sc.check_product(spmv(gp, X, True), Q, X, K, G=G, what="spmv_device + G")
    sc.check_product(gp.EucHessianEta(V), Q, V, K, what="EucHessianEta")
    sc.check_product(gp.EucGrad(X), Q, X, K, G=G, what="EucGrad")
    val, mag = sc.f_ref(Q, G, X)
    sc.check_scalar(gp.f(X), val, mag, K, X.size, "f")

    # Riemannian quantities
    ref, mag, _, _ = sc.rgrad_ref(Q, G, X, d)
    sc.check_elementwise(gp.RieGrad(X), ref, mag, C, "RieGrad")
    gn = np.sqrt(np.sum(ref ** 2))
    bound = np.sqrt(np.sum((C * sc.U * mag) ** 2)) + (X.size + 2) * sc.U * gn
    assert abs(sc.LD(gp.RieGradNorm(X)) - gn) <= bound, "RieGradNorm"
    ref, mag = sc.rhess_ref(Q, G, X, Vt, d)
    sc.check_elementwise(gp.RieHessianEta(X, Vt), ref, mag, C, "RieHessianEta")
    ref, mag = sc.projection_ref(X, V, d)
    sc.check_elementwise(gp.Projection(X, V), ref, mag, C, "Projection")

    # preconditioners
    sc.check_elementwise(gp.PreConditioner(X, V, dp.PRECOND_NONE), ref, mag, C, "PRECOND_NONE")
    ref, mag, cond = sc.jacobi_ref(Q, X, V, d)
    sc.check_elementwise(gp.PreConditioner(X, V, dp.PRECOND_BLOCK_JACOBI), ref, mag, C + 4 * sc.per_elem(cond, r, d),
                         "BLOCK_JACOBI")
    ref, kappa = sc.exact_ref(Q, X, V, d)
    sc.check_exact(gp.PreConditioner(X, V, dp.PRECOND_SPARSE_EXACT), ref, kappa, d, 256, "SPARSE_EXACT")
    if dense:
        sc.check_exact(gp.PreConditioner(X, V, dp.PRECOND_DENSE_EXACT), ref, kappa, d, max(256.0, c.N / 4), "DENSE_EXACT")

    # retraction: orthonormal blocks, translation exactly x + eta
    eta = 0.3 * Vt
    Xr = gp.Retraction(X, eta)
    assert np.abs(Xr - orc.retract(X, eta, d)).max() <= 1e-13
    Xrt = sc.tiles(Xr, d)
    gram = np.einsum("ani,anj->nij", Xrt[:, :, :d], Xrt[:, :, :d])
    assert np.abs(gram - np.eye(d)[None]).max() <= 16 * sc.U * r
    assert np.array_equal(Xrt[:, :, d], sc.tiles(X + eta, d)[:, :, d])


@pytest.mark.parametrize("cluster", [False, True], ids=["grid", "cluster"])
@pytest.mark.parametrize("name", [n for n in sc.CASE_NAMES if n != "single"])      # Q = 0: no step to take
def test_rtr_steps(name, cluster):
    """Three RTR steps with the reference's updateX constants, sparse exact and block-Jacobi preconditioners, against the
    oracle: same tCG iteration count and status, iterate within 1e-8."""
    import dpo_b200 as dp
    d, r = 3, 5
    c, Q, K = case(name, d)
    rng = np.random.default_rng(11)
    X0 = orc.manifold_project(rng.standard_normal((r, c.N)), d)
    op = orc.QuadraticProblem(c.n, d, r)
    op.set_Q(Q)
    gp = make(c, Q, r, cluster, False)
    for precond, pid in (("exact", dp.PRECOND_SPARSE_EXACT), ("jacobi", dp.PRECOND_BLOCK_JACOBI)):
        Xo, Xg = X0, X0
        for it in range(3):
            oo = orc.QuadraticOptimizer(op, precond=precond)
            oo.tr_tolerance, oo.tr_iterations, oo.tr_max_inner, oo.tr_initial_radius = 1e-2, 1, 10, 100.0
            go = dp.QuadraticOptimizer(gp)
            go.setTrustRegionTolerance(1e-2)
            go.setTrustRegionIterations(1)
            go.setTrustRegionMaxInnerIterations(10)
            go.setTrustRegionInitialRadius(100)
            go.setPreconditioner(pid)
            Xo = oo.optimize(Xo)
            Xg = go.optimize(Xg)
            res = go.getOptResult()
            assert res.tcg_iterations == oo.result.tcg_iterations, (precond, it, res.as_dict(), oo.result)
            assert res.tcg_status == oo.result.tcg_status, (precond, it)
            assert np.linalg.norm(Xg - Xo) <= 1e-8 * np.linalg.norm(Xo), (precond, it)


@pytest.mark.parametrize("name", ["multi_edges", "tail_isolated"])
@pytest.mark.parametrize("d", [2, 3])
def test_device_assembly(name, d):
    """Q from block triplets and from raw edges (duplicates, reversed edges, empty rows) assembled on the device: its
    products agree with the host-assembled Q tile by tile (the device sums in its own order)."""
    import dpo_b200 as dp
    c, Q, K = case(name, d)
    r = 5
    rng = np.random.default_rng(5)
    V = rng.standard_normal((r, c.N))
    ref = np.asarray(sc.product_ref(Q, V)[0], dtype=np.float64)
    precs = (dp.PRECOND_BLOCK_JACOBI, dp.PRECOND_SPARSE_EXACT)
    for how in ("blocks", "edges"):
        gp = dp.QuadraticProblem(c.n, d, r, preconditioners=precs)
        if how == "blocks":
            gp.setQ_blocks(*c.triplets())
        else:
            gp.setEdges(c.edges)
        assert gp.num_blocks() == int(c.row_blocks().sum())
        for got in (gp.EucHessianEta(V), spmv(gp, V, False)):
            te = np.sqrt((sc.tiles(got - ref, d) ** 2).sum(axis=(0, 2)))
            tn = np.sqrt((sc.tiles(ref, d) ** 2).sum(axis=(0, 2)))
            assert te.max() <= 1e-13 * tn.max(), (how, int(te.argmax()))
