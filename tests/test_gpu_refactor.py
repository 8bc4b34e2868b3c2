"""Stream-ordered re-weighting: the exact preconditioner refactorised on the device (nd_refactor.cu) after a weight change,
against the synchronous host rebuild (nd::build_numeric) and a SciPy sparse LU of Q + 0.1 I; the single-agent GNC schedule
of the reference (PGOAgent::iterate / updateLoopClosuresWeights, src/PGOAgent.cpp:653-667, 1174-1289; RobustCost,
src/DPGO_robust.cpp:69-103) run with both paths; CUDA-graph capture of the asynchronous calls."""
import ctypes
import os

import numpy as np
import pytest

from oracle import dpgo_oracle as orc

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ASYNC_SYMBOLS = ("dpgo_problem_set_edge_weights_async", "dpgo_problem_robust_reweight_async", "dpgo_problem_device_edge_weights",
                 "dpgo_problem_gnc_counts", "dpgo_nd_node_sizes")


def relerr(a, b):
    return float(np.linalg.norm(np.asarray(a) - np.asarray(b)) / max(np.linalg.norm(b), 1e-300))


# ---- CPU: the boundary exists and rejects bad handles (no device needed) ----------------------------------------------
def test_async_reweight_symbols_and_null_handle():
    from dpo_b200 import _capi
    lib = _capi.load_library()
    header = open(os.path.join(ROOT, "include", "dpgo_b200.h")).read()
    for s in ASYNC_SYMBOLS:
        assert s in header and s in _capi.SIGNATURES and getattr(lib, s) is not None
    w, r2 = ctypes.c_void_p(), ctypes.c_void_p()
    out = (ctypes.c_int64 * 3)()
    cnt = ctypes.c_int64()
    assert lib.dpgo_problem_set_edge_weights_async(None, None) == 1
    assert lib.dpgo_problem_robust_reweight_async(None, 5, 1e-4, 10.0) == 1
    assert lib.dpgo_problem_device_edge_weights(None, ctypes.byref(w), ctypes.byref(r2)) == 1
    assert lib.dpgo_problem_gnc_counts(None, out) == 1
    assert lib.dpgo_nd_node_sizes(None, 0, None, None, None, ctypes.byref(cnt)) == 1


# ---- GPU --------------------------------------------------------------------------------------------------------------
R_OF = {2: 3, 3: 5}


def load(ds, data_dir):
    from dpo_b200 import posegraph as pg
    edges, n = pg.read_g2o_file(os.path.join(data_dir, ds + ".g2o"))
    meas, _ = orc.read_g2o(os.path.join(data_dir, ds + ".g2o"))
    return edges, meas, n


def odometry_flags(edges):
    """The first edge k -> k + 1 of every k: the reference's odometry (isKnownInlier), kept fixed under re-weighting."""
    fx = np.zeros(len(edges), dtype=np.int32)
    seen = set()
    for e in range(len(edges)):
        if edges.p2[e] == edges.p1[e] + 1 and int(edges.p1[e]) not in seen:
            seen.add(int(edges.p1[e]))
            fx[e] = 1
    return fx


def make_problem(edges, n, fixed, mode=0, precond=None):
    import dpo_b200 as dp
    from dpo_b200._capi import PRECOND_BLOCK_JACOBI, PRECOND_SPARSE_EXACT
    d = edges.d
    gp = dp.QuadraticProblem(n, d, R_OF[d], preconditioners=precond or (PRECOND_BLOCK_JACOBI, PRECOND_SPARSE_EXACT))
    gp._lib.dpgo_problem_set_launch_mode(gp._h, mode)
    gp.setEdges(edges, fixed=fixed)
    return gp


def lu_precondition(gp, meas, w, n, X, V):
    """Z = P_X(V (Q + 0.1 I)^-1) with Q from the host construction at weights w, SciPy sparse LU."""
    import scipy.sparse as sp
    import scipy.sparse.linalg as spla
    meas.weight = np.asarray(w, dtype=float).copy()
    Q = sp.csc_matrix(orc.construct_connection_laplacian(meas, n))
    lu = spla.splu((Q + 0.1 * sp.identity(Q.shape[0], format="csc")).tocsc())
    return gp.Projection(X, lu.solve(np.ascontiguousarray(V.T)).T)


def seeded_weights(m, seed):
    rng = np.random.default_rng(seed)
    w = rng.uniform(0.0, 1.0, m)
    w[rng.random(m) < 0.1] = 0.0
    w[rng.random(m) < 0.2] = 1.0
    return w


CASES = [(ds, None, 0) for ds in ("tinyGrid3D", "smallGrid3D", "CSAIL", "sphere2500", "torus3D", "parking-garage", "grid3D")]
CASES += [("sphere2500", levels, mode) for levels in (1, 2, 3, 4) for mode in (0, 1)]
CASES += [(ds, None, 1) for ds in ("smallGrid3D", "CSAIL", "torus3D")]


@pytest.mark.gpu
@pytest.mark.parametrize("ds,levels,mode", CASES)
def test_async_reweight_same_operator(ds, levels, mode, data_dir, monkeypatch):
    import torch
    from dpo_b200._capi import PRECOND_BLOCK_JACOBI
    if levels is not None:
        monkeypatch.setenv("DPGO_ND_CUTS", str(levels - 1))
    edges, meas, n = load(ds, data_dir)
    d, m = edges.d, len(edges)
    fixed = odometry_flags(edges)
    rng = np.random.default_rng(7)
    X = orc.manifold_project(rng.standard_normal((R_OF[d], (d + 1) * n)), d)
    V = rng.standard_normal(X.shape)
    sync, asy = make_problem(edges, n, fixed, mode), make_problem(edges, n, fixed, mode)
    if levels is not None:
        assert sync.nd_info()["levels"] == asy.nd_info()["levels"] == levels
    w1, w = seeded_weights(m, 1), seeded_weights(m, 2)
    asy.setEdgeWeightsAsync(torch.tensor(w1, dtype=torch.float64, device="cuda"))   # first call: builds the structure
    wt = torch.tensor(w, dtype=torch.float64, device="cuda")
    asy.setEdgeWeightsAsync(wt)                                                          # device refactorisation only
    asy.sync()
    sync.setEdgeWeights(w)
    assert np.array_equal(asy.EucGrad(X), sync.EucGrad(X))                             # the same k_assemble_Q
    assert relerr(asy.PreConditioner(X, V, PRECOND_BLOCK_JACOBI), sync.PreConditioner(X, V, PRECOND_BLOCK_JACOBI)) <= 1e-13
    za, zs = asy.PreConditioner(X, V), sync.PreConditioner(X, V)
    assert relerr(za, zs) <= 1e-10
    assert relerr(za, lu_precondition(asy, meas, w, n, X, V)) <= 1e-10


@pytest.mark.gpu
def test_async_reweight_call_order_and_arguments(data_dir):
    import dpo_b200 as dp
    edges, _, n = load("tinyGrid3D", data_dir)
    gp = dp.QuadraticProblem(n, 3, 5)
    w, r2 = ctypes.c_void_p(), ctypes.c_void_p()
    out = (ctypes.c_int64 * 3)()
    buf = gp.device_X_ptr()
    assert gp._lib.dpgo_problem_set_edge_weights_async(gp._h, ctypes.c_void_p(buf)) == 4
    assert gp._lib.dpgo_problem_robust_reweight_async(gp._h, 5, 1e-4, 10.0) == 4
    assert gp._lib.dpgo_problem_device_edge_weights(gp._h, ctypes.byref(w), ctypes.byref(r2)) == 4
    assert gp._lib.dpgo_problem_gnc_counts(gp._h, out) == 4
    gp.setEdges(edges, fixed=odometry_flags(edges))
    assert gp._lib.dpgo_problem_set_edge_weights_async(gp._h, None) == 1
    assert gp._lib.dpgo_problem_device_edge_weights(gp._h, None, ctypes.byref(r2)) == 1
    assert gp._lib.dpgo_problem_gnc_counts(gp._h, None) == 1
    assert gp._lib.dpgo_problem_robust_reweight_async(gp._h, 5, 0.0, 10.0) == 1


# ---- the reference's single-agent GNC schedule -------------------------------------------------------------------------
GNC_MU0, GNC_STEP, GNC_BARC, GNC_MAX = 1e-4, 1.4, 10.0, 100        # RobustCostParameters defaults (DPGO_robust.h:34-55)
STEPS_PER_UPDATE = 30


def with_outliers(edges, fixed, seed):
    """A seeded 10 % of the loop closures replaced with random relative poses."""
    from scipy.spatial.transform import Rotation
    rng = np.random.default_rng(seed)
    lc = np.flatnonzero(fixed == 0)
    bad = np.sort(rng.choice(lc, size=max(1, len(lc) // 10), replace=False))
    e = edges.take(np.arange(len(edges)))
    d = e.d
    if d == 3:
        e.R[bad] = Rotation.random(len(bad), random_state=seed).as_matrix()
    else:
        th = rng.uniform(-np.pi, np.pi, len(bad))
        e.R[bad] = np.stack([np.stack([np.cos(th), -np.sin(th)], 1), np.stack([np.sin(th), np.cos(th)], 1)], 1)
    e.t[bad] = rng.uniform(-10.0, 10.0, (len(bad), d))
    return e, bad


def gnc_loop(gp, X0, use_async, updates, stop_when_binary=False):
    """updateX's RTR constants (src/PGOAgent.cpp:1134-1137) with the exact preconditioner; re-weight every 30 steps.
    stop_when_binary: end after the first update that leaves no weight strictly between 0 and 1."""
    import dpo_b200 as dp
    opt = dp.QuadraticOptimizer(gp)
    opt.setTrustRegionTolerance(1e-2)
    opt.setTrustRegionIterations(1)
    opt.setTrustRegionMaxInnerIterations(10)
    opt.setTrustRegionInitialRadius(100)
    gp.upload_X(X0)
    trace, mu = [], GNC_MU0
    for u in range(updates):
        for _ in range(STEPS_PER_UPDATE):
            opt.optimize_resident_async()
            res = opt.fetch_result()
            trace.append((res.tcg_iterations, res.tcg_status, gp.download_X()))
        if use_async:
            gp.robustReweightAsync("GNC_TLS", mu, GNC_BARC)
        else:
            gp.robustReweight("GNC_TLS", mu, GNC_BARC)
        mu *= GNC_STEP
        if stop_when_binary and gp.gncCounts()[2] == 0:
            break
    counts = gp.gncCounts()
    w, _ = gp.edgeWeightsDevice()
    return trace, w.cpu().numpy().copy(), counts


@pytest.mark.gpu
@pytest.mark.parametrize("ds", ["sphere2500", "torus3D"])
def test_gnc_loop_same_answer_both_paths(ds, data_dir):
    from dpo_b200 import posegraph as pg
    edges, _, n = load(ds, data_dir)
    d = edges.d
    fixed = odometry_flags(edges)
    edges, bad = with_outliers(edges, fixed, 3)
    odo = edges.take(np.flatnonzero(fixed))
    odo = odo.take(np.argsort(odo.p1))
    X0 = pg.fixedStiefelVariable(d, R_OF[d]) @ pg.odometryInitialization(d, n, odo)
    ts, ws, cs = gnc_loop(make_problem(edges, n, fixed), X0, False, GNC_MAX, stop_when_binary=True)
    updates = len(ts) // STEPS_PER_UPDATE
    ta, wa, ca = gnc_loop(make_problem(edges, n, fixed), X0, True, updates)
    assert len(ta) == len(ts)
    for k, ((is_, ss, xs), (ia, sa, xa)) in enumerate(zip(ts, ta)):
        assert (is_, ss) == (ia, sa), k
        assert relerr(xa, xs) <= 1e-8, k
    lc = fixed == 0
    assert np.array_equal(ws[lc] == 0, wa[lc] == 0) and np.array_equal(ws[lc] == 1, wa[lc] == 1)
    assert cs == ca
    print(f"{ds}: {updates} weight updates, {int(np.sum(wa[bad] == 0))} of {len(bad)} injected outliers at weight 0; "
          f"counts (1, 0, between) = {ca}")
    # bit-reproducible: a second asynchronous run gives bitwise the same iterates and weights
    t2, w2, c2 = gnc_loop(make_problem(edges, n, fixed), X0, True, 6)
    for (_, _, x1), (_, _, x2) in zip(ta, t2):
        assert np.array_equal(x1, x2)
    t3, w3, _ = gnc_loop(make_problem(edges, n, fixed), X0, True, 6)
    assert np.array_equal(w2, w3) and all(np.array_equal(a[2], b[2]) for a, b in zip(t2, t3))


# ---- no host synchronisation: CUDA-graph capture -----------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("ds", ["sphere2500", "CSAIL"])
def test_async_reweight_captures(ds, data_dir):
    import torch
    edges, _, n = load(ds, data_dir)
    d = edges.d
    fixed = odometry_flags(edges)
    rng = np.random.default_rng(5)
    X = orc.manifold_project(rng.standard_normal((R_OF[d], (d + 1) * n)), d)
    V = rng.standard_normal(X.shape)
    eager, graphed = make_problem(edges, n, fixed), make_problem(edges, n, fixed)
    for gp in (eager, graphed):
        gp.upload_X(X)
        gp.robustReweightAsync("GNC_TLS", 1e-4, 10.0)          # first call: structure built on the host
        gp.sync()
    s = torch.cuda.Stream()
    graphed.set_stream(s.cuda_stream)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g, stream=s):
        graphed.robustReweightAsync("GNC_TLS", 2e-2, 10.0)
    for _ in range(2):
        g.replay()
    torch.cuda.synchronize()
    graphed.set_stream(None)
    eager.robustReweightAsync("GNC_TLS", 2e-2, 10.0)
    eager.sync()
    we, wg = eager.edgeWeightsDevice()[0].cpu().numpy(), graphed.edgeWeightsDevice()[0].cpu().numpy()
    assert np.array_equal(we, wg)
    assert eager.gncCounts() == graphed.gncCounts()
    assert np.array_equal(eager.PreConditioner(X, V), graphed.PreConditioner(X, V))


@pytest.mark.gpu
def test_async_reweight_and_steps_capture_in_cluster_mode(data_dir):
    import torch
    import dpo_b200 as dp
    edges, _, n = load("smallGrid3D", data_dir)
    fixed = odometry_flags(edges)
    rng = np.random.default_rng(9)
    X = orc.manifold_project(rng.standard_normal((5, 4 * n)), 3)
    probs = [make_problem(edges, n, fixed, mode=1) for _ in range(2)]
    opts = []
    for gp in probs:
        assert gp.launch_info()[1]
        gp.upload_X(X)
        gp.robustReweightAsync("GNC_TLS", 1e-4, 10.0)
        gp.sync()
        opt = dp.QuadraticOptimizer(gp)
        opt.setTrustRegionMaxInnerIterations(10)
        opt.setTrustRegionInitialRadius(100)
        opt.optimize_resident_async()                           # plans the step kernel before capture
        gp.sync()
        gp.upload_X(X)
        opts.append(opt)

    def sequence(gp, opt):
        gp.robustReweightAsync("GNC_TLS", 1e-2, 10.0)
        for _ in range(3):
            opt.optimize_resident_async()

    for _ in range(2):
        sequence(probs[0], opts[0])
    probs[0].sync()
    s = torch.cuda.Stream()
    probs[1].set_stream(s.cuda_stream)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g, stream=s):
        sequence(probs[1], opts[1])
    for _ in range(2):
        g.replay()
    torch.cuda.synchronize()
    probs[1].set_stream(None)
    assert np.array_equal(probs[0].download_X(), probs[1].download_X())
    assert np.array_equal(probs[0].edgeWeightsDevice()[0].cpu().numpy(), probs[1].edgeWeightsDevice()[0].cpu().numpy())


# ---- no stale host copy ------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_no_stale_host_copy_after_async(data_dir):
    import torch
    from dpo_b200._capi import PRECOND_BLOCK_JACOBI, PRECOND_DENSE_EXACT, PRECOND_SPARSE_EXACT
    edges, meas, n = load("smallGrid3D", data_dir)
    fixed = odometry_flags(edges)
    rng = np.random.default_rng(13)
    X = orc.manifold_project(rng.standard_normal((5, 4 * n)), 3)
    V = rng.standard_normal(X.shape)
    pc = (PRECOND_BLOCK_JACOBI, PRECOND_DENSE_EXACT, PRECOND_SPARSE_EXACT)
    gp = make_problem(edges, n, fixed, precond=pc)
    gp.PreConditioner(X, V, PRECOND_DENSE_EXACT)                 # dense inverse of the initial Q prepared
    w = seeded_weights(len(edges), 4)
    gp.setEdgeWeightsAsync(torch.tensor(w, dtype=torch.float64, device="cuda"))
    ref = lu_precondition(gp, meas, w, n, X, V)
    assert relerr(gp.PreConditioner(X, V, PRECOND_DENSE_EXACT), ref) <= 1e-10   # refactorised from the new Q
    assert relerr(gp.PreConditioner(X, V), ref) <= 1e-10
    # a later synchronous re-weight behaves as on a handle that never saw the asynchronous path
    w2 = seeded_weights(len(edges), 6)
    gp.setEdgeWeights(w2)
    fresh = make_problem(edges, n, fixed, precond=pc)
    fresh.setEdgeWeights(w2)
    assert np.array_equal(gp.EucGrad(X), fresh.EucGrad(X))
    for p in pc:
        assert np.array_equal(gp.PreConditioner(X, V, p), fresh.PreConditioner(X, V, p)), p


@pytest.mark.gpu
def test_dense_exact_refactorised_by_a_captured_reweight(data_dir):
    """A prepared dense exact preconditioner is refactorised in place by the asynchronous re-weight, like the sparse one:
    after one eager call the call captures into a CUDA graph, and after a replay with new weights DENSE_EXACT applies the
    re-weighted operator with no further setup."""
    import torch
    from dpo_b200._capi import PRECOND_BLOCK_JACOBI, PRECOND_DENSE_EXACT, PRECOND_SPARSE_EXACT
    edges, meas, n = load("smallGrid3D", data_dir)
    fixed = odometry_flags(edges)
    rng = np.random.default_rng(17)
    X = orc.manifold_project(rng.standard_normal((5, 4 * n)), 3)
    V = rng.standard_normal(X.shape)
    gp = make_problem(edges, n, fixed, precond=(PRECOND_BLOCK_JACOBI, PRECOND_DENSE_EXACT, PRECOND_SPARSE_EXACT))
    gp.PreConditioner(X, V, PRECOND_DENSE_EXACT)                 # the dense exact preconditioner prepared
    prepared = gp.precond_algorithmic_bytes(PRECOND_DENSE_EXACT)
    assert prepared > 0
    w = torch.tensor(seeded_weights(len(edges), 8), dtype=torch.float64, device="cuda")
    gp.setEdgeWeightsAsync(w)                                     # eager: builds the sparse exact structure
    gp.sync()
    s = torch.cuda.Stream()
    gp.set_stream(s.cuda_stream)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g, stream=s):
        gp.setEdgeWeightsAsync(w)
    w2 = seeded_weights(len(edges), 9)
    w.copy_(torch.tensor(w2, dtype=torch.float64, device="cuda"))
    g.replay()
    torch.cuda.synchronize()
    gp.set_stream(None)
    gp.sync()
    assert gp.precond_algorithmic_bytes(PRECOND_DENSE_EXACT) == prepared        # still prepared: nothing to rebuild
    ref = lu_precondition(gp, meas, w2, n, X, V)
    assert relerr(gp.PreConditioner(X, V, PRECOND_DENSE_EXACT), ref) <= 1e-10
    assert relerr(gp.PreConditioner(X, V), ref) <= 1e-10
