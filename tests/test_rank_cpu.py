"""Relaxation ranks d <= r <= 8 without a GPU: the rank bound of dpgo_problem_create and of the hosts over it, the block
solve's plan at the ranks above 5 (host emulation against a sparse LU, inside the per-rank shared-memory capacities), and
the NumPy oracle, the parity reference of the GPU tests at those ranks."""
import ctypes as C
import os

import numpy as np
import pytest

from dpo_b200 import _capi as capi
from dpo_b200 import posegraph as pg
from oracle import dpgo_oracle as orc
from test_nd_plan import dense_reference, relerr

NEW_RANKS = ((2, 4), (2, 6), (2, 7), (2, 8), (3, 6), (3, 7), (3, 8))      # (d, r) compiled since ranks above 5
OPT_SMEM_LIMIT = 227 * 1024
# the step kernel's fixed shared-memory prefix in doubles: warp partials, totals, solver state, block-CSR copy
OPT_SMEM_BASE_DOUBLES = 16 * 4 + 2 * 4 + 32 + 1024


def ycap(r, dh):
    return 600 if r * dh <= 20 else 12000 // (r * dh)


def slot_cap(r):
    return 240 if r <= 5 else 1200 // r


def emulate_info(n, d, r, brow, bcol, blocks, V, **kw):
    """emulate() plus the two residency slots of the info record (bytes read from shared memory per application, and
    the largest resident region of a CTA)"""
    lib = capi.load_library()
    brow = np.ascontiguousarray(brow, dtype=np.int32)
    bcol = np.ascontiguousarray(bcol, dtype=np.int32)
    blocks = np.ascontiguousarray(blocks, dtype=np.float64)
    Vf = np.asfortranarray(V, dtype=np.float64)
    Z = np.asfortranarray(np.full(Vf.shape, np.nan))
    info = (C.c_int64 * 16)()
    capi.check(lib.dpgo_nd_debug_emulate(n, d, r, len(brow), capi.iptr(brow), capi.iptr(bcol), capi.dptr(blocks), 0.1,
                                         kw.get("grid", 148), kw.get("cuts", -1), kw.get("leaf", 0), capi.dptr(Vf),
                                         capi.dptr(Z), info))
    return Z, [int(v) for v in info]


def check_capacities(info, r, dh):
    """the plan stays inside the rank's capacities, and what it stages plus its resident columns fit the kernel's
    227 KB of shared memory"""
    ytiles, slots = info[11], info[12]
    assert 1 <= ytiles <= ycap(r, dh) and slots <= slot_cap(r), (r, dh, info)
    staged = OPT_SMEM_BASE_DOUBLES + ytiles * r * dh + (max(slots, 1) + 1) * 8 * r + 4 * ytiles + 8
    assert 8 * staged + info[14] <= OPT_SMEM_LIMIT, (r, dh, staged, info)


# ---- the rank bound ---------------------------------------------------------------------------------------------------
def test_capacities_keep_the_existing_ranks_and_fit_at_every_rank():
    for d in (2, 3):
        dh = d + 1
        for r in range(d, 9):
            if r <= 5:
                assert (ycap(r, dh), slot_cap(r)) == (600, 240)
            staged = OPT_SMEM_BASE_DOUBLES + ycap(r, dh) * r * dh + (slot_cap(r) + 1) * 8 * r + 4 * ycap(r, dh) + 8
            assert staged <= OPT_SMEM_BASE_DOUBLES + 600 * 20 + 241 * 40 + 4 * 600 + 8       # never above (5, 4)


@pytest.mark.parametrize("d", [2, 3])
def test_rank_above_8_is_refused_before_the_device_probe(d):
    import dpo_b200 as dp
    lib = capi.load_library()
    h = C.c_void_p()
    assert lib.dpgo_problem_create(10, d, 9, 0, C.byref(h)) == 5          # DPGO_ERR_UNSUPPORTED
    assert not h.value
    assert "<= 8" in lib.dpgo_last_error().decode()
    with pytest.raises(dp.DpgoError) as ei:
        dp.QuadraticProblem(10, d, 9)
    assert ei.value.code == 5 and "<= 8" in str(ei.value)
    with pytest.raises(dp.DpgoError) as ei:
        dp.QuadraticProblem(10, d, 40)
    assert ei.value.code == 5


@pytest.mark.parametrize("d,r", NEW_RANKS)
def test_new_ranks_pass_the_argument_checks(d, r):
    """Every d <= r <= 8 passes the argument checks: without a device the call goes on to the device probe."""
    lib = capi.load_library()
    c = C.c_int(-1)
    if lib.dpgo_device_count(C.byref(c)) == 0 and c.value > 0:
        pytest.skip("a CUDA device is present")
    h = C.c_void_p()
    assert lib.dpgo_problem_create(10, d, r, 0, C.byref(h)) == 2           # DPGO_ERR_NO_DEVICE
    assert lib.dpgo_problem_create(10, d, d - 1, 0, C.byref(h)) == 1       # r < d stays an argument error


# ---- the block solve's plan at the new ranks ----------------------------------------------------------------------------
def spd_blocks(rng, n, edge_list, dh):
    """connection-Laplacian-like SPD block matrix: sum over edges of B^T B with B = [M, -I]"""
    brow, bcol, blocks = [], [], []
    for (i, j) in edge_list:
        M = rng.standard_normal((dh, dh))
        brow += [i, j, i, j]
        bcol += [i, j, j, i]
        blocks += [M.T @ M, np.eye(dh), -M.T, -M]
    if not edge_list:
        brow, bcol, blocks = [0], [0], [np.zeros((dh, dh))]
    return np.array(brow), np.array(bcol), np.array(blocks)


def graphs(rng):
    return {
        "single pose": (1, []),
        "chain": (57, [(i, i + 1) for i in range(56)]),
        "two components + isolated pose": (41, [(i, i + 1) for i in range(19)] + [(i, i + 1) for i in range(20, 39)]),
        "dense clique": (30, [(i, j) for i in range(30) for j in range(i + 1, 30)]),
        "star": (64, [(0, i) for i in range(1, 64)]),
        "random sparse": (300, [(int(a), int(b)) for a, b in rng.integers(0, 300, size=(700, 2)) if a != b]),
    }


@pytest.mark.parametrize("d,r", NEW_RANKS)
def test_plan_on_ragged_and_disconnected_graphs(d, r):
    rng = np.random.default_rng(3)
    dh = d + 1
    for name, (n, el) in graphs(rng).items():
        brow, bcol, blocks = spd_blocks(rng, n, el, dh)
        V = rng.standard_normal((r, dh * n))
        ref = dense_reference(n, dh, brow, bcol, blocks, V)
        for grid, leaf, cuts in ((148, 0, -1), (4, 3, -1), (148, 0, 1), (8, 0, 2), (1, 0, -1)):
            Z, info = emulate_info(n, d, r, brow, bcol, blocks, V, grid=grid, leaf=leaf, cuts=cuts)
            assert relerr(Z, ref) <= 1e-11, (name, grid, leaf, cuts, info)
            check_capacities(info, r, dh)


@pytest.mark.parametrize("d,r", NEW_RANKS)
def test_plan_column_chunked_and_slot_limited(d, r):
    """One leaf wider than the rank's tile capacity (column-chunked steps, partial sums carried in the slots), and a
    1-CTA grid whose runs are longer than the slot capacity (split)."""
    rng = np.random.default_rng(5)
    n, dh = 700, d + 1
    el = [(0, i) for i in range(1, n)] + [(i, i + 1) for i in range(1, n - 1)] + [(1, i) for i in range(3, n, 2)]
    brow, bcol, blocks = spd_blocks(rng, n, el, dh)
    V = rng.standard_normal((r, dh * n))
    ref = dense_reference(n, dh, brow, bcol, blocks, V)
    for grid, cuts in ((148, 0), (1, 0), (3, -1), (1, 1)):
        Z, info = emulate_info(n, d, r, brow, bcol, blocks, V, grid=grid, cuts=cuts)
        assert relerr(Z, ref) <= 1e-11, (grid, cuts, info)
        check_capacities(info, r, dh)
        if cuts == 0:
            assert info[5] == dh * n and info[11] == ycap(r, dh)          # one leaf of 700 tiles, chunked at the cap
        if grid == 1 and cuts == 0:
            assert info[12] == slot_cap(r)


def sphere2500_blocks(data_dir):
    edges, n = pg.read_g2o_file(os.path.join(data_dir, "sphere2500.g2o"))
    brow, bcol, blocks = pg.connection_laplacian_blocks(edges)
    return n, edges.d, np.asarray(brow), np.asarray(bcol), np.asarray(blocks)


@pytest.mark.parametrize("cuts", [-1, 1])
def test_plan_sphere2500_single_agent_at_rank_8(cuts, data_dir):
    """The full H100 grid (132 CTAs) at r = 8, cost-model and forced levels."""
    n, d, brow, bcol, blocks = sphere2500_blocks(data_dir)
    dh, r = d + 1, 8
    V = np.random.default_rng(1).standard_normal((r, dh * n))
    Z, info = emulate_info(n, d, r, brow, bcol, blocks, V, grid=132, cuts=cuts)
    assert relerr(Z, dense_reference(n, dh, brow, bcol, blocks, V)) <= 1e-12
    check_capacities(info, r, dh)


@pytest.mark.parametrize("r", [5, 8])
def test_plan_sphere2500_sixteen_agent_clusters(r, data_dir):
    """An agent of a 16-agent contiguous split of sphere2500 (156 poses: its private Q, here the principal block of the
    whole graph's Q) on the grids of the cluster launch mode."""
    n, d, brow, bcol, blocks = sphere2500_blocks(data_dir)
    dh = d + 1
    lo, hi = 5 * (n // 16), 6 * (n // 16)
    keep = (brow >= lo) & (brow < hi) & (bcol >= lo) & (bcol < hi)
    br, bc, bl = brow[keep] - lo, bcol[keep] - lo, blocks[keep]
    m = hi - lo
    V = np.random.default_rng(2).standard_normal((r, dh * m))
    ref = dense_reference(m, dh, br, bc, bl, V)
    for grid in (10, 16):
        Z, info = emulate_info(m, d, r, br, bc, bl, V, grid=grid)
        assert relerr(Z, ref) <= 1e-12, (grid, info)
        check_capacities(info, r, dh)


# ---- the oracle at the new ranks ----------------------------------------------------------------------------------------
def padded(M, r):
    return np.vstack([M, np.zeros((r - M.shape[0], M.shape[1]))])


@pytest.mark.parametrize("ds,r", [("smallGrid3D", 6), ("smallGrid3D", 8), ("input_INTEL_g2o", 4), ("input_INTEL_g2o", 7)])
def test_oracle_is_rank_generic(ds, r, data_dir):
    """A rank-d problem embedded in rank r (zero rows under the iterate, the linear term and the direction) is the same
    problem: the oracle at rank r gives the rank-d values with zero rows below, through f, gradients, Hessian, the exact
    preconditioner, the retraction and an RTR call; the projections at rank r land on the manifold."""
    meas, n = orc.read_g2o(os.path.join(data_dir, ds + ".g2o"))
    d = meas.d
    Q = orc.construct_connection_laplacian(meas, n)
    rng = np.random.default_rng(7)
    T = orc.chordal_initialization(meas, n)
    X = T + 0.05 * rng.standard_normal(T.shape)
    X = orc.manifold_project(X, d)
    G = 0.1 * rng.standard_normal(X.shape)
    V = orc.tangent_project(X, rng.standard_normal(X.shape), d)
    lo, hi = orc.QuadraticProblem(n, d, d), orc.QuadraticProblem(n, d, r)
    for p, g in ((lo, G), (hi, padded(G, r))):
        p.set_Q(Q)
        p.set_G(g)
    Xr, Vr = padded(X, r), padded(V, r)
    assert hi.f(Xr) == pytest.approx(lo.f(X), rel=1e-14)
    assert np.allclose(hi.rie_grad(Xr), padded(lo.rie_grad(X), r), rtol=0, atol=1e-12 * np.abs(lo.rie_grad(X)).max())
    EGl, EGh = lo.euc_grad(X), hi.euc_grad(Xr)
    hv = hi.rie_hess(Xr, EGh, Vr)
    assert np.abs(hv - padded(lo.rie_hess(X, EGl, V), r)).max() <= 1e-11 * np.abs(hv).max()
    pz = hi.precondition(Xr, Vr)
    assert np.abs(pz - padded(lo.precondition(X, V), r)).max() <= 1e-11 * np.abs(pz).max()
    assert np.abs(orc.retract(Xr, 0.3 * Vr, d) - padded(orc.retract(X, 0.3 * V, d), r)).max() <= 1e-13
    def rtr_step(p, X0):
        oo = orc.QuadraticOptimizer(p)
        oo.tr_tolerance, oo.tr_iterations, oo.tr_max_inner, oo.tr_initial_radius = 1e-2, 1, 10, 100.0
        return oo.optimize(X0), oo.result

    (Xl, rl), (Xh, rh) = rtr_step(lo, X), rtr_step(hi, Xr)
    assert (rl.tcg_iterations, rl.tcg_status) == (rh.tcg_iterations, rh.tcg_status)
    assert np.abs(Xh - padded(Xl, r)).max() <= 1e-9
    # a generic rank-r point: the Stiefel projection and the retraction give orthonormal rotation blocks
    M = rng.standard_normal((r, (d + 1) * n))
    for Y in (orc.manifold_project(M, d), orc.retract(orc.manifold_project(M, d), M, d)):
        Yt = Y.reshape(r, n, d + 1)[:, :, :d]
        assert np.abs(np.einsum("ani,anj->nij", Yt, Yt) - np.eye(d)[None]).max() <= 1e-13
