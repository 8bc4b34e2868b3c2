"""The pose-covariance model and the host emulation of its device sweep, without a GPU.

covariance_oracle restates the model; these tests check the oracle itself (Jacobians, null space, cost, a closed-form
case) and then the library's host emulation (same pattern, hierarchy, factorisation and selected-inversion recurrence as
dpgo_pose_covariances) against it."""
import ctypes as C
import os
import sys

import numpy as np
import pytest
import scipy.sparse as sp
import scipy.sparse.linalg as spla

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import covariance_oracle as co  # noqa: E402
from dpo_b200 import posegraph as pg  # noqa: E402


def random_graph(d, n, extra, seed, noise=0.05):
    """A connected random graph (a spanning path plus `extra` random edges) with measurements near a random trajectory."""
    rng = np.random.default_rng(seed)
    Tt = co.random_trajectory(d, n, rng)
    Rt, tt = co.poses(Tt, d)
    p1 = list(range(n - 1))
    p2 = list(range(1, n))
    for _ in range(extra):
        i, j = rng.choice(n, 2, replace=False)
        p1.append(int(i)); p2.append(int(j))
    p1, p2 = np.array(p1), np.array(p2)
    m = len(p1)
    nw = 3 if d == 3 else 1
    R = np.stack([Rt[p1[e]].T @ Rt[p2[e]] @ co.exp_so(d, noise * rng.standard_normal(nw)) for e in range(m)])
    t = np.stack([Rt[p1[e]].T @ (tt[p2[e]] - tt[p1[e]]) + noise * rng.standard_normal(d) for e in range(m)])
    kappa = rng.uniform(50, 200, m)
    tau = rng.uniform(5, 50, m)
    z = np.zeros(m, dtype=np.int64)
    edges = pg.EdgeSet(d, z, z, p1, p2, R, t, kappa, tau)
    T = Tt.copy()
    for p in range(n):                                   # a noisy trajectory: not a critical point
        T = co.perturb(T, d, p, 0.02 * rng.standard_normal(co.tangent_dim(d)))
    return edges, T


def emulate(edges, n, T, anchor=0, pairs=None, force_cuts=-1, leaf_size=0):
    from dpo_b200 import _capi as capi
    lib = capi.load_library()
    d = edges.d
    b = co.tangent_dim(d)
    p1, p2, R, t, kappa, tau, w = co.edge_arrays(edges)
    pr = np.zeros((0, 2), dtype=np.int32) if pairs is None else np.ascontiguousarray(np.asarray(pairs, dtype=np.int32))
    cov = np.zeros((n, b, b))
    pcov = np.zeros((max(len(pr), 1), b, b))
    info = (C.c_int64 * 16)()
    Tf = np.asfortranarray(T)
    code = lib.dpgo_pose_covariances_debug_emulate(n, d, len(p1), capi.iptr(p1), capi.iptr(p2), capi.dptr(R), capi.dptr(t),
                                                   capi.dptr(kappa), capi.dptr(tau), capi.dptr(w), capi.dptr(Tf), anchor,
                                                   force_cuts, leaf_size, len(pr), capi.iptr(pr), capi.dptr(cov),
                                                   capi.dptr(pcov), info)
    capi.check(code)
    return cov, pcov[:len(pr)], list(info)


def rel(a, b):
    return np.linalg.norm(a - b) / max(np.linalg.norm(b), 1e-300)


@pytest.mark.parametrize("d", [2, 3])
def test_jacobians_match_central_differences(d):
    edges, T = random_graph(d, 6, 6, seed=d)
    Ji, Jj = co.jacobians(T, edges)
    h = 1e-6
    b = co.tangent_dim(d)
    for e in range(len(edges)):
        for role, (J, p) in enumerate(((Ji, edges.p1[e]), (Jj, edges.p2[e]))):
            for k in range(b):
                x = np.zeros(b); x[k] = h
                rp, _ = co.residuals(co.perturb(T, d, p, x), edges.take([e]))
                rm, _ = co.residuals(co.perturb(T, d, p, -x), edges.take([e]))
                fd = (rp[0] - rm[0]) / (2 * h)
                assert np.allclose(fd, J[e, :, k], atol=1e-7 * max(1.0, np.abs(fd).max())), (e, role, k)


@pytest.mark.parametrize("d", [2, 3])
@pytest.mark.parametrize("consistent", [True, False])
def test_information_is_psd_with_gauge_null_space(d, consistent):
    """PSD always.  At a trajectory that satisfies every measurement the null space is the whole gauge (b: a global
    rotation and translation leave every residual at zero); at a noisy one a global rotation turns the nonzero
    residuals, so only the d global translations stay in the null space."""
    n = 12
    edges, T = random_graph(d, n, 10, seed=10 + d, noise=0.0 if consistent else 0.05)
    if consistent:
        Rt, tt = co.poses(T, d)
        edges.R = np.einsum("mba,mbc->mac", Rt[edges.p1], Rt[edges.p2])
        edges.t = np.einsum("mba,mb->ma", Rt[edges.p1], tt[edges.p2] - tt[edges.p1])
    H = co.information(T, edges, n).toarray()
    assert np.allclose(H, H.T, atol=1e-9 * np.abs(H).max())
    ev = np.linalg.eigvalsh(H)
    null = co.tangent_dim(d) if consistent else d
    tol = 1e-9 * ev[-1]
    assert ev[0] > -tol
    assert np.sum(ev < tol) == null
    assert ev[null] > 1e-6 * ev[-1]


@pytest.mark.parametrize("d", [2, 3])
def test_half_weighted_residual_is_the_cost(d):
    n = 10
    edges, T = random_graph(d, n, 8, seed=20 + d, noise=0.2)
    edges.weight = np.random.default_rng(3).uniform(0.2, 1.5, len(edges))
    r, om = co.residuals(T, edges)
    Q = pg.constructConnectionLaplacianSE(edges, n)
    f = 0.5 * np.sum((Q @ T.T) * T.T)
    assert abs(0.5 * np.sum(om * r * r) - f) <= 1e-10 * f


@pytest.mark.parametrize("d", [2, 3])
def test_two_poses_one_edge_known_answer(d):
    """Anchor pose 0 at the identity, edge 0 -> 1 measured exactly, T at the measurement.  Then H_11 is block diagonal in
    the body frame of pose 1: the rotation block is kappa |R_1 G_k|_F^2 = 2 kappa I (3D) / 2 kappa (2D) and the translation
    block is tau R_1^T R_1 = tau I, with no rotation-translation coupling (d r_tra / d w_1 = 0).  So
    Sigma_1 = diag(1 / (2 kappa), .., 1 / tau, ..)."""
    rng = np.random.default_rng(7)
    kappa, tau = 37.0, 4.5
    nw = 3 if d == 3 else 1
    R1 = co.exp_so(d, rng.standard_normal(nw))
    t1 = rng.standard_normal(d)
    T = np.zeros((d, 2 * (d + 1)))
    T[:, :d] = np.eye(d)
    T[:, d + 1:2 * d + 1] = R1
    T[:, 2 * d + 1] = t1
    edges = pg.EdgeSet(d, [0], [0], [0], [1], R1[None], t1[None], [kappa], [tau])
    want = np.diag([1 / (2 * kappa)] * nw + [1 / tau] * d)
    S = co.covariances_dense(co.information(T, edges, 2), 2, co.tangent_dim(d), 0)
    b = co.tangent_dim(d)
    assert np.allclose(S[b:, b:], want, rtol=1e-12, atol=1e-15)
    cov, _, _ = emulate(edges, 2, T)
    assert np.allclose(cov[1], want, rtol=1e-12, atol=1e-15)
    assert np.all(cov[0] == 0)


def test_zero_weight_edges_drop_out():
    d, n = 3, 10
    edges, T = random_graph(d, n, 6, seed=31)
    extra = pg.EdgeSet(d, [0, 0], [0, 0], [2, 7], [8, 3], edges.R[:2], edges.t[:2], [500.0, 80.0], [90.0, 7.0],
                       weight=[0.0, 0.0])
    both = pg.EdgeSet.join([edges, extra])
    a, _, _ = emulate(edges, n, T)
    b, _, _ = emulate(both, n, T)
    assert rel(b, a) < 1e-12
    Ha = co.information(T, edges, n).toarray()
    Hb = co.information(T, both, n).toarray()
    assert np.array_equal(Ha, Hb) or np.abs(Ha - Hb).max() <= 1e-12 * np.abs(Ha).max()


def embedded_blocks(H, n, d, anchor):
    """The factorisation's input: H over 3-scalar nodes (d = 3: w_i, v_i; d = 2: the pose), the anchor's nodes an
    identity without coupling, as dpgo_nd_debug_emulate's 3 x 3 blocks (d = 2 there means 3-scalar tiles)."""
    b = co.tangent_dim(d)
    ne = n * b // 3
    A = H.toarray().copy()
    A[anchor * b:(anchor + 1) * b, :] = 0.0
    A[:, anchor * b:(anchor + 1) * b] = 0.0
    A[anchor * b:(anchor + 1) * b, anchor * b:(anchor + 1) * b] = np.eye(b)
    brow, bcol, blocks = [], [], []
    for i in range(ne):
        for j in range(ne):
            blk = A[3 * i:3 * i + 3, 3 * j:3 * j + 3]
            if np.any(blk != 0) or i == j:
                brow.append(i); bcol.append(j); blocks.append(blk)
    return ne, A, np.array(brow, np.int32), np.array(bcol, np.int32), np.ascontiguousarray(np.array(blocks))


@pytest.mark.parametrize("d", [2, 3])
def test_embedded_matrix_through_the_existing_factorisation(d):
    from dpo_b200 import _capi as capi
    lib = capi.load_library()
    n = 40
    edges, T = random_graph(d, n, 30, seed=40 + d)
    H = co.information(T, edges, n)
    ne, A, brow, bcol, blocks = embedded_blocks(H, n, d, anchor=0)
    r = 3
    rng = np.random.default_rng(5)
    V = np.asfortranarray(rng.standard_normal((r, 3 * ne)))
    Z = np.zeros((r, 3 * ne), order="F")
    capi.check(lib.dpgo_nd_debug_emulate(ne, 2, r, len(brow), capi.iptr(brow), capi.iptr(bcol), capi.dptr(blocks), 0.0, 8, -1,
                                         4, capi.dptr(V), capi.dptr(Z), None))
    want = spla.splu(sp.csc_matrix(A)).solve(V.T).T
    assert rel(Z, want) < 1e-10


@pytest.mark.parametrize("d", [2, 3])
@pytest.mark.parametrize("force_cuts", [-1, 0, 1, 2, 3])
def test_host_sweep_matches_the_oracle(d, force_cuts):
    n = 120
    edges, T = random_graph(d, n, 140, seed=50 + d)
    b = co.tangent_dim(d)
    anchor = 5
    rng = np.random.default_rng(9)
    pairs = np.stack([rng.choice(n, 2, replace=False) for _ in range(6)] + [np.array([3, 3]), np.array([anchor, 7])])
    cov, pcov, info = emulate(edges, n, T, anchor=anchor, pairs=pairs, force_cuts=force_cuts, leaf_size=6)
    S = co.covariances_dense(co.information(T, edges, n), n, b, anchor)
    want = co.blocks_of(S, b, [(p, p) for p in range(n)])
    for p in range(n):
        if p == anchor:
            assert np.all(cov[p] == 0)
        else:
            assert rel(cov[p], want[p]) <= 1e-10, p
            assert np.array_equal(cov[p], cov[p].T)
    assert rel(pcov, co.blocks_of(S, b, pairs)) <= 1e-10
    if force_cuts >= 0:
        assert info[0] <= force_cuts + 1
    assert info[2] == n * b // 3


def test_arguments_are_checked():
    edges, T = random_graph(3, 6, 2, seed=60)
    with pytest.raises(Exception, match="anchor"):
        emulate(edges, 6, T, anchor=6)
    with pytest.raises(Exception, match="pair pose"):
        emulate(edges, 6, T, pairs=[[0, 9]])
    part = edges.take(np.nonzero(~((edges.p1 == 2) | (edges.p2 == 2) | (edges.p1 == 3) | (edges.p2 == 3)))[0])
    with pytest.raises(Exception, match="not connected"):
        emulate(part, 6, T)


def test_singular_information_is_reported_by_the_factorisation():
    """A pose whose edges all have tau = 0 is connected (kappa > 0) but its translation is free: the argument check
    passes and the factorisation's zero pivot is reported (DPGO_ERR_CUDA), as on the device."""
    from dpo_b200 import _capi as capi
    d, n = 3, 12
    edges, T = random_graph(d, n, 10, seed=70)
    p = 5
    edges.tau = np.where((edges.p1 == p) | (edges.p2 == p), 0.0, edges.tau)
    with pytest.raises(capi.DpgoError, match="not positive definite") as ei:
        emulate(edges, n, T)
    assert ei.value.code == 3
