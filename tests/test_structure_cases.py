"""CPU checks of the structure cases and comparators of structure_cases.py / pose_references.py:

  * every case reaches the branch it is built for, from host facts only;
  * the componentwise comparators pass a float64 stand-in of each kernel and reject a dropped or a transposed block;
  * the 40-digit references agree with numpy on well-conditioned inputs;
  * the host emulation of the sparse exact preconditioner's plan matches the sparse LU on every case, at the full grid
    of an H100 and at a cluster grid."""
import numpy as np
import pytest
import scipy.sparse as sp
from scipy.sparse.csgraph import connected_components

import pose_references as pr
import structure_cases as sc
from oracle import dpgo_oracle as orc
from test_nd_plan import dense_reference, emulate, relerr

ALL = [(name, d) for name in sc.CASE_NAMES for d in (2, 3)]


@pytest.fixture(scope="module")
def cases():
    return {}


def get(cases, name, d):
    if (name, d) not in cases:
        cases[(name, d)] = sc.make_case(name, d)
    return cases[(name, d)]


@pytest.mark.parametrize("name,d", [(n, d) for (n, d) in ALL if n != "clique700"])
def test_case_reaches_its_branch(name, d, cases):
    c = get(cases, name, d)
    rb = c.row_blocks()
    nb = int(rb.sum())
    groups = sc.tma_groups(rb)
    assert c.n == len(rb) and c.Q().shape == (c.N, c.N)
    if name == "single":
        assert c.n == 1 and nb == 0 and groups is None
    elif name == "single_prior":
        assert c.n == 1 and nb == 1 and len(groups) == 1
    elif name in ("pair", "triple"):
        assert c.n == {"pair": 2, "triple": 3}[name] and nb == 3 * c.n - 2 and len(groups) == 1
    elif name == "hub191":
        assert rb.max() == sc.SPMV_GROUP_BLOCKS and groups is not None
        assert any(g[3] - g[2] == sc.SPMV_GROUP_BLOCKS for g in groups)       # the hub row fills one stage
    elif name == "hub192":
        assert rb.max() == sc.SPMV_GROUP_BLOCKS + 1 and groups is None
    elif name == "hub2100":
        assert 1 + 1 + rb.max() > sc.SP_CACHE_INTS and groups is None      # any CTA holding the hub row
        assert (rb[1:] == 2).all()                                          # every leaf: itself and the hub
    elif name == "tail_isolated":
        trailing = len(rb) - (np.flatnonzero(rb).max() + 1)
        assert nb % 4 == 0 and trailing >= 400 and (rb[:np.flatnonzero(rb).max()] == 0).sum() >= 3
        assert sc.zero_byte_index_groups(groups)
    elif name == "components":
        A = sp.csr_matrix((np.ones(len(c.edges)), (c.edges.p1, c.edges.p2)), shape=(c.n, c.n))
        assert connected_components(A, directed=False)[0] == 4
    elif name == "multi_edges":
        pairs = list(zip(c.edges.p1.tolist(), c.edges.p2.tolist()))
        assert len(pairs) > len(set(pairs))                                 # duplicated
        assert any(a > b for a, b in pairs)                                 # reversed
        assert any((b, a) in set(pairs) for a, b in pairs)                  # both directions
    elif name == "long_chain":
        assert c.n == 5000 and len(c.edges) == 4999
    assert c.N <= sc.DENSE_MAX_N or name == "long_chain"


@pytest.mark.parametrize("d", [2, 3])
def test_clique_reaches_its_branch(d, cases):
    """clique700: every row holds every pose (one dissection leaf, larger than a step's tile capacity), with an even pose
    count for d = 3 and an odd one for d = 2, whose last 8-row panel of the single dense level is half used"""
    c = get(cases, "clique700", d)
    rb = c.row_blocks()
    assert c.n == len(rb) and c.Q().shape == (c.N, c.N)
    assert c.N == {3: 2800, 2: 2103}[d] and rb.min() == c.n
    assert all(c.n > sc.nd_ycap_tiles(r, c.dh) for r in sc.RANKS[d]) and c.n % 2 == {3: 0, 2: 1}[d]
    assert c.N <= sc.DENSE_MAX_N


@pytest.mark.parametrize("name,d", [(n, d) for (n, d) in ALL if n not in ("clique700",)] + [("clique700", 3)])
def test_emulated_plan_on_structure_cases(name, d, cases):
    """dpgo_nd_debug_emulate (the kernel's plan interpreted on the host) against the sparse LU, at the H100's full grid
    (132 CTAs) and at a cluster grid (16 CTAs)"""
    c = get(cases, name, d)
    brow, bcol, blocks = c.triplets()
    if len(brow) == 0:                       # an empty Q: one zero block keeps the triplet arrays non-empty
        brow, bcol, blocks = np.array([0]), np.array([0]), np.zeros((1, c.dh, c.dh))
    rng = np.random.default_rng(7)
    for r in sc.large_ranks(d):
        V = rng.standard_normal((r, c.N))
        ref = dense_reference(c.n, c.dh, brow, bcol, blocks, V)
        for grid in (132, 16):
            Z, info = emulate(c.n, d, r, brow, bcol, blocks, V, grid=grid)
            assert relerr(Z, ref) <= 1e-11, (name, d, r, grid, info)
            if name == "clique700":
                assert info["max_own"] == c.N and info["max_ytiles"] == sc.nd_ycap_tiles(r, c.dh)   # one leaf, chunked
            assert info["max_ytiles"] <= sc.nd_ycap_tiles(r, c.dh) and info["max_slots"] <= sc.nd_slot_cap(r), (r, info)


# ---------------------------------------------------------------------------------------------------------------------
# the comparators have power
# ---------------------------------------------------------------------------------------------------------------------
def _drop_block(Q, dh, i, j):
    Q = sp.lil_matrix(Q)
    Q[i * dh:(i + 1) * dh, j * dh:(j + 1) * dh] = 0.0
    return sp.csr_matrix(Q)


def _transpose_block(Q, dh, i, j):
    Q = sp.lil_matrix(Q)
    B = Q[i * dh:(i + 1) * dh, j * dh:(j + 1) * dh].toarray()
    Q[i * dh:(i + 1) * dh, j * dh:(j + 1) * dh] = B.T
    return sp.csr_matrix(Q)


@pytest.mark.parametrize("d,r", [(3, 5), (2, 3)])
def test_product_comparator_has_power(d, r):
    c = sc.make_case("hub191", d)
    Q = c.Q()
    K = sc.pose_K(c, d)
    rng = np.random.default_rng(1)
    X = orc.manifold_project(rng.standard_normal((r, c.N)), d)
    G = rng.standard_normal((r, c.N))
    sc.check_product((Q @ X.T).T, Q, X, K)                       # float64 stand-in
    sc.check_product((Q @ X.T).T + G, Q, X, K, G=G)
    groups = sc.tma_groups(c.row_blocks())
    last_row = max(g[1] - 1 for g in groups if g[3] > g[2] and g[0] > 0)   # the last row of a later TMA group
    Qb = sp.csr_matrix(Q).tobsr(blocksize=(c.dh, c.dh))
    last_col = int(Qb.indices[Qb.indptr[last_row + 1] - 1])
    off = next(j for j in Qb.indices[Qb.indptr[1]:Qb.indptr[2]] if j != 1)   # an off-diagonal block of row 1
    mutants = {"hub row block dropped": _drop_block(Q, c.dh, 0, 150),
               "last block of a group's last row dropped": _drop_block(Q, c.dh, last_row, last_col),
               "block transposed": _transpose_block(Q, c.dh, 1, int(off))}
    for what, Qm in mutants.items():
        with pytest.raises(AssertionError):
            sc.check_product((Qm @ X.T).T, Q, X, K)
            pytest.fail(what)


def test_riemannian_comparators_have_power():
    d, r = 3, 4
    c = sc.make_case("tail_isolated", d)
    Q = c.Q()
    K = sc.pose_K(c, d)
    rng = np.random.default_rng(2)
    X = orc.manifold_project(rng.standard_normal((r, c.N)), d)
    G = rng.standard_normal((r, c.N))
    V = orc.tangent_project(X, rng.standard_normal((r, c.N)), d)
    op = orc.QuadraticProblem(c.n, d, r)
    op.set_Q(Q)
    op.set_G(G)
    Qm = _drop_block(Q, c.dh, 100, 101)
    opm = orc.QuadraticProblem(c.n, d, r)
    opm.set_Q(Qm)
    opm.set_G(G)
    C = sc.stage_c(K, r, d)
    # projection: the float64 formula passes, a projection without the symmetrisation does not
    ref, mag = sc.projection_ref(X, G, d)
    sc.check_elementwise(orc.tangent_project(X, G, d), ref, mag, C, "projection")
    Xt, Gt = sc.tiles(X, d), sc.tiles(G, d)
    bad = Gt.copy()
    bad[:, :, :d] -= np.einsum("ani,nij->anj", Xt[:, :, :d], np.einsum("ani,anj->nij", Xt[:, :, :d], Gt[:, :, :d]))
    with pytest.raises(AssertionError):
        sc.check_elementwise(bad.reshape(G.shape), ref, mag, C, "projection without sym")
    # Riemannian gradient and Hessian
    ref, mag, _, _ = sc.rgrad_ref(Q, G, X, d)
    sc.check_elementwise(op.rie_grad(X), ref, mag, C, "RieGrad")
    with pytest.raises(AssertionError):
        sc.check_elementwise(opm.rie_grad(X), ref, mag, C, "RieGrad, dropped block")
    ref, mag = sc.rhess_ref(Q, G, X, V, d)
    sc.check_elementwise(op.rie_hess(X, op.euc_grad(X), V), ref, mag, C, "RieHessianEta")
    with pytest.raises(AssertionError):
        sc.check_elementwise(opm.rie_hess(X, opm.euc_grad(X), V), ref, mag, C, "RieHessianEta, dropped block")
    # cost
    val, mag = sc.f_ref(Q, G, X)
    sc.check_scalar(op.f(X), val, mag, K, X.size, "f")
    with pytest.raises(AssertionError):
        sc.check_scalar(opm.f(X), val, mag, K, X.size, "f, dropped block")
    # block-Jacobi and exact preconditioners
    ref, mag, cond = sc.jacobi_ref(Q, X, V, d)
    jc = sc.stage_c(K, r, d) + 4 * sc.per_elem(cond, r, d)
    oo = orc.QuadraticOptimizer(op, precond="jacobi")
    sc.check_elementwise(oo._apply_precond(X, V), ref, mag, jc, "Jacobi")
    opd = orc.QuadraticProblem(c.n, d, r)
    opd.set_Q(_drop_block(Q, c.dh, 100, 100))
    oom = orc.QuadraticOptimizer(opd, precond="jacobi")
    with pytest.raises(AssertionError):
        sc.check_elementwise(oom._apply_precond(X, V), ref, mag, jc, "Jacobi, dropped diagonal block")
    ref, kappa = sc.exact_ref(Q, X, V, d)
    sc.check_exact(op.precondition(X, V), ref, kappa, d, 64, "exact")
    with pytest.raises(AssertionError):
        sc.check_exact(opm.precondition(X, V), ref, kappa, d, 64, "exact, dropped block")


# ---------------------------------------------------------------------------------------------------------------------
# the 40-digit references
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("r,d", [(3, 3), (5, 3), (2, 2), (5, 2)])
def test_mp_references_agree_with_numpy(r, d):
    rng = np.random.default_rng(3)
    for _ in range(5):
        M = pr.with_singular_values(rng, r, d, rng.uniform(0.5, 2.0, d))
        assert np.abs(pr.polar(M) - orc.project_to_stiefel(M)).max() <= 1e-14
        U, S, Vt = np.linalg.svd(M, full_matrices=False)
        assert np.abs(pr.svd(M)[1] - S).max() <= 1e-14
        Qn, Rn = np.linalg.qr(M)
        Qn = Qn * np.sign(np.diag(Rn))[None, :]
        assert np.abs(pr.qf(M) - Qn).max() <= 1e-14
        if r == d:
            for sgn in (1.0, -1.0):
                Md = pr.with_singular_values(rng, d, d, [2.0, 1.0, 0.5][:d], det_sign=sgn)   # separated: well-posed
                assert np.abs(pr.rotation(Md) - orc.project_to_rotation_group(Md)).max() <= 1e-13
