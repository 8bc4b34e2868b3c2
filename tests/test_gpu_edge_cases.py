"""The device's edge-record path on the graphs of edge_cases.py, against long-double references:

  * Q (k_assemble_Q) is read back exactly: with G = 0 and 0/1 selector rows whose picked Q rows have disjoint column
    supports, every entry of X Q is one product by 1.0 plus exact zeros, i.e. bitwise an entry of Q.  Every entry is then
    within gamma_{4 count + 3} sum|terms| of the long-double Q; off-diagonal blocks are bitwise transposes of each other
    (both sum the same products in input order); diagonal blocks are checked against the bound only (kind 0 sums its
    fma chain in the order of its entry's own row, so they need not be bitwise symmetric).  Scaling every weight and
    static block by 2^k scales Q bit for bit; repeated, synchronous and stream-ordered assemblies are bitwise equal.
  * re-weighting (k_edge_weights) at every compiled (d, r) and every loss: r^2 within its bound, weights bitwise equal
    to reference_weight of the device's own r^2 (GM's product rounded on its own), the GNC counts the reference's
    classification, fixed edges untouched, and squared residuals equal to tau exactly at the GNC / Huber / TLS bounds.
"""
import numpy as np
import pytest

import edge_cases as ec
import structure_cases as sc

pytestmark = pytest.mark.gpu

DR = [(d, r) for d in (2, 3) for r in sc.RANKS[d]]
RB = 8                                               # read Q back with 8 selector rows per call
PARAMS = {"L2": (1.0, 1.0), "L1": (1.0, 1.0), "Huber": (1.0, 2.0), "TLS": (1.0, 2.5), "GM": (1.0, 1.0)}


@pytest.fixture(scope="module")
def cases():
    return {}


def get(cases, name, d):
    if (name, d) not in cases:
        cases[(name, d)] = ec.make_case(name, d)
    return cases[(name, d)]


def problem(c, r=RB, edges=None, static_blocks=None, precs=()):
    import dpo_b200 as dp
    gp = dp.QuadraticProblem(c.n, c.d, r, preconditioners=precs)
    gp.setEdges(c.edges if edges is None else edges, static_pose=c.static_pose,
                static_blocks=c.static_blocks if static_blocks is None else static_blocks, fixed=c.fixed)
    return gp


def read_q(gp, c):
    gp.setG(None)
    return ec.read_back(gp.EucGrad, c, gp.r)


def bitwise_equal(a, b):
    return set(a) == set(b) and all(np.array_equal(a[k], b[k]) for k in a)


# ---------------------------------------------------------------------------------------------------------------------
# Q
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", ec.READBACK)
@pytest.mark.parametrize("d", [2, 3])
def test_assembled_q(name, d, cases):
    """within the bound, off-diagonal blocks bitwise transposed, zero-weight-only blocks exactly zero, repeatable, and
    the same as setQ_blocks of the same doubles up to the bound"""
    c = get(cases, name, d)
    qref = ec.q_reference(c)
    gp = problem(c)
    got = read_q(gp, c)
    ec.check_q(got, qref, name)
    if not qref:                                                     # m = 0, no static block: Q = 0
        X = np.random.default_rng(1).standard_normal((RB, c.N))
        assert gp.num_blocks() == 0 and not gp.EucGrad(X).any()
    for (i, j), B in got.items():
        if i != j:
            assert np.array_equal(B, got[(j, i)].T), (i, j)
        if not qref[(i, j)][1].any():                                 # only zero-weight terms
            assert not B.any(), (i, j)
    if name == "wide_weights":
        assert sum(not qref[k][1].any() for k in qref) >= 9             # the zero-weight component's blocks
    assert bitwise_equal(read_q(problem(c), c), got)                  # a second handle: the same bits
    host = problem(c)
    host.setQ_blocks(*c.triplets(), preconditioners=())
    hq = read_q(host, c)
    for ij, (ref, mag, cnt) in qref.items():
        assert (abs(ec.ld(hq[ij]) - ec.ld(got[ij])) <= 2 * ec.LD(ec.gamma(4 * cnt + 3)) * mag).all(), ij


@pytest.mark.parametrize("name", ec.READBACK)
@pytest.mark.parametrize("d", [2, 3])
def test_q_scales_and_permutes(name, d, cases):
    """weights and static blocks times 2^k give Q times 2^k bit for bit (set_edges and set_edge_weights); a permuted
    edge order stays within the bound"""
    c = get(cases, name, d)
    gp = problem(c)
    base = read_q(gp, c)
    for k in (3, -7):
        s = 2.0 ** k
        e = c.edges.take(np.arange(len(c.edges)))
        e.weight = e.weight * s
        sb = None if c.static_blocks is None else c.static_blocks * s
        got = read_q(problem(c, edges=e, static_blocks=sb), c)
        assert bitwise_equal(got, {ij: B * s for ij, B in base.items()}), k
        if c.static_pose is None and len(c.edges):
            gp.setEdgeWeights(e.weight)
            assert bitwise_equal(read_q(gp, c), got), k
            gp.setEdgeWeights(c.edges.weight)
    if len(c.edges) > 1:
        perm = np.random.default_rng(2).permutation(len(c.edges))
        ec.check_q(read_q(problem(c, edges=c.edges.take(perm)), c), ec.q_reference(c), name + " permuted")


@pytest.mark.parametrize("name", ["star2100", "clique60", "repeated_pair", "wide_kappa_tau", "static_twice"])
@pytest.mark.parametrize("d", [2, 3])
def test_sync_and_async_weights_give_the_same_q(name, d, cases):
    import dpo_b200 as dp
    import torch
    c = get(cases, name, d)
    w1 = np.random.default_rng(3).uniform(0.0, 2.0, len(c.edges))
    w1[::5] = 0.0
    precs = (dp.PRECOND_BLOCK_JACOBI, dp.PRECOND_SPARSE_EXACT)
    sync, asy = problem(c, precs=precs), problem(c, precs=precs)
    sync.setEdgeWeights(w1)
    torch.cuda.synchronize()
    asy.setEdgeWeightsAsync(torch.tensor(w1, dtype=torch.float64, device="cuda"))
    asy.sync()
    qs, qa = read_q(sync, c), read_q(asy, c)
    assert bitwise_equal(qs, qa)
    ec.check_q(qs, ec.q_reference(c, weight=w1), name)


# ---------------------------------------------------------------------------------------------------------------------
# re-weighting
# ---------------------------------------------------------------------------------------------------------------------
def random_iterate(c, r, seed):
    rng = np.random.default_rng([seed, c.d, r])
    X = rng.standard_normal((r, c.N))
    Xt = ec.tiles_of(X, c.n, c.dh)
    Y = np.linalg.qr(Xt[:, :, :c.d])[0]                              # a Stiefel point per pose
    Xt[:, :, :c.d] = Y
    Xt[:, :, c.d] *= 3.0
    return np.ascontiguousarray(np.transpose(Xt, (1, 0, 2)).reshape(r, c.N))


def check_reweight(gp, c, X, cost, mu, param, w0):
    """one synchronous re-weight: r^2 within its bound, weights bitwise the reference's, fixed edges untouched, counts"""
    w, r2 = gp.robustReweight(cost, mu=mu, param=param)
    ref, bound = ec.residual_reference(c, X)
    assert (abs(ec.ld(r2) - ref) <= bound).all(), cost
    fixed = np.zeros(len(w), dtype=bool) if c.fixed is None else c.fixed.astype(bool)
    want = ec.reference_weight(cost, r2, mu, param)
    free = ~fixed
    ok = (w == want) | (np.isnan(w) & np.isnan(want))
    assert ok[free].all(), (cost, mu, param, np.flatnonzero(~ok & free)[:5], w[~ok & free][:5], want[~ok & free][:5])
    assert np.array_equal(w[fixed], w0[fixed]), cost
    assert gp.gncCounts() == ec.classify(want[free]), cost
    return w, r2


@pytest.mark.parametrize("d,r", DR)
def test_reweight_every_loss(d, r, cases):
    """clique60 with every third edge fixed and a seeded iterate, every loss, sync and stream-ordered"""
    import dpo_b200 as dp
    c = get(cases, "clique60", d)
    c = ec.EdgeCase(c.name, d, c.n, c.edges, c.target, fixed=(np.arange(len(c.edges)) % 3 == 0).astype(np.int32))
    X = random_iterate(c, r, 5)
    w0 = c.edges.weight.copy()
    precs = (dp.PRECOND_BLOCK_JACOBI,)
    sync, asy = problem(c, r, precs=precs), problem(c, r, precs=precs)
    sync.upload_X(X)
    asy.upload_X(X)
    _, r2 = sync.robustReweight("L2")
    med = float(np.median(r2))
    runs = [(k, *PARAMS[k]) for k in PARAMS] + [("Huber", 1.0, np.sqrt(med)), ("TLS", 1.0, np.sqrt(med)),
                                                ("GNC_TLS", 1.0, np.sqrt(med)), ("GNC_TLS", 0.05, np.sqrt(med)),
                                                ("GNC_TLS", 20.0, np.sqrt(med))]
    classes = set()
    for cost, mu, param in runs:
        w, r2 = check_reweight(sync, c, X, cost, mu, param, w0)
        asy.robustReweightAsync(cost, mu, param)
        asy.sync()
        wd, rd = (t.cpu().numpy() for t in asy.edgeWeightsDevice())
        assert np.array_equal(wd, w) and np.array_equal(rd, r2), cost
        assert asy.gncCounts() == sync.gncCounts(), cost
        if cost == "GNC_TLS":
            classes |= {k for k, v in enumerate(sync.gncCounts()) if v}
        if r == sc.RANKS[d][0] or r == sc.MAX_RANK:
            assert bitwise_equal(read_q(sync, c), read_q(asy, c)), cost
            sync.upload_X(X)                                          # X Q left the selector rows resident
            asy.upload_X(X)
    assert classes == {0, 1, 2}                                       # every GNC class reached


@pytest.mark.parametrize("d,r", DR)
def test_weights_at_the_bounds(d, r):
    """r^2 = tau exactly (R = I, t = 0, one rotation block everywhere, p2 - p1 = e1), tau at every bound either GNC
    formula draws and one ulp either side: the weights, and so the counts, are the reference's.  Huber / TLS at c^2,
    GM over 12 decades (its product rounded on its own) and L1 at r = 0 (+inf) on the same path."""
    gnc = ec.gnc_boundary_set()
    rng = np.random.default_rng(6)
    extra = np.concatenate([[0.0], 10.0 ** rng.uniform(-6, 6, 300)])
    thresholds = (0.5, 3.0)
    for cst in ("Huber", "TLS"):
        for t in thresholds:
            extra = np.concatenate([extra, ec.boundary_probes(cst, 1.0, t)])
    taus = np.unique(np.concatenate([[v for _, _, v in gnc], extra]))
    c = ec.boundary_case(d, taus)
    X = ec.boundary_iterate(r, d, c.n)
    gp = problem(c, r)
    gp.upload_X(X)
    runs = sorted({(mu, cb) for mu, cb, _ in gnc})
    calls = [("GNC_TLS", mu, cb) for mu, cb in runs] + [("GM", 1.0, 1.0), ("L1", 1.0, 1.0), ("L2", 1.0, 1.0)]
    calls += [(cst, 1.0, t) for cst in ("Huber", "TLS") for t in thresholds]
    for cost, mu, param in calls:
        w, r2 = gp.robustReweight(cost, mu=mu, param=param)
        assert np.array_equal(r2, taus)
        want = ec.reference_weight(cost, r2, mu, param)
        bad = ~((w == want) | (np.isnan(w) & np.isnan(want)))
        assert not bad.any(), (cost, mu, param, r2[bad][:4], w[bad][:4], want[bad][:4])
        assert gp.gncCounts() == ec.classify(want), (cost, mu, param)
    w, _ = gp.robustReweight("L1")
    assert w[taus == 0.0][0] == np.inf


@pytest.mark.parametrize("d", [2, 3])
def test_counts_over_a_million_edges(d, cases):
    c = get(cases, "path1e6", d)
    r = d
    rng = np.random.default_rng(8)
    Rp = sc.random_rotations(rng, c.n, d)
    X = np.concatenate([Rp, rng.uniform(-5, 5, (c.n, d, 1))], axis=2)       # (n, d, d+1) pose tiles
    X = np.ascontiguousarray(np.transpose(X, (1, 0, 2)).reshape(d, c.N))
    gp = problem(c, r)
    gp.upload_X(X)
    _, r2 = gp.robustReweight("L2")
    ref, bound = ec.residual_reference(c, X)
    assert (abs(ec.ld(r2) - ref) <= bound).all()
    cb = float(np.sqrt(np.median(r2)))
    free = ~c.fixed.astype(bool)
    for mu in (0.1, 1.0, 10.0):
        w, r2 = gp.robustReweight("GNC_TLS", mu=mu, param=cb)
        want = ec.reference_weight("GNC_TLS", r2, mu, cb)
        assert np.array_equal(w[free], want[free])
        counts = gp.gncCounts()
        assert counts == ec.classify(want[free]) and sum(counts) == int(free.sum()), (mu, counts)
        assert mu < 1.0 or min(counts) > 0, (mu, counts)          # bounds at med/2 .. 2 med and tighter: all three
        gp.robustReweightAsync("GNC_TLS", mu, cb)
        assert gp.gncCounts() == counts
