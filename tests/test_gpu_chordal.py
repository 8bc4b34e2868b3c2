"""Chordal initialisation on the GPU (dpgo_chordal_initialization: two Jacobi-preconditioned CG solves over the hot path's
block-CSR product kernel + SO(d) projection) against the oracle's sparse direct solves and the constants the reference
publishes (vis.ipynb:108746,108748: cost 2f and gradient norm at the chordal point, r = d)."""
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import chordal_reference as cr  # noqa: E402
import structure_cases as sc  # noqa: E402
from oracle import dpgo_oracle as orc  # noqa: E402

pytestmark = pytest.mark.gpu

CHORDAL = {"sphere2500": (1971.17, 265.247), "smallGrid3D": (1561.38, 237.586), "torus3D": (24669.2, 320.591),
           "parking-garage": (1.41536, 2.3906), "CSAIL": (31.4848, 5.44293)}


@pytest.mark.parametrize("ds", ["tinyGrid3D", "smallGrid3D", "CSAIL", "sphere2500", "torus3D", "parking-garage"])
def test_chordal_gpu_matches_oracle_and_published_constants(ds, data_dir):
    from dpo_b200 import posegraph as pg
    edges, n = pg.read_g2o_file(os.path.join(data_dir, ds + ".g2o"))
    meas, _ = orc.read_g2o(os.path.join(data_dir, ds + ".g2o"))
    T, its = pg.chordalInitializationGPU(edges.d, n, edges, return_iterations=True)
    To = orc.chordal_initialization(meas, n)
    d = edges.d
    # rotations are exactly orthonormal with det +1; pose 0 is the gauge
    Rg = np.transpose(T.reshape(d, d + 1, n, order="F")[:, :d, :], (2, 0, 1))        # (n, d, d): R_p
    assert np.abs(np.einsum("nab,nac->nbc", Rg, Rg) - np.eye(d)[None]).max() <= 1e-13
    assert np.all(np.linalg.det(Rg) > 0.99)
    assert np.abs(T[:, :d] - np.eye(d)).max() <= 1e-14 and np.abs(T[:, d]).max() == 0.0
    scale = max(1.0, np.abs(To).max())
    assert np.abs(T - To).max() <= 1e-7 * scale, (its, np.abs(T - To).max())
    if ds in CHORDAL:
        p = orc.QuadraticProblem(n, d, d)
        p.set_Q(orc.construct_connection_laplacian(meas, n))
        cost, gn = CHORDAL[ds]
        assert abs(2 * p.f(T) - cost) <= 6e-6 * cost
        assert abs(p.rie_grad_norm(T) - gn) <= 6e-6 * gn


def test_chordal_gpu_large_synthetic_grid():
    """Size the host direct solves do not like: 64k poses / 256k edges; property check -- the chordal point of a graph with
    small noise is close to the ground truth and has a small cost."""
    from dpo_b200 import posegraph as pg
    edges, n, Tgt = pg.synthetic_grid_graph(40, 40, 40, edges_per_pose=4.0, seed=2)
    T, its = pg.chordalInitializationGPU(3, n, edges, return_iterations=True)
    Rg = np.transpose(T.reshape(3, 4, n, order="F")[:, :3, :], (2, 0, 1))            # (n, 3, 3)
    Rt = np.transpose(np.asarray(Tgt).reshape(3, 4, n, order="F")[:, :3, :], (2, 0, 1))
    Rrel = np.einsum("ba,nbc->nac", Rt[0], Rt)                                       # ground truth in the gauge of pose 0
    ang = np.arccos(np.clip((np.einsum("nab,nab->n", Rg, Rrel) - 1) / 2, -1, 1))
    # measurement noise is 0.05 rad per edge; the chordal point stays within a few noise levels of the ground truth
    assert np.median(ang) < 0.15 and np.max(ang) < 1.0 and its[0] > 0 and its[1] > 0


# ---------------------------------------------------------------------------------------------------------------------
# graphs the datasets never reach, against the high-precision reference of chordal_reference.py
# ---------------------------------------------------------------------------------------------------------------------
TOL = 1e-11                     # dpgo_chordal_initialization's default relative residual


def gpu(d, n, edges, **kw):
    from dpo_b200 import posegraph as pg
    return pg.chordalInitializationGPU(d, n, edges, return_iterations=True, **kw)


def bounds(edges, n, T, ref=None, M=None, R_against=None, t_against=None):
    """Per-pose rotation bounds (NaN: not bounded there) and the translation check of T against the reference (or
    against the unprojected rotations M / translations t_against of a known answer)."""
    ref = cr.chordal_reference(edges, n) if ref is None else ref
    c = cr.gap_constant(edges, n)
    tol_r = cr.rotation_tolerances(ref.rot, ref.M if M is None else M, TOL, c)
    res, bound, err, err_bound = cr.translation_check(edges, n, T, ref.R if R_against is None else R_against, TOL, c,
                                                      t_against)
    return ref, tol_r, (res, bound, err, err_bound)


def check(edges, n, T, ref=None, M=None, R_against=None, t_against=None, min_checked=0.75):
    """T from the GPU against the reference: the gauge and the poses without edges exactly; rotations of the component of
    pose 0 within their bounds, the others exactly I; the translations' certificate and their D^1/2-norm error.
    min_checked: the share of the component's rotations whose projection is well enough determined to be bounded (random
    measured rotations leave some unprojected blocks near rank-deficient)."""
    d = edges.d
    ref, tol_r, (res, bound, err, err_bound) = bounds(edges, n, T, ref, M, R_against, t_against)
    Rg, tg = cr.split_T(T, d)
    I = np.eye(d)
    assert np.array_equal(Rg[0], I) and np.all(tg[0] == 0)
    lonely = np.bincount(np.concatenate([edges.p1, edges.p2]), minlength=n) == 0
    assert np.all(Rg[lonely] == I) and np.all(tg[lonely] == 0)
    comp = ref.rot.free.reshape(n, d * d)[:, 0].copy()
    comp[0] = True
    assert np.all(Rg[~comp] == I), "rotations outside the component of pose 0 are not exactly I"
    Mx = ref.M if M is None else M
    Rx = np.array([cr.project_to_rotation(np.asarray(Mx[p], dtype=np.float64)) for p in range(n)])
    live = np.flatnonzero(comp & np.isfinite(tol_r))
    assert len(live) >= min_checked * comp.sum(), f"only {len(live)} of {comp.sum()} rotations bounded"
    err_r = np.sqrt(((Rg[live] - Rx[live]) ** 2).sum(axis=(1, 2)))
    assert np.all(err_r <= tol_r[live]), \
        f"rotation {live[np.argmax(err_r / tol_r[live])]}: err {err_r.max():.3e}, bound {tol_r[live][np.argmax(err_r / tol_r[live])]:.3e}"
    assert res <= bound, f"translation residual {res:.3e} > certificate {bound:.3e}"
    assert err <= err_bound, f"translation error {err:.3e} > {err_bound:.3e}"
    return ref, tol_r, err_bound


def tiny(d, shape, weights, seed=0):
    rng = np.random.default_rng([seed, d, len(shape)])
    pairs = {"pair": [(0, 1)], "pair_reversed": [(1, 0)], "triple": [(0, 1), (1, 2)], "triangle": [(0, 1), (1, 2), (2, 0)]}[shape]
    e = sc.edge_set(rng, d, pairs)
    if weights != "generic":
        e.kappa[:] = float(weights)
        e.tau[:] = float(weights)
    return 3 if shape in ("triple", "triangle") else 2, e


@pytest.mark.parametrize("d", [2, 3])
@pytest.mark.parametrize("weights", ["generic", "1", "4"])
@pytest.mark.parametrize("shape", ["pair", "pair_reversed", "triple", "triangle"])
def test_tiny_graphs(shape, weights, d):
    """Two and three poses converge before the first residual check (with unit or power-of-two weights the Jacobi
    preconditioner is exact and the first iteration is the answer); the converged solve must stay put, not break down."""
    n, e = tiny(d, shape, weights)
    T, its = gpu(d, n, e)
    assert 0 < its[0] <= 25 and 0 < its[1] <= 25
    check(e, n, T)


def unit_weights(e):
    e.kappa[:] = 1.0
    e.tau[:] = 1.0
    return e


@pytest.mark.parametrize("d", [2, 3])
def test_hub2100_star_is_exact(d):
    """Star rooted at pose 0 with 2100 leaves and unit weights: the Jacobi preconditioner is exact, the hub's row holds
    2101 blocks (the gather product inside CG), and every leaf's answer is proj(R_0j), t_0j."""
    case = sc.make_case("hub2100", d)
    e = unit_weights(case.edges)
    T, its = gpu(d, case.n, e)
    check(e, case.n, T)
    Rg, tg = cr.split_T(T, d)
    leaf = e.p2
    Rx = np.array([cr.project_to_rotation(R) for R in e.R])
    assert np.abs(Rg[leaf] - Rx).max() <= 32 * d * cr.U
    assert np.abs(tg[leaf] - e.t).max() <= 32 * d * cr.U * np.abs(e.t).max()


@pytest.mark.parametrize("d", [2, 3])
@pytest.mark.parametrize("name", ["hub191", "hub192", "multi_edges", "components", "tail_isolated"])
def test_structure_cases(name, d):
    case = sc.make_case(name, d)
    T, _ = gpu(d, case.n, case.edges)
    check(case.edges, case.n, T)


@pytest.mark.parametrize("d", [2, 3])
def test_pose_zero_isolated(d):
    """No edge at pose 0: every rotation is I (the rotations' right-hand side is zero), and the translations of the other
    components solve their singular systems (certificate only)."""
    rng = np.random.default_rng([5, d])
    pairs = sc.chain(range(1, 30)) + sc.chain(range(30, 50)) + [(3, 17), (40, 44)]
    e = sc.edge_set(rng, d, pairs)
    T, its = gpu(d, 52, e)
    assert its[0] == 0
    check(e, 52, T)


@pytest.mark.parametrize("d", [2, 3])
def test_non_orthonormal_measurements(d):
    """Measured rotations scaled by 1 + 1e-3 plus a non-orthogonal perturbation: the i-block is kappa R R^T, not kappa I."""
    case = sc.make_case("multi_edges", d)
    rng = np.random.default_rng([9, d])
    e = case.edges
    e.R[:] = e.R * (1 + 1e-3) + 1e-3 * rng.standard_normal(e.R.shape)
    T, _ = gpu(d, case.n, e)
    check(e, case.n, T)


@pytest.mark.parametrize("d", [2, 3])
def test_weights_over_twelve_decades_and_zero(d):
    """kappa and tau spread log-uniformly over 1e-6 .. 1e6 in one graph, some of them zero (edges whose endpoints stay
    joined by others): ill-conditioned systems, zero Jacobi entries."""
    case = sc.make_case("multi_edges", d)
    rng = np.random.default_rng([13, d])
    e = case.edges
    m = len(e)
    e.kappa[:] = 10.0 ** rng.uniform(-6, 6, m)
    e.tau[:] = 10.0 ** rng.uniform(-6, 6, m)
    e.kappa[[39, 40, 41]] = 0.0                  # the duplicated edges (5, 6), (5, 6), (12, 13)
    e.tau[[40, 42, 43]] = 0.0
    T, _ = gpu(d, case.n, e)
    check(e, case.n, T, min_checked=0.0)           # lambda_min ~ 1e-12 there: the certificate carries the test


def ground_truth(Tgt, d):
    R, t = cr.split_T(sc.in_gauge_of_pose_zero(Tgt, d), d)
    R[0], t[0] = np.eye(d), 0.0                          # the gauge, exactly
    return R, t


@pytest.mark.parametrize("d", [2, 3])
def test_noise_free_chain_20000(d):
    """A 20 000-pose noise-free chain: a deep CG run whose answer is the ground truth in the gauge of pose 0."""
    n, e, Tgt = sc.noise_free_graph(d, sc.chain(range(20000)), 20000, seed=3)
    T, its = gpu(d, n, e)
    Rgt, tgt = ground_truth(Tgt, d)
    rot = cr.rotation_system(e, n)
    ref = cr.Reference(cr.ld(Rgt), Rgt, cr.ld(tgt), rot, None)
    check(e, n, T, ref=ref, M=cr.ld(Rgt), R_against=Rgt, t_against=tgt)
    assert its[0] > 1000 and its[1] > 1000


def test_noise_free_synthetic_grid():
    from dpo_b200 import posegraph as pg
    edges, n, Tgt = pg.synthetic_grid_graph(20, 20, 10, seed=4, rot_sigma=0.0, trans_sigma=0.0)
    T, _ = gpu(3, n, edges)
    Rgt, tgt = ground_truth(Tgt, 3)
    ref = cr.Reference(cr.ld(Rgt), Rgt, cr.ld(tgt), cr.rotation_system(edges, n), None)
    check(edges, n, T, ref=ref, M=cr.ld(Rgt), R_against=Rgt, t_against=tgt)


@pytest.mark.parametrize("d", [2, 3])
def test_iteration_cap(d):
    """A 2000-pose chain needs more than 100 CG iterations: max_iter = 100 is an error that names it, the default cap
    converges."""
    from dpo_b200 import _capi as capi
    rng = np.random.default_rng([17, d])
    e = sc.edge_set(rng, d, sc.chain(range(2000)))
    with pytest.raises(capi.DpgoError, match="did not reach tol in max_iter"):
        gpu(d, 2000, e, max_iter=100)
    T, its = gpu(d, 2000, e)
    assert its[0] > 100 and its[1] > 100
    check(e, 2000, T)


# ---- metamorphic checks --------------------------------------------------------------------------------------------
@pytest.mark.parametrize("d", [2, 3])
def test_weight_scaling_is_exact(d):
    """kappa x 2^40 and tau x 2^-30 scale every operation of both solves exactly: the same T bit for bit."""
    case = sc.make_case("multi_edges", d)
    e = case.edges
    T, its = gpu(d, case.n, e)
    s = e.take(np.arange(len(e)))
    s.kappa *= 2.0 ** 40
    s.tau *= 2.0 ** -30
    Ts, its_s = gpu(d, case.n, s)
    assert its_s == its and np.array_equal(Ts, T)


def test_planar_graph_embedded_in_3d():
    """A d = 2 graph and the same graph in 3-D (R = diag(R2, 1), t = (t2, 0)): the third axis decouples exactly, and the
    planar parts agree within the sum of both runs' bounds."""
    case = sc.make_case("multi_edges", 2)
    e2 = case.edges
    m, n = len(e2), case.n
    R3 = np.zeros((m, 3, 3))
    R3[:, :2, :2] = e2.R
    R3[:, 2, 2] = 1.0
    e3 = pg_edges(3, e2, R3, np.concatenate([e2.t, np.zeros((m, 1))], axis=1))
    T2, _ = gpu(2, n, e2)
    T3, _ = gpu(3, n, e3)
    _, tol2, eb2 = check(e2, n, T2)
    _, tol3, eb3 = check(e3, n, T3)
    R2g, t2g = cr.split_T(T2, 2)
    R3g, t3g = cr.split_T(T3, 3)
    assert np.all(R3g[:, 2, :2] == 0) and np.all(R3g[:, :2, 2] == 0) and np.all(R3g[:, 2, 2] == 1) and np.all(t3g[:, 2] == 0)
    live = np.isfinite(tol2) & np.isfinite(tol3)
    er = np.sqrt(((R3g[:, :2, :2] - R2g) ** 2).sum(axis=(1, 2)))
    assert np.all(er[live] <= tol2[live] + tol3[live])
    D = cr.translation_system(e2, n, R2g).diag().reshape(n, 2)
    assert np.sqrt(np.sum(D * (t3g[:, :2] - t2g) ** 2)) <= eb2 + eb3


def pg_edges(d, e, R, t):
    from dpo_b200 import posegraph as pg
    return pg.EdgeSet(d, e.r1, e.r2, e.p1, e.p2, R, t, e.kappa, e.tau, e.weight)


@pytest.mark.parametrize("d", [2, 3])
def test_edge_order_and_repeatability(d):
    """A permuted edge list gives the same answer within twice the bounds; two runs of one list are bit for bit equal."""
    case = sc.make_case("multi_edges", d)
    e, n = case.edges, case.n
    T, _ = gpu(d, n, e)
    T2, _ = gpu(d, n, e)
    assert np.array_equal(T, T2)
    perm = np.random.default_rng([21, d]).permutation(len(e))
    Tp, _ = gpu(d, n, e.take(perm))
    _, tol_r, eb = check(e, n, T)
    _, tol_p, ebp = check(e.take(perm), n, Tp)
    Rg, tg = cr.split_T(T, d)
    Rp, tp = cr.split_T(Tp, d)
    live = np.isfinite(tol_r) & np.isfinite(tol_p)
    er = np.sqrt(((Rg - Rp) ** 2).sum(axis=(1, 2)))
    assert np.all(er[live] <= tol_r[live] + tol_p[live])
    ref = cr.chordal_reference(e, n)
    D = ref.tra.diag().reshape(n, d)
    comp = ref.tra.free.reshape(n, d)[:, 0]
    assert np.sqrt(np.sum((D * (tg - tp) ** 2)[comp])) <= eb + ebp
