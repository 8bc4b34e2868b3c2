"""RTR steps built to reach every trust-region decision of the step kernel, with the oracle's decision trace to prove it.
Helper module of test_rtr_cases.py (CPU) and test_gpu_rtr_branches.py (GPU); no fixtures.

The reference's updateX constants from a chordal start only ever reach the tCG's residual and iteration-cap exits with
rho > 0.75.  Each case below names the branch it is built for (`RtrCase.target`) and a predicate on the oracle's trace
that decides whether the branch is reached (`REACHES`).  A case is built for one oracle preconditioner ("exact" stands
for both exact operators of the library), d and r; where a start or a radius has to be searched, the search is seeded
and takes the first candidate whose path reaches the branch with every decision clear of its threshold by at least
`margin_floor(precond)` (relative; see `margins`).  With that margin any correct kernel takes the oracle's path.
"""
from __future__ import annotations

import math
from dataclasses import dataclass, field
from typing import Callable, Dict, Optional, Tuple

import numpy as np
import scipy.sparse as sp

import structure_cases as sc
from oracle import dpgo_oracle as orc

RANKS = sc.RANKS
PRECONDS = ("exact", "jacobi", "none")
NEGCURV, EXCREGION, LCON, SCON, MAXITER = orc.TCG_NEGCURV, orc.TCG_EXCREGION, orc.TCG_LCON, orc.TCG_SCON, orc.TCG_MAXITER
SIGMAS = (0.3, 1.0, 0.1)


def margin_floor(precond: str) -> float:
    """un-preconditioned CG amplifies summation-order differences (cf. test_rtr_single_step_sequence's tolerances)"""
    return 1e-4 if precond == "none" else 1e-6


@dataclass
class RtrCase:
    name: str
    d: int
    r: int
    precond: str
    n: int
    Q: sp.csr_matrix
    G: Optional[np.ndarray]
    X: np.ndarray
    tol: float
    iters: int
    inner: int
    radius: float
    target: str
    mutations: Tuple[str, ...] = ()          # oracle mutations of this case's branch that must change what the GPU compares
    trace: list = field(default_factory=list)
    result: Optional[orc.OptResult] = None
    X_out: Optional[np.ndarray] = None

    def attempts(self):
        return attempts(self.trace)


def run(Q, G, X, d, r, precond, tol, iters, inner, radius, mutation=None):
    """the oracle's optimize() with the decision trace on: (X out, result, trace)"""
    n = X.shape[1] // (d + 1)
    op = orc.QuadraticProblem(n, d, r)
    op.set_Q(Q)
    if G is not None:
        op.set_G(G)
    oo = orc.QuadraticOptimizer(op, precond=precond)
    oo.tr_tolerance, oo.tr_iterations, oo.tr_max_inner, oo.tr_initial_radius = tol, iters, inner, radius
    oo.trace, oo.mutation = [], mutation
    Y = oo.optimize(X)
    return Y, oo.result, oo.trace


def attempts(trace):
    return [t[1:] for t in trace if t[0] == "attempt"]            # (status, inner, rho, Delta, accepted)


def margins(trace):
    """relative margin of every comparison on the path: |lhs - rhs| / max(|lhs|, |rhs|, scale); both sides exactly 0
    (sums of exact zeros, the same in any order) count as infinitely clear"""
    out = []
    for t in trace:
        if t[0] != "cmp":
            continue
        _, what, lhs, rhs, scale, _ = t
        den = max(abs(lhs), abs(rhs), scale)
        out.append((what, math.inf if den == 0.0 else abs(lhs - rhs) / den))
    return out


def min_margin(trace):
    return min((m for _, m in margins(trace)), default=math.inf)


def inner_decisions(trace):
    """per attempt, the list of (what, taken) of its tCG comparisons, in order"""
    out, cur = [], []
    for t in trace:
        if t[0] == "cmp" and t[1] in ("d_Hd <= 0", "e_new >= Delta^2", "nr <= n0 min(n0, 0.1)"):
            cur.append((t[1], t[5]))
        elif t[0] == "attempt":
            out.append(cur)
            cur = []
    return out


# ---------------------------------------------------------------------------------------------------------------------
# problems
# ---------------------------------------------------------------------------------------------------------------------
def lattice(d, seed, side=5):
    """side x side lattice: path along the rows plus the column neighbours; measurements of random ground-truth poses
    with small noise, so that a random start sees mostly positive curvature, as on the shipped datasets"""
    from dpo_b200 import posegraph as pg
    rng = np.random.default_rng([seed, d, 77])
    n = side * side
    ids = np.arange(n).reshape(side, side)
    pairs = sc.chain(range(n)) + [(int(ids[i, j]), int(ids[i + 1, j])) for i in range(side - 1) for j in range(side)]
    p1, p2 = np.array(pairs).T
    Rt, tt = sc.random_rotations(rng, n, d), 3.0 * rng.standard_normal((n, d))
    m = len(pairs)
    I = np.eye(d)
    noise = np.array([orc.project_to_rotation_group(I + 0.05 * (Rn - I)) for Rn in sc.random_rotations(rng, m, d)])
    R = np.einsum("mji,mjk->mik", Rt[p1], Rt[p2]) @ noise
    t = np.einsum("mji,mj->mi", Rt[p1], tt[p2] - tt[p1]) + 0.05 * rng.standard_normal((m, d))
    z = np.zeros(m, dtype=np.int64)
    edges = pg.EdgeSet(d, z, z, p1, p2, R, t, rng.uniform(10.0, 100.0, m), rng.uniform(1.0, 10.0, m))
    T = np.concatenate([Rt, tt[:, :, None]], axis=2).transpose(1, 0, 2).reshape(d, (d + 1) * n)
    return n, sc.Case("lattice", d, n, edges, "").Q(), T


def saddle(d, r, seed, n=6):
    """f = 0.5 <Q, X^T X> + <X, G> with a weak chain Q and a rotation-only G: an indefinite Hessian at most points,
    negative curvature near the maximiser of <X, G>"""
    rng = np.random.default_rng([seed, d, r, 78])
    Q = 1e-3 * sc.Case("chain", d, n, sc.edge_set(rng, d, sc.chain(range(n))), "").Q()
    G = rng.standard_normal((r, (d + 1) * n))
    G[:, d::d + 1] = 0.0
    return n, Q, G, rng


def random_start(rng, r, d, n):
    return orc.manifold_project(rng.standard_normal((r, (d + 1) * n)), d)


def near_start(rng, T, r, sigma):
    """the lifted ground truth with noise of size sigma: far enough for long steps, near enough for positive curvature"""
    d = T.shape[0]
    X = orc.fixed_stiefel_variable(d, r) @ T
    return orc.manifold_project(X + sigma * rng.standard_normal(X.shape), d)


# ---------------------------------------------------------------------------------------------------------------------
# the cases
# ---------------------------------------------------------------------------------------------------------------------
def _first(st, inner=None):
    def f(c):
        a = c.attempts()
        return bool(a) and a[0][0] == st and (inner is None or inner(a[0][1]))
    return f


def _reject_then_accept(k):
    def f(c):
        a = c.attempts()
        return c.iters == 1 and len(a) == k + 1 and all(not x[4] for x in a[:k]) and a[k][4]
    return f


def _giveup(c):
    a = c.attempts()
    return c.iters == 1 and len(a) == 12 and not any(x[4] for x in a) and np.array_equal(c.X_out, c.X)


def _negcurv_after_interior(c):
    for dec, a in zip(inner_decisions(c.trace), c.attempts()):
        if a[0] == NEGCURV and dec[-1] == ("d_Hd <= 0", True) and ("nr <= n0 min(n0, 0.1)", False) in dec:
            return True
    return False


def _capped(c):
    """an attempt at 5 Delta0 after a growth that the cap cut (2 Delta > 5 Delta0), which then hits the boundary again"""
    a = c.attempts()
    cap = 5.0 * c.radius
    for i in range(len(a) - 1):
        st, _, rho, De, _ = a[i]
        if st in (NEGCURV, EXCREGION) and rho > 0.75 and 2.0 * De > cap and De < cap and a[i + 1][3] == cap:
            return any(x[3] == cap and x[0] in (NEGCURV, EXCREGION) for x in a[i + 1:])
    return False


def _shrunk_and_accepted(c):
    a = c.attempts()
    return c.iters > 1 and any(0.1 < x[2] < 0.25 and x[4] for x in a[:-1])


def _multi_reject(c):
    a = c.attempts()
    return c.iters > 1 and any(not a[i][4] and a[i][2] > 0.0 and a[i + 1][4] for i in range(len(a) - 1))


def _tol_stop(c):
    a = c.attempts()
    return 1 < len(a) < c.iters and c.trace[-1][1] == "gradnorm < tol" and c.trace[-1][5]


def _early(c):
    return not c.attempts() and np.array_equal(c.X_out, c.X)


def _stationary(c):
    return _giveup(c) and all(x[0] == NEGCURV and x[1] == 1 for x in c.attempts())


REACHES: Dict[str, Tuple[str, Callable]] = {
    "boundary_first": ("tCG boundary exit (EXCREGION) at the first inner iteration", _first(EXCREGION, lambda k: k == 1)),
    "boundary_later": ("tCG boundary exit after >= 2 interior iterations", _first(EXCREGION, lambda k: k >= 3)),
    "negcurv_first": ("negative curvature at the first inner iteration", _first(NEGCURV, lambda k: k == 1)),
    "negcurv_later": ("negative curvature after a positive-curvature interior iteration", _negcurv_after_interior),
    "scon": ("superlinear residual stop (SCON): n0 < 0.1", _first(SCON)),
    "maxiter_1": ("iteration cap with tr_max_inner = 1", _first(MAXITER, lambda k: k == 1)),
    "reject_1": ("single mode: one rejection, Delta / 4, then accepted", _reject_then_accept(1)),
    "reject_3": ("single mode: >= 3 rejections, then accepted", lambda c: any(_reject_then_accept(k)(c) for k in range(3, 12))),
    "giveup": ("single mode: 12 rejections, the input returned", _giveup),
    "multi_cap": ("multi mode: radius growth cut by the 5 Delta0 cap", _capped),
    "multi_shrink": ("multi mode: 0.1 < rho < 0.25, accepted and shrunk, then another attempt", _shrunk_and_accepted),
    "multi_reject": ("multi mode: a rejection at 0 < rho <= 0.1 (z0 reused), then an acceptance", _multi_reject),
    "multi_tol": ("multi mode: stop on the gradient tolerance before tr_iterations", _tol_stop),
    "early_exit": ("gradient norm below the tolerance at the start: no attempt", _early),
    "stationary": ("exactly stationary start, tolerance 0: NaN-free give-up", _stationary),
}
CASE_NAMES = tuple(REACHES)

MUTATIONS = {
    "boundary_first": ("wrong_root",), "boundary_later": ("wrong_root",), "negcurv_first": ("wrong_root",),
    "negcurv_later": ("wrong_root",), "reject_1": ("shrink_half",), "reject_3": ("shrink_half",),
    "giveup": ("giveup_11",), "multi_cap": ("no_cap", "stale_z0"), "multi_shrink": ("shrink_half",),
    "multi_reject": ("shrink_half", "accept_positive", "stale_z0"), "multi_tol": ("stale_z0",),
}


def _finish(c: RtrCase, mutation=None) -> RtrCase:
    c.X_out, c.result, c.trace = run(c.Q, c.G, c.X, c.d, c.r, c.precond, c.tol, c.iters, c.inner, c.radius, mutation)
    return c


# Un-preconditioned CG drifts from another summation order by more than any margin after a few dozen iterations (the
# kernel took one more or fewer iteration than the oracle on 35- to 70-iteration solves), so its solves stay short.
NONE_MAX_INNER = 15


def _ok(c):
    short = c.precond != "none" or all(a[1] <= NONE_MAX_INNER for a in c.attempts())
    return REACHES[c.name][1](c) and short and min_margin(c.trace) >= margin_floor(c.precond)


def _search(make, tries=40):
    """first of the seeded candidates make(seed) that reaches its branch with sufficient margins"""
    for seed in range(tries):
        c = make(seed)
        if c is not None and _ok(_finish(c)):
            return c
    raise RuntimeError("no candidate reaches the branch")


def e_new_sequence(Q, G, X, d, r, precond, inner):
    """the first attempt's e_new at each interior iteration, with a radius no step reaches"""
    _, _, tr = run(Q, G, X, d, r, precond, 0.0, 1, inner, 1e8)
    out = []
    for t in tr:
        if t[0] == "attempt":
            break
        if t[0] == "cmp" and t[1] == "e_new >= Delta^2":
            out.append(t[2])
    return out


def make_case(name: str, d: int, r: int, precond: str) -> RtrCase:
    target = REACHES[name][0]
    muts = MUTATIONS.get(name, ())
    pi = PRECONDS.index(precond)

    def mk(n, Q, G, X, tol, iters, inner, radius):
        return RtrCase(name, d, r, precond, n, Q, G, X, tol, iters, inner, radius, target, muts)

    def lat(seed):
        """a lattice problem and a start near its ground truth, the distance cycling through SIGMAS"""
        n, Q, T = lattice(d, seed)
        rng = np.random.default_rng([seed, d, r, pi, CASE_NAMES.index(name)])
        return n, Q, near_start(rng, T, r, SIGMAS[seed % len(SIGMAS)])

    if name in ("boundary_first", "boundary_later"):
        k = 1 if name == "boundary_first" else 3

        def make(seed):
            n, Q, X = lat(seed)
            e = e_new_sequence(Q, None, X, d, r, precond, 20)
            if len(e) < k + 1:
                return None
            # the boundary between iterations k - 1 and k (e_new grows monotonically along preconditioned CG)
            rad = math.sqrt(e[k - 1] * (0.5 if k == 1 else math.sqrt(e[k - 2] / e[k - 1])))
            return mk(n, Q, None, X, 1e-2, 1, 20, rad)
        return _search(make)
    if name in ("negcurv_first", "giveup"):
        def make(seed):
            n, Q, G, rng = saddle(d, r, seed)
            X = orc.manifold_project(G + 1e-3 * rng.standard_normal(G.shape), d)     # near the maximiser of <X, G>
            if name == "giveup":
                return mk(n, Q, G, X, 1e-6, 1, 10, 1e12)
            return mk(n, Q, G, X, 1e-6, 1, 10, 0.1)
        return _search(make)
    if name == "negcurv_later":
        def make(seed):
            n, Q, G, rng = saddle(d, r, seed)
            return mk(n, Q, G, random_start(rng, r, d, n), 1e-6, 1, 50, 1e6)
        return _search(make, 200)
    if name == "scon":
        def make(seed):
            n, Q, X = lat(seed)
            for _ in range(40):                    # towards a critical point
                X, res, _ = run(Q, None, X, d, r, "exact", 0.0, 1, 50, 100.0)
                if res.gradNormOpt < 1e-4:
                    break
            else:
                return None
            # then out to a gradient norm of about 0.08: n0 < 0.1, and the residual stop n0^2 is a reduction by n0 only
            E = np.random.default_rng([seed, d, r, pi, 81]).standard_normal(X.shape)
            op = orc.QuadraticProblem(n, d, r)
            op.set_Q(Q)
            eps = 1e-3 * 0.08 / op.rie_grad_norm(orc.manifold_project(X + 1e-3 * E, d))
            X = orc.manifold_project(X + eps * E, d)
            return mk(n, Q, None, X, 1e-3 * op.rie_grad_norm(X), 1, NONE_MAX_INNER if precond == "none" else 200, 100.0)
        return _search(make, 5)
    if name == "maxiter_1":
        def make(seed):
            n, Q, X = lat(seed)
            return mk(n, Q, None, X, 1e-2, 1, 1, 100.0)
        return _search(make)
    if name in ("reject_1", "reject_3"):
        radii = 4.0 * 1.5 ** np.arange(0, 40)

        def make(i):
            seed, rad = divmod(i, len(radii))
            n, Q, X = lat(seed)
            return mk(n, Q, None, X, 1e-2, 1, 10, float(radii[rad]))
        return _search(make, 10 * len(radii))
    if name in ("multi_cap", "multi_shrink", "multi_reject"):
        # few outer iterations: near a critical point f1 - f2 cancels and rho is noise
        radii = {"multi_cap": (1.0, 0.5, 0.25), "multi_shrink": (2.0, 4.0, 8.0, 16.0, 32.0, 1.0), "multi_reject": tuple(4.0 * 1.4 ** np.arange(12))}[name]

        def make(i):
            seed, rad = divmod(i, len(radii))
            n, Q, X = lat(seed)
            return mk(n, Q, None, X, 1e-8, 6, NONE_MAX_INNER if precond == "none" else 50, radii[rad])
        return _search(make, 40 * len(radii))
    if name == "multi_tol":
        def make(seed):
            n, Q, X = lat(seed)
            inner = NONE_MAX_INNER if precond == "none" else 50
            _, _, tr = run(Q, None, X, d, r, precond, 0.0, 10, inner, 1.0)
            gns = [t[2] for t in tr if t[0] == "cmp" and t[1] == "gradnorm < tol"]
            if len(gns) < 6 or not gns[4] < gns[3]:
                return None
            return mk(n, Q, None, X, math.sqrt(gns[3] * gns[4]), 10, inner, 1.0)     # stops after the 4th attempt
        return _search(make)
    if name == "early_exit":
        n, Q, X = lat(0)
        op = orc.QuadraticProblem(n, d, r)
        op.set_Q(Q)
        return _finish(mk(n, Q, None, X, 2.0 * op.rie_grad_norm(X), 1, 10, 100.0))
    if name == "stationary":
        n = 5
        rng = np.random.default_rng([d, r, pi, 79])
        N = (d + 1) * n
        return _finish(mk(n, sp.csr_matrix((N, N)), np.zeros((r, N)), random_start(rng, r, d, n), 0.0, 1, 10, 100.0))
    raise KeyError(name)


BATCH_DR = ((2, 3), (3, 5))


def batch_agents(d, r):
    """three single-mode steps with one parameter set (tolerance 0, radius 10, sparse exact preconditioner) and no G, as
    one batched round runs them: an exactly stationary agent that gives up, a lattice agent rejected once and then
    accepted, and one accepted at once"""
    key = ("batch", d, r)
    if key in _CACHE:
        return _CACHE[key]
    tol, iters, inner, radius = 0.0, 1, 10, 10.0
    stat = case("stationary", d, r, "exact")
    out = [_finish(RtrCase("batch_giveup", d, r, "exact", stat.n, stat.Q, None, stat.X, tol, iters, inner, radius,
                           REACHES["giveup"][0]))]
    for want in (1, 0):
        for seed in range(60):
            n, Q, T = lattice(d, seed)
            rng = np.random.default_rng([seed, d, r, want, 80])
            X = near_start(rng, T, r, SIGMAS[seed % len(SIGMAS)])
            c = _finish(RtrCase(f"batch_reject{want}", d, r, "exact", n, Q, None, X, tol, iters, inner, radius, ""))
            if c.result.rejections == want and len(c.attempts()) == want + 1 and min_margin(c.trace) >= 1e-6:
                out.append(c)
                break
        else:
            raise RuntimeError("no lattice start with %d rejections" % want)
    _CACHE[key] = out
    return out


def grad_norm(c: RtrCase, X) -> float:
    """the oracle's Riemannian gradient norm of case c's problem at X"""
    op = orc.QuadraticProblem(c.n, c.d, c.r)
    op.set_Q(c.Q)
    if c.G is not None:
        op.set_G(c.G)
    return op.rie_grad_norm(np.asarray(X))


def differs(a: RtrCase, X_b, res_b, tol) -> bool:
    """what the GPU test compares tells run b from case a's oracle run: an exactly compared field, or the iterate or f_opt
    beyond the tolerances of that preconditioner"""
    ra = a.result
    exact = ("success", "tcg_status", "tcg_iterations", "outer_iterations", "rejections")
    if any(getattr(ra, k) != getattr(res_b, k) for k in exact):
        return True
    xtol, ftol = tol
    return (np.linalg.norm(X_b - a.X_out) > xtol * np.linalg.norm(a.X_out)
            or abs(res_b.fOpt - ra.fOpt) > ftol * abs(ra.fOpt))


def tolerances(precond: str):
    """(iterate, f_opt) relative tolerances of test_rtr_single_step_sequence"""
    return {"exact": (1e-8, 1e-9), "jacobi": (1e-9, 1e-9), "none": (1e-5, 1e-7)}[precond]


_CACHE: Dict[tuple, RtrCase] = {}


def case(name, d, r, precond) -> RtrCase:
    key = (name, d, r, precond)
    if key not in _CACHE:
        _CACHE[key] = make_case(*key)
    return _CACHE[key]
