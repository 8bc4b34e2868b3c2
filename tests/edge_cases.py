"""Edge-record graphs the datasets never reach, and references for the device's edge-record path in the reference's
arithmetic.  Helper module of test_edge_cases_cpu.py (CPU) and test_gpu_edge_cases.py (GPU); no fixtures.

The path is `dpgo_problem_set_edges` / `_set_edge_weights[_async]` / `_robust_reweight[_async]`: k_assemble_Q sums every
block's contribution list (edge kinds 0-3 and static blocks), k_edge_weights evaluates each edge's squared residual, its
robust weight and the GNC counts.  Each case names what it is built for (`EdgeCase.target`); test_edge_cases_cpu.py checks
from host facts that it gets there.

  * Q: T Om T^T, -T Om, -Om T^T, Om and the static blocks in long double from the doubles the library receives, with the
    bound gamma_k sum|terms| per entry, k = 4 (block's contribution count) + 3: it holds for any summation order.
  * r^2: computeMeasurementError (ref src/DPGO_utils.cpp:494-500) in long double, with its forward-error bound.
  * weights: `reference_weight` is RobustCost::weight(sqrt(r2)) (ref src/DPGO_robust.cpp:23-66) with the operations in the
    reference's order, in float64.  GM's `1 + r * r` may be contracted to an fma by a compiler allowed to (the reference's
    own build uses -march=native), so both variants are given; the device computes the product rounded on its own
    (GM_DEVICE), as ISO C++ and the host port do.  GNC has no contractable expression: one expected value.
"""
from __future__ import annotations

from dataclasses import dataclass
from fractions import Fraction
from typing import Optional

import numpy as np

import structure_cases as sc
from dpo_b200 import posegraph as pg

U = sc.U
LD = np.longdouble
COSTS = ("L2", "L1", "Huber", "TLS", "GM", "GNC_TLS")
GM_DEVICE = "separate"                 # 1 + r*r with the product rounded first (no fma)

# the reference's default GNC schedule (RobustCostParameters: mu0 = 1e-4, mu *= 1.4, 100 updates; barc = 5) and the barc
# of the GNC loops in test_gpu_refactor.py
GNC_MU0, GNC_STEP, GNC_ITERS = 1e-4, 1.4, 100
GNC_BARCS = (5.0, 10.0)


def gnc_schedule():
    mu, out = GNC_MU0, []
    for _ in range(GNC_ITERS + 1):
        out.append(mu)
        mu = GNC_STEP * mu                # RobustCost::update: mu = GNCMuStep * mu
    return out


# ---------------------------------------------------------------------------------------------------------------------
# cases
# ---------------------------------------------------------------------------------------------------------------------
@dataclass
class EdgeCase(sc.Case):
    fixed: Optional[np.ndarray] = None             # per-edge flags: weights robust re-weighting leaves alone


CASE_NAMES = ("static_only", "no_edges", "static_on_edge_pose", "static_on_free_pose", "static_twice",
              "static_nonsymmetric", "star2100", "clique60", "repeated_pair", "wide_weights", "wide_kappa_tau",
              "non_orthonormal", "path1e6")
READBACK = tuple(nm for nm in CASE_NAMES if nm != "path1e6")      # Q read back and checked entry by entry
HUB_LEAVES = 2100


def _spd(rng, dh):
    M = rng.standard_normal((dh, dh))
    return M @ M.T + np.eye(dh)


def _edges(rng, d, pairs):
    e = sc.edge_set(rng, d, pairs)
    e.weight = rng.uniform(0.25, 4.0, len(e))
    return e


def make_case(name: str, d: int, seed: int = 0) -> EdgeCase:
    rng = np.random.default_rng([seed, d, 100 + CASE_NAMES.index(name)])
    dh = d + 1
    spose, sblk, fixed = [], [], None
    if name == "static_only":
        n, pairs, target = 1, [], "n = 1, m = 0, one static block: Q is that block"
        spose, sblk = [0], [_spd(rng, dh)]
    elif name == "no_edges":
        n, pairs, target = 6, [], "m = 0, n > 1, no static block: no contribution at all, Q = 0"
    elif name == "static_on_edge_pose":
        n, pairs, target = 4, sc.chain(range(4)), "a static block summed after the edge terms of its pose"
        spose, sblk = [2], [_spd(rng, dh)]
    elif name == "static_on_free_pose":
        n, pairs, target = 5, sc.chain(range(4)), "a static block on a pose without edges: its block is the static block"
        spose, sblk = [4], [_spd(rng, dh)]
    elif name == "static_twice":
        n, pairs, target = 4, sc.chain(range(4)), "two static blocks on one pose, summed in input order"
        spose, sblk = [1, 3, 1], [_spd(rng, dh), _spd(rng, dh), _spd(rng, dh)]
    elif name == "static_nonsymmetric":
        n, pairs, target = 3, sc.chain(range(3)), "a non-symmetric static block, summed as given (not symmetrised)"
        spose, sblk = [1], [rng.standard_normal((dh, dh))]
    elif name == "star2100":
        n = HUB_LEAVES + 1
        pairs = [(0, i) if i % 2 else (i, 0) for i in range(1, n)]        # the hub as p1 (kind 0) and as p2 (kind 1)
        target = f"hub diagonal block of {HUB_LEAVES} kind-0/1 contributions"
    elif name == "clique60":
        n, pairs, target = 60, [tuple(p) for p in sc._clique(60)], "60-pose clique: every block of Q present"
    elif name == "repeated_pair":
        n = 3
        pairs = [(0, 1) if k % 2 == 0 else (1, 0) for k in range(100)] + [(1, 2)]
        target = "one pair 50 times in each direction: kind 2 and kind 3 contributions in one block"
    elif name == "wide_weights":
        n = 46
        pairs = sc.chain(range(40)) + [(3, 17), (5, 30), (11, 39), (0, 39)] + sc.chain(range(40, 45))
        target = "weights over +-100 decades, exact zeros; poses 40-44 touched by zero-weight edges only"
    elif name == "wide_kappa_tau":
        n, pairs, target = 30, sc.chain(range(30)) + [(0, 29), (4, 20), (7, 13)], "kappa and tau over +-8 decades"
    elif name == "non_orthonormal":
        n, pairs, target = 25, sc.chain(range(25)) + [(2, 24), (9, 3)], "non-orthonormal R, |t| up to 1e6"
    elif name == "path1e6":
        n, pairs, target = 1_000_001, None, "10^6 edges: the counters' atomics from ~7800 CTAs"
    else:
        raise KeyError(name)
    if name == "path1e6":
        m = n - 1
        z = np.zeros(m, dtype=np.int64)
        e = pg.EdgeSet(d, z, z, np.arange(m), np.arange(1, n), sc.random_rotations(rng, m, d),
                       rng.standard_normal((m, d)), rng.uniform(1.0, 100.0, m), rng.uniform(0.5, 10.0, m))
        fixed = (np.arange(m) % 7 == 0).astype(np.int32)
    elif pairs:
        e = _edges(rng, d, pairs)
    else:
        e = pg.EdgeSet.empty(d)
    m = len(e)
    if name == "wide_weights":
        e.weight = 10.0 ** rng.uniform(-100.0, 100.0, m)
        e.weight[[2, 9, 41]] = 0.0                                       # zeros inside the main component
        e.weight[np.flatnonzero(e.p1 >= 40)] = 0.0                       # the last component: zero weights only
    elif name == "wide_kappa_tau":
        e.kappa = 10.0 ** rng.uniform(-8.0, 8.0, m)
        e.tau = 10.0 ** rng.uniform(-8.0, 8.0, m)
    elif name == "non_orthonormal":
        e.R = rng.standard_normal((m, d, d)) * 10.0 ** rng.uniform(-2.0, 2.0, (m, 1, 1))
        e.t = rng.uniform(-1.0, 1.0, (m, d)) * 10.0 ** rng.uniform(0.0, 6.0, (m, 1))
        e.t[0] = 1e6
    c = EdgeCase(name, d, n, e, target, fixed=fixed)
    if spose:
        c.static_pose, c.static_blocks = np.array(spose, dtype=np.int32), np.array(sblk, dtype=np.float64)
    return c


def zero_only_poses(c: EdgeCase) -> np.ndarray:
    """Poses whose every edge has weight 0 (and that have at least one edge and no static block)."""
    e = c.edges
    touched = np.zeros(c.n, dtype=bool)
    nonzero = np.zeros(c.n, dtype=bool)
    for p in (e.p1, e.p2):
        touched[p] = True
        nonzero[p[e.weight != 0]] = True
    if c.static_pose is not None:
        nonzero[c.static_pose] = True
    return np.flatnonzero(touched & ~nonzero)


# ---------------------------------------------------------------------------------------------------------------------
# Q in long double, block by block
# ---------------------------------------------------------------------------------------------------------------------
def contributions(c: EdgeCase, weight=None, static_blocks=None):
    """(brow, bcol, values, magnitudes, count) per contribution in long double, (d+1)x(d+1) each: the terms k_assemble_Q
    sums, with the absolute-value evaluation of each.  `weight` / `static_blocks` override the case's."""
    e, d, dh = c.edges, c.d, c.dh
    m = len(e)
    w = ld(e.weight if weight is None else weight)
    T = ld(e.homogeneous()) if m else np.zeros((0, dh, dh), dtype=LD)
    om = np.zeros((m, dh), dtype=LD)
    om[:, :d] = ld(e.kappa)[:, None]
    om[:, d] = ld(e.tau)
    omw = om * w[:, None]
    TOm = T * omw[:, None, :]
    aTOm = abs(T) * abs(omw)[:, None, :]
    diag = np.zeros((m, dh, dh), dtype=LD)
    diag[:, np.arange(dh), np.arange(dh)] = omw
    vals = [TOm @ np.transpose(T, (0, 2, 1)), diag, -TOm, -np.transpose(TOm, (0, 2, 1))]
    mags = [aTOm @ np.transpose(abs(T), (0, 2, 1)), abs(diag), aTOm, np.transpose(aTOm, (0, 2, 1))]
    brow = [e.p1, e.p2, e.p1, e.p2]
    bcol = [e.p1, e.p2, e.p2, e.p1]
    if c.static_pose is not None and len(c.static_pose):
        S = ld(c.static_blocks if static_blocks is None else static_blocks)
        vals.append(S)
        mags.append(abs(S))
        brow.append(c.static_pose)
        bcol.append(c.static_pose)
    cat = lambda xs, dt: np.concatenate([np.asarray(x, dtype=dt) for x in xs]) if xs else np.zeros(0, dt)
    return (cat(brow, np.int64), cat(bcol, np.int64), np.concatenate(vals).reshape(-1, dh, dh),
            np.concatenate(mags).reshape(-1, dh, dh))


def q_reference(c: EdgeCase, weight=None, static_blocks=None):
    """{(i, j): (Q_ij in long double, sum of |terms|, contribution count)} over the block pattern of the case."""
    brow, bcol, vals, mags = contributions(c, weight, static_blocks)
    key = brow * c.n + bcol
    uniq, inv, cnt = np.unique(key, return_inverse=True, return_counts=True)
    ref = np.zeros((len(uniq), c.dh, c.dh), dtype=LD)
    mag = np.zeros_like(ref)
    np.add.at(ref, inv, vals)
    np.add.at(mag, inv, mags)
    return {(int(k // c.n), int(k % c.n)): (ref[q], mag[q], int(cnt[q])) for q, k in enumerate(uniq)}


def gamma(k):
    return k * U / (1.0 - k * U)


def check_q(blocks, qref, what="Q"):
    """blocks: {(i, j): float64 (d+1)x(d+1)} read from the device.  Every block of the pattern, every entry within
    gamma_{4 count + 3} sum|terms|; no block outside the pattern."""
    assert set(blocks) == set(qref), f"{what}: block pattern differs"
    worst = (0.0, None)
    for ij, (ref, mag, cnt) in qref.items():
        err = abs(ld(blocks[ij]) - ref)
        bound = LD(gamma(4 * cnt + 3)) * mag
        bad = err > bound
        if bad.any():
            k, cc = np.unravel_index(int(np.argmax(err - bound)), err.shape)
            raise AssertionError(f"{what}: block {ij} entry ({k}, {cc}) got {blocks[ij][k, cc]!r}, ref {float(ref[k, cc])!r}, "
                                 f"err {float(err[k, cc]):.3e} > bound {float(bound[k, cc]):.3e} ({cnt} contributions)")
        rel = float(np.max(np.where(mag > 0, err / np.where(mag > 0, mag, 1), 0)))
        if rel > worst[0]:
            worst = (rel, ij)
    return worst


def q_dense(blocks, n, dh):
    import scipy.sparse as sp
    if not blocks:
        return sp.csr_matrix((n * dh, n * dh))
    keys = list(blocks)
    rows = np.concatenate([np.repeat(np.arange(dh), dh) + i * dh for i, _ in keys])
    cols = np.concatenate([np.tile(np.arange(dh), dh) + j * dh for _, j in keys])
    vals = np.concatenate([np.asarray(blocks[k], dtype=np.float64).ravel() for k in keys])
    return sp.csr_matrix((vals, (rows, cols)), shape=(n * dh, n * dh))


# ---------------------------------------------------------------------------------------------------------------------
# reading Q back exactly through X Q
# ---------------------------------------------------------------------------------------------------------------------
def pattern(c: EdgeCase):
    """sorted block columns of every block row"""
    nbr = [set() for _ in range(c.n)]
    for a, b in zip(c.edges.p1.tolist(), c.edges.p2.tolist()):
        nbr[a].update((a, b))
        nbr[b].update((a, b))
    if c.static_pose is not None:
        for p in c.static_pose.tolist():
            nbr[p].add(p)
    return [sorted(s) for s in nbr]


def selector_classes(c: EdgeCase):
    """Poses grouped so that no two poses of a group share a block column (a distance-2 colouring of the block graph):
    one 0/1 row of X that picks row k of every pose in a group makes each entry of X Q one product by 1.0 plus exact
    zeros, i.e. bitwise that entry of Q."""
    nbr = pattern(c)
    colour = np.full(c.n, -1, dtype=np.int64)
    classes = []
    for p in np.argsort([-len(s) for s in nbr], kind="stable").tolist():
        if not nbr[p]:
            continue
        used = {int(colour[q]) for j in nbr[p] for q in nbr[j] if colour[q] >= 0}     # the pattern is symmetric
        k = 0
        while k in used:
            k += 1
        colour[p] = k
        if k == len(classes):
            classes.append([])
        classes[k].append(p)
    return [np.array(cl, dtype=np.int64) for cl in classes], nbr


def read_back(product, c: EdgeCase, r: int):
    """Q's blocks from calls product(X) = X Q with r selector rows each.  {(i, j): (d+1)x(d+1) float64}."""
    dh = c.dh
    classes, nbr = selector_classes(c)
    probes = [(cl, k) for cl in classes for k in range(dh)]
    out = {}
    for s in range(0, len(probes), r):
        X = np.zeros((r, c.N))
        chunk = probes[s:s + r]
        for a, (cl, k) in enumerate(chunk):
            X[a, cl * dh + k] = 1.0
        Y = product(X)
        for a, (cl, k) in enumerate(chunk):
            for p in cl.tolist():
                for j in nbr[p]:
                    out.setdefault((p, j), np.zeros((dh, dh)))[k] = Y[a, j * dh:(j + 1) * dh]
    return out


# ---------------------------------------------------------------------------------------------------------------------
# squared residuals and weights
# ---------------------------------------------------------------------------------------------------------------------
def ld(a):
    return np.asarray(a, dtype=LD)


def tiles_of(X, n, dh):
    """(n, r, d+1) pose tiles of an r x (d+1) n iterate"""
    r = X.shape[0]
    return np.transpose(np.asarray(X).reshape(r, n, dh), (1, 0, 2))


def residual_reference(c: EdgeCase, X):
    """computeMeasurementError (ref src/DPGO_utils.cpp:494-500) in long double, and its bound: every squared term's
    base as |X2| + sum |X1| |T| is a dot of d + 1 terms, r d + r of them are squared and summed, kappa and tau scale."""
    e, d, dh = c.edges, c.d, c.dh
    r = X.shape[0]
    Xt = ld(tiles_of(X, c.n, dh))
    Y1, Y2 = Xt[e.p1][:, :, :d], Xt[e.p2][:, :, :d]
    q1, q2 = Xt[e.p1][:, :, d], Xt[e.p2][:, :, d]
    R, t = ld(e.R), ld(e.t)
    rot = np.sum((np.einsum("mab,mbc->mac", Y1, R) - Y2) ** 2, axis=(1, 2))
    tra = np.sum((q2 - q1 - np.einsum("mab,mb->ma", Y1, t)) ** 2, axis=1)
    rotm = np.sum((np.einsum("mab,mbc->mac", abs(Y1), abs(R)) + abs(Y2)) ** 2, axis=(1, 2))
    tram = np.sum((abs(q2) + abs(q1) + np.einsum("mab,mb->ma", abs(Y1), abs(t))) ** 2, axis=1)
    ka, ta = ld(e.kappa), ld(e.tau)
    k = 2 * (d + 2) + r * dh + 2
    return ka * rot + ta * tra, LD(gamma(k)) * (abs(ka) * rotm + abs(ta) * tram)


def _gm_fused(r):
    """1 / (a a) with a = fma(r, r, 1): the exact r r + 1, rounded once"""
    fr = Fraction(float(r))
    a = float(fr * fr + 1) if np.isfinite(r) else float(r) * float(r) + 1.0
    return 1.0 / (a * a) if a != 0 else np.inf


def reference_weight(cost, r2, mu=1.0, param=1.0, gm=GM_DEVICE):
    """RobustCost::weight(sqrt(r2)) (ref src/DPGO_robust.cpp:23-66) in float64, every operation in the reference's order.
    r2: scalar or array; returns float64 of the same shape.  gm: "separate" (1 + r*r with r*r rounded first) or "fused"
    (one fma)."""
    r2 = np.asarray(r2, dtype=np.float64)
    mu, c = np.float64(mu), np.float64(param)
    with np.errstate(divide="ignore", invalid="ignore", over="ignore"):
        r = np.sqrt(r2)
        if cost == "L2":
            w = np.ones_like(r)
        elif cost == "L1":
            w = np.float64(1.0) / r
        elif cost == "Huber":
            w = np.where(r < c, 1.0, c / r)
        elif cost == "TLS":
            w = np.where(r < c, 1.0, 0.0)
        elif cost == "GM":
            if gm == "fused":
                w = np.vectorize(_gm_fused, otypes=[np.float64])(r)
            else:
                a = 1.0 + r * r
                w = 1.0 / (a * a)
        elif cost == "GNC_TLS":
            rsq = r * r
            c2 = c * c
            upper = (mu + 1.0) / mu * c2
            lower = mu / (mu + 1.0) * c2
            w = np.where(rsq >= upper, 0.0, np.where(rsq <= lower, 1.0, np.sqrt(c2 * mu * (mu + 1.0) / rsq) - mu))
        else:
            raise KeyError(cost)
    return np.asarray(w, dtype=np.float64)


def prefix_device_weight(cost, r2, mu=1.0, param=1.0):
    """What k_edge_weights computed before it took r = sqrt(r2) for every loss: GM from 1 + r2, GNC from r2 against
    bounds evaluated as c2 (mu + 1) / mu and c2 mu / (mu + 1).  Kept to show which residuals it classified differently."""
    r2 = np.asarray(r2, dtype=np.float64)
    mu, c = np.float64(mu), np.float64(param)
    with np.errstate(divide="ignore", invalid="ignore", over="ignore"):
        if cost == "GM":
            s = 1.0 + r2
            return 1.0 / (s * s)
        if cost == "GNC_TLS":
            c2 = c * c
            return np.where(r2 >= c2 * (mu + 1.0) / mu, 0.0,
                            np.where(r2 <= c2 * mu / (mu + 1.0), 1.0, np.sqrt(c2 * mu * (mu + 1.0) / r2) - mu))
    return reference_weight(cost, r2, mu, param)


def classify(w):
    """(weight exactly 1, exactly 0, anything else) as computeConvergedLoopClosureRatio counts (ref src/PGOAgent.cpp:1247-1289)"""
    w = np.asarray(w)
    one, zero = int(np.sum(w == 1.0)), int(np.sum(w == 0.0))
    return one, zero, int(w.size) - one - zero


def _around(v):
    v = np.float64(v)
    return [np.nextafter(v, -np.inf), v, np.nextafter(v, np.inf)]


def boundary_probes(cost, mu, param):
    """Squared residuals at every bound either formula draws for (cost, mu, param), and one ulp either side: the GNC
    bounds in the reference's order and in the pre-fix device order, and c^2 for Huber and TLS.  Finite and >= 0 only."""
    mu, c = np.float64(mu), np.float64(param)
    c2 = c * c
    vals = []
    with np.errstate(over="ignore", divide="ignore", invalid="ignore"):
        if cost == "GNC_TLS":
            for b in ((mu + 1.0) / mu * c2, mu / (mu + 1.0) * c2, c2 * (mu + 1.0) / mu, c2 * mu / (mu + 1.0)):
                vals += _around(b)
        elif cost in ("Huber", "TLS"):
            vals += _around(c2)
    v = np.unique(np.array(vals, dtype=np.float64))
    return v[np.isfinite(v) & (v >= 0)]


def gnc_boundary_set():
    """(mu, barc, r2) of every GNC probe: the default schedule at barc 5 and 10, mu = 1e-300 and 1e300, and barc = 0"""
    out = []
    for c in GNC_BARCS:
        for mu in gnc_schedule() + [1e-300, 1e300]:
            out += [(mu, c, v) for v in boundary_probes("GNC_TLS", mu, c)]
    for mu in (1e-4, 1.0, 1e300):
        out += [(mu, 0.0, v) for v in boundary_probes("GNC_TLS", mu, 0.0)]
    return out


def boundary_iterate(r, d, n):
    """An r x (d+1) n iterate whose rotation blocks are all one Stiefel point and whose translations are k e_1 at pose k:
    with R = I and t = 0 on an edge k -> k + 1, every squared term but one is exactly 0 and r^2 is exactly tau."""
    rng = np.random.default_rng([r, d])
    Y = np.linalg.qr(rng.standard_normal((r, d)))[0]
    X = np.zeros((r, (d + 1) * n))
    for k in range(n):
        X[:, k * (d + 1):k * (d + 1) + d] = Y
        X[0, k * (d + 1) + d] = float(k)
    return X


def boundary_case(d, taus):
    """A path whose edge k -> k + 1 has R = I, t = 0, kappa = 1 and tau = taus[k]: at boundary_iterate, r^2 = tau."""
    m = len(taus)
    z = np.zeros(m, dtype=np.int64)
    R = np.broadcast_to(np.eye(d), (m, d, d)).copy()
    e = pg.EdgeSet(d, z, z, np.arange(m), np.arange(1, m + 1), R, np.zeros((m, d)), np.ones(m), np.asarray(taus, dtype=np.float64))
    return EdgeCase("boundary", d, m + 1, e, "r^2 = tau exactly at each probe")
